"""GPU: mixed-size uint8 augmentation (byol_augment_params_ragged / byol_augment_apply_ragged) against torchvision and
the fp32 kernels, GPU JPEG decoding, and byol_b200.data.get_loader feeding the reference's own main.py step loop."""
import functools
import os

import numpy as np
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder
from tests.test_gpu_augment import _reference

pytestmark = pytest.mark.gpu


@pytest.fixture
def folder(tmp_path):
    return tmp_path, make_image_folder(tmp_path, seed=11)


def _decoded(root, made, cuda, split="train"):
    from byol_b200.data import _read, decode_batch
    rels = sorted(r for r in made if r.startswith(split))
    return rels, decode_batch([_read(os.path.join(root, r)) for r in rels], cuda)


def test_ragged_matches_torchvision(folder, cuda):
    from byol_b200.augment import TwoViewAugment
    root, made = folder
    _, imgs = _decoded(root, made, cuda)
    n, R = len(imgs), 64
    aug = TwoViewAugment(image_size=R, seed=123)
    sizes = [tuple(t.shape[1:]) for t in imgs]
    params = aug.sample_params_ragged(sizes, cuda)
    # every branch at least once, whatever the sampler drew
    params[0, 0, 4] = 1.0; params[0, 0, 5] = 1.0; params[0, 0, 14] = 0.0; params[0, 0, 15] = 1.3
    params[0, 1, 5] = 1.0; params[0, 1, 14] = 1.0; params[0, 1, 15] = 0.0
    params[1, 2, 5] = 0.0; params[1, 2, 4] = 0.0; params[1, 2, 15] = 0.4
    h3, w3 = sizes[3]
    params[1, 3, 0:4] = torch.tensor([0.0, 0.0, float(h3), float(w3)])          # whole image
    v1, v2 = aug.apply_ragged(imgs, params)
    torch.cuda.synchronize()
    out = torch.stack([v1, v2]).cpu()
    pc = params.cpu().numpy()
    worst = 0.0
    for view in range(2):
        for i in range(n):
            hs, ws = sizes[i]
            top, left, ch, cw = [int(v) for v in pc[view, i, :4]]
            assert 0 <= top and 0 <= left and top + ch <= hs and left + cw <= ws, (i, sizes[i], pc[view, i, :4])
            ref = _reference(imgs[i].cpu().float() / 255, pc[view, i], R, aug.ksize)
            err = float((out[view, i] - ref).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, (view, i, sizes[i], err, pc[view, i])
    print("ragged augment vs torchvision: worst abs error %.2e over %d images" % (worst, n))
    assert float(out.min()) >= 0.0 and float(out.max()) <= 1.0 + 1e-6


def test_ragged_equal_sizes_bit_equal_to_dense(cuda):
    from byol_b200.augment import TwoViewAugment
    g = torch.Generator().manual_seed(3)
    n, hs, ws, R = 40, 90, 130, 64
    u8 = torch.randint(0, 256, (n, 3, hs, ws), dtype=torch.uint8, generator=g).to(cuda)
    a = TwoViewAugment(image_size=R, seed=9)
    b = TwoViewAugment(image_size=R, seed=9)
    for call in range(2):
        pd = a.sample_params(n, hs, ws, cuda)
        pr = b.sample_params_ragged([(hs, ws)] * n, cuda)
        assert torch.equal(pd, pr), call
    # chunks of one batch, sampled with one step, give the single call's records
    sizes = [(50 + 7 * i, 60 + 5 * i) for i in range(n)]
    whole = b.sample_params_ragged(sizes, cuda, step=17)
    parts = [b.sample_params_ragged(sizes[s:s + 16], cuda, n0=s, total=n, step=17) for s in range(0, n, 16)]
    assert torch.equal(torch.cat(parts, dim=1), whole)
    # uint8 images read as v / 255 give apply's bits on the same fp32 values.  The table is the correctly rounded
    # quotient, as the kernel computes it; torch's CUDA `u8.float() / 255` multiplies by a rounded reciprocal instead
    # and can differ in the last bit.
    lut = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255)).to(cuda)
    dense = lut[u8.long()]
    assert float((dense - u8.float() / 255).abs().max()) < 1e-7
    imgs = [u8[i] for i in range(n)]
    r1, r2 = b.apply_ragged(imgs, pd)
    d1, d2 = a.apply(dense, pd)
    assert torch.equal(r1, d1) and torch.equal(r2, d2)
    # the list form of the call draws the same records as sample_params
    c = TwoViewAugment(image_size=R, seed=4)
    e = TwoViewAugment(image_size=R, seed=4)
    l1, l2 = c(imgs)
    t1, t2 = e(dense)
    assert torch.equal(l1, t1) and torch.equal(l2, t2)


def test_ragged_input_checks(cuda):
    from byol_b200.augment import TwoViewAugment
    aug = TwoViewAugment(image_size=32)
    ok = torch.zeros(3, 40, 40, dtype=torch.uint8, device=cuda)
    bad = [[], [ok.float()], [ok.cpu()], [ok[:1]], [ok.transpose(1, 2).contiguous()[:, :, ::2]], [ok, ok[None]]]
    for images in bad:
        with pytest.raises(ValueError):
            aug(images)
    with pytest.raises(ValueError):
        aug.sample_params_ragged([(0, 5)], cuda)
    with pytest.raises(ValueError):
        aug.sample_params_ragged([(5, 5)] * 3, cuda, n0=2, total=4)
    with pytest.raises(ValueError):
        aug.apply_ragged([ok], torch.zeros(2, 2, 16, device=cuda))


def test_resize_records_match_resize(folder, cuda):
    import torchvision.transforms.v2.functional as F
    from byol_b200.augment import TwoViewAugment
    root, made = folder
    _, imgs = _decoded(root, made, cuda)
    for R in (64, 96):
        aug = TwoViewAugment(image_size=R)
        v1, v2 = aug.apply_ragged(imgs, aug.resize_params([tuple(t.shape[1:]) for t in imgs], cuda))
        assert torch.equal(v1, v2)
        for i, t in enumerate(imgs):
            ref = F.resize(t.cpu().float() / 255, [R, R], interpolation=F.InterpolationMode.BILINEAR, antialias=True)
            err = float((v1[i].cpu() - ref).abs().max())
            assert err < 2e-4, (R, i, tuple(t.shape), err)


def test_decoding_png_and_grayscale(folder, cuda):
    from PIL import Image
    root, made = folder
    rels, imgs = _decoded(root, made, cuda)
    for rel, t in zip(rels, imgs):
        kind = made[rel][1]
        pil = np.asarray(Image.open(os.path.join(root, rel)).convert("RGB"))
        assert t.is_cuda and t.dtype == torch.uint8 and tuple(t.shape) == (3,) + pil.shape[:2], rel
        got = t.permute(1, 2, 0).cpu().numpy()
        if kind == "png":
            assert np.array_equal(got, pil), rel                      # lossless
        else:
            # nvJPEG and libjpeg upsample the chroma planes differently: close, not equal
            assert np.abs(got.astype(int) - pil.astype(int)).mean() < 8.0, rel
        if kind == "gray":
            assert np.array_equal(got[..., 0], got[..., 1]) and np.array_equal(got[..., 0], got[..., 2]), rel


def test_loader_batches_reproducible(folder, cuda):
    from byol_b200.data import get_loader
    root, _ = folder
    runs = []
    for _ in range(2):
        ld = get_loader(**loader_kwargs(root, batch_size=5))
        ld.set_all_epochs(2)
        runs.append([[t.clone() for t in b] for b in ld.train_loader] + [[t.clone() for t in b] for b in ld.test_loader])
    assert len(runs[0]) == 2 + 1
    for ba, bb in zip(*runs):
        for x, y in zip(ba, bb):
            assert torch.equal(x, y)
    a1, a2, lab = runs[0][0]
    assert a1.is_cuda and a1.shape == (5, 3, 64, 64) and a1.dtype == torch.float32 and lab.dtype == torch.int64
    assert float(a1.min()) >= 0 and float(a1.max()) <= 1 and not torch.equal(a1, a2)
    t1, t2, tl = runs[0][2]
    assert torch.equal(t1, t2) and tl.tolist() == [0, 1, 2, 2, 2]
    # another epoch: another order and other views
    ld = get_loader(**loader_kwargs(root, batch_size=5))
    ld.set_all_epochs(3)
    b3 = next(iter(ld.train_loader))
    assert not torch.equal(b3[0], a1)


def test_reference_main_trains_on_image_folder(folder, cuda):
    """The reference's own lazy_generate_modules and execute_graph (train and test) on the folder, fed by get_loader."""
    import byol_b200.lars
    import byol_b200.model
    import byol_b200.objective
    import byol_b200.wiring
    from byol_b200.data import get_loader
    from tests.test_gpu_zz_dropin import _import_reference_main
    root, _ = folder
    main = _import_reference_main("resnet18", 512, 4, 64)
    main.BYOL = functools.partial(byol_b200.model.BYOL, arch=main.args.arch,
                                  head_latent_size=main.args.head_latent_size)
    main.loss_function = byol_b200.objective.loss_function
    main.LARS = byol_b200.lars.LARS
    main.layers.DistributedDataParallelPassthrough = byol_b200.wiring.DistributedDataParallelPassthrough
    main.args.data_dir = str(root)
    main.args.seed = 1
    loader = get_loader(train_transform=[], test_transform=[], **vars(main.args))
    assert loader.num_train_samples // main.args.num_replicas // main.args.batch_size == len(loader.train_loader) == 3
    assert loader.output_size == 3
    torch.manual_seed(1)
    # main.py:598 takes the top-5 accuracy, which needs at least 5 classifier outputs; the fixture has 3 classes
    model = main.BYOL(base_network_output_size=512, projection_output_size=256, classifier_output_size=10,
                      total_training_steps=6, base_decay=0.996).cuda()
    main.lazy_generate_modules(model, loader.train_loader)
    opt = main.LARS(torch.optim.SGD(main.layers.add_weight_decay(model, 1e-6), lr=0.1, momentum=0.9), eps=0.0)
    losses = []
    for epoch in range(2):      # --debug-step: one minibatch per call
        losses.append(main.execute_graph(epoch, model, loader.train_loader, None, optimizer=opt, prefix="train"))
        losses.append(main.execute_graph(epoch, model, loader.test_loader, None, optimizer=None, prefix="test"))
        loader.set_all_epochs(epoch + 1)
    print("reference execute_graph on the image folder:", losses)
    assert all(np.isfinite(losses))
