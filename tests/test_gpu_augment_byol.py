"""GPU: the BYOL paper's augmentation recipe (TwoViewAugment(recipe="byol"), csrc/augment.cu) against
torchvision.transforms.v2.functional on identical records, its sampler's distribution, reproducibility, and
get_loader(augmentation="byol") feeding a training step.

The oracle for one (sample, view): resized_crop(BICUBIC, antialias=True) (BILINEAR when the record's bicubic bit is
clear), clamp(0, 1) after a bicubic resize, flip, the colour jitter in the record's order, grayscale, gaussian_blur,
solarize(0.5)."""
import numpy as np
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder

pytestmark = pytest.mark.gpu

GRAY, SOLARIZE, BICUBIC = 1, 2, 4


def _oracle(img, q, R, ksize):
    import torchvision.transforms.v2.functional as F
    flags = int(q[14])
    top, left, ch, cw = [int(v) for v in q[:4]]
    mode = F.InterpolationMode.BICUBIC if flags & BICUBIC else F.InterpolationMode.BILINEAR
    x = F.resized_crop(img, top, left, ch, cw, [R, R], interpolation=mode, antialias=True)
    if flags & BICUBIC:
        x = x.clamp(0.0, 1.0)
    if q[4] != 0:
        x = F.hflip(x)
    if q[5] != 0:
        for op in [int(v) for v in q[6:10]]:
            if op == 0:
                x = F.adjust_brightness(x, float(q[10]))
            elif op == 1:
                x = F.adjust_contrast(x, float(q[11]))
            elif op == 2:
                x = F.adjust_saturation(x, float(q[12]))
            else:
                x = F.adjust_hue(x, float(q[13]))
    if flags & GRAY:
        x = F.rgb_to_grayscale(x, num_output_channels=3)
    if ksize and q[15] > 0:
        x = F.gaussian_blur(x, [ksize, ksize], [float(q[15]), float(q[15])])
    if flags & SOLARIZE:
        x = F.solarize(x, 0.5)
    return x


def _force_branches(params, up_crop):
    """Every branch at least once, whatever the sampler drew.  params: [2, n, 16] (n >= 6), edited in place."""
    p = params
    # view 1, sample 0: jitter, blur and solarize (solarize after the blur)
    p[0, 0, 4] = 1.0; p[0, 0, 5] = 1.0; p[0, 0, 14] = BICUBIC | SOLARIZE; p[0, 0, 15] = 1.3
    # view 1, sample 1: jitter, grayscale, solarize without blur
    p[0, 1, 5] = 1.0; p[0, 1, 14] = BICUBIC | GRAY | SOLARIZE; p[0, 1, 15] = 0.0
    # view 2, sample 2: no colour op at all (no jitter, grayscale, blur or solarize), no flip
    p[1, 2, 4] = 0.0; p[1, 2, 5] = 0.0; p[1, 2, 14] = BICUBIC; p[1, 2, 15] = 0.0
    # view 2, sample 3: the whole image (the strongest down-scaling the image allows), jitter on
    p[1, 3, 0:2] = 0.0; p[1, 3, 5] = 1.0
    # view 1, sample 4: a crop smaller than the output (up-scaling), blur on
    p[0, 4, 0:4] = torch.tensor(up_crop, dtype=torch.float32); p[0, 4, 15] = 0.7
    # view 2, sample 5: a bilinear record that solarizes: the flag word is read bit by bit
    p[1, 5, 14] = SOLARIZE; p[1, 5, 15] = 0.0


def _check_views(out, srcs, pc, R, ksize):
    worst = 0.0
    for view in range(2):
        for i, img in enumerate(srcs):
            ref = _oracle(img, pc[view, i], R, ksize)
            err = float((out[view, i] - ref).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, (view, i, err, pc[view, i])
    assert float(out.min()) >= 0.0 and float(out.max()) <= 1.0
    return worst


@pytest.mark.parametrize("hs,ws,R", [(96, 128, 64), (300, 260, 224), (400, 300, 48)])
def test_byol_views_match_torchvision_dense(cuda, hs, ws, R):
    from byol_b200.augment import TwoViewAugment
    g = torch.Generator().manual_seed(hs + ws)
    n = 7
    imgs = torch.rand(n, 3, hs, ws, generator=g)
    aug = TwoViewAugment(image_size=R, seed=21, recipe="byol")
    params = aug.sample_params(n, hs, ws, cuda)
    _force_branches(params, [5.0, 7.0, 20.0, 24.0])
    params[1, 3, 2:4] = torch.tensor([float(hs), float(ws)])
    v1, v2 = aug.apply(imgs.to(cuda), params)
    torch.cuda.synchronize()
    worst = _check_views(torch.stack([v1, v2]).cpu(), imgs, params.cpu().numpy(), R, aug.ksize)
    print("byol recipe, dense fp32 vs torchvision: worst abs error %.2e" % worst)


def test_byol_views_match_torchvision_ragged(cuda):
    from byol_b200.augment import TwoViewAugment
    g = torch.Generator().manual_seed(5)
    sizes = [(375, 500), (500, 375), (20, 30), (333, 500), (480, 640), (64, 48), (16, 200), (281, 300)]
    u8 = [torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g) for h, w in sizes]
    R = 224
    aug = TwoViewAugment(image_size=R, seed=8, recipe="byol")
    params = aug.sample_params_ragged(sizes, cuda)
    _force_branches(params, [2.0, 3.0, 15.0, 20.0])
    params[1, 3, 0:4] = torch.tensor([0.0, 0.0, float(sizes[3][0]), float(sizes[3][1])])
    v1, v2 = aug.apply_ragged([t.to(cuda) for t in u8], params)
    torch.cuda.synchronize()
    lut = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255))   # v / 255, correctly rounded
    worst = _check_views(torch.stack([v1, v2]).cpu(), [lut[t.long()] for t in u8], params.cpu().numpy(), R,
                         aug.ksize)
    print("byol recipe, ragged uint8 vs torchvision: worst abs error %.2e" % worst)


def test_byol_sampler_distribution(cuda):
    from byol_b200.augment import TwoViewAugment
    n, hs, ws = 20000, 256, 320
    aug = TwoViewAugment(image_size=224, seed=7, recipe="byol")
    p = aug.sample_params(n, hs, ws, cuda).cpu().numpy()
    flags = p[:, :, 14].astype(np.int64)
    assert np.array_equal(p[:, :, 14], flags.astype(np.float32)) and ((flags & ~7) == 0).all()
    assert (flags & BICUBIC).all()
    v1, v2 = p[0], p[1]
    assert abs((v1[:, 15] > 0).mean() - 1.0) < 0.02 and abs((v2[:, 15] > 0).mean() - 0.1) < 0.02
    assert abs((flags[0] & SOLARIZE != 0).mean() - 0.0) < 0.02 and abs((flags[1] & SOLARIZE != 0).mean() - 0.2) < 0.02
    sig = p[:, :, 15][p[:, :, 15] > 0]
    assert 0.1 <= sig.min() and sig.max() <= 2.0
    both = p.reshape(-1, 16)
    for col, prob in ((4, 0.5), (5, 0.8)):
        assert abs((both[:, col] != 0).mean() - prob) < 0.02, col
    assert abs(((flags & GRAY) != 0).mean() - 0.2) < 0.02
    for col, lo, hi in ((10, 0.6, 1.4), (11, 0.6, 1.4), (12, 0.8, 1.2), (13, -0.1, 0.1)):
        assert lo - 1e-6 <= both[:, col].min() and both[:, col].max() <= hi + 1e-6, col
        assert abs(both[:, col].min() - lo) < 0.01 and abs(both[:, col].max() - hi) < 0.01, col
        assert abs(both[:, col].mean() - 0.5 * (lo + hi)) < 0.02, col
    # crops and colour-op order are the reference recipe's: the same draws, hence the same values, for the same seed
    ref = TwoViewAugment(image_size=224, seed=7).sample_params(n, hs, ws, cuda).cpu().numpy()
    assert np.array_equal(ref[:, :, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9]], p[:, :, [0, 1, 2, 3, 4, 5, 6, 7, 8, 9]])
    assert np.array_equal(ref[:, :, 14].astype(np.int64) & GRAY, flags & GRAY)
    # color_jitter_strength scales the paper's factors
    half = TwoViewAugment(image_size=224, seed=7, color_jitter_strength=0.5, recipe="byol")
    ph = half.sample_params(n, hs, ws, cuda).cpu().numpy().reshape(-1, 16)
    for col, lo, hi in ((10, 0.8, 1.2), (12, 0.9, 1.1), (13, -0.05, 0.05)):
        assert lo - 1e-6 <= ph[:, col].min() and ph[:, col].max() <= hi + 1e-6, col


def test_byol_records_reproducible_and_chunked(cuda):
    from byol_b200.augment import TwoViewAugment
    n, hs, ws = 50, 120, 90
    a = TwoViewAugment(image_size=64, seed=3, recipe="byol")
    b = TwoViewAugment(image_size=64, seed=3, recipe="byol")
    pa0, pa1 = a.sample_params(n, hs, ws, cuda), a.sample_params(n, hs, ws, cuda)
    assert torch.equal(pa0, b.sample_params(n, hs, ws, cuda)) and not torch.equal(pa0, pa1)
    # equal sizes through the ragged sampler: the dense sampler's records
    assert torch.equal(b.sample_params_ragged([(hs, ws)] * n, cuda), pa1)
    sizes = [(40 + 11 * i, 300 - 5 * i) for i in range(n)]
    whole = a.sample_params_ragged(sizes, cuda, step=9)
    for chunk in (7, 16):
        parts = [b.sample_params_ragged(sizes[s:s + chunk], cuda, n0=s, total=n, step=9) for s in range(0, n, chunk)]
        assert torch.equal(torch.cat(parts, dim=1), whole), chunk
    # the same images and records give the same bits
    u8 = [torch.randint(0, 256, (3, h, w), dtype=torch.uint8, device=cuda) for h, w in sizes]
    x1, x2 = a.apply_ragged(u8, whole)
    y1, y2 = b.apply_ragged(u8, whole.clone())
    assert torch.equal(x1, y1) and torch.equal(x2, y2)


def test_byol_loader_views_and_step(tmp_path, cuda):
    from byol_b200 import wiring
    from byol_b200.data import get_loader
    from byol_b200.model import BYOL
    make_image_folder(tmp_path, seed=11)
    runs = []
    for _ in range(2):
        ld = get_loader(**loader_kwargs(tmp_path, batch_size=4, augmentation="byol"))
        ld.set_all_epochs(1)
        assert ld.train_loader.augment.recipe == "byol" and ld.test_loader.augment.recipe == "reference"
        runs.append([[t.clone() for t in b] for b in ld.train_loader] + [[t.clone() for t in b] for b in ld.test_loader])
    assert len(runs[0]) == 3 + 2
    for ba, bb in zip(*runs):
        for x, y in zip(ba, bb):
            assert torch.equal(x, y)
    for a1, a2, _ in runs[0][:3]:
        assert a1.shape == (4, 3, 64, 64) and not torch.equal(a1, a2)
        for v in (a1, a2):
            assert float(v.min()) >= 0.0 and float(v.max()) <= 1.0
    # the test split keeps its resize; the training views are the recipe's own
    ref = get_loader(**loader_kwargs(tmp_path, batch_size=4))
    ref.set_all_epochs(1)
    ref_batches = [[t.clone() for t in b] for b in ref.train_loader] + [[t.clone() for t in b] for b in ref.test_loader]
    for ba, bb in zip(runs[0][3:], ref_batches[3:]):
        for x, y in zip(ba, bb):
            assert torch.equal(x, y)
    assert not torch.equal(runs[0][0][0], ref_batches[0][0])
    torch.manual_seed(0)
    model = BYOL(512, 256, 10, 10, arch="resnet18").cuda().train()
    opt = wiring.build_optimizer(model, global_batch_size=4)
    out = wiring.train_step(model, opt, *runs[0][0])
    torch.cuda.synchronize()
    assert np.isfinite(float(out["loss_mean"]))
