"""GPU: the BYOL paper's test transform (eval_transform="byol": the shorter side resized to (8R + 3) // 7 by antialiased
bicubic, then the centre R x R crop) on the window records of csrc/augment.cu, against torchvision; the loader's test
split and knn_accuracy reading it.

The oracle for one image: F.center_crop(F.resize(x, S, BICUBIC, antialias=True).clamp(0, 1), R) (BILINEAR and no
clamp when the record's bicubic bit is clear), then the record's flip and grayscale."""
import numpy as np
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder
from tests.test_eval_transform_host import SIZES

pytestmark = pytest.mark.gpu

GRAY, BICUBIC, WINDOW = 1, 4, 8


def _oracle(img, q, R):
    import torchvision.transforms.v2.functional as F
    flags = int(q[14])
    mode = F.InterpolationMode.BICUBIC if flags & BICUBIC else F.InterpolationMode.BILINEAR
    x = F.resize(img, (8 * R + 3) // 7, interpolation=mode, antialias=True)
    if flags & BICUBIC:
        x = x.clamp(0.0, 1.0)
    x = F.center_crop(x, [R, R])
    if q[4] != 0:
        x = F.hflip(x)
    if flags & GRAY:
        x = F.rgb_to_grayscale(x, num_output_channels=3)
    return x


def _records(aug, sizes, device, bicubic=True):
    """centre_crop_params with view 2 flipped and every third view-2 record grayscale; bicubic=False clears the
    bicubic bit (a bilinear resize + centre crop)."""
    p = aug.centre_crop_params(sizes, "cpu")
    p[1, :, 4] = 1.0
    p[1, ::3, 14] += GRAY
    if not bicubic:
        p[:, :, 14] -= BICUBIC
    return p.to(device)


def _check(out, srcs, p, R, tol=2e-4):
    worst = 0.0
    for view in range(2):
        for i, img in enumerate(srcs):
            ref = _oracle(img, p[view, i], R)
            err = float((out[view][i].cpu() - ref).abs().max())
            worst = max(worst, err)
            assert err < tol, (view, i, tuple(img.shape), err)
    return worst


@pytest.mark.parametrize("bicubic", [True, False])
@pytest.mark.parametrize("R", [64, 96, 224])
def test_window_records_match_torchvision_ragged(cuda, R, bicubic):
    from byol_b200.augment import TwoViewAugment
    g = torch.Generator().manual_seed(R)
    u8 = [torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g) for h, w in SIZES]
    aug = TwoViewAugment(image_size=R, seed=1, eval_transform="byol")
    p = _records(aug, SIZES, cuda, bicubic)
    v1, v2 = aug.apply_ragged([t.to(cuda) for t in u8], p)
    torch.cuda.synchronize()
    lut = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255))   # v / 255, correctly rounded
    worst = _check((v1, v2), [lut[t.long()] for t in u8], p.cpu().numpy(), R)
    if bicubic:
        assert float(torch.stack([v1, v2]).min()) >= 0.0 and float(torch.stack([v1, v2]).max()) <= 1.0
    print("window records (%s), ragged uint8 at R %d vs torchvision: worst abs error %.2e"
          % ("bicubic" if bicubic else "bilinear", R, worst))


@pytest.mark.parametrize("bicubic", [True, False])
@pytest.mark.parametrize("R", [64, 96, 224])
def test_window_records_match_torchvision_dense(cuda, R, bicubic):
    from byol_b200.augment import TwoViewAugment
    aug = TwoViewAugment(image_size=R, seed=1, eval_transform="byol")
    worst = 0.0
    for hs, ws in SIZES[::2]:
        imgs = torch.rand(3, 3, hs, ws, generator=torch.Generator().manual_seed(hs * 1000 + ws))
        p = _records(aug, [(hs, ws)] * 3, cuda, bicubic)
        v1, v2 = aug.apply(imgs.to(cuda), p)
        torch.cuda.synchronize()
        worst = max(worst, _check((v1, v2), imgs, p.cpu().numpy(), R))
    print("window records (%s), dense fp32 at R %d vs torchvision: worst abs error %.2e"
          % ("bicubic" if bicubic else "bilinear", R, worst))


def _decoded(samples, device):
    from byol_b200.data import _read, decode_batch
    return decode_batch([_read(path) for path, _ in samples], device)


def _batches(ld):
    return [[t.clone() for t in b] for b in ld]


def test_loader_test_split_takes_the_centre_crop(tmp_path, cuda):
    from byol_b200.data import get_loader
    make_image_folder(tmp_path, seed=13)
    runs = {}
    for name, kw in (("byol", dict(eval_transform="byol")), ("default", dict())):
        ld = get_loader(**loader_kwargs(tmp_path, batch_size=4, **kw))
        ld.set_all_epochs(1)
        runs[name] = (ld, _batches(ld.train_loader), _batches(ld.test_loader))
    ld, train, test = runs["byol"]
    # training batches: the default loader's bits
    assert len(train) == len(runs["default"][1]) == 3
    for a, b in zip(train, runs["default"][1]):
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    # test batches: the "byol" records applied to the decoded images, both views the same, in [0, 1]
    aug, samples = ld.test_loader.augment, ld.test_loader.samples
    assert len(test) == 2
    for k, (v1, v2, lab) in enumerate(test):
        chunk = samples[4 * k:4 * k + 4]
        imgs = _decoded(chunk, cuda)
        e1, e2 = aug.apply_ragged(imgs, aug.centre_crop_params([tuple(t.shape[1:]) for t in imgs], cuda))
        assert v1.shape == (len(chunk), 3, 64, 64)
        assert torch.equal(v1, e1) and torch.equal(v2, e2) and torch.equal(v1, v2)
        assert lab.tolist() == [c for _, c in chunk]
        assert float(v1.min()) >= 0.0 and float(v1.max()) <= 1.0
    # not the default loader's whole-image resize
    assert not torch.equal(test[0][0], runs["default"][2][0][0])


def test_knn_accuracy_reads_the_eval_transform(tmp_path, cuda, monkeypatch):
    from byol_b200 import knn
    from byol_b200.data import get_loader
    from byol_b200.model import BYOL
    make_image_folder(tmp_path, seed=4)
    loader = get_loader(**loader_kwargs(tmp_path, eval_transform="byol"))
    torch.manual_seed(12)
    model = BYOL(512, 64, loader.output_size, 10, arch="resnet18", head_latent_size=128).cuda()
    seen = {}
    classify = knn.knn_classify

    def spy(bank, bank_labels, queries, *args, **kw):
        seen.update(bank=bank.clone(), queries=queries.clone())
        return classify(bank, bank_labels, queries, *args, **kw)

    monkeypatch.setattr(knn, "knn_classify", spy)
    acc = knn.knn_accuracy(model, loader, k=3)
    monkeypatch.undo()

    aug, bs = loader.test_loader.augment, loader.test_loader.batch_size

    def features(samples, records):
        feats, labels = [], []
        for s in range(0, len(samples), bs):
            imgs = _decoded(samples[s:s + bs], cuda)
            v1, _ = aug.apply_ragged(imgs, records([tuple(t.shape[1:]) for t in imgs], cuda))
            feats.append(model.representations(v1))
            labels += [c for _, c in samples[s:s + bs]]
        return torch.cat(feats), torch.tensor(labels, dtype=torch.int64, device=cuda)

    bank, bank_labels = features(loader.train_loader.samples, aug.centre_crop_params)
    queries, query_labels = features(loader.test_loader.samples, aug.centre_crop_params)
    assert torch.equal(seen["bank"], knn.l2_normalize_rows(bank))
    assert torch.equal(seen["queries"], knn.l2_normalize_rows(queries))
    pred = knn.knn_classify(bank, bank_labels, queries, loader.output_size, k=3)
    hit = pred.long() == query_labels.view(-1, 1)
    assert acc == {"knn_top1": 100.0 * float(hit[:, 0].float().mean()),
                   "knn_top5": 100.0 * float(hit.any(1).float().mean())}
    # the whole-image resize gives other features: the evaluation did read the centre crops
    resized, _ = features(loader.train_loader.samples, aug.resize_params)
    assert not torch.equal(seen["bank"], knn.l2_normalize_rows(resized))
