"""GPU: the on-device two-view augmentation (csrc/augment.cu, byol_b200/augment.py) against
torchvision.transforms.v2.functional on identical parameters (/root/reference/main.py:386-397 builds this recipe from
torchvision transforms), plus distribution checks of the parameter sampler."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _reference(img, q, R, ksize):
    """One (sample, view): the torchvision functional pipeline on the CPU with the record's parameters."""
    import torchvision.transforms.v2.functional as F
    top, left, ch, cw = [int(v) for v in q[:4]]
    x = F.resized_crop(img, top, left, ch, cw, [R, R], interpolation=F.InterpolationMode.BILINEAR, antialias=True)
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
    if q[14] != 0:
        x = F.rgb_to_grayscale(x, num_output_channels=3)
    if ksize and q[15] > 0:
        x = F.gaussian_blur(x, [ksize, ksize], [float(q[15]), float(q[15])])
    return x


@pytest.mark.parametrize("hs,ws,R", [(96, 128, 64), (300, 260, 224)])
def test_augment_matches_torchvision(cuda, hs, ws, R):
    from byol_b200.augment import TwoViewAugment
    g = torch.Generator().manual_seed(hs)
    n = 6
    imgs = torch.rand(n, 3, hs, ws, generator=g)
    aug = TwoViewAugment(image_size=R, seed=123)
    params = aug.sample_params(n, hs, ws, cuda)
    # make sure every branch is exercised at least once, whatever the sampler drew
    params[0, 0, 4] = 1.0; params[0, 0, 5] = 1.0; params[0, 0, 14] = 0.0; params[0, 0, 15] = 1.3
    params[0, 1, 5] = 1.0; params[0, 1, 14] = 1.0; params[0, 1, 15] = 0.0
    params[1, 2, 5] = 0.0; params[1, 2, 4] = 0.0; params[1, 2, 15] = 0.4
    params[1, 3, 0:4] = torch.tensor([0.0, 0.0, float(hs), float(ws)])          # whole image: pure down-scaling
    v1, v2 = aug.apply(imgs.to(cuda), params)
    torch.cuda.synchronize()
    out = torch.stack([v1, v2]).cpu()
    pc = params.cpu().numpy()
    worst = 0.0
    for view in range(2):
        for i in range(n):
            ref = _reference(imgs[i], pc[view, i], R, aug.ksize)
            err = float((out[view, i] - ref).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, (view, i, err, pc[view, i])
    print("augment vs torchvision: worst abs error %.2e" % worst)
    assert float(out.min()) >= 0.0 and float(out.max()) <= 1.0 + 1e-6


def test_augment_parameter_distribution(cuda):
    """RandomResizedCrop.get_params / ColorJitter.get_params / the Bernoulli switches: ranges and frequencies."""
    from byol_b200.augment import TwoViewAugment
    n, hs, ws = 20000, 256, 320
    aug = TwoViewAugment(image_size=224, seed=7)
    p = aug.sample_params(n, hs, ws, cuda).cpu().numpy().reshape(-1, 16)
    p2 = aug.sample_params(n, hs, ws, cuda).cpu().numpy().reshape(-1, 16)
    assert not np.array_equal(p, p2)                                   # a fresh draw per call
    aug_b = TwoViewAugment(image_size=224, seed=7)
    assert np.array_equal(aug_b.sample_params(n, hs, ws, cuda).cpu().numpy().reshape(-1, 16), p)   # reproducible
    top, left, ch, cw = p[:, 0], p[:, 1], p[:, 2], p[:, 3]
    assert (top >= 0).all() and (left >= 0).all() and (top + ch <= hs).all() and (left + cw <= ws).all()
    area = ch * cw / (hs * ws)
    ratio = cw / ch
    assert area.min() > 0.07 and area.max() <= 1.0 and 0.70 < ratio.min() and ratio.max() < 1.40
    # against torchvision's own sampler (RandomResizedCrop.get_params: 10 attempts, then a centre crop)
    import torchvision.transforms as T
    torch.manual_seed(0)
    dummy = torch.zeros(3, hs, ws)
    ref = np.array([T.RandomResizedCrop.get_params(dummy, (0.08, 1.0), (3. / 4., 4. / 3.)) for _ in range(4000)])
    ref_area = ref[:, 2] * ref[:, 3] / (hs * ws)
    assert abs(area.mean() - ref_area.mean()) < 0.02 and abs(area.std() - ref_area.std()) < 0.02
    assert abs(np.log(ratio).std() - np.log(ref[:, 3] / ref[:, 2]).std()) < 0.02
    for col, prob in ((4, 0.5), (5, 0.8), (14, 0.2)):
        assert abs((p[:, col] != 0).mean() - prob) < 0.02, col
    assert abs((p[:, 15] > 0).mean() - 0.5) < 0.02
    sig = p[p[:, 15] > 0, 15]
    assert 0.1 <= sig.min() and sig.max() <= 2.0 and abs(sig.mean() - 1.05) < 0.05
    for col, lo, hi in ((10, 0.2, 1.8), (11, 0.2, 1.8), (12, 0.2, 1.8), (13, -0.2, 0.2)):
        assert lo - 1e-6 <= p[:, col].min() and p[:, col].max() <= hi + 1e-6
        assert abs(p[:, col].mean() - 0.5 * (lo + hi)) < 0.02
    order = p[:, 6:10].astype(int)
    assert (np.sort(order, 1) == np.arange(4)).all()                    # a permutation
    first = np.bincount(order[:, 0], minlength=4) / len(order)
    assert np.abs(first - 0.25).max() < 0.02
    # the two views of a sample are drawn independently
    a, b = p[:n, 0], p[n:, 0]
    assert abs(np.corrcoef(a, b)[0, 1]) < 0.05


def test_augment_throughput_and_step(cuda):
    """Feeds the training step: 2 x [N, 3, 224, 224] views straight into BYOL."""
    from byol_b200.augment import TwoViewAugment
    n = 256
    imgs = torch.rand(n, 3, 256, 256, device=cuda)
    aug = TwoViewAugment(image_size=224, seed=1)
    for _ in range(2):
        v1, v2 = aug(imgs)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        v1, v2 = aug(imgs)
    e1.record()
    torch.cuda.synchronize()
    rate = 5 * n / (e0.elapsed_time(e1) / 1000.0)
    print("two-view augmentation: %.0f images/s (2 views each)" % rate)
    assert rate > 20000
    assert v1.shape == (n, 3, 224, 224) and torch.isfinite(v1).all() and not torch.equal(v1, v2)
