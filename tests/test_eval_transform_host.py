"""CPU: the evaluation transforms' records (byol_b200.augment: centre_crop_params, eval_params) and their choice in
get_loader (eval_transform).  The "byol" geometry is torchvision's own, read off F.resize and F.center_crop on small
index images (no kernel runs)."""
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder

# (H, W): landscape, portrait and square photographs; resized long sides of 257 / 259 at R = 224 (half-pixel centre
# offsets 16.5 -> 16 and 17.5 -> 18, Python's round half to even), images smaller than S = (8R + 3) // 7 (up-scaled),
# an extreme aspect ratio, and sizes whose long side lands on a rounding boundary
SIZES = [(375, 500), (500, 375), (333, 500), (480, 640), (256, 256), (224, 224), (300, 300), (256, 257), (257, 256),
         (256, 259), (259, 256), (512, 514), (100, 150), (150, 100), (40, 52), (20, 30), (64, 48), (16, 200), (200, 16),
         (281, 300), (97, 131), (73, 110), (110, 73), (600, 450), (1, 7)]
RES = [32, 64, 96, 224]


def _torchvision_geometry(h, w, R):
    """(top, left, Sh, Sw) of CenterCrop(R)(Resize(S)(img)) on an h x w image, read from torchvision's outputs."""
    import torchvision.transforms.v2.functional as F
    S = (8 * R + 3) // 7
    sh, sw = F.resize(torch.zeros(1, h, w), S, antialias=False).shape[-2:]
    index = torch.arange(sh * sw, dtype=torch.float64).reshape(1, sh, sw)
    window = F.center_crop(index, [R, R])
    assert window.shape[-2:] == (R, R)
    top, left = divmod(int(window[0, 0, 0]), sw)
    assert torch.equal(window[0], index[0, top:top + R, left:left + R])
    return top, left, sh, sw


@pytest.mark.parametrize("R", RES)
def test_geometry_is_torchvision_resize_then_center_crop(R):
    from byol_b200.augment import centre_crop_geometry
    for h, w in SIZES:
        assert centre_crop_geometry(h, w, R) == _torchvision_geometry(h, w, R), (h, w, R)


def test_geometry_at_224():
    from byol_b200.augment import centre_crop_geometry
    assert (8 * 224 + 3) // 7 == 256
    assert centre_crop_geometry(375, 500, 224) == (16, 58, 256, 341)
    assert centre_crop_geometry(256, 257, 224) == (16, 16, 256, 257)      # 16.5 -> 16
    assert centre_crop_geometry(256, 259, 224) == (16, 18, 256, 259)      # 17.5 -> 18
    assert centre_crop_geometry(100, 150, 224) == (16, 80, 256, 384)      # up-scaled


def test_centre_crop_records():
    from byol_b200.augment import (FLAG_BICUBIC, FLAG_WINDOW, RECORD, TwoViewAugment, centre_crop_geometry)
    aug = TwoViewAugment(image_size=96, seed=3, eval_transform="byol")
    p = aug.centre_crop_params(SIZES, "cpu")
    assert p.shape == (2, len(SIZES), RECORD) and p.dtype == torch.float32
    assert torch.equal(p[0], p[1])
    geo = torch.tensor([centre_crop_geometry(h, w, 96) for h, w in SIZES], dtype=torch.float32)
    assert torch.equal(p[0, :, 0:4], geo)
    assert (p[:, :, 14] == FLAG_BICUBIC | FLAG_WINDOW).all()
    assert (p[:, :, 6:10] == torch.arange(4, dtype=torch.float32)).all()
    # no flip, jitter, colour factors or blur
    assert not p[:, :, 4:6].any() and not p[:, :, 10:14].any() and not p[:, :, 15].any()
    assert torch.equal(aug.eval_params(SIZES, "cpu"), p)
    # the default transform is today's whole-image resize records
    ref = TwoViewAugment(image_size=96, seed=3)
    assert ref.eval_transform == "resize"
    assert torch.equal(ref.eval_params(SIZES, "cpu"), ref.resize_params(SIZES, "cpu"))


@pytest.mark.parametrize("bad", ["centre", "BYOL", None, "reference"])
def test_two_view_augment_rejects_eval_transform(bad):
    from byol_b200.augment import TwoViewAugment
    with pytest.raises(ValueError):
        TwoViewAugment(64, eval_transform=bad)


def test_get_loader_eval_transform(tmp_path):
    from byol_b200.data import get_loader
    make_image_folder(tmp_path, seed=2)
    for kw in (dict(), dict(eval_transform=None)):          # key absent (or None): today's loader
        ld = get_loader(**loader_kwargs(tmp_path, **kw))
        assert ld.eval_transform == "resize"
        assert ld.test_loader.augment.eval_transform == "resize" and ld.test_loader.augment.recipe == "reference"
    ld = get_loader(**loader_kwargs(tmp_path, eval_transform="byol"))
    assert ld.eval_transform == "byol" and ld.augmentation == "reference"
    assert ld.test_loader.augment.eval_transform == "byol"
    # the training split is untouched, and the choice is independent of the training recipe
    assert ld.train_loader.augment.recipe == "reference" and ld.train_loader.augment.eval_transform == "resize"
    ld = get_loader(**loader_kwargs(tmp_path, eval_transform="byol", augmentation="byol"))
    assert ld.train_loader.augment.recipe == "byol" and ld.test_loader.augment.eval_transform == "byol"
    ld = get_loader(**loader_kwargs(tmp_path, augmentation="byol"))
    assert ld.test_loader.augment.eval_transform == "resize"
    for bad in ("centre_crop", "reference", "BYOL"):
        with pytest.raises(ValueError, match="eval_transform"):
            get_loader(**loader_kwargs(tmp_path, eval_transform=bad))
