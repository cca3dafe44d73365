"""CPU: the host logic of transfer linear evaluation (byol_b200.logreg): the regularisation grid, head selection,
"mean_per_class", argument checks that run before any kernel, and the "byol_transfer" eval transform (the shorter side
resized to R by bicubic, then the centre R x R crop) against torchvision's Resize(R) + CenterCrop(R)."""
import numpy as np
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder
from tests.test_eval_transform_host import SIZES

RES = [32, 64, 96, 224]


def test_l2_grid():
    from byol_b200.logreg import L2_GRID, check_l2s
    assert np.array_equal(L2_GRID, np.logspace(-6, 5, 45))
    assert L2_GRID[0] == 1e-6 and L2_GRID[-1] == 1e5 and len(L2_GRID) == 45
    assert check_l2s(L2_GRID) == tuple(float(v) for v in L2_GRID)
    for bad in ((), (1.0, -1.0), (float("nan"),), (float("inf"),), 3.0):
        with pytest.raises(ValueError):
            check_l2s(bad)


def test_selection_ties_and_non_finite_heads():
    from byol_b200.linear_eval import select_head
    assert select_head([50.0, 70.0, 70.0, 10.0]) == 1                  # ties: the earlier value of the grid
    assert select_head([50.0, 70.0, 70.0], [True, False, True]) == 2   # a non-finite head is never chosen
    assert select_head([90.0, 10.0], [False, True]) == 1
    with pytest.raises(ValueError, match="diverged"):
        select_head([90.0, 10.0], [False, False])


def test_mean_per_class_by_hand():
    from byol_b200.logreg import class_metric
    # 3 classes with 4, 1 and 5 images; head 0 hits 4 / 0 / 1, head 1 hits 2 / 1 / 5
    hits = [[4, 0, 1], [2, 1, 5]]
    counts = [4, 1, 5]
    np.testing.assert_allclose(class_metric(hits, counts, "top1"), [50.0, 80.0])
    np.testing.assert_allclose(class_metric(hits, counts, "mean_per_class"),
                               [100.0 * (1.0 + 0.0 + 0.2) / 3, 100.0 * (0.5 + 1.0 + 1.0) / 3])
    # a class absent from the split does not count
    np.testing.assert_allclose(class_metric([[3, 0, 1]], [3, 0, 2], "mean_per_class"), [100.0 * (1.0 + 0.5) / 2])
    np.testing.assert_allclose(class_metric([[3, 0, 1]], [3, 0, 2], "top1"), [80.0])
    with pytest.raises(ValueError, match="no images"):
        class_metric([[0, 0]], [0, 0], "top1")
    with pytest.raises(ValueError, match="metric"):
        class_metric(hits, counts, "top5")


def test_fit_rejects_bad_arguments():
    """Shapes, dtypes and arguments are checked before any device access (CPU tensors reach the device check last)."""
    from byol_b200.logreg import fit_logistic_regression
    x, y = torch.zeros(8, 64), torch.zeros(8, dtype=torch.int64)
    with pytest.raises(ValueError, match="multiple of 64"):
        fit_logistic_regression(torch.zeros(8, 96), y, 3)
    with pytest.raises(ValueError, match="multiple of 64"):
        fit_logistic_regression(torch.zeros(8, 0), y, 3)
    with pytest.raises(ValueError, match="num_classes"):
        fit_logistic_regression(x, y, 1)
    with pytest.raises(ValueError, match="num_classes"):
        fit_logistic_regression(x, y, True)
    with pytest.raises(ValueError, match="empty"):
        fit_logistic_regression(torch.zeros(0, 64), torch.zeros(0, dtype=torch.int64), 3)
    with pytest.raises(ValueError, match="fp32"):
        fit_logistic_regression(x.bfloat16(), y, 3)
    with pytest.raises(ValueError, match="labels"):
        fit_logistic_regression(x, y.int(), 3)
    with pytest.raises(ValueError, match="max_iter"):
        fit_logistic_regression(x, y, 3, max_iter=0)
    with pytest.raises(ValueError, match="tol"):
        fit_logistic_regression(x, y, 3, tol=0.0)
    with pytest.raises(ValueError, match="l2s"):
        fit_logistic_regression(x, y, 3, l2s=())
    with pytest.raises(RuntimeError, match="CPU path"):
        fit_logistic_regression(x, y, 3)


def test_transfer_accuracy_rejects_bad_arguments(tmp_path):
    from byol_b200.data import get_loader
    from byol_b200.logreg import transfer_accuracy

    class Model(object):
        base_network_output_size = 512

    make_image_folder(tmp_path, seed=1)
    loader = get_loader(**loader_kwargs(tmp_path))
    with pytest.raises(ValueError, match="metric"):
        transfer_accuracy(Model(), loader, metric="top5")
    with pytest.raises(ValueError, match="network"):
        transfer_accuracy(Model(), loader, network="ema")
    with pytest.raises(ValueError, match="l2s"):
        transfer_accuracy(Model(), loader, l2s=[-1.0])
    bad = Model()
    bad.base_network_output_size = 100
    with pytest.raises(ValueError, match="multiple of 64"):
        transfer_accuracy(bad, loader)
    loader.test_loader.samples = []
    with pytest.raises(ValueError, match="test split is empty"):
        transfer_accuracy(Model(), loader)
    loader.train_loader.samples = []
    with pytest.raises(ValueError, match="training split is empty"):
        transfer_accuracy(Model(), loader)


def _torchvision_transfer_geometry(h, w, R):
    """(top, left, Sh, Sw) of CenterCrop(R)(Resize(R)(img)), read from torchvision's outputs."""
    import torchvision.transforms.v2.functional as F
    sh, sw = F.resize(torch.zeros(1, h, w), R, antialias=False).shape[-2:]
    index = torch.arange(sh * sw, dtype=torch.float64).reshape(1, sh, sw)
    window = F.center_crop(index, [R, R])
    assert window.shape[-2:] == (R, R)
    top, left = divmod(int(window[0, 0, 0]), sw)
    assert torch.equal(window[0], index[0, top:top + R, left:left + R])
    return top, left, sh, sw


@pytest.mark.parametrize("R", RES)
def test_transfer_geometry_is_torchvision_resize_then_center_crop(R):
    """Odd, portrait, landscape, square and up-scaled sizes (SIZES) at four resolutions."""
    from byol_b200.augment import centre_crop_geometry
    for h, w in SIZES:
        assert centre_crop_geometry(h, w, R, resize=R) == _torchvision_transfer_geometry(h, w, R), (h, w, R)
    # the default resize target is still the "byol" one
    assert centre_crop_geometry(375, 500, 224) == centre_crop_geometry(375, 500, 224, resize=256)


def test_transfer_geometry_by_hand():
    from byol_b200.augment import centre_crop_geometry
    assert centre_crop_geometry(375, 500, 224, resize=224) == (0, 37, 224, 298)
    assert centre_crop_geometry(500, 375, 224, resize=224) == (37, 0, 298, 224)
    assert centre_crop_geometry(224, 225, 224, resize=224) == (0, 0, 224, 225)     # 0.5 -> 0
    assert centre_crop_geometry(100, 150, 224, resize=224) == (0, 56, 224, 336)    # up-scaled
    with pytest.raises(ValueError):
        centre_crop_geometry(100, 150, 224, resize=200)


def test_transfer_records():
    from byol_b200.augment import EVAL_TRANSFORMS, FLAG_BICUBIC, FLAG_WINDOW, TwoViewAugment, centre_crop_geometry
    assert set(EVAL_TRANSFORMS) == {"resize", "byol", "byol_transfer"}
    aug = TwoViewAugment(image_size=96, seed=3, eval_transform="byol_transfer")
    p = aug.eval_params(SIZES, "cpu")
    assert torch.equal(p, aug.transfer_crop_params(SIZES, "cpu")) and torch.equal(p[0], p[1])
    geo = torch.tensor([centre_crop_geometry(h, w, 96, resize=96) for h, w in SIZES], dtype=torch.float32)
    assert torch.equal(p[0, :, 0:4], geo)
    assert (p[:, :, 14] == FLAG_BICUBIC | FLAG_WINDOW).all()
    assert not p[:, :, 4:6].any() and not p[:, :, 10:14].any() and not p[:, :, 15].any()
    # the other transforms' records are unchanged
    byol = TwoViewAugment(image_size=96, seed=3, eval_transform="byol")
    assert torch.equal(byol.eval_params(SIZES, "cpu")[0, :, 0:4],
                       torch.tensor([centre_crop_geometry(h, w, 96) for h, w in SIZES], dtype=torch.float32))
    for bad in ("centre", "centre_crop", "BYOL", "reference", None, "transfer", "BYOL_TRANSFER"):
        with pytest.raises(ValueError):
            TwoViewAugment(64, eval_transform=bad)


def test_get_loader_transfer_transform(tmp_path):
    import shutil
    from byol_b200.data import get_loader
    make_image_folder(tmp_path, seed=2)
    shutil.copytree(tmp_path / "test", tmp_path / "valid")
    ld = get_loader(**loader_kwargs(tmp_path, eval_transform="byol_transfer"))
    assert ld.eval_transform == "byol_transfer"
    assert ld.test_loader.augment.eval_transform == "byol_transfer"
    assert ld.valid_loader is not None and ld.valid_loader.augment.eval_transform == "byol_transfer"
    # the training split keeps its augmentation
    assert ld.train_loader.augment.eval_transform == "resize" and ld.train_loader.augment.recipe == "reference"
