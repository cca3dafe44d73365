"""On-device two-view augmentation (SURVEY.md §8 f4) — the torchvision branch of the reference's
``build_train_and_test_transforms`` (/root/reference/main.py:386-397) for a batch of decoded images that already live
in HBM: ``RandomResizedCrop(R)``, ``RandomHorizontalFlip(0.5)``, ``RandomApply([ColorJitter(0.8s, 0.8s, 0.8s, 0.2s)], 0.8)``,
``RandomGrayscale(0.2)``, ``GaussianBlur(kernel 0.1 R, p 0.5)``.

    aug = TwoViewAugment(image_size=224, seed=0)
    aug1, aug2 = aug(images)            # images: fp32 CUDA [N, 3, H, W] in [0, 1] -> two fp32 [N, 3, 224, 224]
    aug1, aug2 = aug([u8_0, u8_1])      # or a list of CUDA uint8 [3, H_i, W_i] images of any sizes (read as v / 255)

``recipe="byol"`` gives the BYOL paper's views instead (Grill et al. 2020, Appendix B, Table 6): the crop resized with
an antialiased bicubic filter (clamped to [0, 1]), ``ColorJitter(0.4s, 0.4s, 0.2s, 0.1s)``, blur with p 1.0 on view 1
and 0.1 on view 2, and ``solarize(0.5)`` last with p 0.0 on view 1 and 0.2 on view 2; crop, flip, jitter p and
grayscale are the reference's.  The views are asymmetric: the first output is always the paper's view 1.

Every call draws fresh parameters from a counter-based RNG (seed, call counter, sample, view), so a run is
reproducible and the two views of a sample are independent.  ``apply(images, params)`` and
``apply_ragged(images, params)`` run the pipeline on explicit parameter records (tests/test_gpu_augment.py checks every stage against torchvision on identical parameters).

Test and validation images take no random draw: ``eval_params(sizes, device)`` builds, on the host, the records of
the object's ``eval_transform`` (``EVAL_TRANSFORMS``), and both views are the same image.  "resize" (the default) is
the reference's ``Resize((R, R))`` of the whole image (antialiased bilinear, ``resize_params``).  "byol" is the BYOL
paper's test transform (Grill et al. 2020, Appendix C.1; ``centre_crop_params``): the shorter side resized to
S = (8R + 3) // 7 (256 at R = 224) by antialiased bicubic (clamped to [0, 1]), then the centre R x R crop, i.e.
torchvision's ``CenterCrop(R)(Resize(S, BICUBIC)(x))`` on float images, the geometry computed as torchvision computes it
(``centre_crop_geometry``).  "byol_transfer" is the preprocessing of the paper's transfer evaluation (Appendix C.2,
after Kornblith et al. 2019; ``transfer_crop_params``): the shorter side resized to R itself by the same filter, then
the centre R x R crop.  Their records are window records: flag bit 3 says that floats 0-3 are (top, left, Sh, Sw),
the R x R window at (top, left) of the whole image resized to Sh x Sw, whose border pixels take taps from outside the
window; without the bit they are a crop box (top, left, h, w) resized to R x R.
"""
import ctypes

import torch

from . import _lib, ops
from ._lib import lib, check

RECORD = lib.byol_augment_record_floats()
# record float 14: a flag word (bit 3: floats 0-3 are a window of the resized image, see the module docstring)
FLAG_GRAY, FLAG_SOLARIZE, FLAG_BICUBIC, FLAG_WINDOW = 1, 2, 4, 8

# name -> colour-jitter factors (brightness, contrast, saturation, hue; times color_jitter_strength), blur and
# solarize probabilities of (view 1, view 2), bicubic crop resize
RECIPES = {
    "reference": dict(jitter=(0.8, 0.8, 0.8, 0.2), p_blur=(0.5, 0.5), p_solarize=(0.0, 0.0), bicubic=False),
    "byol": dict(jitter=(0.4, 0.4, 0.2, 0.1), p_blur=(1.0, 0.1), p_solarize=(0.0, 0.2), bicubic=True),
}


def _probability(name, v):
    v = float(v)
    if not 0.0 <= v <= 1.0:
        raise ValueError("TwoViewAugment: %s must lie in [0, 1], got %r" % (name, v))
    return v


def _per_view(name, v):
    """A probability for both views, or a (view 1, view 2) pair."""
    if isinstance(v, (tuple, list)):
        if len(v) != 2:
            raise ValueError("TwoViewAugment: %s must be a probability or a (view 1, view 2) pair" % name)
        return (_probability(name, v[0]), _probability(name, v[1]))
    p = _probability(name, v)
    return (p, p)


def centre_crop_geometry(h, w, image_size, resize=None):
    """(top, left, Sh, Sw) of a centre-crop eval transform for an h x w image: torchvision's ``Resize(S)`` (the shorter
    side to S, the longer one to ``int(S * long / short)``), then ``CenterCrop(R)`` (offsets
    ``int(round((size - R) / 2.0))``, Python's round half to even).  ``resize`` is S: by default (8R + 3) // 7, the
    "byol" transform; R for "byol_transfer"."""
    R = int(image_size)
    S = (8 * R + 3) // 7 if resize is None else int(resize)
    if S < R:
        raise ValueError("centre_crop_geometry: the resize target %d is smaller than the crop %d" % (S, R))
    short, long = (w, h) if w <= h else (h, w)
    new_short, new_long = S, int(S * long / short)
    sh, sw = (new_long, new_short) if w <= h else (new_short, new_long)
    return int(round((sh - R) / 2.0)), int(round((sw - R) / 2.0)), sh, sw


class TwoViewAugment(object):
    def __init__(self, image_size=224, color_jitter_strength=1.0, seed=0, p_flip=0.5, p_jitter=0.8, p_gray=0.2,
                 p_blur=None, blur=True, recipe="reference", p_solarize=None, eval_transform="resize"):
        """``recipe``: "reference" or "byol" (module docstring).  ``p_blur`` / ``p_solarize``: a probability for both
        views or a (view 1, view 2) pair; None takes the recipe's.  ``eval_transform``: what ``eval_params`` builds,
        "resize", "byol" or "byol_transfer" (``EVAL_TRANSFORMS``)."""
        if recipe not in RECIPES:
            raise ValueError("TwoViewAugment: unknown recipe %r (expected one of %s)" % (recipe, sorted(RECIPES)))
        if eval_transform not in EVAL_TRANSFORMS:
            raise ValueError("TwoViewAugment: unknown eval_transform %r (expected one of %s)"
                             % (eval_transform, sorted(EVAL_TRANSFORMS)))
        rc = RECIPES[recipe]
        self.recipe = recipe
        self.eval_transform = eval_transform
        self.R = int(image_size)
        self.strength = float(color_jitter_strength)
        self.seed = int(seed)
        self.p = (_probability("p_flip", p_flip), _probability("p_jitter", p_jitter), _probability("p_gray", p_gray))
        self.p_blur = _per_view("p_blur", rc["p_blur"] if p_blur is None else p_blur)
        self.p_solarize = _per_view("p_solarize", rc["p_solarize"] if p_solarize is None else p_solarize)
        self._recipe = _lib.AugmentRecipe(rc["jitter"], self.p[0], self.p[1], self.p[2], self.p_blur,
                                          self.p_solarize, int(rc["bicubic"]))
        k = int(0.1 * self.R) if blur else 0      # main.py:396 kernel_size = int(0.1 * image_size); made odd
        self.ksize = (k | 1) if k > 0 else 0
        self.calls = 0

    def sample_params(self, n, hs, ws, device):
        params = torch.empty((2, n, RECORD), dtype=torch.float32, device=device)
        check(lib.byol_augment_params_recipe(params.data_ptr(), n, hs, ws, self.seed, self.calls, self.strength,
                                             ctypes.byref(self._recipe), ops._stream()), "byol_augment_params_recipe")
        self.calls += 1
        return params

    def apply(self, images, params):
        if not images.is_cuda or images.dtype != torch.float32 or images.dim() != 4 or images.shape[1] != 3:
            raise ValueError("TwoViewAugment: expected a CUDA fp32 [N, 3, H, W] batch in [0, 1] (no CPU path)")
        images = images.contiguous()
        n, _, hs, ws = images.shape
        if tuple(params.shape) != (2, n, RECORD) or params.dtype != torch.float32 or not params.is_contiguous():
            raise ValueError("TwoViewAugment: params must be a contiguous fp32 [2, N, %d] tensor" % RECORD)
        out = torch.empty((2, n, 3, self.R, self.R), dtype=torch.float32, device=images.device)
        tmp = torch.empty_like(out) if self.ksize else None
        gray = torch.empty(2 * n, dtype=torch.float64, device=images.device)
        check(lib.byol_augment_apply(images.data_ptr(), params.data_ptr(), out.data_ptr(),
                                     0 if tmp is None else tmp.data_ptr(), gray.data_ptr(), n, hs, ws, self.R, self.ksize,
                                     ops._stream()), "byol_augment_apply", kernels=4 if self.ksize else 2)
        return out[0], out[1]

    def sample_params_ragged(self, sizes, device, n0=0, total=None, step=None):
        """Records for images of their own sizes ``sizes`` (a list of ``(H, W)``): samples ``[n0, n0 + len(sizes))`` of
        a ``total``-image batch (default: just these).  ``step`` keys the draw (default: the call counter, which then
        advances), so the chunks of one batch, sampled with one ``step``, get the records of a single call; equal
        sizes with ``n0 = 0`` reproduce ``sample_params``."""
        hw = _sizes_table(sizes, device)
        n = hw.shape[0]
        total = n if total is None else int(total)
        if n0 < 0 or n0 + n > total:
            raise ValueError("TwoViewAugment: samples [%d, %d) are not part of a %d-image batch" % (n0, n0 + n, total))
        if step is None:
            step = self.calls
            self.calls += 1
        params = torch.empty((2, n, RECORD), dtype=torch.float32, device=device)
        check(lib.byol_augment_params_ragged_recipe(params.data_ptr(), hw.data_ptr(), n, int(n0), total, self.seed,
                                                    int(step), self.strength, ctypes.byref(self._recipe),
                                                    ops._stream()),
              "byol_augment_params_ragged_recipe")
        return params

    def resize_params(self, sizes, device):
        """Records that take the whole image, with no flip, jitter, grayscale, blur or solarize: ``Resize((R, R))``,
        antialiased bilinear whatever the recipe, as the reference's test transform (main.py:398), through the same
        kernels as the training views."""
        params = torch.zeros((2, len(sizes), RECORD), dtype=torch.float32)
        params[:, :, 2:4] = torch.tensor([[float(h), float(w)] for h, w in sizes], dtype=torch.float32)
        params[:, :, 6:10] = torch.arange(4, dtype=torch.float32)
        return params.to(device)

    def centre_crop_params(self, sizes, device, resize=None):
        """Window records of the BYOL paper's test transform (Appendix C.1): the shorter side resized to
        (8R + 3) // 7 (or to ``resize``) with antialiased bicubic resampling (clamped to [0, 1]), then the centre R x R
        crop (``centre_crop_geometry``); no flip, jitter, grayscale, blur or solarize."""
        params = torch.zeros((2, len(sizes), RECORD), dtype=torch.float32)
        params[:, :, 0:4] = torch.tensor([[float(v) for v in centre_crop_geometry(h, w, self.R, resize)]
                                          for h, w in sizes], dtype=torch.float32).reshape(-1, 4)
        params[:, :, 6:10] = torch.arange(4, dtype=torch.float32)
        params[:, :, 14] = float(FLAG_BICUBIC | FLAG_WINDOW)
        return params.to(device)

    def transfer_crop_params(self, sizes, device):
        """Window records of the paper's transfer-evaluation preprocessing (Appendix C.2): the shorter side resized to
        R by antialiased bicubic, then the centre R x R crop."""
        return self.centre_crop_params(sizes, device, resize=self.R)

    def eval_params(self, sizes, device):
        """The records of this object's ``eval_transform`` for test / validation images of sizes ``sizes``."""
        return EVAL_TRANSFORMS[self.eval_transform](self, sizes, device)

    def apply_ragged(self, images, params):
        """``images``: a list of CUDA uint8 ``[3, H_i, W_i]`` tensors (values read as v / 255) -> two fp32
        ``[N, 3, R, R]`` views, computed exactly as ``apply`` computes them on ``[u8.float() / 255]``."""
        device = _check_ragged(images)
        n = len(images)
        if tuple(params.shape) != (2, n, RECORD) or params.dtype != torch.float32 or not params.is_contiguous() \
                or params.device != device:
            raise ValueError("TwoViewAugment: params must be a contiguous fp32 [2, N, %d] tensor on %s" % (RECORD, device))
        hw = _sizes_table([tuple(t.shape[1:]) for t in images], device)
        ptrs = torch.tensor([t.data_ptr() for t in images], dtype=torch.int64).to(device)
        out = torch.empty((2, n, 3, self.R, self.R), dtype=torch.float32, device=device)
        tmp = torch.empty_like(out) if self.ksize else None
        check(lib.byol_augment_apply_ragged(ptrs.data_ptr(), hw.data_ptr(), params.data_ptr(), out.data_ptr(),
                                            0 if tmp is None else tmp.data_ptr(), n, self.R, self.ksize, ops._stream()),
              "byol_augment_apply_ragged", kernels=4 if self.ksize else 2)
        return out[0], out[1]

    def __call__(self, images):
        if isinstance(images, (list, tuple)):
            device = _check_ragged(images)
            return self.apply_ragged(images, self.sample_params_ragged([tuple(t.shape[1:]) for t in images], device))
        n, _, hs, ws = images.shape
        return self.apply(images, self.sample_params(n, hs, ws, images.device))


# name -> the record maker of a test / validation transform (TwoViewAugment.eval_params)
EVAL_TRANSFORMS = {
    "resize": TwoViewAugment.resize_params,          # the reference's Resize((R, R)) (main.py:398)
    "byol": TwoViewAugment.centre_crop_params,       # Resize((8R + 3) // 7, BICUBIC) + CenterCrop(R)
    "byol_transfer": TwoViewAugment.transfer_crop_params,   # Resize(R, BICUBIC) + CenterCrop(R)
}


def _check_ragged(images):
    """A non-empty list of contiguous CUDA uint8 [3, H, W] tensors on one device; returns that device."""
    if not isinstance(images, (list, tuple)) or len(images) == 0:
        raise ValueError("TwoViewAugment: expected a non-empty list of CUDA uint8 [3, H, W] tensors")
    device = images[0].device if isinstance(images[0], torch.Tensor) else None
    for t in images:
        if not isinstance(t, torch.Tensor) or not t.is_cuda or t.dtype != torch.uint8 or t.dim() != 3 \
                or t.shape[0] != 3 or t.shape[1] < 1 or t.shape[2] < 1:
            raise ValueError("TwoViewAugment: every image must be a CUDA uint8 [3, H, W] tensor (no CPU path)")
        if not t.is_contiguous():
            raise ValueError("TwoViewAugment: every image must be contiguous")
        if t.device != device:
            raise ValueError("TwoViewAugment: all images must be on one device")
    return device


def _sizes_table(sizes, device):
    """``[(H, W), ...]`` -> device int32 [n, 2]"""
    hw = torch.tensor([[int(h), int(w)] for h, w in sizes], dtype=torch.int32).reshape(-1, 2)
    if hw.shape[0] == 0 or int(hw.min()) < 1:
        raise ValueError("TwoViewAugment: sizes must be a non-empty list of (H, W) with H, W >= 1")
    return hw.to(device)
