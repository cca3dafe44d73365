"""Linear evaluation of the frozen encoder (the BYOL paper's headline protocol): linear classifiers trained on the
frozen representation, a sweep of hyperparameters chosen on held-out data, test top-1 / top-5 of the chosen one.

    from byol_b200.linear_eval import linear_accuracy
    acc = linear_accuracy(model, loader)     # {"linear_top1": %, "linear_top5": %, "lr", "weight_decay", "heads": [...]}

H = len(lrs) * len(weight_decays) heads, one per (lr, weight decay) pair in lr-major order, train together on the same
bf16 features (``LinearHeads``).  Their weights are one [H * Cp, D] matrix (Cp = C rounded up to a multiple of 8), so
one training step is five launches with no host synchronisation:

1. ``ops.linear_fprop``: fp32 logits [B, H * Cp] of every head in one tensor-core GEMM (with the biases);
2. ``byol_linprobe_ce``: per (row, head) softmax cross-entropy, the bf16 gradient (softmax - onehot) / B and the
   per-head loss sums (csrc/linear_eval.cu);
3. ``ops.linear_wgrad``: dW += dlogits^T @ feats (deterministic fixed-point wgrad);
4. ``ops.col_sum``: db += the column sums of the same bf16 dlogits, so W and b get the gradient of one rounded matrix;
5. ``byol_linprobe_sgd``: Nesterov SGD of every head with its own lr and weight decay, the bf16 weight copy for the
   next GEMM, and dW / db zeroed.

Every reduction is fixed-point or integer, so a run gives the same bits every time.  The features are bf16 and the
logits their fp32-accumulated products, not fp32-accurate ones.
"""
import math

import numpy as np
import torch

from . import ops
from ._lib import check, lib

HOLDOUT_MAX = 10000           # the BYOL paper holds out about 10 000 ImageNet training images for its sweep
EVAL_ROWS = 8192              # feature rows per evaluation GEMM
DEFAULT_LRS = (0.4, 0.3, 0.2, 0.1, 0.05)


def _cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("byol_b200.linear_eval: %s must be a CUDA tensor (no CPU path)" % name)


def _finite_list(values, name):
    try:
        out = tuple(float(v) for v in values)
    except TypeError:
        raise ValueError("%s must be a sequence of numbers, got %r" % (name, values))
    if not out:
        raise ValueError("%s must not be empty" % name)
    for v in out:
        if not (v >= 0.0 and math.isfinite(v)):
            raise ValueError("%s must be finite and >= 0, got %r" % (name, values))
    return out


def _positive_int(v, name):
    if not isinstance(v, int) or isinstance(v, bool) or v < 1:
        raise ValueError("%s must be a positive int, got %r" % (name, v))


def check_hyperparameters(lrs, weight_decays, momentum):
    """(lrs, weight_decays) as float tuples; raises ValueError unless lrs is non-empty, both are finite and >= 0 and
    momentum is in [0, 1)."""
    lrs = _finite_list(lrs, "lrs")
    weight_decays = _finite_list(weight_decays, "weight_decays")
    if not (0.0 <= float(momentum) < 1.0):
        raise ValueError("momentum must be in [0, 1), got %r" % (momentum,))
    return lrs, weight_decays


def head_grid(lrs, weight_decays):
    """The (lr, weight decay) pair of each head, lr-major: head i has lrs[i // len(wds)], wds[i % len(wds)]."""
    return [(lr, wd) for lr in lrs for wd in weight_decays]


def cosine_factor(step, total_steps):
    """lr multiplier of 0-based step `step` of `total_steps`: 0.5 (1 + cos(pi step / total)), in fp64, rounded once
    to fp32.  Cosine decay to 0 over all steps with no warm-up (this module's choice)."""
    return np.float32(0.5 * (1.0 + math.cos(math.pi * step / total_steps)))


def holdout_split(n, seed):
    """(fit, held out) sorted int64 index arrays of n training images: a seeded draw of max(1, min(10 000, n // 10))
    images is held out for the selection; the rest are trained on."""
    if n < 1:
        raise ValueError("the training split is empty")
    k = max(1, min(HOLDOUT_MAX, n // 10))
    perm = np.random.default_rng([int(seed), 0x6c696e]).permutation(n)
    return np.sort(perm[k:]), np.sort(perm[:k])


def select_head(val_top1, finite=None):
    """Index of the head with the best validation top-1 (ties: the earlier head in the grid) among the heads whose
    `finite` flag is set (default: all).  A head with non-finite weights or biases has diverged and is never chosen;
    ValueError when every head has."""
    v = np.asarray(val_top1)
    if v.size == 0:
        raise ValueError("no heads to select from")
    ok = np.ones(v.shape, dtype=bool) if finite is None else np.asarray(finite, dtype=bool)
    if not ok.any():
        raise ValueError("every head diverged (non-finite weights or biases): no head can be selected; check the "
                         "features for non-finite values or lower the learning rates")
    return int(np.argmax(np.where(ok, v, np.iinfo(np.int64).min if v.dtype.kind in "iu" else -np.inf)))


def multihead_ce(logits, labels, num_heads, num_classes, dlogits=None, loss_sum=None, hits=None):
    """Softmax cross-entropy of H = num_heads heads side by side (byol_linprobe_ce).  logits: fp32 [B, >= H * Cp]
    (unit column stride, row pitch a multiple of 4), head h in columns h * Cp .. h * Cp + C - 1, Cp = C rounded up
    to a multiple of 8; labels: int64 [B] (a row whose label is outside [0, C) counts for nothing: no loss, no hit, a
    zero gradient).  Outputs, each optional: dlogits bf16
    [B, H * Cp] = (softmax - onehot) / B (0 in the padding columns); loss_sum fp32 [H] += the per-head sums of the row
    losses; hits int64 [H, 2] += the rows whose label is in the top 1 / top 5 (a NaN label logit is a miss)."""
    _cuda(logits, "logits"); _cuda(labels, "labels")
    if not isinstance(num_heads, int) or num_heads < 1 or not isinstance(num_classes, int) or num_classes < 2:
        raise ValueError("need num_heads >= 1 and num_classes >= 2, got %r, %r" % (num_heads, num_classes))
    cp = (num_classes + 7) // 8 * 8
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or \
            logits.shape[1] < num_heads * cp or logits.stride(0) % 4 != 0:
        raise ValueError("logits must be an fp32 [B, >= %d] matrix with unit column stride and a row pitch that is a "
                         "multiple of 4" % (num_heads * cp))
    b = logits.shape[0]
    if labels.dtype != torch.int64 or tuple(labels.shape) != (b,) or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous int64 [%d] vector" % b)
    for t, name, dtype, shape in ((dlogits, "dlogits", torch.bfloat16, (b, num_heads * cp)),
                                  (loss_sum, "loss_sum", torch.float32, (num_heads,)),
                                  (hits, "hits", torch.int64, (num_heads, 2))):
        if t is None:
            continue
        _cuda(t, name)
        if t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError("%s must be a contiguous %s %s tensor" % (name, dtype, list(shape)))
    if dlogits is None and loss_sum is None and hits is None:
        raise ValueError("multihead_ce: no output requested")
    if b:
        check(lib.byol_linprobe_ce(logits.data_ptr(), logits.stride(0), labels.data_ptr(), b, num_heads, num_classes,
                                   cp, 0 if dlogits is None else dlogits.data_ptr(),
                                   0 if loss_sum is None else loss_sum.data_ptr(),
                                   0 if hits is None else hits.data_ptr(), ops._stream()),
              "byol_linprobe_ce", kernels=1 if loss_sum is None else 2)


class LinearHeads(object):
    """H = len(lrs) * len(weight_decays) linear classifiers over the same D-dimensional features, one per (lr, weight
    decay) pair in ``head_grid`` order, trained by Nesterov SGD with momentum ``momentum``.

    ``params`` is one flat fp32 buffer: the weights [H, Cp, D] (``weight``) followed by the biases [H, Cp] (``bias``),
    Cp = C rounded up to a multiple of 8; the padding rows c >= C are zero and stay zero.  ``momentum_buf`` and
    ``grads`` have the same layout; ``weight_bf16`` is the [H * Cp, D] bf16 copy the logit GEMM reads (each update rewrites it; an edit
    of ``weight`` by hand reaches the logits only once it is copied there too).  Every head
    starts from the same seeded init, weights N(0, 0.01^2) and bias 0, so heads differ only by their hyperparameters."""

    def __init__(self, dim, num_classes, lrs, weight_decays, momentum=0.9, seed=0, device=None):
        lrs, weight_decays = check_hyperparameters(lrs, weight_decays, momentum)
        _positive_int(dim, "dim")
        if dim % 64 != 0:
            raise ValueError("the feature width D=%d must be a positive multiple of 64" % dim)
        if not isinstance(num_classes, int) or isinstance(num_classes, bool) or num_classes < 2:
            raise ValueError("num_classes must be an int >= 2, got %r" % (num_classes,))
        device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("byol_b200.linear_eval: LinearHeads lives on a CUDA device (no CPU path)")
        self.grid = head_grid(lrs, weight_decays)
        self.H, self.C, self.D = len(self.grid), num_classes, dim
        self.Cp = (num_classes + 7) // 8 * 8
        self.momentum = float(momentum)
        H, Cp, D = self.H, self.Cp, self.D
        nw = H * Cp * D
        w0 = torch.randn(num_classes, dim, generator=torch.Generator().manual_seed(int(seed))) * 0.01
        params = torch.zeros(nw + H * Cp, dtype=torch.float32)
        params[:nw].view(H, Cp, D)[:, :num_classes] = w0
        self.params = params.to(device)
        self.grads = torch.zeros_like(self.params)
        self.momentum_buf = torch.zeros_like(self.params)
        self.weight = self.params[:nw].view(H, Cp, D)
        self.bias = self.params[nw:].view(H, Cp)
        self.weight_bf16 = ops.cast_bf16(self.params[:nw].view(H * Cp, D))
        self.lr = torch.tensor([lr for lr, _ in self.grid], dtype=torch.float32, device=device)
        self.wd = torch.tensor([wd for _, wd in self.grid], dtype=torch.float32, device=device)
        self._logits = None
        self._dlogits = None

    @property
    def device(self):
        return self.params.device

    def _buffers(self, rows, want_grad):
        n = self.H * self.Cp
        if self._logits is None or self._logits.shape[0] < rows:
            self._logits = torch.empty((rows, n), dtype=torch.float32, device=self.device)
        if want_grad and (self._dlogits is None or self._dlogits.shape[0] < rows):
            self._dlogits = torch.empty((rows, n), dtype=torch.bfloat16, device=self.device)
        return self._logits[:rows], (self._dlogits[:rows] if want_grad else None)

    def _check_batch(self, feats, labels):
        _cuda(feats, "feats"); _cuda(labels, "labels")
        if feats.dtype != torch.bfloat16 or feats.dim() != 2 or feats.shape[1] != self.D or not feats.is_contiguous():
            raise ValueError("feats must be a contiguous bf16 [B, %d] matrix, got %s %s"
                             % (self.D, feats.dtype, tuple(feats.shape)))
        if labels.dtype != torch.int64 or tuple(labels.shape) != (feats.shape[0],) or not labels.is_contiguous():
            raise ValueError("labels must be a contiguous int64 [%d] vector" % feats.shape[0])
        if feats.device != self.device or labels.device != self.device:
            raise ValueError("feats / labels must be on %s" % self.device)

    def logits(self, feats, out=None):
        """fp32 [B, H * Cp] logits of every head (head h in columns h * Cp .. h * Cp + C - 1)."""
        return ops.linear_fprop(feats, self.weight_bf16, bias=self.params[self.H * self.Cp * self.D:], out_fp32=True,
                                out=out)

    def step(self, feats, labels, lr_scale):
        """One SGD step of every head on bf16 feats [B, D] and int64 labels [B] (rows labelled outside [0, C) are ignored), with
        head h's learning rate fp32(lr_h * lr_scale).  Returns the per-head mean loss before the step, fp32 [H] on the
        device; nothing waits for the GPU."""
        self._check_batch(feats, labels)
        b = feats.shape[0]
        logits, dlogits = self._buffers(b, True)
        self.logits(feats, out=logits)
        loss = torch.zeros(self.H, dtype=torch.float32, device=self.device)
        multihead_ce(logits, labels, self.H, self.C, dlogits=dlogits, loss_sum=loss)
        nw = self.H * self.Cp * self.D
        ops.linear_wgrad(feats, dlogits, self.grads[:nw].view(self.H * self.Cp, self.D))
        ops.col_sum(dlogits, self.grads[nw:])
        self.apply_gradients(lr_scale)
        return loss.div_(b)

    def apply_gradients(self, lr_scale):
        """The Nesterov-SGD update of every head from ``grads`` (byol_linprobe_sgd), which it leaves zeroed; refreshes
        ``weight_bf16``."""
        check(lib.byol_linprobe_sgd(self.params.data_ptr(), self.grads.data_ptr(), self.momentum_buf.data_ptr(),
                                    self.weight_bf16.data_ptr(), self.lr.data_ptr(), self.wd.data_ptr(),
                                    float(np.float32(lr_scale)), self.momentum, self.H, self.C, self.Cp, self.D,
                                    ops._stream()), "byol_linprobe_sgd")

    def finite_heads(self):
        """bool numpy [H]: True where every weight and bias of the head is finite (waits for the GPU)."""
        ok = torch.isfinite(self.weight[:, :self.C]).flatten(1).all(1) & torch.isfinite(self.bias[:, :self.C]).all(1)
        return ok.cpu().numpy()

    def evaluate(self, feats, labels):
        """Per-head top-1 / top-5 hit counts, int64 [H, 2] on the device, of bf16 feats [N, D] with int64 labels [N]
        (top-k: fewer than k other logits strictly larger than the label's or NaN; a NaN label logit, or a label outside
        [0, C), is a miss)."""
        self._check_batch(feats, labels)
        hits = torch.zeros((self.H, 2), dtype=torch.int64, device=self.device)
        n = feats.shape[0]
        for r0 in range(0, n, EVAL_ROWS):
            rows = min(EVAL_ROWS, n - r0)
            logits, _ = self._buffers(rows, False)
            self.logits(feats[r0:r0 + rows], out=logits)
            multihead_ce(logits, labels[r0:r0 + rows], self.H, self.C, hits=hits)
        return hits


def _fit(heads, epochs, steps_per_epoch, batches):
    """Runs epochs x steps_per_epoch steps; batches(epoch) yields that epoch's (bf16 feats, labels)."""
    total = epochs * steps_per_epoch
    t = 0
    for epoch in range(epochs):
        for feats, labels in batches(epoch):
            heads.step(feats, labels, cosine_factor(t, total))
            t += 1


def select_heads(heads, val_feats, val_labels):
    """Validation accuracy of every head of `heads` and the selected one: {"best": head index, "lr", "weight_decay",
    "val_top1", "val_top5", "heads": [{"lr", "weight_decay", "val_top1", "val_top5", "finite"}, ...]} (accuracies in
    %).  "finite" is False for a head whose weights or biases hold a NaN or an infinity; such a head is not selected
    (ValueError when no head is finite)."""
    val = heads.evaluate(val_feats, val_labels).cpu().numpy()
    finite = heads.finite_heads()
    n = val_feats.shape[0]
    entries = [{"lr": lr, "weight_decay": wd, "val_top1": 100.0 * float(v[0]) / n, "val_top5": 100.0 * float(v[1]) / n,
                "finite": bool(f)} for (lr, wd), v, f in zip(heads.grid, val, finite)]
    best = select_head(val[:, 0], finite)
    return {"best": best, "lr": heads.grid[best][0], "weight_decay": heads.grid[best][1],
            "val_top1": entries[best]["val_top1"], "val_top5": entries[best]["val_top5"], "heads": entries}


def _check_features(feats, labels, name, d=None):
    """Shape and dtype of one (features, labels) pair, no device access; returns (rows, D)."""
    if not isinstance(feats, torch.Tensor) or not isinstance(labels, torch.Tensor):
        raise TypeError("%s features and labels must be torch.Tensors" % name)
    if feats.dim() != 2 or feats.dtype not in (torch.bfloat16, torch.float32):
        raise ValueError("%s features must be a bf16 or fp32 [rows, D] matrix, got %s %s"
                         % (name, feats.dtype, tuple(feats.shape)))
    n, dim = feats.shape
    if dim == 0 or dim % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % dim)
    if d is not None and dim != d:
        raise ValueError("%s features have width %d, the training features %d" % (name, dim, d))
    if labels.dtype != torch.int64 or tuple(labels.shape) != (n,):
        raise ValueError("%s labels must be int64 [%d], got %s %s" % (name, n, labels.dtype, tuple(labels.shape)))
    return n, dim


def _check_labels(labels, num_classes, name):
    if labels.numel():
        lo, hi = (int(v) for v in torch.aminmax(labels))
        if lo < 0 or hi >= num_classes:
            raise ValueError("%s labels span [%d, %d], outside [0, %d)" % (name, lo, hi, num_classes))


def _bf16(feats):
    return feats.contiguous() if feats.dtype == torch.bfloat16 else ops.cast_bf16(feats.contiguous())


def train_linear_heads(train_feats, train_labels, val_feats, val_labels, num_classes, epochs=80, batch_size=1024,
                       lrs=DEFAULT_LRS, weight_decays=(0.0,), momentum=0.9, seed=0):
    """Trains a ``LinearHeads`` grid on cached features and selects on the validation features:
    (heads, ``select_heads``'s report).

    Features: bf16 or fp32 (cast to bf16 once) [rows, D] CUDA matrices, D a multiple of 64; labels int64 in
    [0, num_classes).  Each epoch is a permutation of the training rows seeded from (seed, epoch), cut into full
    batches of batch_size (the remainder is dropped, as ImageFolderLoader does).  Head h's learning rate decays from
    lrs[...] to 0 by a cosine over all steps, with no warm-up; the factor is computed in fp64 on the host and rounded
    to fp32 once per step.  The selected head has the best validation top-1, ties going to the earlier head; a head
    whose weights went non-finite is never selected, and ValueError says so when every head did (non-finite features
    make every head diverge)."""
    lrs, weight_decays = check_hyperparameters(lrs, weight_decays, momentum)
    _positive_int(epochs, "epochs")
    _positive_int(batch_size, "batch_size")
    if not isinstance(num_classes, int) or isinstance(num_classes, bool) or num_classes < 2:
        raise ValueError("num_classes must be an int >= 2, got %r" % (num_classes,))
    n, d = _check_features(train_feats, train_labels, "training")
    nv, _ = _check_features(val_feats, val_labels, "validation", d)
    if n < batch_size:
        raise ValueError("%d training rows cannot fill one batch of %d" % (n, batch_size))
    if nv < 1:
        raise ValueError("the validation split is empty")
    for t, name in ((train_feats, "train_feats"), (train_labels, "train_labels"), (val_feats, "val_feats"),
                    (val_labels, "val_labels")):
        _cuda(t, name)
    if len({t.device for t in (train_feats, train_labels, val_feats, val_labels)}) != 1:
        raise ValueError("features and labels must be on one device")
    _check_labels(train_labels, num_classes, "training")
    _check_labels(val_labels, num_classes, "validation")
    train_feats, val_feats = _bf16(train_feats), _bf16(val_feats)
    train_labels, val_labels = train_labels.contiguous(), val_labels.contiguous()
    with torch.cuda.device(train_feats.device):
        heads = LinearHeads(d, num_classes, lrs, weight_decays, momentum, seed, train_feats.device)
        steps = n // batch_size

        def batches(epoch):
            perm = torch.from_numpy(np.random.default_rng([int(seed), epoch]).permutation(n)).to(train_feats.device)
            for i in range(steps):
                idx = perm[i * batch_size:(i + 1) * batch_size]
                yield train_feats.index_select(0, idx), train_labels.index_select(0, idx)

        _fit(heads, epochs, steps, batches)
        return heads, select_heads(heads, val_feats, val_labels)


def _extract(model, samples, batch_size, augment, network, fp32=False):
    """(bf16 features [len(samples), D], int64 labels) of one pass over `samples` in file order, view 1 (the
    eval transform of `augment`, as knn._extract); fp32=True keeps the fp32 representations."""
    from .data import ImageFolderLoader
    feats, labels = [], []
    for img, _, lab in ImageFolderLoader(samples, batch_size, augment, train=False):
        rep = model.representations(img, network)
        feats.append(rep if fp32 else ops.cast_bf16(rep))
        labels.append(lab)
    return torch.cat(feats), torch.cat(labels)


def linear_accuracy(model, loader, epochs=80, batch_size=1024, lrs=DEFAULT_LRS, weight_decays=(0.0,), momentum=0.9,
                    augment=False, network="online", seed=0):
    """Linear-evaluation top-1 / top-5 accuracy (%) of `model`'s frozen encoder on the test split of `loader` (the
    ``ImageFolderTwoView`` from ``byol_b200.data.get_loader``):
    {"linear_top1", "linear_top5", "lr", "weight_decay", "heads": [{"lr", "weight_decay", "val_top1", "val_top5",
    "finite", "test_top1", "test_top5"}, ...]}.

    Selection split: ``loader.valid_loader`` when it holds images; otherwise a seeded hold-out of
    max(1, min(10 000, N // 10)) training images (``holdout_split``), which are then not trained on.  The reported
    head is the one with the best validation top-1 (ties: the earlier head) among the heads with finite weights (a
    NaN logit never counts as a hit; ValueError if every head diverged); every head's validation and test accuracy
    is returned as well.  Validation and test images come from the loader's eval transform
    (``loader.test_loader.augment``, as in ``knn_accuracy``), and their features from
    ``model.representations(images, network)``.  By default that transform resizes the whole image to R x R; for the
    paper's protocol, the shorter side resized to 256 (at R = 224) by bicubic and the centre R x R crop, build the
    loader with ``get_loader(..., eval_transform="byol")``.

    augment=False (the default): the training features are extracted once the same way, kept on the device as bf16
    (5.25 GB for ImageNet-1k at D = 2048) and trained on for `epochs` (``train_linear_heads``).
    augment=True (the paper's protocol): every epoch reads the training images again through an ``ImageFolderLoader``
    whose augmentation is only the random resized crop and flip, one view per image.  That mode is bound by the JPEG
    decode, not by the heads: 773-907 images/s for decode + crop / flip + ResNet-50 @224 representations on one
    H100 80GB HBM3 (700 W), about 27 minutes per ImageNet-1k epoch (README).

    The model is not changed (running statistics, weights, the EMA and its step, captured CUDA graphs).  Under
    torch.distributed it runs on the calling rank alone, with no collective."""
    lrs, weight_decays = check_hyperparameters(lrs, weight_decays, momentum)
    _positive_int(epochs, "epochs")
    _positive_int(batch_size, "batch_size")
    if network not in ("online", "target"):
        raise ValueError("network must be 'online' or 'target', got %r" % (network,))
    d = int(model.base_network_output_size)
    if d < 1 or d % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % d)
    num_classes = int(loader.output_size)
    if num_classes < 2:
        raise ValueError("linear evaluation needs at least 2 classes, got %d" % num_classes)
    train_samples = loader.train_loader.samples
    if loader.valid_loader is not None and len(loader.valid_loader.samples) > 0:
        fit, val = list(train_samples), list(loader.valid_loader.samples)
    else:
        fit_idx, val_idx = holdout_split(len(train_samples), seed)
        fit, val = [train_samples[i] for i in fit_idx], [train_samples[i] for i in val_idx]
    test = list(loader.test_loader.samples)
    if not test:
        raise ValueError("linear_accuracy: the test split is empty")
    if len(fit) < batch_size:
        raise ValueError("%d training images cannot fill one batch of %d" % (len(fit), batch_size))
    resize, ext_bs = loader.test_loader.augment, loader.test_loader.batch_size
    val_feats, val_labels = _extract(model, val, ext_bs, resize, network)
    test_feats, test_labels = _extract(model, test, ext_bs, resize, network)
    if not augment:
        train_feats, train_labels = _extract(model, fit, ext_bs, resize, network)
        heads, report = train_linear_heads(train_feats, train_labels, val_feats, val_labels, num_classes, epochs,
                                           batch_size, lrs, weight_decays, momentum, seed)
        train_feats = train_labels = None
    else:
        from .augment import TwoViewAugment
        from .data import ImageFolderLoader
        crop = TwoViewAugment(image_size=resize.R, seed=seed, p_jitter=0.0, p_gray=0.0, p_blur=0.0, blur=False)
        train = ImageFolderLoader(fit, batch_size, crop, train=True, seed=seed, workers=loader.train_loader.workers)
        heads = LinearHeads(d, num_classes, lrs, weight_decays, momentum, seed)

        def batches(epoch):
            train.set_epoch(epoch)
            for view1, _, lab in train:
                yield ops.cast_bf16(model.representations(view1, network)), lab

        _fit(heads, epochs, len(train), batches)
        report = select_heads(heads, val_feats, val_labels)
    test_hits = heads.evaluate(test_feats, test_labels).cpu().numpy()
    nt = test_feats.shape[0]
    for entry, v in zip(report["heads"], test_hits):
        entry["test_top1"] = 100.0 * float(v[0]) / nt
        entry["test_top5"] = 100.0 * float(v[1]) / nt
    best = report["heads"][report["best"]]
    return {"linear_top1": best["test_top1"], "linear_top5": best["test_top5"], "lr": best["lr"],
            "weight_decay": best["weight_decay"], "heads": report["heads"]}
