"""Transfer linear evaluation (the BYOL paper's Table 3 "Linear evaluation" protocol, after Kornblith et al. 2019): an
L2-regularised multinomial logistic regression on the frozen fp32 features, minimised to convergence by full-batch
L-BFGS, its regularisation strength chosen on a validation split from 45 log-spaced values, then refitted on train +
validation and scored on the test split.

    from byol_b200.logreg import transfer_accuracy
    acc = transfer_accuracy(model, loader)   # {"transfer_accuracy": %, "metric", "l2", "refit": {...}, "heads": [...]}

Head h with strength l2_h minimises f_h(W, b) = (1/N) sum_i CE(softmax(W x_i + b), y_i) + (l2_h / 2) ||W||_F^2 from
W = 0, b = 0 (the bias is not penalised).  All H heads are fitted together (csrc/logreg.cu): their weights are one fp32
[H * Cp, D] matrix (Cp = C rounded up to a multiple of 8) followed by the [H, Cp] biases, so one function evaluation
of every head is, per chunk of at most ``EVAL_ROWS`` rows:

1. ``ops.linear_fprop`` on split-bf16 planes (T = 6, fp32-accurate): the fp32 logits [rows, H * Cp] of every head;
2. ``byol_logreg_ce``: softmax cross-entropy, (softmax - onehot) / N as six bf16 planes, the bias gradient and the
   loss sums (fixed point);
3. ``ops.conv_wgrad_planes`` as a 1x1 convolution: dW += dlogits^T x over the same planes;

then ``byol_logreg_grad`` adds l2_h W and reduces max |g| and ||W||^2 per head.  The features are split into their
planes once (12 D bytes per row) and the weights once per evaluation.  No split-K: a head's logits, loss and gradient do
not depend on the heads beside it.

L-BFGS, one per head (history m = 10): the first direction is -g / ||g||_2, later ones the two-loop recursion scaled by
gamma = s.y / y.y of the newest pair; a pair with s.y <= 1e-10 y.y is not stored.  Backtracking Armijo line search from
t = 1 (c1 = 1e-4, halving).  A head stops when ||g||_inf <= tol (converged), after max_iter iterations, or when no
decrease is found after 40 halvings.  The objective is fp32-accurate, not exact: near the optimum f carries rounding
noise of about 1e-7 relative, and an Armijo test can fail, or pass, on that noise alone.  So a search also fails once
the decrease it asks for, t |g.d|, is below 1e-7 max(1, |f|) (``NOISE``); a failed search (and a direction that is not
a descent direction, which only rounding can produce) ends the head, which counts as converged when its
||g||_inf <= 10 tol.  A stopped head's parameters are never written again.

The host makes the per-head decisions: once per function evaluation it reads 32 bytes per head (the loss sum, max |g|,
||W||^2 and g.d) and uploads the heads' modes and step sizes.  Nothing else synchronises.
"""
import ctypes
import math

import numpy as np
import torch

from . import ops
from ._lib import check, lib
from .linear_eval import EVAL_ROWS, _check_labels, _cuda, _extract, holdout_split, select_head

L2_GRID = np.logspace(-6, 5, 45)
HISTORY = 10
ARMIJO_C1 = 1e-4
MAX_HALVINGS = 40
CURVATURE_EPS = 1e-10
NOISE = 1e-7        # relative rounding noise of the fp32-accurate objective: smaller predicted decreases are not searched
T_PLANES = 6
METRICS = ("top1", "mean_per_class")

# per-head modes of the device kernels (csrc/logreg.cu)
_STOPPED, _SEARCH, _ACCEPT, _START, _FINAL = 0, 1, 2, 3, 4


def _bit(*modes):
    return sum(1 << m for m in modes)


def _padded(num_classes):
    return (num_classes + 7) // 8 * 8


def check_metric(metric):
    if metric not in METRICS:
        raise ValueError("metric must be one of %s, got %r" % (METRICS, metric))
    return metric


def check_l2s(l2s):
    try:
        out = tuple(float(v) for v in l2s)
    except TypeError:
        raise ValueError("l2s must be a sequence of numbers, got %r" % (l2s,))
    if not out:
        raise ValueError("l2s must not be empty")
    for v in out:
        if not (v >= 0.0 and math.isfinite(v)):
            raise ValueError("l2s must be finite and >= 0, got %r" % (l2s,))
    return out


def class_metric(hits, counts, metric):
    """Accuracy (%) of each head from per-(head, class) top-1 hits [H, C] and per-class image counts [C]: "top1" is
    all hits over all images; "mean_per_class" the mean over the classes with at least one image of each class's
    top-1.  ValueError when there is no image."""
    check_metric(metric)
    hits = np.asarray(hits, dtype=np.float64)
    counts = np.asarray(counts, dtype=np.float64)
    if hits.ndim != 2 or counts.shape != (hits.shape[1],):
        raise ValueError("hits must be [H, C] and counts [C]")
    if counts.sum() <= 0:
        raise ValueError("no images to score")
    if metric == "top1":
        return 100.0 * hits.sum(1) / counts.sum()
    present = counts > 0
    return 100.0 * (hits[:, present] / counts[present]).mean(1)


def _check_fp32(feats, labels, name, d=None):
    if not isinstance(feats, torch.Tensor) or not isinstance(labels, torch.Tensor):
        raise TypeError("%s features and labels must be torch.Tensors" % name)
    if feats.dtype != torch.float32 or feats.dim() != 2:
        raise ValueError("%s features must be an fp32 [rows, D] matrix, got %s %s" % (name, feats.dtype,
                                                                                   tuple(feats.shape)))
    n, dim = feats.shape
    if dim == 0 or dim % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % dim)
    if d is not None and dim != d:
        raise ValueError("%s features have width %d, the training features %d" % (name, dim, d))
    if n < 1:
        raise ValueError("the %s split is empty" % name)
    if labels.dtype != torch.int64 or tuple(labels.shape) != (n,):
        raise ValueError("%s labels must be int64 [%d], got %s %s" % (name, n, labels.dtype, tuple(labels.shape)))
    _cuda(feats, "%s features" % name)
    _cuda(labels, "%s labels" % name)
    return n, dim


def _num_classes(num_classes):
    if not isinstance(num_classes, int) or isinstance(num_classes, bool) or num_classes < 2:
        raise ValueError("num_classes must be an int >= 2, got %r" % (num_classes,))
    return num_classes


# ---------------------------------------------------------------------------------------------------------------------
# thin wrappers over csrc/logreg.cu
# ---------------------------------------------------------------------------------------------------------------------
def vec_blocks(num_classes, dim):
    """Blocks per head of the vector kernels (the fixed slicing of a head's Cp * D + Cp parameters)."""
    return int(lib.byol_logreg_vec_blocks(_padded(num_classes), dim))


def logreg_ce(logits, labels, num_heads, num_classes, n_total=None, planes=None, loss_acc=None, bias_acc=None,
              class_hits=None, class_count=None):
    """byol_logreg_ce on fp32 logits [B, >= H * Cp] and int64 labels [B].  Fit: planes bf16 [B, 6 * H * Cp] receive the
    split planes of (softmax - onehot) / n_total; loss_acc int64 [H, 3] and bias_acc int64 [H * Cp, 3] (zeroed
    fixed-point records) the loss and bias-gradient sums.  Evaluation: class_hits int64 [H, Cp] and class_count int64
    [Cp] += top-1 hits per label and images per label."""
    _cuda(logits, "logits"); _cuda(labels, "labels")
    cp = _padded(num_classes)
    b = logits.shape[0]
    if logits.dtype != torch.float32 or logits.dim() != 2 or logits.stride(1) != 1 or \
            logits.shape[1] < num_heads * cp or logits.stride(0) % 4 != 0:
        raise ValueError("logits must be an fp32 [B, >= %d] matrix with unit column stride" % (num_heads * cp))
    if labels.dtype != torch.int64 or tuple(labels.shape) != (b,) or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous int64 [%d] vector" % b)
    for t, name, dtype, shape in ((planes, "planes", torch.bfloat16, (b, T_PLANES * num_heads * cp)),
                                  (loss_acc, "loss_acc", torch.int64, (num_heads, 3)),
                                  (bias_acc, "bias_acc", torch.int64, (num_heads * cp, 3)),
                                  (class_hits, "class_hits", torch.int64, (num_heads, cp)),
                                  (class_count, "class_count", torch.int64, (cp,))):
        if t is not None:
            _cuda(t, name)
            if t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
                raise ValueError("%s must be a contiguous %s %s tensor" % (name, dtype, list(shape)))
    p = lambda t: 0 if t is None else t.data_ptr()
    if b:
        check(lib.byol_logreg_ce(logits.data_ptr(), logits.stride(0), labels.data_ptr(), b, num_heads, num_classes, cp,
                                 float(n_total if n_total is not None else b), p(planes), p(loss_acc), p(bias_acc),
                                 p(class_hits), p(class_count), ops._stream()), "byol_logreg_ce")


class _Solver(object):
    """Device state of H heads over one feature matrix: x (accepted point), g (its gradient), xt / gt (the trial point
    and its gradient), d (the direction), the ring of m + 1 (s, y) slots, and the per-head scalars."""

    def __init__(self, planes, labels, n, d, num_classes, l2s, device):
        self.planes, self.labels, self.N, self.D = planes, labels, n, d
        self.C, self.Cp, self.H = num_classes, _padded(num_classes), len(l2s)
        self.l2 = np.asarray(l2s, dtype=np.float64)
        H, Cp, D, m = self.H, self.Cp, self.D, HISTORY
        self.nw = H * Cp * D
        size = self.nw + H * Cp
        z = lambda *s, **k: torch.zeros(*s, device=device, **k)
        self.x, self.xt, self.g, self.gt, self.d = (z(size) for _ in range(5))
        self.S, self.Y = z((m + 1, size)), z((m + 1, size))
        self.hist = z((H, 2), dtype=torch.int32)
        self.rho = z((H, m + 1), dtype=torch.float64)
        self.gamma = z(H, dtype=torch.float64)
        self.alpha = z((H, m + 1), dtype=torch.float64)
        self.part = z(8 * H * vec_blocks(num_classes, d), dtype=torch.float64)
        self.scalars = z((H, 4), dtype=torch.float64)        # loss sum, max |g|, ||W||^2, g.d
        self.l2_dev = torch.tensor(self.l2, dtype=torch.float64, device=device)
        self.mode = z(H, dtype=torch.int32)
        self.t = z(H, dtype=torch.float64)
        self.fix = z((H + H * Cp, 3), dtype=torch.int64)
        self.w_planes = torch.empty((H * Cp, T_PLANES * D), dtype=torch.bfloat16, device=device)
        rows = min(EVAL_ROWS, n)
        self.logits = torch.empty((rows, H * Cp), dtype=torch.float32, device=device)
        self.dplanes = torch.empty((rows, T_PLANES * H * Cp), dtype=torch.bfloat16, device=device)
        self.evals = 0

    def _shape(self):
        return self.H, self.C, self.Cp, self.D

    def evaluate(self, mask):
        """f and g at xt for every head (the data term of all, l2 term and reductions for the heads in mask)."""
        H, C, Cp, D = self._shape()
        self.fix.zero_()
        self.gt[:self.nw].zero_()
        ops.prep_weight_planes(self.xt[:self.nw].view(H * Cp, D), T_PLANES, D, self.w_planes)
        bias = self.xt[self.nw:]
        dw = self.gt[:self.nw].view(H * Cp, D, 1, 1)
        loss_acc, bias_acc = self.fix[:H], self.fix[H:]
        for r0 in range(0, self.N, EVAL_ROWS):
            rows = min(EVAL_ROWS, self.N - r0)
            xp = self.planes[r0:r0 + rows]
            logits, dp = self.logits[:rows], self.dplanes[:rows]
            ops.linear_fprop(xp, self.w_planes, bias=bias, out_fp32=True, out=logits)
            logreg_ce(logits, self.labels[r0:r0 + rows], H, C, self.N, planes=dp, loss_acc=loss_acc, bias_acc=bias_acc)
            ops.conv_wgrad_planes(xp.view(rows, 1, 1, -1), dp.view(rows, 1, 1, -1), dw, 1, 1, 1, 0, T_PLANES)
        check(lib.byol_logreg_grad(self.xt.data_ptr(), self.gt.data_ptr(), loss_acc.data_ptr(), bias_acc.data_ptr(),
                                   self.l2_dev.data_ptr(), self.mode.data_ptr(), mask, H, C, Cp, D,
                                   self.part.data_ptr(), self.scalars.data_ptr(), 4, ops._stream()),
              "byol_logreg_grad", kernels=2)
        self.evals += 1

    def set_modes(self, mode, t):
        self.mode.copy_(torch.from_numpy(np.asarray(mode, dtype=np.int32)))
        self.t.copy_(torch.from_numpy(np.asarray(t, dtype=np.float64)))

    def step(self):
        """Accept / store pairs, new directions with their g.d, trial points (modes already set)."""
        H, C, Cp, D = self._shape()
        s = ops._stream()
        check(lib.byol_logreg_accept(self.x.data_ptr(), self.xt.data_ptr(), self.g.data_ptr(), self.gt.data_ptr(),
                                     self.S.data_ptr(), self.Y.data_ptr(), self.hist.data_ptr(), self.rho.data_ptr(),
                                     self.gamma.data_ptr(), self.mode.data_ptr(), HISTORY, H, C, Cp, D,
                                     self.part.data_ptr(), s), "byol_logreg_accept", kernels=2)
        new_dir = _bit(_ACCEPT, _START)
        check(lib.byol_logreg_twoloop(self.g.data_ptr(), self.d.data_ptr(), self.S.data_ptr(), self.Y.data_ptr(),
                                      self.hist.data_ptr(), self.rho.data_ptr(), self.gamma.data_ptr(),
                                      self.alpha.data_ptr(), self.part.data_ptr(), self.mode.data_ptr(), new_dir,
                                      HISTORY, H, C, Cp, D, s), "byol_logreg_twoloop", kernels=2 * (HISTORY + 1))
        dots(self, [(self.g, self.d)], new_dir, self.scalars[:, 3:])
        check(lib.byol_logreg_trial(self.x.data_ptr(), self.d.data_ptr(), self.xt.data_ptr(), self.t.data_ptr(),
                                    self.mode.data_ptr(), _bit(_SEARCH, _ACCEPT, _START), H, C, Cp, D, s),
              "byol_logreg_trial")


def dots(solver, pairs, mask, out):
    """out[h, k] (fp64, row pitch out.stride(0)) = head h's part of pairs[k][0] . pairs[k][1] for the heads whose
    mode is in mask (byol_logreg_dots; at most 8 pairs of parameter-shaped fp32 vectors)."""
    k = len(pairs)
    u = (ctypes.c_void_p * k)(*[a.data_ptr() for a, _ in pairs])
    v = (ctypes.c_void_p * k)(*[b.data_ptr() for _, b in pairs])
    check(lib.byol_logreg_dots(u, v, k, solver.mode.data_ptr(), mask, solver.H, solver.C, solver.Cp, solver.D,
                               solver.part.data_ptr(), out.data_ptr(), out.stride(0), ops._stream()),
          "byol_logreg_dots", kernels=2)


def _lbfgs(solver, max_iter, tol):
    """Runs every head to its stop; returns the per-head report list."""
    H = solver.H
    f = np.full(H, np.nan)
    ginf = np.full(H, np.nan)
    t = np.ones(H)
    halvings = np.zeros(H, dtype=np.int64)
    iters = np.zeros(H, dtype=np.int64)
    active = np.ones(H, dtype=bool)
    converged = np.zeros(H, dtype=bool)
    mode = np.full(H, _SEARCH, dtype=np.int32)
    solver.set_modes(mode, t)
    solver.evaluate(_bit(_SEARCH))
    while True:
        sc = solver.scalars.cpu().numpy()           # the one synchronisation per function evaluation
        ft = sc[:, 0] / solver.N + 0.5 * solver.l2 * sc[:, 2]
        gt_inf, gtd = sc[:, 1], sc[:, 3]
        first = np.isnan(f)
        mode[:] = _STOPPED
        for h in np.flatnonzero(active):
            if not first[h] and not gtd[h] < 0.0:
                # not a descent direction (only rounding produces one): ends the head like a failed search
                active[h], converged[h] = False, ginf[h] <= 10.0 * tol
            elif first[h] or (np.isfinite(ft[h]) and ft[h] <= f[h] + ARMIJO_C1 * t[h] * gtd[h]):
                if not first[h]:
                    iters[h] += 1
                f[h], ginf[h] = ft[h], gt_inf[h]
                if not (np.isfinite(ft[h]) and np.isfinite(gt_inf[h])):
                    mode[h], active[h] = _FINAL, False
                elif ginf[h] <= tol:
                    mode[h], active[h], converged[h] = _FINAL, False, True
                elif iters[h] >= max_iter:
                    mode[h], active[h] = _FINAL, False
                else:
                    mode[h], t[h], halvings[h] = (_START if first[h] else _ACCEPT), 1.0, 0
            elif halvings[h] >= MAX_HALVINGS or t[h] * -gtd[h] <= NOISE * max(1.0, abs(f[h])):
                active[h], converged[h] = False, ginf[h] <= 10.0 * tol
            else:
                mode[h], t[h] = _SEARCH, 0.5 * t[h]
                halvings[h] += 1
        solver.set_modes(mode, t)
        solver.step()
        if not active.any():
            break
        solver.evaluate(_bit(_SEARCH, _ACCEPT, _START))
    return [{"iterations": int(iters[h]), "objective": float(f[h]), "converged": bool(converged[h]),
             "grad_inf": float(ginf[h])} for h in range(H)]


class LogisticRegressionFit(object):
    """H fitted heads: ``weight`` fp32 [H, C, D], ``bias`` [H, C] (views of the solver's parameters), ``l2s`` and
    ``heads``: per head {"l2", "iterations", "objective", "converged", "finite"}; ``evaluations`` counts the
    function evaluations of the fit."""

    def __init__(self, solver, l2s, reports):
        H, C, Cp, D = solver.H, solver.C, solver.Cp, solver.D
        self.H, self.C, self.Cp, self.D = H, C, Cp, D
        self.params = solver.x
        self.weight = solver.x[:solver.nw].view(H, Cp, D)[:, :C]
        self.bias = solver.x[solver.nw:].view(H, Cp)[:, :C]
        self.l2s = tuple(l2s)
        finite = (torch.isfinite(self.weight).flatten(1).all(1) & torch.isfinite(self.bias).all(1)).cpu().numpy()
        self.heads = [dict(l2=l, finite=bool(fin), **{k: r[k] for k in ("iterations", "objective", "converged")})
                      for l, r, fin in zip(self.l2s, reports, finite)]
        self.evaluations = solver.evals
        self.rows = solver.N

    def finite_heads(self):
        return np.array([e["finite"] for e in self.heads], dtype=bool)

    def class_hits(self, feats, labels):
        """(top-1 hits per (head, class) int64 [H, C], images per class [C]) of fp32 feats [N, D] and labels [N]
        (a NaN label logit is a miss)."""
        n, _ = _check_fp32(feats, labels, "evaluation", self.D)
        _check_labels(labels, self.C, "evaluation")
        dev = self.params.device
        H, Cp, D = self.H, self.Cp, self.D
        w_planes = torch.empty((H * Cp, T_PLANES * D), dtype=torch.bfloat16, device=dev)
        ops.prep_weight_planes(self.params[:H * Cp * D].view(H * Cp, D), T_PLANES, D, w_planes)
        bias = self.params[H * Cp * D:]
        hits = torch.zeros((H, Cp), dtype=torch.int64, device=dev)
        count = torch.zeros(Cp, dtype=torch.int64, device=dev)
        feats, labels = feats.contiguous(), labels.contiguous()
        for r0 in range(0, n, EVAL_ROWS):
            rows = min(EVAL_ROWS, n - r0)
            xp, _ = ops.split_planes(feats[r0:r0 + rows], T_PLANES)
            logits = ops.linear_fprop(xp, w_planes, bias=bias, out_fp32=True)
            logreg_ce(logits, labels[r0:r0 + rows], H, self.C, class_hits=hits, class_count=count)
        return hits[:, :self.C].cpu().numpy(), count[:self.C].cpu().numpy()

    def evaluate(self, feats, labels, metric="top1"):
        """Accuracy (%) of every head, numpy [H], on fp32 feats [N, D] with int64 labels [N] in [0, C): "top1" or
        "mean_per_class" (``class_metric``)."""
        check_metric(metric)
        return class_metric(*self.class_hits(feats, labels), metric)


def fit_logistic_regression(train_feats, train_labels, num_classes, l2s=L2_GRID, max_iter=1000, tol=1e-5):
    """Fits one head per value of ``l2s`` on fp32 CUDA features [N, D] (D a positive multiple of 64) with int64 labels
    in [0, num_classes), every head from zero, by the batched L-BFGS of this module; returns a
    ``LogisticRegressionFit``.  Every class needs at least one training row (ValueError otherwise: an absent class's
    bias has no finite minimiser)."""
    l2s = check_l2s(l2s)
    num_classes = _num_classes(num_classes)
    if not isinstance(max_iter, int) or isinstance(max_iter, bool) or max_iter < 1:
        raise ValueError("max_iter must be a positive int, got %r" % (max_iter,))
    if not (float(tol) > 0.0 and math.isfinite(float(tol))):
        raise ValueError("tol must be finite and > 0, got %r" % (tol,))
    n, d = _check_fp32(train_feats, train_labels, "training")
    if train_feats.device != train_labels.device:
        raise ValueError("features and labels must be on one device")
    _check_labels(train_labels, num_classes, "training")
    present = torch.bincount(train_labels, minlength=num_classes)
    if int((present == 0).sum()):
        missing = torch.nonzero(present == 0).flatten().tolist()
        raise ValueError("classes %s have no training image: their biases have no finite minimiser" % missing[:10])
    with torch.cuda.device(train_feats.device):
        planes, _ = ops.split_planes(train_feats.contiguous(), T_PLANES)
        solver = _Solver(planes, train_labels.contiguous(), n, d, num_classes, l2s, train_feats.device)
        reports = _lbfgs(solver, max_iter, float(tol))
        return LogisticRegressionFit(solver, l2s, reports)


def transfer_accuracy(model, loader, l2s=L2_GRID, metric="top1", network="online", max_iter=1000, tol=1e-5, seed=0):
    """Transfer linear-evaluation accuracy (%) of `model`'s frozen encoder on the test split of `loader` (the
    ``ImageFolderTwoView`` of ``byol_b200.data.get_loader``; for the paper's preprocessing, build it with
    ``eval_transform="byol_transfer"``):
    {"transfer_accuracy", "metric", "l2", "refit": {"iterations", "objective", "converged"},
     "heads": [{"l2", "val_metric", "finite", "iterations", "objective", "converged"}, ...]}.

    Features: fp32 ``model.representations(images, network)`` of every split, through the loader's eval transform
    (``loader.test_loader.augment``); no augmentation.  One head per value of ``l2s`` (default the paper's 45 values
    from 1e-6 to 1e5) is fitted on the training split and scored on the validation split: ``loader.valid_loader`` when
    it holds images, otherwise a seeded hold-out of the training split (``linear_eval.holdout_split``), which is then
    not fitted on.  The chosen value has the best validation `metric` ("top1", or "mean_per_class": the mean over the
    classes present of each class's top-1), ties going to the earlier value; a head with non-finite weights is never
    chosen (ValueError when none is finite).  One head with the chosen value is then refitted from zero on train +
    validation (the whole training split after a hold-out), and its test `metric` is the result.

    The model is not changed (weights, running statistics, the EMA and its step, captured CUDA graphs).  Under
    torch.distributed it runs on the calling rank alone, with no collective."""
    check_metric(metric)
    l2s = check_l2s(l2s)
    if network not in ("online", "target"):
        raise ValueError("network must be 'online' or 'target', got %r" % (network,))
    d = int(model.base_network_output_size)
    if d < 1 or d % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % d)
    num_classes = int(loader.output_size)
    if num_classes < 2:
        raise ValueError("transfer evaluation needs at least 2 classes, got %d" % num_classes)
    train_samples = list(loader.train_loader.samples)
    if not train_samples:
        raise ValueError("transfer_accuracy: the training split is empty")
    if loader.valid_loader is not None and len(loader.valid_loader.samples) > 0:
        fit, val = train_samples, list(loader.valid_loader.samples)
        refit = fit + val
    else:
        fit_idx, val_idx = holdout_split(len(train_samples), seed)
        fit, val = [train_samples[i] for i in fit_idx], [train_samples[i] for i in val_idx]
        refit = train_samples
    test = list(loader.test_loader.samples)
    if not test:
        raise ValueError("transfer_accuracy: the test split is empty")
    aug, bs = loader.test_loader.augment, loader.test_loader.batch_size
    extract = lambda samples: _extract(model, samples, bs, aug, network, fp32=True)
    fit_x, fit_y = extract(fit)
    val_x, val_y = extract(val)
    sweep = fit_logistic_regression(fit_x, fit_y, num_classes, l2s, max_iter, tol)
    val_metric = sweep.evaluate(val_x, val_y, metric)
    best = select_head(val_metric, sweep.finite_heads())
    heads = [dict(e, val_metric=float(v)) for e, v in zip(sweep.heads, val_metric)]
    sweep = None
    if len(refit) == len(fit) + len(val):
        ref_x, ref_y = torch.cat([fit_x, val_x]), torch.cat([fit_y, val_y])
    else:
        ref_x, ref_y = extract(refit)
    fit_x = val_x = None
    final = fit_logistic_regression(ref_x, ref_y, num_classes, (l2s[best],), max_iter, tol)
    ref_x = ref_y = None
    test_x, test_y = extract(test)
    acc = float(final.evaluate(test_x, test_y, metric)[0])
    r = final.heads[0]
    return {"transfer_accuracy": acc, "metric": metric, "l2": l2s[best],
            "refit": {"iterations": r["iterations"], "objective": r["objective"], "converged": r["converged"],
                      "rows": int(final.rows)},
            "heads": heads}
