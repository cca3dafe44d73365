"""Semi-supervised evaluation (the BYOL paper's 1 % / 10 % label tables): copies of the pretrained encoder are
fine-tuned, each with a fresh linear classifier, on a labelled subset of the training images; the run to report is
chosen on held-out images and scored on the test split.

    from byol_b200.finetune import finetune_accuracy
    acc = finetune_accuracy(model, loader, label_fraction=0.01)
    # {"finetune_top1": %, "finetune_top5": %, "lr", "weight_decay", "labelled": n, "runs": [...]}

H = len(lrs) * len(weight_decays) runs, one per (lr, weight decay) pair in lr-major order (``linear_eval.head_grid``).
Each run (``FineTune``) owns an independent copy of the encoder and trains it with one-lane supervised steps of the
engine: the train-mode forward of one lane stopping after the average pool, the classifier (``ops.linear_fprop``, the
cross-entropy of ``byol_linprobe_ce`` with one head, ``linear_wgrad`` / ``col_sum`` for its gradient, ``linear_dgrad``
for the representation's), the engine's encoder backward (``Engine.backward_online``) and a Nesterov-SGD kernel over
the encoder and the classifier (``byol_sgd_nesterov_step``).  Every reduction is fixed-point, so a run gives the same
bits every time, alone or in a sweep.  The step stays eager (no CUDA graph): it is bound by the JPEG decode, and a
graph per run would pin one activation pool per run.

Protocol (this module's choices):

* labelled subset: ``label_fraction`` f in (0, 1] draws k_c = max(1, floor(f n_c + 0.5)) images of each class c
  (seeded); or ``subset`` names the training images by file base name, as SimCLR's ``1percent.txt`` /
  ``10percent.txt`` do.  Exactly one of the two must be given;
* selection split: ``valid/`` when it holds images, else a seeded hold-out of max(1, min(10 000, M // 10)) of the M
  training images outside the labelled subset;
* training: every epoch a (seed, epoch) permutation of the labelled images in full batches, random resized crop + flip
  only (as ``linear_accuracy(augment=True)``); each decoded batch feeds all H runs one after another, so the decode is
  paid once per batch.  Nesterov SGD, momentum 0.9, the weight decay on every fine-tuned parameter, the lr decayed to 0
  by a cosine over all steps with no warm-up; BatchNorm in train mode (batch statistics, running statistics updated once
  per step);
* evaluation: validation and test images through the loader's eval transform (as k-NN and linear evaluation:
  the whole image resized to R x R by default; ``get_loader(..., eval_transform="byol")`` gives the paper's resize to
  (8R + 3) // 7 = 256 at R = 224 and centre R x R crop), features from the copy's ``representations()`` (eval-mode
  BatchNorm), then its classifier;
* selection: the best validation top-1, ties to the earlier run; a run whose parameters went non-finite is never chosen.
"""
import math
import os

import numpy as np
import torch

from . import ops
from .lars import chunk_table
from .linear_eval import (HOLDOUT_MAX, _cuda, _positive_int, check_hyperparameters, cosine_factor, head_grid,
                          multihead_ce, select_head)

DEFAULT_LRS = (0.1, 0.05, 0.02, 0.01, 0.005)


def label_subset(samples, num_classes, label_fraction=None, subset=None, seed=0):
    """Sorted int64 indices into `samples` ([(path, class index)], the training split) of the labelled images.

    label_fraction f in (0, 1]: from each class c with n_c images, k_c = max(1, floor(f * n_c + 0.5)) drawn by a
    generator seeded from `seed`.  subset: an iterable of file base names (e.g. the lines of SimCLR's 1percent.txt;
    surrounding white space and empty names are ignored); ValueError for a name that matches no training image or more
    than one.  Exactly one of the two must be given (ValueError otherwise)."""
    if (label_fraction is None) == (subset is None):
        raise ValueError("give exactly one of label_fraction and subset (the paper uses label_fraction=0.01 and 0.1)")
    if label_fraction is not None:
        if isinstance(label_fraction, bool) or not isinstance(label_fraction, (int, float, np.floating)) or \
                not (0.0 < float(label_fraction) <= 1.0):
            raise ValueError("label_fraction must be a number in (0, 1], got %r" % (label_fraction,))
        f = float(label_fraction)
        labels = np.array([c for _, c in samples], dtype=np.int64)
        rng = np.random.default_rng([int(seed), 0x6c6162])
        picked = []
        for c in range(num_classes):
            idx = np.flatnonzero(labels == c)
            if idx.size:
                k = min(idx.size, max(1, int(math.floor(f * idx.size + 0.5))))
                picked.append(rng.permutation(idx)[:k])
        return np.sort(np.concatenate(picked)) if picked else np.zeros(0, dtype=np.int64)
    if isinstance(subset, (str, bytes)):
        raise ValueError("subset must be an iterable of file names, not a single string")
    where = {}
    for i, (path, _) in enumerate(samples):
        where.setdefault(os.path.basename(path), []).append(i)
    picked = set()
    for name in subset:
        name = str(name).strip()
        if not name:
            continue
        found = where.get(name, [])
        if not found:
            raise ValueError("subset: %r matches no training image" % name)
        if len(found) > 1:
            raise ValueError("subset: %r matches %d training images (%s)" %
                             (name, len(found), ", ".join(samples[i][0] for i in found[:3])))
        picked.add(found[0])
    if not picked:
        raise ValueError("subset names no image")
    return np.array(sorted(picked), dtype=np.int64)


def holdout_indices(n, labelled, seed):
    """Sorted int64 indices of the selection hold-out when there is no ``valid/``: a seeded draw of
    max(1, min(10 000, M // 10)) of the M training images outside `labelled`; ValueError when M = 0."""
    rest = np.setdiff1d(np.arange(n, dtype=np.int64), np.asarray(labelled, dtype=np.int64))
    if rest.size == 0:
        raise ValueError("every training image is labelled and there is no valid/ split: no image is left to select "
                         "the run on")
    k = max(1, min(HOLDOUT_MAX, rest.size // 10))
    return np.sort(np.random.default_rng([int(seed), 0x686f6c]).permutation(rest)[:k])


def _check_network(network):
    if network not in ("online", "target"):
        raise ValueError("network must be 'online' or 'target', got %r" % (network,))


def _model_device(model):
    dev = next(model.parameters()).device
    if dev.type != "cuda":
        raise RuntimeError("byol_b200.finetune: the model must be on a CUDA device (no CPU path)")
    return dev


class FineTune(object):
    """One fine-tuned copy of `model`'s encoder (online weights, or ``target_network.mean`` with network="target",
    and `model`'s BatchNorm running statistics) with a fresh linear classifier over `num_classes` classes (weights
    N(0, 0.01^2) from a generator seeded with `seed`, bias 0), trained by Nesterov SGD with learning rate `lr`, weight
    decay `weight_decay` on every fine-tuned parameter and `momentum`.

    The copy (``self.model``) is a new ``BYOL`` of `model`'s arch and layer widths with ``classifier_output_size =
    num_classes``; its projector and predictor never run.  It always runs precision="bf16", whatever `model`'s
    precision is.  `model` itself is only read."""

    def __init__(self, model, num_classes, lr, weight_decay=0.0, momentum=0.9, network="online", seed=0):
        from .model import BYOL
        (lr,), (weight_decay,) = check_hyperparameters((lr,), (weight_decay,), momentum)
        if not isinstance(num_classes, int) or isinstance(num_classes, bool) or num_classes < 2:
            raise ValueError("num_classes must be an int >= 2, got %r" % (num_classes,))
        _check_network(network)
        dev = _model_device(model)
        d = int(model.base_network_output_size)
        if d < 1 or d % 64 != 0:
            raise ValueError("the feature width D=%d must be a positive multiple of 64" % d)
        self.C, self.Cp, self.D = num_classes, (num_classes + 7) // 8 * 8, d
        self.lr, self.weight_decay, self.momentum = lr, weight_decay, float(momentum)
        with torch.random.fork_rng(devices=[]):           # the copy's (discarded) initialisation draws from torch's RNG
            copy = BYOL(d, model.head[-1].out_features, num_classes, 1, arch=model.arch,
                        head_latent_size=model.head[0].out_features, norm=model.norm)
        self.model = copy.to(dev).train()
        eng = self.eng = copy._engine
        eng.flatten()
        eng.build_plan()
        with torch.no_grad():
            src = list(model.base_network.parameters())
            n_enc = sum(p.numel() for p in src)
            if network == "target":
                eng.theta[:n_enc].copy_(model.target_network.mean[:n_enc])
            else:
                eng.theta[:n_enc].copy_(torch.cat([p.detach().reshape(-1) for p in src]))
            for dst, b in zip(copy.base_network.buffers(), model.base_network.buffers()):
                dst.copy_(b)
            u = eng.cls
            w0 = torch.randn(num_classes, d, generator=torch.Generator().manual_seed(int(seed))) * 0.01
            eng.theta[u.w_off:u.w_off + u.w_numel].copy_(w0.reshape(-1))
            eng.theta[u.b_off:u.b_off + num_classes].zero_()
        # the fine-tuned ranges of the flat buffers: the encoder prefix and the classifier (weight, then bias)
        assert u.b_off == u.w_off + u.w_numel
        n_cls = u.w_numel + num_classes
        self.ranges = [(0, n_enc), (u.w_off, n_cls)]
        # momentum buffers with the 16-byte phase of their range in theta, so the update runs on float4
        self.momentum_buf = [torch.zeros(n + 3, dtype=torch.float32, device=dev)[off % 4:off % 4 + n]
                             for off, n in self.ranges]
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device=dev)
        self.table = chunk_table([n for _, n in self.ranges], dev)
        self.table.update({
            "p_ptrs": i64([eng.theta[off:].data_ptr() for off, _ in self.ranges]),
            "g_ptrs": i64([eng.grad[off:].data_ptr() for off, _ in self.ranges]),
            "m_ptrs": i64([m.data_ptr() for m in self.momentum_buf]),
            "lr": torch.full((2,), lr, dtype=torch.float32, device=dev),
            "wd": torch.full((2,), weight_decay, dtype=torch.float32, device=dev)})
        # the classifier's tensor-core layouts with the classes padded to Cp (zero rows): fprop [Cp, D] for [B, Cp]
        # logits (byol_linprobe_ce's layout) and dgrad [D, Cp] for d_rep = dlogits @ W, made from a padded fp32 copy
        self._stage = torch.zeros((self.Cp, d), dtype=torch.float32, device=dev)
        self._bias = torch.zeros(self.Cp, dtype=torch.float32, device=dev)
        self._wf = torch.empty((self.Cp, d), dtype=torch.bfloat16, device=dev)
        self._wd = torch.empty((d, self.Cp), dtype=torch.bfloat16, device=dev)

    @property
    def device(self):
        return self.eng.theta.device

    @property
    def classifier_weight(self):
        u = self.eng.cls
        return self.eng.theta[u.w_off:u.w_off + u.w_numel].view(self.C, self.D)

    @property
    def classifier_bias(self):
        u = self.eng.cls
        return self.eng.theta[u.b_off:u.b_off + self.C]

    def _prep_classifier(self):
        self._stage[:self.C].copy_(self.classifier_weight)
        self._bias[:self.C].copy_(self.classifier_bias)
        ops.prep_weight(self._stage, cpad=self.D, want_dgrad=True, out_f=self._wf, out_d=self._wd)

    def _check_batch(self, images, labels):
        _cuda(images, "images"); _cuda(labels, "labels")
        if images.dtype != torch.float32 or images.dim() != 4 or images.shape[0] < 1 or not images.is_contiguous():
            raise ValueError("images must be a contiguous fp32 [B, C, H, W] batch, got %s %s"
                             % (images.dtype, tuple(images.shape)))
        if labels.dtype != torch.int64 or tuple(labels.shape) != (images.shape[0],) or not labels.is_contiguous():
            raise ValueError("labels must be a contiguous int64 [%d] vector" % images.shape[0])
        if images.device != self.device or labels.device != self.device:
            raise ValueError("images / labels must be on %s" % self.device)

    def gradients(self, images, labels):
        """The gradient of the mean cross-entropy of one train-mode step on fp32 NCHW `images` (values in [0, 1]) and
        int64 `labels`, accumulated into the copy's flat gradient (``self.eng.grad``: encoder and classifier).  Updates
        the copy's BatchNorm running statistics and ``num_batches_tracked``.  Returns (the summed loss, fp32 [1];
        d_rep, the bf16 [B, D] gradient of the representation that entered the encoder's backward pass); nothing
        waits for the GPU."""
        self._check_batch(images, labels)
        eng, u = self.eng, self.eng.cls
        eng.prep_weights(eng.theta, eng.w_online, want_dgrad=True)
        self._prep_classifier()
        saved = {}
        _, reps_b = eng.forward_lanes([images], [(eng.theta, eng.w_online, saved)], True, reps_only=True)
        rep = reps_b[0]
        b = rep.shape[0]
        logits = ops.linear_fprop(rep, self._wf, bias=self._bias, out_fp32=True)
        dlogits = torch.empty((b, self.Cp), dtype=torch.bfloat16, device=self.device)
        loss = torch.zeros(1, dtype=torch.float32, device=self.device)
        multihead_ce(logits, labels, 1, self.C, dlogits=dlogits, loss_sum=loss)
        ops.col_sum(dlogits[:, :self.C], eng._gview(u.b_off, self.C))
        eng._wgrad(u, [rep], [dlogits])                  # dW on the side stream; the backward below joins it
        d_rep = ops.linear_dgrad(dlogits, self._wd)
        # one lane on this stream; notify=False: no flat-gradient all-reduce, this copy is the calling rank's own
        eng.backward_online([saved], [d_rep], [None], [None], notify=False)
        eng._join_side_stream()
        return loss, d_rep

    def apply_gradients(self, lr_scale):
        """Nesterov-SGD update of the encoder and the classifier from the flat gradient, with learning rate
        fp32(lr * lr_scale); leaves the gradient zeroed."""
        ops.sgd_nesterov_step(self.table, float(np.float32(lr_scale)), self.momentum)

    def step(self, images, labels, lr_scale):
        """One training step (``gradients`` + ``apply_gradients``).  Returns the mean loss before the step, fp32 [1]
        on the device; nothing waits for the GPU."""
        loss, _ = self.gradients(images, labels)
        self.apply_gradients(lr_scale)
        return loss.div_(images.shape[0])

    def evaluate(self, images, labels, hits=None):
        """Top-1 / top-5 hit counts, int64 [1, 2] on the device (added to `hits` when given), of fp32 NCHW `images`
        with int64 `labels`: the copy's eval-mode representations, then its classifier (a NaN label logit, or a label
        outside [0, C), is a miss)."""
        self._check_batch(images, labels)
        if hits is None:
            hits = torch.zeros((1, 2), dtype=torch.int64, device=self.device)
        feats = ops.cast_bf16(self.model.representations(images))
        self._prep_classifier()
        logits = ops.linear_fprop(feats, self._wf, bias=self._bias, out_fp32=True)
        multihead_ce(logits, labels, 1, self.C, hits=hits)
        return hits

    def finite(self):
        """True when every fine-tuned parameter (encoder and classifier) is finite (waits for the GPU)."""
        th = self.eng.theta
        return bool(all(torch.isfinite(th[off:off + n]).all() for off, n in self.ranges))


def _split_hits(runs, samples, loader):
    """int64 numpy [H, 2] top-1 / top-5 hits of every run over `samples`, each batch decoded once for all runs."""
    from .data import ImageFolderLoader
    hits = [torch.zeros((1, 2), dtype=torch.int64, device=r.device) for r in runs]
    for img, _, lab in ImageFolderLoader(samples, loader.test_loader.batch_size, loader.test_loader.augment,
                                         train=False, workers=loader.test_loader.workers):
        for r, h in zip(runs, hits):
            r.evaluate(img, lab, h)
    return torch.cat(hits).cpu().numpy()


def finetune_accuracy(model, loader, label_fraction=None, subset=None, epochs=30, batch_size=1024, lrs=DEFAULT_LRS,
                      weight_decays=(0.0,), momentum=0.9, network="online", seed=0):
    """Semi-supervised top-1 / top-5 accuracy (%) on the test split of `loader` (the ``ImageFolderTwoView`` from
    ``byol_b200.data.get_loader``) of `model`'s encoder fine-tuned on a labelled subset of the training images (see the
    module docstring for the protocol):
    {"finetune_top1", "finetune_top5", "lr", "weight_decay", "labelled": the number of labelled images,
    "runs": [{"lr", "weight_decay", "val_top1", "val_top5", "finite", "test_top1", "test_top5"}, ...]} in lr-major
    order.  Exactly one of `label_fraction` (the paper: 0.01 or 0.1) and `subset` (training-image base names) is
    given.  ValueError when every run diverged.

    Validation and test images come from the loader's eval transform (``loader.test_loader.augment``): the whole
    image resized to R x R by default; ``get_loader(..., eval_transform="byol")`` gives the paper's protocol, the
    shorter side resized to 256 (at R = 224) by bicubic and the centre R x R crop.

    The copies run precision="bf16" whatever `model`'s precision is.  `model` is not changed (weights, running
    statistics, num_batches_tracked, the EMA and its step, captured CUDA graphs).  Under torch.distributed it runs on
    the calling rank alone, with no collective.  Arguments are checked before any device work."""
    lrs, weight_decays = check_hyperparameters(lrs, weight_decays, momentum)
    _positive_int(epochs, "epochs")
    _positive_int(batch_size, "batch_size")
    _check_network(network)
    d = int(model.base_network_output_size)
    if d < 1 or d % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % d)
    num_classes = int(loader.output_size)
    if num_classes < 2:
        raise ValueError("fine-tuning needs at least 2 classes, got %d" % num_classes)
    train_samples = list(loader.train_loader.samples)
    labelled = label_subset(train_samples, num_classes, label_fraction, subset, seed)
    if loader.valid_loader is not None and len(loader.valid_loader.samples) > 0:
        val = list(loader.valid_loader.samples)
    else:
        val = [train_samples[i] for i in holdout_indices(len(train_samples), labelled, seed)]
    test = list(loader.test_loader.samples)
    if not test:
        raise ValueError("finetune_accuracy: the test split is empty")
    if len(labelled) < batch_size:
        raise ValueError("%d labelled images cannot fill one batch of %d" % (len(labelled), batch_size))
    dev = _model_device(model)

    from .augment import TwoViewAugment
    from .data import ImageFolderLoader
    with torch.cuda.device(dev):
        grid = head_grid(lrs, weight_decays)
        runs = [FineTune(model, num_classes, lr, wd, momentum, network, seed) for lr, wd in grid]
        crop = TwoViewAugment(image_size=loader.test_loader.augment.R, seed=seed, p_jitter=0.0, p_gray=0.0,
                              p_blur=0.0, blur=False)
        train = ImageFolderLoader([train_samples[i] for i in labelled], batch_size, crop, train=True, seed=seed,
                                  workers=loader.train_loader.workers)
        total, t = epochs * len(train), 0
        for epoch in range(epochs):
            train.set_epoch(epoch)
            for view1, _, lab in train:
                scale = cosine_factor(t, total)
                for r in runs:
                    r.step(view1, lab, scale)
                t += 1
        val_hits = _split_hits(runs, val, loader)
        test_hits = _split_hits(runs, test, loader)
        finite = [r.finite() for r in runs]
    best = select_head(val_hits[:, 0], finite)
    nv, nt = len(val), len(test)
    entries = [{"lr": lr, "weight_decay": wd, "val_top1": 100.0 * float(v[0]) / nv, "val_top5": 100.0 * float(v[1]) / nv,
                "finite": bool(f), "test_top1": 100.0 * float(s[0]) / nt, "test_top5": 100.0 * float(s[1]) / nt}
               for (lr, wd), v, f, s in zip(grid, val_hits, finite, test_hits)]
    return {"finetune_top1": entries[best]["test_top1"], "finetune_top5": entries[best]["test_top5"],
            "lr": entries[best]["lr"], "weight_decay": entries[best]["weight_decay"], "labelled": int(len(labelled)),
            "runs": entries}
