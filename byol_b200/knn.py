"""Weighted k-nearest-neighbour evaluation of the learned representation (Wu et al. 2018; k = 20, T = 0.07 as in
DINO): the training split's features are the bank, the test split's the queries, and each query votes with its k most
similar bank rows, weighted by exp(similarity / T).  Nothing is trained and nothing needs tuning, so it is the usual
way to follow self-supervised training.

    from byol_b200.knn import knn_accuracy
    acc = knn_accuracy(model, loader)            # {"knn_top1": %, "knn_top5": %} on the test split

Features are L2-normalised to bf16 rows (``byol_l2_normalize_rows``).  Cosine similarities of Qc queries against Nc
bank rows come from the tensor-core GEMM as an fp32 chunk (``ops.linear_fprop``: the bank rows are the [Cout][K]
weight layout of the convolution kernel); ``byol_knn_topk`` merges each chunk into a running list of the k best
neighbours per query, and ``byol_knn_vote`` turns the lists into the five best classes (csrc/knn.cu).  The order of the
selection is total (similarity descending, then bank index ascending), so the neighbours do not depend on the chunk
sizes.  The similarities are those of the bf16 features accumulated in fp32, not fp32-accurate ones.
"""
import torch

from . import ops
from ._lib import check, lib

MAX_K = 256
SIM_BUDGET = 1 << 30           # bytes of fp32 similarities per chunk
QUERY_CHUNK = 4096


def _cuda(t, name):
    if not isinstance(t, torch.Tensor):
        raise TypeError("%s must be a torch.Tensor" % name)
    if not t.is_cuda:
        raise RuntimeError("byol_b200.knn: %s must be a CUDA tensor (no CPU path)" % name)


def _same_device(*ts):
    devs = {t.device for t in ts}
    if len(devs) != 1:
        raise ValueError("byol_b200.knn: tensors on different devices: %s" % sorted(str(d) for d in devs))


def _check_k(k):
    if not isinstance(k, int) or isinstance(k, bool) or not 1 <= k <= MAX_K:
        raise ValueError("k must be an int in [1, %d], got %r" % (MAX_K, k))


def l2_normalize_rows(x, out=None):
    """fp32 [R, D] (unit column stride) -> bf16 [R, D] rows of unit L2 norm (zero rows stay zero)."""
    _cuda(x, "x")
    if x.dtype != torch.float32 or x.dim() != 2 or x.stride(1) != 1:
        raise ValueError("l2_normalize_rows: need an fp32 [R, D] matrix with unit column stride, got %s %s"
                         % (x.dtype, tuple(x.shape)))
    r, d = x.shape
    if out is None:
        out = torch.empty((r, d), dtype=torch.bfloat16, device=x.device)
    if r:
        check(lib.byol_l2_normalize_rows(x.data_ptr(), out.data_ptr(), r, d, x.stride(0), ops._stream()),
              "byol_l2_normalize_rows")
    return out


def topk_update(sim, n0, vals, idx, merge):
    """Merge the fp32 similarity chunk sim [Q, Nc] (unit column stride; column j is bank row n0 + j) into the running
    lists vals fp32 / idx int32 [Q, k] (best first; -inf / -1 in empty slots).  merge=False: the lists are only written
    (first chunk)."""
    _cuda(sim, "sim"); _cuda(vals, "vals"); _cuda(idx, "idx")
    _same_device(sim, vals, idx)
    if sim.dtype != torch.float32 or sim.dim() != 2 or sim.stride(1) != 1:
        raise ValueError("topk_update: sim must be an fp32 [Q, Nc] matrix with unit column stride")
    q, nc = sim.shape
    if vals.dtype != torch.float32 or idx.dtype != torch.int32 or vals.dim() != 2 or vals.shape != idx.shape or \
            vals.shape[0] != q or not vals.is_contiguous() or not idx.is_contiguous():
        raise ValueError("topk_update: vals / idx must be contiguous fp32 / int32 [Q, k] with Q = %d" % q)
    _check_k(vals.shape[1])
    if n0 < 0 or n0 + nc > 2 ** 31 - 1:
        raise ValueError("topk_update: bank rows [%d, %d) outside [0, 2^31 - 1)" % (n0, n0 + nc))
    if q and nc:
        check(lib.byol_knn_topk(sim.data_ptr(), q, nc, sim.stride(0), int(n0), vals.shape[1], int(bool(merge)),
                                vals.data_ptr(), idx.data_ptr(), ops._stream()), "byol_knn_topk")
    return vals, idx


def vote(vals, idx, bank_labels, num_classes, temperature=0.07, want_scores=False):
    """Top-5 classes int32 [Q, 5] of the neighbour lists (see byol_knn_vote); with want_scores also their scores
    fp32 [Q, 5].  bank_labels: int64 [N], every label in [0, num_classes) (checked by the caller)."""
    _cuda(vals, "vals"); _cuda(idx, "idx"); _cuda(bank_labels, "bank_labels")
    _same_device(vals, idx, bank_labels)
    if vals.dtype != torch.float32 or idx.dtype != torch.int32 or vals.dim() != 2 or vals.shape != idx.shape or \
            not vals.is_contiguous() or not idx.is_contiguous():
        raise ValueError("vote: vals / idx must be contiguous fp32 / int32 [Q, k]")
    if bank_labels.dtype != torch.int64 or bank_labels.dim() != 1 or not bank_labels.is_contiguous():
        raise ValueError("vote: bank_labels must be a contiguous int64 vector")
    _check_k(vals.shape[1])
    if not isinstance(num_classes, int) or num_classes < 1:
        raise ValueError("num_classes must be a positive int, got %r" % (num_classes,))
    if not (float(temperature) > 0.0 and float(temperature) < float("inf")):
        raise ValueError("temperature must be positive and finite, got %r" % (temperature,))
    q = vals.shape[0]
    pred = torch.empty((q, 5), dtype=torch.int32, device=vals.device)
    scores = torch.empty((q, 5), dtype=torch.float32, device=vals.device) if want_scores else None
    if q:
        check(lib.byol_knn_vote(vals.data_ptr(), idx.data_ptr(), bank_labels.data_ptr(), q, vals.shape[1], num_classes,
                                float(temperature), pred.data_ptr(), 0 if scores is None else scores.data_ptr(),
                                ops._stream()), "byol_knn_vote")
    return (pred, scores) if want_scores else pred


def _features(x, name):
    """bf16 rows as given (taken as L2-normalised), fp32 rows normalised here."""
    _cuda(x, name)
    if x.dim() != 2 or x.dtype not in (torch.bfloat16, torch.float32):
        raise ValueError("%s must be a bf16 or fp32 [rows, D] matrix, got %s %s" % (name, x.dtype, tuple(x.shape)))
    if x.dtype == torch.float32:
        return l2_normalize_rows(x.contiguous())
    return x.contiguous()


def _check_scalars(k, query_chunk, bank_chunk):
    _check_k(k)
    for name, v in (("query_chunk", query_chunk), ("bank_chunk", bank_chunk)):
        if v is not None and (not isinstance(v, int) or isinstance(v, bool) or v < 1):
            raise ValueError("%s must be a positive int, got %r" % (name, v))


def _check_features(bank_feats, query_feats):
    """Shapes and dtypes of the two feature matrices (no device access); returns (N, D, Q)."""
    for name, t in (("bank_feats", bank_feats), ("query_feats", query_feats)):
        if not isinstance(t, torch.Tensor):
            raise TypeError("%s must be a torch.Tensor" % name)
        if t.dim() != 2 or t.dtype not in (torch.bfloat16, torch.float32):
            raise ValueError("%s must be a bf16 or fp32 [rows, D] matrix, got %s %s" % (name, t.dtype, tuple(t.shape)))
    n, d = bank_feats.shape
    if query_feats.shape[1] != d:
        raise ValueError("bank and query features differ in width: %d vs %d" % (d, query_feats.shape[1]))
    if d == 0 or d % 64 != 0:
        raise ValueError("the feature width D=%d must be a positive multiple of 64" % d)
    if n < 1 or n > 2 ** 31 - 1:
        raise ValueError("the bank must hold between 1 and 2^31 - 1 rows, got %d" % n)
    return n, d, query_feats.shape[0]


def _search(bank, queries, k, query_chunk, bank_chunk, budget_bytes):
    n, q = bank.shape[0], queries.shape[0]
    dev = bank.device
    vals = torch.empty((q, k), dtype=torch.float32, device=dev)
    idx = torch.empty((q, k), dtype=torch.int32, device=dev)
    if q == 0:
        return vals, idx
    qc = min(q, query_chunk or QUERY_CHUNK)
    nc = min(n, bank_chunk or max(128, budget_bytes // (4 * qc) // 128 * 128))
    sim = torch.empty(qc * nc, dtype=torch.float32, device=dev)
    for q0 in range(0, q, qc):
        qn = min(qc, q - q0)
        for n0 in range(0, n, nc):
            bn = min(nc, n - n0)
            s = sim[:qn * bn].view(qn, bn)
            ops.linear_fprop(queries[q0:q0 + qn], bank[n0:n0 + bn], out_fp32=True, out=s)
            topk_update(s, n0, vals[q0:q0 + qn], idx[q0:q0 + qn], merge=n0 > 0)
    return vals, idx


def knn_search(bank_feats, query_feats, k=20, query_chunk=None, bank_chunk=None, budget_bytes=SIM_BUDGET):
    """The k most similar bank rows of every query: (similarities fp32 [Q, k], bank indices int32 [Q, k]), best
    first (similarity descending, then bank index ascending; -inf / -1 in the slots of a bank shorter than k).

    bank_feats [N, D] / query_feats [Q, D]: bf16 rows already L2-normalised (as l2_normalize_rows makes them), or fp32
    rows, normalised here; D % 64 == 0; 1 <= k <= 256.  The fp32 similarities are computed in chunks of query_chunk x
    bank_chunk rows (by default at most `budget_bytes` of them); the result does not depend on the chunk sizes."""
    _check_scalars(k, query_chunk, bank_chunk)
    _check_features(bank_feats, query_feats)
    _cuda(bank_feats, "bank_feats"); _cuda(query_feats, "query_feats")
    _same_device(bank_feats, query_feats)
    return _search(_features(bank_feats, "bank_feats"), _features(query_feats, "query_feats"), k, query_chunk,
                   bank_chunk, budget_bytes)


def knn_classify(bank_feats, bank_labels, query_feats, num_classes, k=20, temperature=0.07, query_chunk=None,
                 bank_chunk=None, budget_bytes=SIM_BUDGET):
    """Top-5 predicted classes, int32 [Q, 5], of the weighted k-NN vote (w = exp(s / temperature)) over the bank:
    knn_search, then byol_knn_vote.  bank_labels: int64 [N] in [0, num_classes); with fewer than 5 classes the
    remaining places hold -1.  Arguments are checked before anything runs: scalars and shapes first, then devices (CPU
    tensors raise RuntimeError), then the label range."""
    _check_scalars(k, query_chunk, bank_chunk)
    if not isinstance(num_classes, int) or isinstance(num_classes, bool) or num_classes < 1:
        raise ValueError("num_classes must be a positive int, got %r" % (num_classes,))
    if not (float(temperature) > 0.0 and float(temperature) < float("inf")):
        raise ValueError("temperature must be positive and finite, got %r" % (temperature,))
    n, _, q = _check_features(bank_feats, query_feats)
    if not isinstance(bank_labels, torch.Tensor):
        raise TypeError("bank_labels must be a torch.Tensor")
    if bank_labels.dtype != torch.int64 or tuple(bank_labels.shape) != (n,):
        raise ValueError("bank_labels must be int64 [%d], got %s %s" % (n, bank_labels.dtype,
                                                                         tuple(bank_labels.shape)))
    _cuda(bank_feats, "bank_feats"); _cuda(bank_labels, "bank_labels"); _cuda(query_feats, "query_feats")
    _same_device(bank_feats, bank_labels, query_feats)
    lo, hi = (int(v) for v in torch.aminmax(bank_labels))
    if lo < 0 or hi >= num_classes:
        raise ValueError("bank labels span [%d, %d], outside [0, %d)" % (lo, hi, num_classes))
    if q == 0:
        return torch.empty((0, 5), dtype=torch.int32, device=bank_feats.device)
    vals, idx = _search(_features(bank_feats, "bank_feats"), _features(query_feats, "query_feats"), k, query_chunk,
                        bank_chunk, budget_bytes)
    return vote(vals, idx, bank_labels.contiguous(), num_classes, temperature)


def _extract(model, samples, batch_size, augment, network):
    """(bf16 normalised features [len(samples), D], int64 labels) of one pass over `samples` in file order, view 1
    (the eval transform of `augment`)."""
    from .data import ImageFolderLoader
    feats, labels = [], []
    for img, _, lab in ImageFolderLoader(samples, batch_size, augment, train=False):
        feats.append(l2_normalize_rows(model.representations(img, network)))
        labels.append(lab)
    return torch.cat(feats), torch.cat(labels)


def knn_accuracy(model, loader, k=20, temperature=0.07, network="online", batch_size=None):
    """k-NN top-1 / top-5 accuracy (%) of `model`'s frozen encoder on the test split of `loader` (the
    ``ImageFolderTwoView`` from ``byol_b200.data.get_loader``): {"knn_top1": float, "knn_top5": float}.

    The bank is the whole training split in file order, unsharded, each image taken through the loader's eval
    transform as the test split is (``loader.test_loader.augment``; not augmented): the whole image resized to R x R
    by default, or with ``get_loader(..., eval_transform="byol")`` the paper's protocol, the shorter side resized to
    256 (at R = 224) by bicubic and the centre R x R crop.  Features come from ``model.representations(images,
    network)`` and are kept as L2-normalised bf16 rows with int64 labels (5.25 GB for ImageNet-1k at D = 2048).
    Under torch.distributed it runs on the calling rank alone, with no collective, so every rank that calls it gets the
    same result."""
    _check_k(k)
    if not (float(temperature) > 0.0 and float(temperature) < float("inf")):
        raise ValueError("temperature must be positive and finite, got %r" % (temperature,))
    if network not in ("online", "target"):
        raise ValueError("network must be 'online' or 'target', got %r" % (network,))
    bs = int(batch_size or loader.test_loader.batch_size)
    if bs < 1:
        raise ValueError("batch_size must be positive, got %r" % (batch_size,))
    augment = loader.test_loader.augment
    bank, bank_labels = _extract(model, loader.train_loader.samples, bs, augment, network)
    queries, query_labels = _extract(model, loader.test_loader.samples, bs, augment, network)
    if queries.shape[0] == 0:
        raise ValueError("knn_accuracy: the test split is empty")
    pred = knn_classify(bank, bank_labels, queries, loader.output_size, k=k, temperature=temperature)
    hit = pred.long() == query_labels.view(-1, 1)
    return {"knn_top1": 100.0 * float(hit[:, 0].float().mean()), "knn_top5": 100.0 * float(hit.any(1).float().mean())}
