"""numpy restatement of one step of byol_b200.linear_eval.LinearHeads (the GPU tests compare against it): bf16-rounded
features and weights, logits and the cross-entropy gradient in float64, and the Nesterov-SGD update in its exact fp32
operation order (every product and sum rounded to fp32 on its own)."""
import numpy as np


def bf16(x):
    """Round-to-nearest-even to bf16, returned as float32 (finite inputs)."""
    u = np.ascontiguousarray(np.asarray(x, dtype=np.float32)).view(np.uint32).astype(np.uint64)
    u = (u + 0x7FFF + ((u >> 16) & 1)) & 0xFFFF0000
    return u.astype(np.uint32).view(np.float32)


def padded(c):
    return (c + 7) // 8 * 8


def logits(feats, w, b):
    """float64 [B, H * Cp] = bf16(feats) @ bf16(w)^T + b; w fp32 [H, Cp, D], b [H, Cp]."""
    h, cp, d = w.shape
    return bf16(feats).astype(np.float64) @ bf16(w).reshape(h * cp, d).astype(np.float64).T + \
        np.asarray(b, np.float64).reshape(-1)


MISS = 1 << 30    # the rank of a row that is in no top k


def rank(s, labels):
    """Rank of each row's label among the columns of s [B, C]: the number of other columns whose value is not <= the
    label's (strictly larger, or NaN); MISS when the label's value is NaN or the label is outside [0, C)."""
    s = np.asarray(s, dtype=np.float64)
    bsz, c = s.shape
    ok = (labels >= 0) & (labels < c)
    lab = np.where(ok, labels, 0)
    xl = s[np.arange(bsz), lab]
    other = np.arange(c)[None, :] != lab[:, None]
    r = (~(s <= xl[:, None]) & other).sum(1)
    return np.where(ok & ~np.isnan(xl), r, MISS)


def cross_entropy(z, labels, h, c):
    """Per (row, head) of logits z [B, >= H * Cp] (columns c < C of each segment): (loss float64 [B, H],
    rank int64 [B, H] (see `rank`), grad float64 [B, H * Cp] = (softmax - onehot) / B with 0 in the padding columns).
    A row whose label is outside [0, C) has loss 0, rank MISS and a zero gradient."""
    z = np.asarray(z, dtype=np.float64)
    labels = np.asarray(labels)
    cp = padded(c)
    bsz = z.shape[0]
    loss = np.zeros((bsz, h))
    ranks = np.zeros((bsz, h), dtype=np.int64)
    grad = np.zeros((bsz, h * cp))
    rows = np.arange(bsz)
    ok = (labels >= 0) & (labels < c)
    lab = np.where(ok, labels, 0)
    with np.errstate(invalid="ignore", over="ignore"):     # non-finite logits give NaN losses and gradients
        for k in range(h):
            s = z[:, k * cp:k * cp + c]
            xl = s[rows, lab]
            m = s.max(1, keepdims=True)
            e = np.exp(s - m)
            se = e.sum(1)
            loss[:, k] = np.where(ok, np.log(se) + m[:, 0] - xl, 0.0)
            ranks[:, k] = rank(s, labels)
            p = e / se[:, None]
            p[rows, lab] -= 1.0
            grad[:, k * cp:k * cp + c] = np.where(ok[:, None], p / bsz, 0.0)
    return loss, ranks, grad


def sgd(w, buf, grad, lr, wd, mu):
    """One Nesterov-SGD step in fp32, the kernel's order: g = dW + wd w; buf = mu buf + g; d = g + mu buf;
    w = w - lr d.  All arguments fp32 (lr, wd broadcast against w); returns (w, buf)."""
    f = np.float32
    w, buf, grad = (np.asarray(a, dtype=f) for a in (w, buf, grad))
    lr, wd, mu = np.asarray(lr, dtype=f), np.asarray(wd, dtype=f), f(mu)
    g = grad + wd * w
    buf = mu * buf + g
    d = g + mu * buf
    return w - lr * d, buf
