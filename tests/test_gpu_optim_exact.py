"""GPU: the BYOL loss, the LARS + SGD-momentum step and the classifier cross-entropy (csrc/optim.cu) exactly against
float64, on every branch inside their kernels.

* Exact operands.  Predictions, targets, parameters and gradients are small integers times a power of two and weight
  decays are powers of two, so every fp32 product, sum of squares and dot product the kernels accumulate is exact
  whatever the order: each row checks that the sum of the magnitudes of the terms one fp32 accumulator can see (one
  loss block, one 32 768-element LARS chunk) stays below 2^24 grid units.  The six loss sums, the per-chunk LARS
  partials and their fp64 re-addition are then exact, and what follows them is fp32 sqrt, division, multiplication
  and fused multiply-add (built with -O3 and no fast-math: sqrtf and / are IEEE).
* Restatement.  That remainder is restated in numpy in nvcc's order, with the contractions `cuobjdump -sass` shows
  for sm_90a (loss_bwd_kernel and lars_update_kernel hold 45 FFMA each; the others are the division and square-root
  sequences):
    - loss_bwd_kernel: `a1 * d + b1 * a` is FMUL a1*d, then FFMA b1*a + that, so dq1 = fma(b1, q1, rn(a1 * z2)) and
      dq2 = fma(b2, q2, rn(a2 * z1)).  a1, b1, a2, b2 and k are FMUL / division only.
    - loss_finalize_kernel: no contraction.  The loss is rn(rn(t12 + t21) / rows) with t12 = rn(rn(-2 s12) /
      rn(nq1 nz2)), and the norms are sqrtf of the fp32 roundings of the exact sums.
    - lars_update_kernel: `gv += w * pv` is FFMA w*pv + gv (exact for these operands), `gv *= ratio` an FMUL,
      `pv -= rate * b` FFMA -rate*b + pv.  The momentum `momentum * mv + gv` is FFMA momentum*mv + rn(ratio*gv) on
      the float4 path and on the scalar path with weight decay, but on the scalar path without weight decay nvcc
      fuses the other product: FMUL momentum*mv, then FFMA ratio*g + that.
    - lars_norms_kernel: ratio = rn(rn(trust * pn) / rn(gn + eps)), pn = sqrtf(fp32(sum p^2)), gn likewise.
  Loss, the six saved scalars, dq1 / dq2, parameters and momentum must equal the restatement bit for bit; they are
  also compared with float64 evaluations of objective.py and lars.py within the bounds stated below.
* Cross-entropy.  expf / logf are library functions and are not restated: the per-row loss, the mean and dlogits are
  compared with float64 within CE_TOL; the label's rank is restated exactly (the number of other columns c with
  !(x_c <= x_label); a NaN label logit or a label outside [0, C) is a miss), and top-1 / top-5 must be exactly
  fp32(100 * hits) / R.
* Row table.  Each row names the kernel branches it is meant for; the test restates their predicates (aligned16 on
  the chunk pointers, grid-stride passes, chunk counts) and checks that the row is on that side, and one
  torch.profiler test checks that every row launches exactly its kernels.
* Scale.  The loss is bit-identical under power-of-two scaling of its inputs down to an RMS of ~1e-11.
* Replay.  One eager wiring.train_step of a ResNet-18 and of a small bottleneck net, in bf16 and fp32, records the
  shapes and options of every loss, cross-entropy and LARS call (for LARS each tensor's length and 16-byte phases),
  and every distinct call is replayed with exact operands.
"""
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests.exact import (Case, bits_same, byol_kernel_sequence, byol_train_step, check_in_fresh_process, expect_bits,
                         expect_within, NO_EVENTS, recording, replay, row_case, run_and_check)
from tests.util import _rn32, fma32, gen, ints

pytestmark = pytest.mark.gpu
F32, F64, I64 = torch.float32, torch.float64, torch.int64
f32 = np.float32

CHUNK = 32768             # lars.chunk_table
SENTINEL = 1234.5         # fills the LARS buffers around the tensors: must survive the step
# float64 bounds, in fp32 units (2^-24) of the stated magnitude
LOSS_ULPS = 16            # loss: of |t12| + |t21| (the two cosine terms); saved norms / sums: of the value
DQ_ULPS = 16              # dq: of |a1 z2| + |b1 q1|
LARS_ULPS = 16            # momentum: of M = sum over steps of momentum^age * |ratio * g'|; p: of |p| + |lr| M
CE_TOL = 2.0 ** -16       # row loss / lse: of 1 + |max| + |x_label|; dlogits: |k| (CE_TOL p (1 + |max| + |x|) + 2^-23)


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def _grid(shape, dev, g, amp, k):
    """fp32 integers in [-amp, amp] times 2^-k (exact)."""
    return (ints(shape, dev, g, amp) * 2.0 ** -k).float()


def _units(x64, unit):
    """Sum of |terms| in grid units (an exact fp64 integer): below 2^24 every partial sum in fp32 is exact."""
    return float(x64.abs().sum() / unit)


# ------------------------------------------------------------------------------------------------------------------
# BYOL loss
# ------------------------------------------------------------------------------------------------------------------
LOSS_K = 4                # operands on the 2^-4 grid, |q| <= 1/2, |z| <= 3/4: products on the 2^-8 grid


def loss_restated(sums, rows, go, q1, q2, z1, z2):
    """loss_finalize_kernel and loss_bwd_kernel as compiled, from the six exact sums (Fractions)."""
    v = [_rn32(s) for s in sums]
    nq1, nq2, nz1, nz2 = (np.sqrt(f32(x)) for x in v[:4])
    s12, s21 = v[4], v[5]
    t12 = (f32(-2) * s12) / (nq1 * nz2)
    t21 = (f32(-2) * s21) / (nq2 * nz1)
    loss = (t21 + t12) / f32(rows)
    saved = np.array([nq1, nq2, nz1, nz2, s12, s21], dtype=np.float32)
    k = (f32(go) * f32(-2)) / f32(rows)
    a1, a2 = k / (nq1 * nz2), k / (nq2 * nz1)
    b1 = ((-k) * s12) / (((nq1 * nq1) * nq1) * nz2)
    b2 = ((-k) * s21) / (((nq2 * nq2) * nq2) * nz1)
    dq1 = fma32(b1, q1, f32(a1) * z2)
    dq2 = fma32(b2, q2, f32(a2) * z1)
    return f32(loss), saved, dq1, dq2, (a1, b1, a2, b2)


def loss_branch(rows, dim):
    n4 = rows * dim // 4
    nb = min(max(-(-n4 // 256), 1), 132)
    return {"fwd_blocks": nb, "fwd_passes": -(-n4 // (nb * 256)), "sub_block": n4 < 256,
            "bwd_passes": -(-n4 // (min(max(-(-n4 // 256), 1), 528) * 256))}


def loss_case(dev, g, rows, dim, go=0.75):
    """One loss forward + backward; go None: the backward without grad_out (1)."""
    from byol_b200 import ops
    q1 = _grid((rows, dim), dev, g, 8, LOSS_K)
    q2 = _grid((rows, dim), dev, g, 8, LOSS_K)
    # targets correlated with the predictions: the two cosine terms stay away from zero, as in training
    z2 = q1 + _grid((rows, dim), dev, g, 4, LOSS_K)
    z1 = q2 + _grid((rows, dim), dev, g, 4, LOSS_K)
    ops_ = [q1, q2, z1, z2]
    n4 = rows * dim // 4
    br = loss_branch(rows, dim)
    x64 = [x.double() for x in ops_]
    unit = 2.0 ** (-2 * LOSS_K)
    blk = ((torch.arange(n4, device=dev) // 256) % br["fwd_blocks"]).repeat_interleave(4)
    terms = [x64[0] * x64[0], x64[1] * x64[1], x64[2] * x64[2], x64[3] * x64[3], x64[0] * x64[3], x64[1] * x64[2]]
    worst = max(float(torch.zeros(br["fwd_blocks"], device=dev, dtype=F64).index_add_(
        0, blk, t.reshape(-1).abs()).max()) / unit for t in terms)
    assert worst < 2 ** 24, "a loss block sums %.0f grid units: fp32 partial sums would round" % worst
    gout = None if go is None else torch.full((1,), go, device=dev)

    def run():
        ws = torch.empty(6, dtype=F64, device=dev)
        out = torch.full((7,), float("nan"), device=dev)
        ops.loss_fwd(q1, q2, z1, z2, ws, out[0:1], out[1:7])
        dq1, dq2 = torch.empty_like(q1), torch.empty_like(q2)
        ops.loss_bwd(q1, q2, z1, z2, out[1:7], gout, dq1, dq2)
        return out, dq1, dq2

    def check(outs):
        out, dq1, dq2 = outs
        sums = [Fraction(int(round(float(t.sum()) / unit))) * Fraction(unit) for t in terms]
        np_ = [x.cpu().numpy() for x in ops_]
        loss, saved, r1, r2, (a1, b1, a2, b2) = loss_restated(sums, rows, 1.0 if go is None else go,
                                                              np_[0], np_[1], np_[2], np_[3])
        expect_bits("loss", out[0:1], [loss])
        expect_bits("saved", out[1:7], saved)
        expect_bits("dq1", dq1, r1)
        expect_bits("dq2", dq2, r2)
        # float64 evaluation of objective.py (regression_loss of whole-matrix norms, symmetric, mean over rows)
        s = [float(x) for x in sums]
        n = [s[0] ** 0.5, s[1] ** 0.5, s[2] ** 0.5, s[3] ** 0.5]
        c12, c21 = -2 * s[4] / (n[0] * n[3]), -2 * s[5] / (n[1] * n[2])
        expect_within("loss vs float64", out[0:1], [(c12 + c21) / rows],
                      LOSS_ULPS * 2.0 ** -24 * (abs(c12) + abs(c21)) / rows)
        expect_within("saved vs float64", out[1:7], n + s[4:], LOSS_ULPS * 2.0 ** -24 * np.abs(n + s[4:]))
        gv = 1.0 if go is None else float(f32(go))
        kk = gv * -2 / rows
        for name, got, q, z, nq, nz, sqz in (("dq1", dq1, x64[0], x64[3], n[0], n[3], s[4]),
                                            ("dq2", dq2, x64[1], x64[2], n[1], n[2], s[5])):
            ta, tb = kk / (nq * nz) * z, -kk * sqz / (nq ** 3 * nz) * q
            expect_within(name + " vs float64", got.reshape(-1), (ta + tb).reshape(-1).cpu().numpy(),
                          DQ_ULPS * 2.0 ** -24 * (ta.abs() + tb.abs()).reshape(-1).cpu().numpy())

    return Case(run, check, launches=["loss_fwd_partial_kernel", "loss_finalize_kernel", "loss_bwd_kernel"],
                branch=dict(br, grad_out=go is not None))


# ------------------------------------------------------------------------------------------------------------------
# LARS + SGD momentum
# ------------------------------------------------------------------------------------------------------------------
class T:
    """One tensor of a LARS call: length, weight decay, learning rate, ignore flag and the 16-byte phases (in floats)
    of its parameter, gradient and momentum storage."""

    def __init__(self, n, wd=0.0, lr=0.3, ignore=0, pp=0, pg=0, pm=0, grad=None):
        self.n, self.wd, self.lr, self.ignore, self.ph = n, wd, lr, ignore, (pp, pg, pm)
        self.grad = grad          # None | "nan" | "inf" | "zero": a non-finite or zero gradient element set
        self.zero_p = False


def _layout(ts, role):
    offs, cur = [], 0
    for t in ts:
        cur = -(-cur // 4) * 4 + t.ph[role]
        offs.append(cur)
        cur += t.n + 1
    return offs, cur + 8


P_K, G_K = 4, 6           # parameters on the 2^-4 grid (|p| <= 1/4), gradients on the 2^-6 grid (|g| <= 1/16)


def lars_branch(ts, mom):
    """The restated in-kernel predicates: aligned16(p, g) in lars_norms_kernel, aligned16(p, g, m) in update_chunk,
    and the chunk count of every tensor (the lane loop of lars_update_kernel takes chunks l, l + 32, ...)."""
    norm_vec = [t.ph[0] == 0 and t.ph[1] == 0 for t in ts if t.n]
    upd_vec = [t.ph[0] == 0 and t.ph[1] == 0 and (not mom or t.ph[2] == 0) for t in ts if t.n]
    kind = lambda v: "vec" if all(v) else "scalar" if not any(v) else "both"
    return {"norms": kind(norm_vec), "update": kind(upd_vec), "chunks": max(-(-t.n // CHUNK) for t in ts),
            "tails": sorted({t.n % CHUNK % 4 for t in ts if t.n}), "empty": any(t.n == 0 for t in ts)}


def lars_restated(ps, gs, ms, ts, momentum, eps, trust, first_step):
    """lars_norms_kernel + lars_update_kernel as compiled.  ps / gs / ms: numpy fp32 per tensor (ms None: no
    momentum buffers).  Returns (new ps, new ms)."""
    out_p, out_m = [], []
    for i, t in enumerate(ts):
        p, g = ps[i], gs[i]
        w, rate = f32(t.wd), f32(t.lr)
        gw = fma32(w, p, g) if w > 0 else g
        ratio = f32(1)
        if not t.ignore and t.n:
            with np.errstate(invalid="ignore", over="ignore"):
                sp = np.sum(p.astype(np.float64) ** 2)
                sg = np.sum(gw.astype(np.float64) ** 2)
                pn, gn = np.sqrt(f32(sp)), np.sqrt(f32(sg))
                if pn > 0 and gn > 0:
                    ratio = (f32(trust) * pn) / (gn + f32(eps))
        with np.errstate(invalid="ignore", over="ignore"):
            rg = f32(ratio) * gw
            if ms is None or first_step:
                b = rg
            else:
                m = ms[i]
                vec = t.ph[0] == 0 and t.ph[1] == 0 and t.ph[2] == 0
                idx = np.arange(t.n) % CHUNK
                clen = np.minimum(CHUNK, t.n - (np.arange(t.n) // CHUNK) * CHUNK)
                in_vec = vec & (idx < clen // 4 * 4)
                if w > 0:
                    b = fma32(f32(momentum), m, rg)
                else:
                    # scalar path without weight decay: FMUL momentum*m, FFMA ratio*g + that
                    b = np.where(in_vec, fma32(f32(momentum), m, rg), fma32(f32(ratio), g, f32(momentum) * m))
            out_p.append(fma32(-rate, b, p))
            out_m.append(None if ms is None else b.astype(np.float32))
    return out_p, out_m


def lars_float64(ps, gs, m64, ts, momentum, eps, trust, first_step, mag):
    """/root/reference lars.py (apply_adaptive_lrs + torch.optim.SGD momentum step) in float64 on the same fp32
    inputs and hyperparameters.  m64 / mag: per-tensor fp64 momentum and its magnitude bound M, updated in place."""
    out = []
    for i, t in enumerate(ts):
        p, g = ps[i].astype(np.float64), gs[i].astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            if t.wd > 0:
                g = g + float(f32(t.wd)) * p
            if not t.ignore and t.n:
                pn, gn = np.sqrt(np.sum(p * p)), np.sqrt(np.sum(g * g))
                if pn > 0 and gn > 0:
                    g = g * (float(f32(trust)) * pn / (gn + float(f32(eps))))
            mu = float(f32(momentum))
            if m64 is None:
                b, mag_b = g, np.abs(g)
            elif first_step or m64[i] is None:
                m64[i], mag[i] = g, np.abs(g)
                b, mag_b = g, mag[i]
            else:
                m64[i], mag[i] = mu * m64[i] + g, mu * mag[i] + np.abs(g)
                b, mag_b = m64[i], mag[i]
            out.append((p - float(f32(t.lr)) * b, mag_b))
    return out


def lars_case(dev, g, ts, momentum=0.9, eps=0.0, trust=0.001, first_step=False, steps=1, m_nan=False):
    """A LARS step over tensors `ts` laid out at their phases in three flat buffers (sentinel-filled around them);
    momentum None: no momentum buffers (m_ptrs null).  Each step draws fresh exact p and g and carries the momentum.
    m_nan: the momentum buffers start as NaN (first_step must not read them)."""
    from byol_b200 import ops
    from byol_b200.lars import chunk_table
    mom = momentum is not None
    lay = [_layout(ts, r) for r in range(3)]
    gens = [gen(dev, 100 + 7 * s + int(g.initial_seed()) % 1000) for s in range(steps)]
    for t in ts:
        assert t.wd == 0 or float(np.log2(t.wd)).is_integer(), "weight decays are powers of two"

    def draw(s):
        gg = gens[s]
        ps = [_grid((t.n,), dev, gg, 4, P_K) for t in ts]
        gs = [_grid((t.n,), dev, gg, 4, G_K) for t in ts]
        for i, t in enumerate(ts):
            if t.zero_p:
                ps[i].zero_()
            if t.grad == "zero":
                gs[i].zero_()
            elif t.grad in ("nan", "inf") and t.n:
                gs[i][t.n // 3] = float(t.grad)
                gs[i][(2 * t.n) // 3] = -float("inf") if t.grad == "inf" else float("nan")
        return ps, gs

    def bound_check(ps, gs):
        for i, t in enumerate(ts):
            if t.ignore or not t.n or t.grad in ("nan", "inf"):
                continue
            p, gr = ps[i].double(), gs[i].double()
            gw = gr + t.wd * p if t.wd > 0 else gr
            unit = min(2.0 ** -G_K, t.wd * 2.0 ** -P_K if t.wd else 1.0) ** 2
            for c0 in range(0, t.n, CHUNK):
                for name, x in (("p", p), ("g + wd p", gw)):
                    u = _units(x[c0:c0 + CHUNK] ** 2, 2.0 ** (-2 * P_K) if name == "p" else unit)
                    assert u < 2 ** 24, "a LARS chunk sums %.0f grid units of |%s|^2" % (u, name)

    def run():
        bufs = [torch.full((lay[r][1],), SENTINEL, device=dev) for r in range(3)]
        views = [[bufs[r][o:o + t.n] for o, t in zip(lay[r][0], ts)] for r in range(3)]
        if mom:
            for v in views[2]:
                v.fill_(float("nan") if m_nan else 0.0)
        tb = chunk_table([t.n for t in ts], dev)
        ptr = lambda vs: torch.tensor([v.data_ptr() for v in vs], dtype=I64, device=dev)
        tb.update({"p_ptrs": ptr(views[0]), "g_ptrs": ptr(views[1]), "m_ptrs": ptr(views[2]) if mom else None,
                   "wd": torch.tensor([t.wd for t in ts], device=dev),
                   "lr": torch.tensor([t.lr for t in ts], device=dev),
                   "ignore": torch.tensor([t.ignore for t in ts], dtype=torch.int32, device=dev),
                   "partial": torch.full((2 * max(tb["chunk_start"].numel(), 1),), float("nan"), dtype=F64,
                                         device=dev)})
        hist = []
        for s in range(steps):
            ps, gs = draw(s)
            for v, x in zip(views[0], ps):
                v.copy_(x)
            for v, x in zip(views[1], gs):
                v.copy_(x)
            ms = [v.clone() for v in views[2]] if mom else None
            ops.lars_sgd_step(tb, trust, eps, 0.0 if not mom else momentum, first_step=first_step)
            hist.append((ps, gs, ms, [v.clone() for v in views[0]], [v.clone() for v in views[2]] if mom else None))
        return hist, bufs, views

    def check(outs):
        hist, bufs, views = outs
        m64, mag = ([None] * len(ts) if mom else None), [None] * len(ts)
        for s, (ps, gs, ms, got_p, got_m) in enumerate(hist):
            bound_check(ps, gs)
            np_p, np_g = [x.cpu().numpy() for x in ps], [x.cpu().numpy() for x in gs]
            np_m = [x.cpu().numpy() for x in ms] if mom else None
            if mom and s > 0:
                # the carried buffer is the one the previous step wrote
                for i in range(len(ts)):
                    expect_bits("step %d momentum in, tensor %d" % (s, i), ms[i], hist[s - 1][4][i])
            want_p, want_m = lars_restated(np_p, np_g, np_m, ts, momentum or 0.0, eps, trust, first_step)
            ref = lars_float64(np_p, np_g, m64, ts, momentum or 0.0, eps, trust, first_step, mag)
            for i, t in enumerate(ts):
                expect_bits("step %d p[%d] (n=%d)" % (s, i, t.n), got_p[i], want_p[i])
                if mom:
                    expect_bits("step %d m[%d] (n=%d)" % (s, i, t.n), got_m[i], want_m[i])
                p64, mag_b = ref[i]
                if not t.n:
                    continue
                expect_within("step %d p[%d] vs float64" % (s, i), got_p[i], p64,
                              LARS_ULPS * 2.0 ** -24 * np.nan_to_num(np.abs(p64) + float(f32(t.lr)) * mag_b))
                if mom:
                    expect_within("step %d m[%d] vs float64" % (s, i), got_m[i], m64[i],
                                  LARS_ULPS * 2.0 ** -24 * np.nan_to_num(mag[i]))
        # nothing outside the tensors was written
        for r, buf in enumerate(bufs):
            keep = torch.ones_like(buf, dtype=torch.bool)
            for o, t in zip(lay[r][0], ts):
                keep[o:o + t.n] = False
            if r < 2 or mom:
                assert bool((buf[keep] == SENTINEL).all()), "LARS wrote outside its tensors (buffer %d)" % r

    return Case(run, check, launches=["lars_norms_kernel", "lars_update_kernel"] * steps,
                branch=dict(lars_branch(ts, mom), momentum=mom, first_step=bool(first_step)))


# ------------------------------------------------------------------------------------------------------------------
# classifier cross-entropy
# ------------------------------------------------------------------------------------------------------------------
MISS = 1 << 30


def ce_reference(x32, labels, R, C):
    """Per row, in float64 with the kernel's handling of non-finite values (the max ignores NaN):
    (loss, lse, rank, max, x_label).  rank MISS: a miss for every k."""
    x = x32.astype(np.float64)
    lab = np.array([labels[r % len(labels)] for r in range(R)], dtype=np.int64)
    ok = (lab >= 0) & (lab < C)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        allnan = np.isnan(x).all(1)
        mx = np.where(allnan, -np.inf, np.nanmax(np.where(allnan[:, None], 0, x), 1))
        se = np.exp(x - mx[:, None]).sum(1)
        lse = mx + np.log(se)
        xl = np.where(ok, x[np.arange(R), np.where(ok, lab, 0)], -np.inf)
        loss = lse - xl
        other = np.ones((R, C), dtype=bool)
        other[np.arange(R)[ok], lab[ok]] = False
        rank = (other & ~(x <= xl[:, None])).sum(1)
    rank = np.where(ok & ~np.isnan(xl), rank, MISS)
    return loss, lse, rank, mx, xl, lab, ok


def ce_branch(x32, labels, R, C, ld):
    loss, lse, rank, mx, xl, lab, ok = ce_reference(x32, labels, R, C)
    return {"R>256": R > 256, "R%8": R % 8 != 0, "repeat": len(labels) < R, "pitched": ld > C,
            "nan_label": bool((ok & np.isnan(xl)).any()), "out_of_range": bool((~ok).any()),
            "nan_column": bool((np.isnan(x32).any(1) & ~np.isnan(xl) & ok).any()),
            "inf": bool(np.isinf(x32).any()), "tie": bool(((x32 == xl[:, None]).sum(1) > 1).any())}


def ce_case(dev, g, R, C, LR=None, ld=None, edits=None, labels=None, go=0.37):
    """logits [R, C] (a column slice of [R, ld] when ld > C) of normal values * 3 on the 2^-10 grid; labels [LR]
    (row r uses labels[r % LR]); edits(x, lab): in-place special values on the numpy logits / labels."""
    from byol_b200 import ops
    from byol_b200._lib import check as lib_check, lib
    LR = LR or R
    ld = ld or C
    gg = torch.Generator().manual_seed(int(g.initial_seed()) % (2 ** 31))
    full = torch.round(torch.randn(R, ld, generator=gg, dtype=F64) * 3 * 1024) / 1024
    lab = torch.randint(0, C, (LR,), generator=gg) if labels is None else torch.tensor(labels, dtype=I64)
    xn, labn = full.float().numpy(), lab.numpy().copy()
    if edits is not None:
        edits(xn, labn)
    base = torch.from_numpy(xn).to(dev)
    logits = base[:, :C]
    labels_d = torch.from_numpy(labn).to(dev)
    x32 = xn[:, :C].copy()
    gout = torch.full((1,), go, device=dev)

    def run():
        fl = torch.full((2 * R + 3,), float("nan"), device=dev)
        it = torch.zeros(R + 1, dtype=torch.int32, device=dev)
        lib_check(lib.byol_ce_topk_fwd(logits.data_ptr(), labels_d.data_ptr(), LR, R, C, logits.stride(0),
                                       fl.data_ptr(), fl[R:].data_ptr(), it.data_ptr(), it[R:].data_ptr(),
                                       fl[2 * R:].data_ptr(),
                                       torch.cuda.current_stream().cuda_stream), "byol_ce_topk_fwd")
        out2, lse2 = ops.ce_topk_fwd(logits, labels_d)
        d = ops.ce_bwd(logits, labels_d, fl[:R], gout)
        d2 = ops.ce_bwd(logits, labels_d, lse2, gout)
        return fl, it, out2, lse2, d, d2

    def check(outs):
        fl, it, out2, lse2, d, d2 = outs
        loss, lse, rank, mx, xl, labr, ok = ce_reference(x32, labn, R, C)
        # two launches, the same bits; the ticket is reset
        assert bits_same(out2, fl[2 * R:].cpu().numpy()) and bits_same(lse2, fl[:R].cpu().numpy())
        assert bits_same(d, d2.cpu().numpy()), "two backward launches differ"
        assert int(it[R]) == 0, "ticket not reset"
        got_rank = it[:R].cpu().numpy().astype(np.int64)
        got_rank = np.where(got_rank == 0x7fffffff, MISS, got_rank)
        bad = np.nonzero(got_rank != rank)[0]
        assert not bad.size, "rank of rows %s: kernel %s, rule %s" % (bad[:8].tolist(), got_rank[bad][:8].tolist(),
                                                                      rank[bad][:8].tolist())
        tol = CE_TOL * (1 + np.abs(np.nan_to_num(mx, posinf=0, neginf=0)) + np.abs(np.nan_to_num(xl, posinf=0,
                                                                                                neginf=0)))
        expect_within("row_loss", fl[R:2 * R], loss, tol)
        expect_within("row_lse", fl[:R], lse, tol)
        # the mean: exactly the kernel's fp64 reduction of its own row losses (thread i: rows i, i + 256, ...; then
        # the shared-memory tree), and within the row bounds of float64
        rl = fl[R:2 * R].cpu().numpy().astype(np.float64)
        part = np.zeros(256)
        with np.errstate(invalid="ignore"):
            for i in range(256):
                for r in range(i, R, 256):
                    part[i] += rl[r]
            o = 128
            while o:
                part[:o] = part[:o] + part[o:2 * o]
                o >>= 1
            mean = f32(part[0] / R)
        expect_bits("mean loss (row reduction)", fl[2 * R:2 * R + 1], [mean])
        expect_within("mean loss vs float64", fl[2 * R:2 * R + 1], [loss.mean()], [tol.mean()])
        hits1, hits5 = int((rank < 1).sum()), int((rank < 5).sum())
        expect_bits("top1", fl[2 * R + 1:2 * R + 2], [f32(100) * f32(hits1) / f32(R)])
        expect_bits("top5", fl[2 * R + 2:2 * R + 3], [f32(100) * f32(hits5) / f32(R)])
        # dlogits = go / R * (softmax - onehot); a label outside [0, C) has no one-hot term
        k = float(f32(go) / f32(R))
        with np.errstate(invalid="ignore", over="ignore"):
            x = x32.astype(np.float64)
            p = np.exp(x - lse[:, None])
            onehot = np.zeros((R, C))
            onehot[np.arange(R)[ok], labr[ok]] = 1.0
            ref = k * (p - onehot)
            fin = lambda v: np.abs(np.nan_to_num(v, posinf=0, neginf=0))
            dtol = abs(k) * (CE_TOL * np.nan_to_num(p, nan=0) * (1 + fin(mx)[:, None] + fin(x)) + 2.0 ** -23)
        expect_within("dlogits", d.reshape(-1), ref.reshape(-1), dtol.reshape(-1))

    return Case(run, check, launches=["ce_topk_fwd_kernel"] * 2 + ["ce_bwd_kernel"] * 2,
                branch=ce_branch(x32, labn, R, C, ld))


def _nan_label(x, lab):
    x[1, lab[1 % len(lab)]] = np.nan


def _nan_column(x, lab):
    c = (lab[2 % len(lab)] + 1) % x.shape[1]
    x[2, c] = np.nan


def _all_nan(x, lab):
    x[3, :] = np.nan


def _infs(x, lab):
    x[0, lab[0]] = np.inf            # label +inf: rank 0, loss NaN (inf - inf)
    x[4, (lab[4 % len(lab)] + 1) % x.shape[1]] = np.inf
    x[5, :] = -np.inf
    x[5, lab[5 % len(lab)]] = 0.0    # only the label finite
    x[6, lab[6 % len(lab)]] = -np.inf


def _ties(x, lab):
    for r in range(0, x.shape[0], 3):
        c = lab[r % len(lab)]
        x[r, (c + 1) % x.shape[1]] = x[r, c]          # the label tied with another column
        x[r, (c + 2) % x.shape[1]] = x[r, c] + 1.0    # and one strictly above


def _bad_labels(x, lab):
    C = x.shape[1]
    lab[0], lab[1], lab[2], lab[3] = -1, C, (1 << 32) + 3, -(1 << 32) + 3


def _everything(x, lab):
    for f in (_nan_label, _nan_column, _all_nan):
        f(x, lab)
    x[7, lab[7 % len(lab)]] = -np.inf
    C = x.shape[1]
    lab[8], lab[9], lab[10], lab[11] = -1, C, (1 << 32) + 3, -(1 << 32) + 3


# ------------------------------------------------------------------------------------------------------------------
# the row table: (builder, kwargs, the branch predicates the row is meant for)
# ------------------------------------------------------------------------------------------------------------------
def _lars_rows():
    r = {}
    one = lambda n, **kw: [T(n, wd=0.25, **kw)]
    r["lars 1 chunk"] = (dict(ts=one(1000)), {"chunks": 1, "update": "vec"})
    r["lars 32 chunks"] = (dict(ts=one(32 * CHUNK)), {"chunks": 32})
    r["lars 33 chunks"] = (dict(ts=one(32 * CHUNK + 5)), {"chunks": 33})
    r["lars 65 chunks"] = (dict(ts=one(64 * CHUNK + 4097)), {"chunks": 65})
    r["lars tails 0-3, empty tensor"] = (dict(ts=[T(CHUNK + 4, wd=0.5), T(CHUNK + 5, wd=0.5, lr=0.1), T(0),
                                                  T(CHUNK + 6, wd=1.0, lr=0.05), T(7, wd=2.0, lr=0.2)]),
                                         {"tails": [0, 1, 2, 3], "empty": True, "update": "vec"})
    r["lars all misaligned"] = (dict(ts=[T(5000, wd=0.25, pp=1, pg=2, pm=3), T(300, pp=3, pg=3, pm=1, ignore=1)]),
                                {"norms": "scalar", "update": "scalar"})
    r["lars p misaligned"] = (dict(ts=[T(5001, wd=0.25, pp=2), T(77, ignore=1, pp=1)]),
                              {"norms": "scalar", "update": "scalar"})
    r["lars g misaligned"] = (dict(ts=[T(5002, wd=0.25, pg=1), T(78, ignore=1, pg=3)]),
                              {"norms": "scalar", "update": "scalar"})
    r["lars m misaligned"] = (dict(ts=[T(5003, wd=0.25, pm=2), T(79, ignore=1, pm=1), T(4096, pm=3)]),
                              {"norms": "vec", "update": "scalar"})
    r["lars ignore wd=0 and wd>0"] = (dict(ts=[T(3000, ignore=1), T(3001, ignore=1, wd=0.5, pm=1),
                                               T(3002, ignore=1, wd=0.25), T(40, ignore=1, pp=2, pg=2, pm=2)]),
                                      {"update": "both"})
    for eps in (0.0, 1e-3):
        zp, zg = T(2000, wd=0.0), T(2001, wd=0.0, pp=1, pg=1, pm=1)
        zp.zero_p, zg.grad = True, "zero"
        r["lars zero p / zero g, eps=%g" % eps] = (dict(ts=[zp, zg, T(1500, wd=0.5)], eps=eps), {})
    r["lars eps>0, no wd, scalar"] = (dict(ts=[T(9000, pp=1, pg=1, pm=1), T(9001)], eps=2.0 ** -10),
                                      {"update": "both"})
    r["lars first_step=1 (NaN momentum in)"] = (dict(ts=[T(4000, wd=0.25), T(33, ignore=1, pm=1)], first_step=True,
                                                     m_nan=True), {"first_step": True})
    r["lars no momentum"] = (dict(ts=[T(4000, wd=0.25), T(4001, pp=2, pg=2), T(10, ignore=1)], momentum=None),
                             {"momentum": False, "update": "both"})
    r["lars per-tensor lr, 3 steps"] = (dict(ts=[T(6000, wd=0.25, lr=0.3), T(10, ignore=1, lr=0.7),
                                                 T(6001, wd=0.5, lr=0.011, pm=2), T(503, lr=1.5, pp=1, pg=1, pm=1),
                                                 T(7000, lr=0.2, ignore=0)], steps=3),
                                        {"update": "both"})
    nan_g, inf_g = T(3000, wd=0.25), T(3001, wd=0.25, pm=1)
    nan_g.grad, inf_g.grad = "nan", "inf"
    r["lars non-finite gradients"] = (dict(ts=[nan_g, inf_g, T(500, wd=0.25)], steps=2), {})
    return {k: (lars_case, kw, want) for k, (kw, want) in r.items()}


def _loss_rows():
    r = {
        "loss n4 < one block": (dict(rows=8, dim=64), {"sub_block": True}),
        "loss dim % 4 != 0": (dict(rows=12, dim=37), {}),
        "loss [8, 256]": (dict(rows=8, dim=256), {"fwd_passes": 1}),
        "loss [256, 256]": (dict(rows=256, dim=256), {"fwd_passes": 1}),
        "loss [512, 256]": (dict(rows=512, dim=256), {"fwd_passes": 1}),
        "loss [512, 256] grad_out null": (dict(rows=512, dim=256, go=None), {"grad_out": False}),
        "loss [4096, 256] grid-stride": (dict(rows=4096, dim=256), {"fwd_passes": 8, "bwd_passes": 2}),
        "loss [8, 256] grad_out null": (dict(rows=8, dim=256, go=None), {"grad_out": False}),
    }
    return {k: (loss_case, kw, want) for k, (kw, want) in r.items()}


def _ce_rows():
    r = {}
    for C in (2, 5, 10, 37, 1000, 1001):
        r["ce C=%d" % C] = (dict(R=24, C=C), {"R%8": False})
    r["ce R=300 (R % 8, R > 256)"] = (dict(R=300, C=10), {"R>256": True, "R%8": True})
    r["ce R=1030, LR=515"] = (dict(R=1030, C=37, LR=515), {"R>256": True, "repeat": True})
    r["ce R=2 LR, pitched ld"] = (dict(R=16, C=10, LR=8, ld=16), {"repeat": True, "pitched": True})
    r["ce pitched ld, C=1000"] = (dict(R=40, C=1000, ld=1003), {"pitched": True})
    r["ce label tied"] = (dict(R=33, C=37, edits=_ties), {"tie": True})
    r["ce +-inf logits"] = (dict(R=8, C=10, edits=_infs), {"inf": True})
    r["ce NaN label logit"] = (dict(R=8, C=37, edits=_nan_label), {"nan_label": True})
    r["ce NaN label logit, C=2"] = (dict(R=8, C=2, edits=_nan_label), {"nan_label": True})
    r["ce NaN column"] = (dict(R=8, C=10, edits=_nan_column), {"nan_column": True})
    r["ce all-NaN row"] = (dict(R=8, C=10, edits=_all_nan), {"nan_label": True})
    r["ce labels -1, C, 2^32+3, -2^32+3"] = (dict(R=8, C=10, edits=_bad_labels), {"out_of_range": True})
    r["ce labels out of range, repeated"] = (dict(R=16, C=1000, LR=8, edits=_bad_labels),
                                             {"out_of_range": True, "repeat": True})
    r["ce everything, R=264"] = (dict(R=264, C=37, LR=132, edits=_everything),
                                 {"R>256": True, "nan_label": True, "out_of_range": True, "nan_column": True})
    return {k: (ce_case, kw, want) for k, (kw, want) in r.items()}


ROWS = {**_loss_rows(), **_lars_rows(), **_ce_rows()}


def _build(dev, name):
    return row_case(dev, name, *ROWS[name][:2])


def _check_branch(name, case):
    want = ROWS[name][2]
    wrong = {k: (case.branch.get(k), v) for k, v in want.items() if case.branch.get(k) != v}
    assert not wrong, "%s is meant for %s, the restated predicates give %s" % (name, want, case.branch)


@pytest.mark.parametrize("name", list(ROWS))
def test_row_exact(cuda, name):
    case = _build(cuda, name)
    _check_branch(name, case)
    run_and_check(case)


def _check_launches():
    """All rows in one profiler session, one after the other with a device synchronisation between them: the byol::
    kernels in device-time order must be the rows' launch lists one after the other."""
    cases = {name: _build(torch.device("cuda:0"), name) for name in ROWS}
    for case in cases.values():
        case.run()
    torch.cuda.synchronize()
    got = byol_kernel_sequence([case.run for case in cases.values()])
    if not got:
        print(NO_EVENTS)
        return
    at = 0
    for name, case in cases.items():
        seen = got[at:at + len(case.launches)]
        assert seen == case.launches, "%s: launched %s, expected %s" % (name, seen, case.launches)
        at += len(case.launches)
    assert at == len(got), "kernels after the last row: %s" % got[at:at + 8]
    print("%d rows launched their %d kernels" % (len(cases), at))


def test_rows_launch_their_kernels(cuda):
    """Every row launches exactly its kernels: loss_fwd_partial + loss_finalize + loss_bwd, lars_norms + lars_update
    per step, ce_topk_fwd twice + ce_bwd twice, and no other byol:: kernel.  Checked in a fresh Python process: one
    that has already held many profiler sessions (the rest of the GPU suite) can drop CUDA kernel events."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# the loss's small-scale limit
# ------------------------------------------------------------------------------------------------------------------
# The loss is invariant under power-of-two scaling of its four inputs in exact arithmetic, and the kernels keep that
# bit for bit: the fp32 block partials scale exactly, their fp64 block-ordered sum has relative precision, and sqrt,
# products and quotients of exactly scaled values scale exactly.  The test scales general (randn) operands by 2^-e,
# e = 0 .. SCALE_E (RMS down to ~1e-11; their squares stay fp32-normal), and asserts the same loss bits and exactly
# scaled saved scalars.  A fixed-point accumulator with absolute resolution does not have this property.  The Fix128
# sums this kernel used before (2^-50 per block addend), measured the same way on an H100 80GB HBM3 (700 W) with
# these operands, at 8x256 and at 512x256: the loss first moved (1 ulp) at an operand RMS of 8.3e-7 (2^-20.2) and by
# more than one fp32 ulp at 4.2e-7 (2^-21.2; 3 ulp, then 7 and 459 at the next two halvings).  The target projections
# z of the replayed training steps (test_replay_engine_calls_exactly) have an RMS of 3.5e-5 (2^-14.8), only 2^6.4
# above that, hence the block-ordered fp64 sum.
SCALE_E = 36


def test_loss_is_scale_invariant(cuda):
    from byol_b200 import ops
    for rows in (8, 512):
        g = torch.Generator(device=cuda).manual_seed(rows)
        q1, q2 = (torch.randn(rows, 256, generator=g, device=cuda) for _ in range(2))
        z2 = q1 * 0.5 + torch.randn(rows, 256, generator=g, device=cuda) * 0.5
        z1 = q2 * 0.5 + torch.randn(rows, 256, generator=g, device=cuda) * 0.5
        base = None
        for e in range(0, SCALE_E + 1):
            xs = [x * 2.0 ** -e for x in (q1, q2, z1, z2)]     # exact: a power of two
            ws, out = torch.empty(6, dtype=F64, device=cuda), torch.empty(7, device=cuda)
            ops.loss_fwd(*xs, ws, out[0:1], out[1:7])
            scaled = torch.cat([out[0:1], out[1:5] * 2.0 ** e, out[5:7] * 4.0 ** e]).cpu()
            if base is None:
                base = scaled
            expect_bits("%dx256 loss and saved, inputs scaled by 2^-%d" % (rows, e), scaled, base)
    print("loss bit-identical under scaling by 2^0 .. 2^-%d at 8x256 and 512x256" % SCALE_E)


# ------------------------------------------------------------------------------------------------------------------
# replay of one training step's calls
# ------------------------------------------------------------------------------------------------------------------
def _lars_signature(table, trust, eps, momentum, first_step):
    tf = table["tensor_first_chunk"].cpu().tolist()
    cl = table["chunk_len"].cpu().tolist()
    pp, gp = table["p_ptrs"].cpu().tolist(), table["g_ptrs"].cpu().tolist()
    mp = table["m_ptrs"].cpu().tolist() if table.get("m_ptrs") is not None else None
    wd, ig, lr = table["wd"].cpu().tolist(), table["ignore"].cpu().tolist(), table["lr"].cpu().tolist()
    ts = tuple((sum(cl[tf[t]:tf[t + 1]]), pp[t] % 16 // 4, gp[t] % 16 // 4, 0 if mp is None else mp[t] % 16 // 4,
                wd[t] > 0, ig[t], lr[t]) for t in range(len(wd)))
    return ("lars", ts, mp is not None, float(f32(trust)), float(f32(eps)), float(f32(momentum)), bool(first_step))


def _recorders(calls, rms):
    """ops function name -> recorder noting the call's shapes and options (for LARS: lengths and 16-byte phases)."""
    def loss_fwd(q1, q2, z1, z2, workspace, loss, saved):
        calls.add(("loss", q1.shape[0], q1.shape[1]))
        for nm, t in (("q", q1), ("q", q2), ("z", z1), ("z", z2)):
            rms[nm].append(float(t.double().pow(2).mean().sqrt()))

    def loss_bwd(q1, q2, z1, z2, saved, grad_out, dq1, dq2):
        calls.add(("loss_bwd", q1.shape[0], q1.shape[1], grad_out is not None))

    def ce_topk_fwd(logits, labels, scratch=None):
        calls.add(("ce", logits.shape[0], logits.shape[1], labels.numel(), logits.stride(0)))

    def ce_bwd(logits, labels, row_lse, grad_out):
        calls.add(("ce_bwd", logits.shape[0], logits.shape[1], labels.numel(), logits.stride(0)))

    def lars_sgd_step(table, trust_coef, eps, momentum, first_step):
        calls.add(_lars_signature(table, trust_coef, eps, momentum, first_step))
    return {k: v for k, v in locals().items() if callable(v)}


def _replay_case(dev, g, sig):
    op = sig[0]
    if op == "loss":
        return loss_case(dev, g, sig[1], sig[2])
    if op == "loss_bwd":
        return loss_case(dev, g, sig[1], sig[2], go=0.75 if sig[3] else None)
    if op in ("ce", "ce_bwd"):
        R, C, LR, ld = sig[1:]
        return ce_case(dev, g, R, C, LR=LR, ld=ld)
    if op == "lars":
        _, ts, mom, trust, eps, momentum, first = sig
        # exact operands: a power-of-two weight decay where the step has one; the recorded phases and lengths
        tensors = [T(n, wd=0.25 if wdp else 0.0, lr=lr, ignore=ig, pp=pp, pg=pg, pm=pm)
                   for n, pp, gp_, pm, wdp, ig, lr in ts for pg in (gp_,)]
        return lars_case(dev, g, tensors, momentum=momentum if mom else None, eps=eps, trust=trust,
                         first_step=first)
    raise AssertionError("no replay for %s" % (sig,))


# (arch, representation size, classes, batch, resolution, precision)
NETS = [("resnet18", 512, 1000, 8, 64, "bf16"), ("resnet:bottleneck:1,1,1,1", 2048, 10, 8, 64, "bf16"),
        ("resnet18", 512, 10, 4, 64, "fp32")]


def test_replay_engine_calls_exactly(cuda):
    calls, rms = set(), {"q": [], "z": []}
    with recording(_recorders(calls, rms)):
        for arch, rep, classes, b, r, precision in NETS:
            byol_train_step(cuda, arch, rep, b, r, classes, precision=precision, backward_precision=precision)
            torch.cuda.empty_cache()
    kinds = {sig[0] for sig in calls}
    assert kinds == {"loss", "loss_bwd", "ce", "ce_bwd", "lars"}, kinds
    phases = {(t[1], t[2], t[3]) for sig in calls if sig[0] == "lars" for t in sig[1]}
    print("LARS 16-byte phases (p, g, m) seen: %s" % sorted(phases))
    print("loss operand RMS in these steps: q %.3g .. %.3g, z %.3g .. %.3g" % (
        min(rms["q"]), max(rms["q"]), min(rms["z"]), max(rms["z"])))
    assert min(rms["q"] + rms["z"]) >= 2.0 ** -SCALE_E, "loss operands below the range test_loss_is_scale_invariant " \
        "asserts"
    replay(cuda, calls, _replay_case, 3000)
