"""GPU: the BatchNorm, pooling, layout and cast kernels bit for bit against float64, on every kernel variant.

* Exact operands.  Activations, gradients and residuals are integers in a small range (a few of them even integers in
  [256, 510], so that outputs need the bf16 round-to-nearest-even); scale, shift-side powers (rscale, gamma, invstd)
  are signed powers of two, shifts and means integers, `count` a power of two and the backward sums multiples of it.
  Every fp32 intermediate is then exact, with or without FMA contraction, so an output must equal the float64
  reference rounded once to its dtype (torch.equal; NaN matches NaN).
* The statistics -> coefficients kernels (bn_finalize_lanes, bn_eval_coeffs) take sqrt and divisions: they are
  compared bit for bit with a numpy restatement of the same fp32 / fp64 operations, in the order and with the FMA
  contractions nvcc emits for them, and with float64 within a stated ulp bound.
* Route table.  One row per (kernel, variant, options) at the edge of its host predicate (fixed_grid in csrc/bn.cu,
  the 2x2-block max-pool backward in csrc/elementwise.cu); one test checks under torch.profiler that each row
  launches the kernel named for it and no other variant of the same kernel family.
* Replay.  One eager training step of a few small nets records the engine's own calls of these kernels (shapes and
  options only; byol_avgpool_fwd at the ops.lib level, where the engine calls it) and replays every distinct call with
  exact operands.
"""
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.exact import (Case, byol_train_step, check_in_fresh_process, check_row_launches, expect, expect_same,
                         recording, replay, row_case, run_and_check)
from tests.util import _fma32, fma32, fma64, gen, ints, pack_bits, pow2, unpack_bits

pytestmark = pytest.mark.gpu
BF, F32, F64, U8 = torch.bfloat16, torch.float32, torch.float64, torch.uint8


# ------------------------------------------------------------------------------------------------------------------
# operands and comparison
# ------------------------------------------------------------------------------------------------------------------
def acts(shape, dev, g, amp=4, big=0.05):
    """fp64 integers in [-amp, amp]; a fraction `big` of them even integers of either sign in [256, 510] (exact in
    bf16, while their sums with small integers are not: the bf16 output rounding is exercised)."""
    v = ints(shape, dev, g, amp)
    if big:
        b = 2.0 * torch.randint(128, 256, shape, generator=g, device=dev).to(F64)
        b = b * (torch.randint(0, 2, shape, generator=g, device=dev) * 2 - 1)
        v = torch.where(torch.rand(shape, generator=g, device=dev) < big, b, v)
    return v


def _fine(shape, dev, g, amp=4):
    """fp64 integers in [-amp, amp] plus multiples of 2^-14: 17 significant bits, more than two bf16 planes hold."""
    return ints(shape, dev, g, amp) + torch.randint(0, 1 << 14, shape, generator=g, device=dev).to(F64) * 2.0 ** -14


def _pos2(n, dev, g):
    return pow2(n, dev, g)


# ------------------------------------------------------------------------------------------------------------------
# the host's kernel choice, restated
# ------------------------------------------------------------------------------------------------------------------
def fixed_grid(nvec, groups):
    """csrc/bn.cu fixed_grid: > 0 when every thread of the grid can stay on one 8-channel group."""
    unit = groups // 256 if groups > 256 else 1
    if (groups % 256 != 0) if groups > 256 else (256 % groups != 0):
        return 0
    b = min((nvec + 255) // 256, 132 * 8)
    return max(-(-b // unit) * unit, unit)


def maxpool_bwd_fast(h, w, k, s, p):
    """byol_maxpool_bwd: the 2x2-block kernel serves k3 / s2 / p1 with H = 2 Ho and W = 2 Wo."""
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    return k == 3 and s == 2 and p == 1 and h == 2 * ho and w == 2 * wo


_K = r"(?<![A-Za-z0-9_])"      # kernel names: no longer name may end in the pattern
ROUTE_KERNEL = {
    "apply_fixed_ff": _K + r"bn_apply_fixed_kernel<false,false>",
    "apply_fixed_tf": _K + r"bn_apply_fixed_kernel<true,false>",
    "apply_fixed_tt": _K + r"bn_apply_fixed_kernel<true,true>",
    "apply_generic": _K + r"bn_apply_kernel",
    "finalize": _K + r"bn_finalize_lanes_kernel",
    "eval": _K + r"bn_eval_coeffs_kernel",
    "maxpool": _K + r"maxpool_fwd_kernel",
    "bnpool_idx": _K + r"bn_relu_maxpool_fwd_kernel",
    "bnpool_noidx": _K + r"bn_relu_maxpool_fwd_noidx_kernel",
    "pool_bwd_k3s2": _K + r"maxpool_bwd_k3s2_kernel",
    "pool_bwd_generic": _K + r"maxpool_bwd_kernel",
    "avgpool_fwd": _K + r"avgpool_fwd_kernel",
    "avgpool_bwd": _K + r"avgpool_bwd_kernel",
    "avgpool_f32": _K + r"avgpool_f32_kernel",
    "avgpool_bwd_f32": _K + r"avgpool_bwd_f32_kernel",
    "nhwc8": _K + r"nchw_to_nhwc8_kernel",
    "stem4": _K + r"nchw_to_stem4_kernel",
    "cast": _K + r"cast_f32_bf16_kernel",
    "cast2d": _K + r"cast_f32_bf16_2d_kernel",
    "subsample2": _K + r"subsample2_kernel",
    "apply_f32": _K + r"bn_apply_f32_kernel",
    "maxpool_f32": _K + r"maxpool_f32_kernel",
    "maxpool_bwd_f32": _K + r"maxpool_bwd_f32_kernel",
    "finalize_f64": _K + r"bn_finalize_lanes_f64_kernel",
    "split_planes": _K + r"split_planes_kernel",
    "nchw_to_planes": _K + r"nchw_to_planes_kernel",
    "prep_weight_planes": _K + r"prep_weight_planes_kernel",
    "prep_weight_dgrad_planes": _K + r"prep_weight_dgrad_planes_kernel",
}
for _m in range(4):
    ROUTE_KERNEL["bwd_apply_fixed%d" % _m] = _K + r"bn_bwd_apply_fixed_kernel<%d>" % _m
    ROUTE_KERNEL["bwd_apply_generic%d" % _m] = _K + r"bn_bwd_apply_kernel<%d>" % _m
    ROUTE_KERNEL["reduce_fixed%d" % _m] = _K + r"bn_bwd_reduce_fixed_kernel<%d>" % _m
    ROUTE_KERNEL["reduce_rows%d" % _m] = _K + r"bn_bwd_reduce_kernel<%d>" % _m
    ROUTE_KERNEL["bwd_apply_f32_%d" % _m] = _K + r"bn_bwd_apply_f32_kernel<%d>" % _m
# kernels with more than one variant: every launched kernel of the family must be the row's variant
FAMILY = [_K + r"bn_apply(_fixed)?_kernel", _K + r"bn_bwd_apply(_fixed)?_kernel", _K + r"bn_bwd_reduce(_fixed)?_kernel",
          _K + r"bn_relu_maxpool_fwd(_noidx)?_kernel", _K + r"maxpool_bwd(_k3s2)?_kernel"]


# ------------------------------------------------------------------------------------------------------------------
# BatchNorm
# ------------------------------------------------------------------------------------------------------------------
def bn_apply_case(dev, g, m, c, resid=None, relu=False, mask=False, out=True, out_f32=False):
    """y = act(x*scale + shift (+ r | r*rscale + rshift)); resid None / "plain" / "affine"; any of y, y_f32, mask."""
    from byol_b200 import ops
    x, sc, sh = acts((m, c), dev, g), pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    r = acts((m, c), dev, g) if resid else None
    rs, rb = (pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)) if resid == "affine" else (None, None)
    xd, rd = x.to(BF), (r.to(BF) if resid else None)
    f = [t.float() if t is not None else None for t in (sc, sh, rs, rb)]

    def run():
        y = torch.empty((m, c), dtype=BF, device=dev) if out else None
        y32 = torch.empty((m, c), dtype=F32, device=dev) if out_f32 else None
        mo = torch.full((m * c // 8,), 0xA5, dtype=U8, device=dev) if mask else None
        ops.bn_apply(xd, f[0], f[1], relu, resid=rd, rscale=f[2], rshift=f[3], out=y, out_f32=y32, mask_out=mo)
        return [y, y32, mo]

    def check(outs):
        y, y32, mo = outs
        ref = x * sc + sh
        if resid:
            ref = ref + (r * rs + rb if resid == "affine" else r)
        if relu:
            ref = torch.relu(ref)
        if out:
            expect("y", y, ref)
        if out_f32:
            expect("y_f32", y32, ref)
        if mask:
            assert torch.equal(unpack_bits(mo, (m, c)), ref > 0), "mask_out differs"

    fixed = out and not out_f32 and fixed_grid(m * c // 8, c // 8) > 0
    route = "apply_fixed_" + {None: "ff", "plain": "tf", "affine": "tt"}[resid] if fixed else "apply_generic"
    return Case(run, check, route)


def _bwd_operands(dev, g, m, c, mask_mode):
    x, gr = acts((m, c), dev, g), acts((m, c), dev, g, 3)
    mean, invstd, gamma = ints((c,), dev, g, 3), _pos2(c, dev, g), pow2(c, dev, g, signed=True)
    scale, shift = pow2(c, dev, g, signed=True), ints((c,), dev, g, 2)
    act = keep = None
    if mask_mode == 1:
        keep = x * scale + shift > 0
    elif mask_mode == 2:
        act = ints((m, c), dev, g, 2)
        keep = act > 0
        act = act.to(BF)
    elif mask_mode == 3:
        keep = torch.rand((m, c), generator=g, device=dev) > 0.4
        act = pack_bits(keep)
    coeffs = torch.stack([scale, shift, mean, invstd]).float()
    dz = gr * keep if keep is not None else gr
    return x, gr, mean, invstd, gamma, coeffs, act, dz


def bn_bwd_apply_case(dev, g, m, c, mask_mode, dz_out=False, grads=False, count=1024):
    """dy = gamma*invstd*(dz - s1/n - xhat*s2/n) with n = count (a power of two independent of m) and s1, s2 multiples
    of it.  grads: dgamma / dbeta from two calls (the two online lanes) with rank-local sums s12_local != s12, added
    onto one zeroed gradient."""
    from byol_b200 import ops
    x, gr, mean, invstd, gamma, coeffs, act, dz = _bwd_operands(dev, g, m, c, mask_mode)
    s1, s2 = count * ints((c,), dev, g, 2), count * ints((c,), dev, g, 2)
    loc = [ints((2 * c,), dev, g, 50) for _ in range(2)]
    xd, gd, gf = x.to(BF), gr.to(BF), gamma.float()
    s12 = torch.cat([s1, s2]).float()

    def run():
        dy = torch.empty((m, c), dtype=BF, device=dev)
        dzo = torch.empty((m, c), dtype=BF, device=dev) if dz_out else None
        dg = db = None
        if grads:
            dg, db = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
            for lo in loc:
                ops.bn_bwd_apply(gd, xd, coeffs, gf, s12, count, mask_mode, act=act, dy=dy, dz_out=dzo,
                                 s12_local=lo.float(), dgamma=dg, dbeta=db)
        else:
            ops.bn_bwd_apply(gd, xd, coeffs, gf, s12, count, mask_mode, act=act, dy=dy, dz_out=dzo)
        return [dy, dzo, dg, db]

    def check(outs):
        dy, dzo, dg, db = outs
        xhat = (x - mean) * invstd
        expect("dy", dy, gamma * invstd * (dz - s1 / count - xhat * s2 / count))
        if dz_out:
            expect("dz", dzo, dz)
        if grads:
            expect("dgamma", dg, loc[0][c:] + loc[1][c:])
            expect("dbeta", db, loc[0][:c] + loc[1][:c])

    fixed = fixed_grid(m * c // 8, c // 8) > 0
    return Case(run, check, ("bwd_apply_fixed%d" if fixed else "bwd_apply_generic%d") % mask_mode)


def bn_bwd_reduce_case(dev, g, m, c, mask_mode):
    """s12 += [sum dz, sum dz * (x - mean) * invstd] (fixed-point sums: exact in any order)."""
    from byol_b200 import ops
    x, gr = ints((m, c), dev, g, 4), ints((m, c), dev, g, 3)
    mean, invstd = ints((c,), dev, g, 2), _pos2(c, dev, g)
    scale, shift = pow2(c, dev, g, signed=True), ints((c,), dev, g, 2)
    keep, act = None, None
    if mask_mode == 1:
        keep = x * scale + shift > 0
    elif mask_mode == 2:
        a = ints((m, c), dev, g, 2)
        keep, act = a > 0, a.to(BF)
    elif mask_mode == 3:
        keep = torch.rand((m, c), generator=g, device=dev) > 0.4
        act = pack_bits(keep)
    coeffs = torch.stack([scale, shift, mean, invstd]).float()
    xd, gd = x.to(BF), gr.to(BF)

    def run():
        s12 = torch.zeros(2 * c, device=dev)
        ops.bn_bwd_reduce(gd, xd, coeffs, s12, mask_mode, act=act)
        return [s12]

    def check(outs):
        dz = gr * keep if keep is not None else gr
        expect("s12", outs[0], torch.cat([dz.sum(0), (dz * (x - mean) * invstd).sum(0)]))

    fixed = fixed_grid(m * c // 8, c // 8) > 0
    return Case(run, check, ("reduce_fixed%d" if fixed else "reduce_rows%d") % mask_mode)


# --- statistics -> coefficients: numpy restatement of the compiled arithmetic ------------------------------------
def finalize_restated(stats, count, gammas, betas, rm, rv, momentum, eps):
    """bn_finalize_lanes_kernel as compiled (fp64 statistics, fp32 coefficients; nvcc contracts
    q/n - mean^2, beta - mean*scale and both running-statistic updates into FMAs)."""
    C = gammas[0].size
    mom, eps32 = np.float32(momentum), np.float32(eps)
    one_m = np.float32(1) - mom
    co = []
    rm, rv = rm.copy(), rv.copy()
    for l in range(len(gammas)):
        st = stats[l * 2 * C:(l + 1) * 2 * C].astype(np.float64)
        mean = st[:C] / count
        var = np.maximum(fma64(-mean, mean, st[C:] / count), 0.0)
        invstd = (1.0 / np.sqrt(var + np.float64(eps32))).astype(np.float32)
        sc = gammas[l] * invstd
        mean32 = mean.astype(np.float32)
        shift = _fma32(-sc, mean32, betas[l])
        unb = var * count / (count - 1.0) if count > 1 else var
        rm = _fma32(rm, np.full(C, one_m), mom * mean32)
        rv = _fma32(rv, np.full(C, one_m), mom * unb.astype(np.float32))
        co.append(np.stack([sc, shift, mean32, invstd]))
    return np.stack(co), rm, rv


def eval_restated(gamma, beta, rm, rv, eps):
    """bn_eval_coeffs_kernel as compiled: fp32 IEEE sqrt and division, shift = fma(-scale, running_mean, beta)."""
    invstd = np.float32(1) / np.sqrt(rv + np.float32(eps))
    sc = gamma * invstd
    return sc, _fma32(-sc, rm, beta)


def _ulps(got, exact):
    """|got - exact| in units of the fp32 ulp of exact."""
    exact = np.asarray(exact, dtype=np.float64)
    ulp = np.spacing(np.abs(exact).astype(np.float32)).astype(np.float64)
    return np.abs(got.astype(np.float64) - exact) / ulp


def finalize_case(dev, g, c, lanes, count, momentum=0.1, eps=1e-5):
    """Coefficients and running statistics of `lanes` lock-step lanes from general fp32 sums (|mean| / std <= 3)."""
    from byol_b200 import ops
    cnt = float(count)
    mean = torch.randn((lanes, c), generator=g, device=dev, dtype=F64)
    var = torch.rand((lanes, c), generator=g, device=dev, dtype=F64) * 2 + 0.1
    stats = torch.cat([torch.cat([mean[l] * cnt, (var[l] + mean[l] ** 2) * cnt]) for l in range(lanes)]).float()
    gammas = [torch.randn(c, generator=g, device=dev) for _ in range(lanes)]
    betas = [torch.randn(c, generator=g, device=dev) for _ in range(lanes)]
    rm0, rv0 = torch.randn(c, generator=g, device=dev), torch.rand(c, generator=g, device=dev) + 0.5

    def run():
        rm, rv = rm0.clone(), rv0.clone()
        co = torch.empty((lanes, 4, c), device=dev)
        ops.bn_finalize_lanes(stats, cnt, gammas, betas, rm, rv, momentum, eps, co)
        return [co, rm, rv]

    def check(outs):
        co, rm, rv = [t.cpu().numpy() for t in outs]
        st = stats.cpu().numpy()
        want, wrm, wrv = finalize_restated(st, cnt, [t.cpu().numpy() for t in gammas],
                                           [t.cpu().numpy() for t in betas], rm0.cpu().numpy(), rv0.cpu().numpy(),
                                           momentum, eps)
        for name, a, b in (("coeffs", co, want), ("running_mean", rm, wrm), ("running_var", rv, wrv)):
            bad = a.view(np.uint32) != b.view(np.uint32)
            assert not bad.any(), "%s: %d of %d values differ from the restatement (first at %s: %r vs %r)" % (
                name, int(bad.sum()), bad.size, np.argwhere(bad)[0].tolist(), a[bad][0], b[bad][0])
        # float64: invstd within 1 ulp of the exact value for these sums (no cancellation here), the scale within 2,
        # the shift within 3 ulps of the larger of |beta| and |mean * scale|
        for l in range(lanes):
            s = st[l * 2 * c:(l + 1) * 2 * c].astype(np.float64)
            m64 = s[:c] / cnt
            inv64 = 1.0 / np.sqrt(s[c:] / cnt - m64 * m64 + np.float64(np.float32(eps)))
            gam = gammas[l].cpu().numpy().astype(np.float64)
            assert _ulps(co[l, 3], inv64).max() <= 1.0, "invstd further than 1 ulp from float64"
            assert _ulps(co[l, 0], gam * inv64).max() <= 2.0, "scale further than 2 ulps from float64"
            sh64 = betas[l].cpu().numpy().astype(np.float64) - m64 * gam * inv64
            scale_of = np.maximum(np.abs(betas[l].cpu().numpy()), np.abs(m64 * gam * inv64))
            assert (np.abs(co[l, 1] - sh64) / np.spacing(scale_of.astype(np.float32))).max() <= 3.0, \
                "shift further than 3 ulps from float64"

    return Case(run, check, "finalize")


def finalize_f64_restated(stats, count, gammas, betas, rm, rv, momentum, eps):
    """bn_finalize_lanes_f64_kernel as compiled: fp64 mean, var = fma(-mean, mean, q/n) clamped at 0, invstd =
    fp32(1 / sqrt(var + eps)) with IEEE fp64 sqrt and division, scale = gamma * invstd in fp32, shift =
    fp32(fma(-mean, scale, beta)) in fp64; unbiased = var * n / (n - 1) (var when n <= 1); the running statistics
    rm = fma(rm, 1 - m, m * mean) and rv = fma(rv, 1 - m, m * unbiased) in fp32 (rm, rv None: not kept)."""
    C = gammas[0].size
    mom = np.float32(momentum)
    one_m = np.float32(1) - mom
    rm = np.zeros(C, np.float32) if rm is None else rm.copy()
    rv = np.zeros(C, np.float32) if rv is None else rv.copy()
    co = []
    for l in range(len(gammas)):
        st = stats[l * 2 * C:(l + 1) * 2 * C]
        mean = st[:C] / count
        var = np.maximum(fma64(-mean, mean, st[C:] / count), 0.0)
        invstd = (1.0 / np.sqrt(var + np.float64(np.float32(eps)))).astype(np.float32)
        sc = gammas[l] * invstd
        shift = fma64(-mean, sc.astype(np.float64), betas[l].astype(np.float64)).astype(np.float32)
        mean32 = mean.astype(np.float32)
        unb = var * count / (count - 1.0) if count > 1 else var
        rm = fma32(rm, one_m, mom * mean32)
        rv = fma32(rv, one_m, mom * unb.astype(np.float32))
        co.append(np.stack([sc, shift, mean32, invstd]))
    return np.stack(co), rm, rv


def finalize_f64_case(dev, g, c, lanes, count, running=True, negvar=False, momentum=0.1, eps=1e-5):
    """bn_finalize_lanes_f64 (the fp32 path) from fp64 sums; negvar: a few channels whose sums give a variance just
    below zero (clamped)."""
    from byol_b200 import ops
    cnt = float(count)
    mean = torch.randn((lanes, c), generator=g, device=dev, dtype=F64)
    var = torch.rand((lanes, c), generator=g, device=dev, dtype=F64) * 2 + 0.1
    q = (var + mean ** 2) * cnt
    if negvar:
        q[:, :5] = mean[:, :5] ** 2 * cnt * (1 - 2.0 ** -40)
    stats = torch.cat([torch.cat([mean[l] * cnt, q[l]]) for l in range(lanes)])
    gammas = [torch.randn(c, generator=g, device=dev) for _ in range(lanes)]
    betas = [torch.randn(c, generator=g, device=dev) for _ in range(lanes)]
    rm0, rv0 = torch.randn(c, generator=g, device=dev), torch.rand(c, generator=g, device=dev) + 0.5

    def run():
        rm, rv = (rm0.clone(), rv0.clone()) if running else (None, None)
        co = torch.empty((lanes, 4, c), device=dev)
        ops.bn_finalize_lanes_f64(stats, cnt, gammas, betas, rm, rv, momentum, eps, co)
        return [co, rm, rv]

    def check(outs):
        co, rm, rv = [None if t is None else t.cpu().numpy() for t in outs]
        st = stats.cpu().numpy()
        want, wrm, wrv = finalize_f64_restated(st, cnt, [t.cpu().numpy() for t in gammas],
                                               [t.cpu().numpy() for t in betas], rm0.cpu().numpy(),
                                               rv0.cpu().numpy(), momentum, eps)
        if negvar:
            m64 = st[:c] / cnt
            assert (fma64(-m64[:5], m64[:5], st[c:c + 5] / cnt) < 0).all(), "no negative variance to clamp"
        checks = [("coeffs", co, want)] + ([("running_mean", rm, wrm), ("running_var", rv, wrv)] if running else [])
        for name, a, b in checks:
            bad = a.view(np.uint32) != b.view(np.uint32)
            assert not bad.any(), "%s: %d of %d values differ from the restatement (first at %s: %r vs %r)" % (
                name, int(bad.sum()), bad.size, np.argwhere(bad)[0].tolist(), a[bad][0], b[bad][0])

    return Case(run, check, "finalize_f64")


def eval_case(dev, g, c, eps=1e-5):
    from byol_b200 import ops
    gamma, beta = torch.randn(c, generator=g, device=dev), torch.randn(c, generator=g, device=dev)
    rm, rv = torch.randn(c, generator=g, device=dev), torch.rand(c, generator=g, device=dev) * 4 + 1e-3

    def run():
        co = torch.full((2, c), float("nan"), device=dev)
        ops.bn_eval_coeffs(gamma, beta, rm, rv, eps, co)
        return [co]

    def check(outs):
        co = outs[0].cpu().numpy()
        sc, sh = eval_restated(*[t.cpu().numpy() for t in (gamma, beta, rm, rv)], eps)
        assert (co[0].view(np.uint32) == sc.view(np.uint32)).all(), "eval scale differs from the restatement"
        assert (co[1].view(np.uint32) == sh.view(np.uint32)).all(), "eval shift differs from the restatement"
        inv64 = 1.0 / np.sqrt(rv.cpu().numpy().astype(np.float64) + np.float64(np.float32(eps)))
        assert _ulps(co[0], gamma.cpu().numpy().astype(np.float64) * inv64).max() <= 3.0, \
            "eval scale further than 3 ulps from float64"

    return Case(run, check, "eval")


# ------------------------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------------------------
def _with_edges(x, k, s, p):
    """x [n, h, w, c] fp64 integers with the pooling edges added: an all-negative corner region, NaNs, and a top-left
    window whose in-image values are all -inf (its argmax is the first in-image position, as in ATen)."""
    x = x.clone()
    x[0, :3, :3, :] = -1.0 - x[0, :3, :3, :].abs()
    x[-1, 1, 1, 3] = float("nan")
    x[-1, 2, 2, 3] = float("nan")
    x[-1, 0, 0, 5] = float("nan")
    x[0, :k - p, :k - p, 8:16] = float("-inf")
    return x


def aten_pool(x64, k, s, p):
    """float64 NHWC -> (values NHWC, flat input index h*W + w NHWC) of torch.nn.functional.max_pool2d."""
    y, i = F.max_pool2d(x64.permute(0, 3, 1, 2), k, s, p, return_indices=True)
    return y.permute(0, 2, 3, 1), i.permute(0, 2, 3, 1)


def flat_index(idx, w, k, s, p):
    """window position (kh*k + kw) -> flat input index ih*W + iw, as ATen reports it."""
    n, ho, wo, c = idx.shape
    i = idx.long()
    oh = torch.arange(ho, device=idx.device).view(1, -1, 1, 1)
    ow = torch.arange(wo, device=idx.device).view(1, 1, -1, 1)
    return (oh * s - p + i // k) * w + (ow * s - p + i % k)


def maxpool_case(dev, g, n, h, w, c, k, s, p, edges=False, fp32=False):
    """maxpool_fwd (bf16) / maxpool_f32: small integers (ties everywhere: the first maximum in scan order wins)."""
    from byol_b200 import ops
    x = ints((n, h, w, c), dev, g, 3)
    if edges:
        x = _with_edges(x, k, s, p)
    xd = x.float() if fp32 else x.to(BF)

    def run():
        return list(ops.maxpool_f32(xd, k, s, p) if fp32 else ops.maxpool_fwd(xd, k, s, p))

    def check(outs):
        y, idx = outs
        ry, ri = aten_pool(x, k, s, p)
        expect("y", y, ry)
        fi = flat_index(idx, w, k, s, p)
        bad = fi != ri
        assert not bad.any(), "argmax differs at %d of %d outputs (first %s: %d vs ATen %d)" % (
            int(bad.sum()), bad.numel(), bad.nonzero()[0].tolist(), int(fi[bad][0]), int(ri[bad][0]))

    return Case(run, check, "maxpool_f32" if fp32 else "maxpool")


def bnpool_case(dev, g, n, h, w, c, k, s, p, want_idx):
    """bn_relu_maxpool_fwd == bn_apply(relu) then maxpool_fwd, values and argmax bit for bit; values also against
    float64 (scales of both signs: many windows are all zeros after the ReLU)."""
    from byol_b200 import ops
    x, sc, sh = acts((n, h, w, c), dev, g), pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    x[-1, 1, 1, 3] = float("nan")         # NaN * scale + shift -> fmaxf(NaN, 0) = 0 on both paths
    xd, scf, shf = x.to(BF), sc.float(), sh.float()

    def run():
        return list(ops.bn_relu_maxpool_fwd(xd, scf, shf, k, s, p, want_idx=want_idx))

    def check(outs):
        y, idx = outs
        a = ops.bn_apply(xd.view(-1, c), scf, shf, True).view(n, h, w, c)
        y2, i2 = ops.maxpool_fwd(a, k, s, p)
        expect_same("y vs bn_apply + maxpool_fwd", y, y2)
        if want_idx:
            assert torch.equal(idx, i2), "argmax differs from bn_apply + maxpool_fwd"
        a64 = torch.relu(torch.nan_to_num(x * sc + sh, nan=0.0)).float().to(BF).to(F64)
        expect("y", y, aten_pool(a64, k, s, p)[0])

    return Case(run, check, "bnpool_idx" if want_idx else "bnpool_noidx")


def pool_bwd_case(dev, g, n, h, w, c, k, s, p, fp32=False):
    """maxpool_bwd (bf16: 2x2-block or generic kernel) / maxpool_bwd_f32 against a float64 scatter-add of the saved
    argmax (overlapping windows add onto one pixel)."""
    from byol_b200 import ops
    x = _with_edges(ints((n, h, w, c), dev, g, 3), k, s, p)
    ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
    dy = ints((n, ho, wo, c), dev, g, 3)
    if fp32:
        _, idx = ops.maxpool_f32(x.float(), k, s, p)
        dyd = dy.float()
    else:
        _, idx = ops.maxpool_fwd(x.to(BF), k, s, p)
        dyd = dy.to(BF)

    def run():
        return [(ops.maxpool_bwd_f32 if fp32 else ops.maxpool_bwd)(dyd, idx, h, w, k, s, p)]

    def check(outs):
        fi = flat_index(idx, w, k, s, p).permute(0, 3, 1, 2).reshape(n, c, -1)
        assert bool(((fi >= 0) & (fi < h * w)).all()), "a saved argmax points outside the image"
        ref = torch.zeros((n, c, h * w), dtype=F64, device=dev)
        ref.scatter_add_(2, fi, dy.permute(0, 3, 1, 2).reshape(n, c, -1))
        expect("dx", outs[0], ref.view(n, c, h, w).permute(0, 2, 3, 1))

    if fp32:
        return Case(run, check, "maxpool_bwd_f32")
    return Case(run, check, "pool_bwd_k3s2" if maxpool_bwd_fast(h, w, k, s, p) else "pool_bwd_generic")


def _times_inv(v32, hw):
    """RN(v * RN(1/HW)) in fp32: the bf16 path's averaging (an exact power of two when HW is one)."""
    return v32 * (torch.ones((), dtype=F32) / hw).to(v32.device)


def avgpool_case(dev, g, n, h, w, c, want_f32=True, want_bf16=True):
    """avgpool_fwd: fp32 sums of bf16 integers (exact), times fl(1/HW) -> fp32 RN(sum * RN(1/HW)), bf16 of that."""
    from byol_b200 import ops
    x = acts((n, h, w, c), dev, g)
    xd = x.to(BF)

    def run():
        return list(ops.avgpool_fwd(xd, want_f32, want_bf16))

    def check(outs):
        yf, yb = outs
        sm = x.sum((1, 2))
        want = _times_inv(sm.float(), h * w)
        if (h * w) & (h * w - 1) == 0:
            assert torch.equal(want.to(F64), sm / (h * w))        # a power of two: the average itself
        if want_f32:
            expect_same("y_f32", yf, want)
        if want_bf16:
            expect_same("y_bf16", yb, want.to(BF))

    return Case(run, check, "avgpool_fwd")


def avgpool_bwd_case(dev, g, n, h, w, c, ga=True, gb=True):
    """avgpool_bwd: dx = bf16(RN((g_a + g_b) * RN(1/HW))), g_a bf16, g_b fp32, either absent."""
    from byol_b200 import ops
    a, b = acts((n, c), dev, g), ints((n, c), dev, g, 5)
    ad, bf = (a.to(BF) if ga else None), (b.float() if gb else None)

    def run():
        return [ops.avgpool_bwd(ad, bf, n, h, w, c)]

    def check(outs):
        v = (a if ga else 0) + (b if gb else 0)
        want = _times_inv(v.float(), h * w).to(BF)
        expect_same("dx", outs[0], want.view(n, 1, 1, c).expand(n, h, w, c).contiguous())

    return Case(run, check, "avgpool_bwd")


def avgpool_f32_case(dev, g, n, h, w, c):
    """avgpool_f32: fp32 sum (exact for integers) divided by HW -> RN(sum / HW)."""
    from byol_b200 import ops
    x = acts((n, h, w, c), dev, g)
    xf = x.float()

    def run():
        return [ops.avgpool_f32(xf)]

    def check(outs):
        want = x.sum((1, 2)).float().cpu() / float(h * w)       # IEEE fp32 division
        expect_same("y", outs[0].cpu(), want)

    return Case(run, check, "avgpool_f32")


def avgpool_bwd_f32_case(dev, g, n, h, w, c, ga=True, gb=True):
    from byol_b200 import ops
    a, b = acts((n, c), dev, g).float(), ints((n, c), dev, g, 5).float()

    def run():
        return [ops.avgpool_bwd_f32(a if ga else None, b if gb else None, n, h, w, c)]

    def check(outs):
        v = ((a if ga else 0) + (b if gb else 0)).cpu() / float(h * w)
        expect_same("dx", outs[0].cpu(), v.view(n, 1, 1, c).expand(n, h, w, c).contiguous())

    return Case(run, check, "avgpool_bwd_f32")


# ------------------------------------------------------------------------------------------------------------------
# layout and casts
# ------------------------------------------------------------------------------------------------------------------
def _special_f32(dev, n, g):
    """fp32 values at the edges of the bf16 rounding: ties to even both ways, the largest finite values, both sides of
    0x7F7F8000 (the smallest finite value that rounds to inf) and FLT_MAX, +-inf, NaN, fp32 subnormals (which bf16
    keeps), signed zeros, values whose third split plane x2 is a bf16 subnormal (exact down to 2^-110, inexact below),
    and random normals."""
    one = 1.0
    sp = [one + 2 ** -8, one + 3 * 2 ** -8, -(one + 2 ** -8), 256 + 1, 256 + 3, 2 ** 126 * (1 + 2 ** -8),
          3.3895313892515355e38, 3.3961e38, float("inf"), float("-inf"), float("nan"), 2 ** -130, 2 ** -149,
          3 * 2 ** -140, -(2 ** -133) * (1 + 2 ** -8), 2 ** -126 * (1 - 2 ** -8), 0.0, -0.0, 1.0 + 2 ** -9 + 2 ** -20,
          2 ** -110 * (1 + 2 ** -9 + 2 ** -23), -(2 ** -108) * (1 + 2 ** -5 + 2 ** -13 + 2 ** -21),
          2 ** -111 * (1 + 2 ** -23), -(2 ** -115) * (1 + 2 ** -3 + 2 ** -17 + 2 ** -22)]
    bits = [0x7F7F7FFF, 0x7F7F8000, 0x7F7F8001, 0x7F7FC000, 0x7F7FFFFF]
    big = torch.tensor(bits, dtype=torch.int32).view(F32)
    v = torch.randn(n, generator=g, device=dev, dtype=F32)
    sp = torch.cat([torch.tensor(sp, dtype=F32), big, -big])
    v[:len(sp)] = sp[:n].to(dev)
    return v


def _bits_equal(got, want):
    """bf16 bit patterns equal (any NaN matches any NaN)."""
    gn, wn = torch.isnan(got), torch.isnan(want)
    return torch.equal(gn, wn) and torch.equal(got.view(torch.int16)[~gn], want.view(torch.int16)[~wn])


def cast_case(dev, g, n):
    from byol_b200 import ops
    x = _special_f32(dev, n, g)

    def run():
        return [ops.cast_bf16(x)]

    def check(outs):
        assert _bits_equal(outs[0], x.to(BF)), "cast_bf16 differs from tensor.to(torch.bfloat16)"

    return Case(run, check, "cast")


def cast2d_case(dev, g, rows, cols, ldx, ldy, guard=256):
    """byol_cast_f32_bf16_2d: rows of pitch ldx -> bf16 rows of pitch ldy, padding columns zero, nothing written
    outside the [rows, ldy] output (guard bands keep their value)."""
    from byol_b200 import ops
    big = _special_f32(dev, rows * ldx, g).view(rows, ldx)
    x = big[:, :cols]

    def run():
        buf = torch.full((guard + rows * ldy + guard,), 7.0, dtype=BF, device=dev)   # padding too must be written
        ops.check(ops.lib.byol_cast_f32_bf16_2d(x.data_ptr(), buf[guard:].data_ptr(), rows, cols, ldx, ldy,
                                                ops._stream()), "byol_cast_f32_bf16_2d")
        return [buf]

    def check(outs):
        buf = outs[0]
        y = buf[guard:guard + rows * ldy].view(rows, ldy)
        assert _bits_equal(y[:, :cols].contiguous(), x.to(BF)), "cast_bf16_pitched data differs"
        assert bool((y[:, cols:].float() == 0).all()) and not torch.signbit(y[:, cols:].float()).any(), \
            "cast_bf16_pitched padding columns not +0"
        assert bool((buf[:guard] == 7).all() and (buf[guard + rows * ldy:] == 7).all()), \
            "cast_bf16_pitched wrote outside its output"

    return Case(run, check, "cast2d")


def nhwc8_case(dev, g, n, cin, h, w):
    from byol_b200 import ops
    x = _special_f32(dev, n * cin * h * w, g).view(n, cin, h, w)

    def run():
        out = torch.full((n, h, w, 8), float("nan"), dtype=BF, device=dev)
        return [ops.nchw_to_nhwc8(x, out=out)]

    def check(outs):
        want = torch.zeros((n, h, w, 8), dtype=BF, device=dev)
        want[..., :cin] = x.permute(0, 2, 3, 1).to(BF)
        assert _bits_equal(outs[0], want), "nchw_to_nhwc8 differs (data or zero padding channels)"

    return Case(run, check, "nhwc8")


def stem4_case(dev, g, n, cin, h, w):
    from byol_b200 import ops
    x = _special_f32(dev, n * cin * h * w, g).view(n, cin, h, w)
    wp = ops.lib.byol_stem4_row_pixels()

    def run():
        out = torch.full((n, h + 6, wp, 4), float("nan"), dtype=BF, device=dev)
        return [ops.nchw_to_stem4(x, out=out)]

    def check(outs):
        want = torch.zeros((n, h + 6, wp, 4), dtype=BF, device=dev)
        want[:, 3:3 + h, 3:3 + w, :cin] = x.permute(0, 2, 3, 1).to(BF)
        assert _bits_equal(outs[0], want), "nchw_to_stem4 differs (data, padding rows / pixels or channels)"

    return Case(run, check, "stem4")


def subsample2_case(dev, g, n, h, w, c):
    from byol_b200 import ops
    x = acts((n, h, w, c), dev, g)
    xd = x.to(BF)

    def run():
        return [ops.subsample2(xd)]

    def check(outs):
        expect("y", outs[0], x[:, ::2, ::2, :])

    return Case(run, check, "subsample2")


# ------------------------------------------------------------------------------------------------------------------
# fp32 path
# ------------------------------------------------------------------------------------------------------------------
# the plane of each term (csrc/split.cu make_pattern): activation side (A) and weight side (B)
PATTERN = {3: (0, 0, 1), 6: (0, 0, 1, 1, 0, 2)}
WPATTERN = {3: (0, 1, 0), 6: (0, 1, 0, 1, 2, 0)}
EXACT_FROM = 2.0 ** -110     # the planes sum back to x for every finite |x| >= this (test_split_algebra)


def _split3(o32):
    """split3 (csrc/split.cu): x0 = bf16(x), or the largest finite bf16 of x's sign when a finite x rounds to inf;
    x1 = bf16(x - x0), x2 = bf16(x - x0 - x1).  +-inf gives (+-inf, NaN, NaN), NaN three NaNs."""
    p0 = o32.to(BF)
    over = torch.isinf(p0) & torch.isfinite(o32)
    p0 = torch.where(over, (torch.sign(o32) * torch.finfo(BF).max).to(BF), p0)
    r1 = o32 - p0.float()
    p1 = r1.to(BF)
    return p0, p1, (r1 - p1.float()).to(BF)


def _check_plane_stack(name, got, x, pattern):
    """got [R, T, C] bf16 planes of the fp32 values x [R, C] in `pattern`: each plane equals the restated split, and
    where the pattern holds all three planes, they sum back to every finite x with |x| >= 2^-110 (or 0)."""
    pl = _split3(x)
    for j, a in enumerate(pattern):
        expect_same("%s plane %d" % (name, j), got[:, j].contiguous(), pl[a])
    if 2 in pattern:
        back = sum(got[:, pattern.index(a)].double() for a in range(3))
        keep = torch.isfinite(x) & ((x.abs() >= EXACT_FROM) | (x == 0))
        assert torch.equal(back[keep], x.double()[keep]), "%s: the planes do not sum back to the fp32 value" % name


def _check_planes(name, planes, o32, T):
    m, c = o32.shape
    _check_plane_stack(name, planes.view(m, T, c), o32, PATTERN[T])


def _is_pos_zero(t):
    return bool((t.view(torch.int16) == 0).all())


def split_planes_case(dev, g, m, c, T, cpad=None, ldx=None, copy=False, guard=256):
    """byol_split_planes: fp32 rows of pitch ldx -> bf16 [m, T*cpad], column j*cpad + c = plane PATTERN[j] of x[:, c],
    padding channels c >= C +0 in every plane; the optional bf16 copy is x0.  Nothing is written outside the outputs."""
    from byol_b200 import ops
    cpad, ldx = cpad or c, ldx or c
    big = torch.full((m, ldx), float("nan"), device=dev)
    big[:, :c] = _special_f32(dev, m * c, g).view(m, c)
    x = big[:, :c]

    def run():
        buf = torch.full((2 * guard + m * T * cpad,), float("nan"), dtype=BF, device=dev)
        cbuf = torch.full((2 * guard + m * c,), float("nan"), dtype=BF, device=dev) if copy else None
        ops.check(ops.lib.byol_split_planes(x.data_ptr(), buf[guard:].data_ptr(),
                                            cbuf[guard:].data_ptr() if copy else 0, m, c, cpad, ldx, T,
                                            ops._stream()), "byol_split_planes")
        return [buf, cbuf]

    def check(outs):
        buf, cbuf = outs
        got = buf[guard:guard + m * T * cpad].view(m, T, cpad)
        _check_plane_stack("planes", got[..., :c], x, PATTERN[T])
        assert _is_pos_zero(got[..., c:]), "split_planes: padding channels not +0"
        guards = [buf[:guard], buf[guard + m * T * cpad:]]
        if copy:
            expect_same("copy", cbuf[guard:guard + m * c].view(m, c), _split3(x)[0])
            guards += [cbuf[:guard], cbuf[guard + m * c:]]
        assert all(bool(torch.isnan(t).all()) for t in guards), "split_planes wrote outside its outputs"

    return Case(run, check, "split_planes")


def nchw_to_planes_case(dev, g, n, cin, h, w, T, cpad=8):
    """byol_nchw_to_planes: fp32 NCHW -> bf16 NHWC [n, h, w, T*cpad], channel j*cpad + c = plane PATTERN[j] of x[:, c],
    channels c >= cin +0 in every plane."""
    from byol_b200 import ops
    x = _special_f32(dev, n * cin * h * w, g).view(n, cin, h, w)

    def run():
        out = torch.full((n, h, w, T * cpad), float("nan"), dtype=BF, device=dev)
        return [ops.nchw_to_planes(x, T, cpad, out=out)]

    def check(outs):
        got = outs[0].view(-1, T, cpad)
        _check_plane_stack("planes", got[..., :cin], x.permute(0, 2, 3, 1).reshape(-1, cin), PATTERN[T])
        assert _is_pos_zero(got[..., cin:]), "nchw_to_planes: padding channels not +0"

    return Case(run, check, "nchw_to_planes")


def prep_weight_planes_case(dev, g, cout, cin, taps, T, cpad=None):
    """byol_prep_weight_planes: fp32 [cout, cin, taps] -> bf16 [cout, taps*T*cpad], column (tap*T + j)*cpad + c =
    plane WPATTERN[j] of w[co, c, tap], channels c >= cin +0."""
    from byol_b200 import ops
    cpad = cpad or cin
    w = _special_f32(dev, cout * cin * taps, g).view(cout, cin, taps)

    def run():
        out = torch.full((cout, taps * T * cpad), float("nan"), dtype=BF, device=dev)
        return [ops.prep_weight_planes(w, T, cpad, out)]

    def check(outs):
        got = outs[0].view(cout, taps, T, cpad)
        _check_plane_stack("planes", got[..., :cin].reshape(-1, T, cin), w.permute(0, 2, 1).reshape(-1, cin),
                           WPATTERN[T])
        assert _is_pos_zero(got[..., cin:]), "prep_weight_planes: padding channels not +0"

    return Case(run, check, "prep_weight_planes")


def prep_weight_dgrad_planes_case(dev, g, cout, cin, taps, T):
    """byol_prep_weight_dgrad_planes: fp32 [cout, cin, taps] -> bf16 [cin, taps*T*cout], column (tap*T + j)*cout + co
    = plane WPATTERN[j] of w[co, ci, tap]."""
    from byol_b200 import ops
    w = _special_f32(dev, cout * cin * taps, g).view(cout, cin, taps)

    def run():
        out = torch.full((cin, taps * T * cout), float("nan"), dtype=BF, device=dev)
        return [ops.prep_weight_dgrad_planes(w, T, out)]

    def check(outs):
        got = outs[0].view(cin * taps, T, cout)
        _check_plane_stack("dgrad planes", got, w.permute(1, 2, 0).reshape(-1, cout), WPATTERN[T])

    return Case(run, check, "prep_weight_dgrad_planes")


def apply_f32_case(dev, g, m, c, T, out32=True, planes=True, copy=False, mask=False, resid=None, relu=True):
    """bn_apply_f32: o = act(y*scale + shift (+ residual)) exact in fp32 (17-bit operands); every output subset."""
    from byol_b200 import ops
    y, sc, sh = _fine((m, c), dev, g), pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    r = _fine((m, c), dev, g) if resid else None
    rs, rb = (pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)) if resid == "affine" else (None, None)
    f = [t.float() if t is not None else None for t in (y, sc, sh, r, rs, rb)]

    def run():
        return list(ops.bn_apply_f32(f[0], f[1], f[2], relu, T, resid=f[3], rscale=f[4], rshift=f[5],
                                     want_out32=out32, want_planes=planes, want_copy=copy, want_mask=mask))

    def check(outs):
        o32, pl, cp, mk = outs
        ref = y * sc + sh
        if resid:
            ref = ref + (r * rs + rb if resid == "affine" else r)
        if relu:
            ref = torch.relu(ref)
        ref32 = ref.float()
        assert torch.equal(ref32.double(), ref), "operands not exact in fp32"
        if out32:
            expect("out32", o32, ref)
        if planes:
            _check_planes("planes", pl, ref32, T)
        if copy:
            expect_same("copy", cp, ref32.to(BF))
        if mask:
            assert torch.equal(unpack_bits(mk, (m, c)), ref > 0), "mask differs"

    return Case(run, check, "apply_f32")


def bwd_apply_f32_case(dev, g, m, c, mask_mode, T, want_f32=True, want_planes=True, want_dz=True, count=1024):
    """bn_bwd_apply_f32 with s12_local != s12 (two lanes onto one zeroed dgamma / dbeta)."""
    from byol_b200 import ops
    y, gr = _fine((m, c), dev, g), _fine((m, c), dev, g, 3)
    mean, invstd, gamma = ints((c,), dev, g, 3), _pos2(c, dev, g), pow2(c, dev, g, signed=True)
    scale, shift = pow2(c, dev, g, signed=True), ints((c,), dev, g, 2)
    keep = mk = None
    if mask_mode == 1:
        keep = y * scale + shift > 0
    elif mask_mode == 3:
        keep = torch.rand((m, c), generator=g, device=dev) > 0.4
        mk = pack_bits(keep)
    coeffs = torch.stack([scale, shift, mean, invstd]).float()
    s12 = count * torch.cat([ints((c,), dev, g, 2), ints((c,), dev, g, 2)])
    loc = [ints((2 * c,), dev, g, 50) for _ in range(2)]
    yf, gf, gam = y.float(), gr.float(), gamma.float()

    def run():
        dg, db = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        for lo in loc:
            out = ops.bn_bwd_apply_f32(gf, yf, coeffs, gam, s12, count, mask_mode, T, mask=mk, want_planes=want_planes,
                                       want_f32=want_f32, want_dz=want_dz, s12_local=lo, dgamma=dg, dbeta=db)
        return list(out) + [dg, db]

    def check(outs):
        pl, d32, dz, dg, db = outs
        dzr = gr * keep if keep is not None else gr
        ref = gamma * invstd * (dzr - s12[:c] / count - (y - mean) * invstd * s12[c:] / count)
        assert torch.equal(ref.float().double(), ref), "operands not exact in fp32"
        if want_f32:
            expect("dy32", d32, ref)
        if want_planes:
            _check_planes("dy planes", pl, ref.float(), T)
        if want_dz:
            expect("dz", dz, dzr)
        expect("dgamma", dg, loc[0][c:] + loc[1][c:])
        expect("dbeta", db, loc[0][:c] + loc[1][:c])

    return Case(run, check, "bwd_apply_f32_%d" % mask_mode)


# ------------------------------------------------------------------------------------------------------------------
# the route table
# ------------------------------------------------------------------------------------------------------------------
A, BA, R, FN = bn_apply_case, bn_bwd_apply_case, bn_bwd_reduce_case, finalize_case
MP, BP, PB = maxpool_case, bnpool_case, pool_bwd_case
ROWS = {
    # bn_apply, fixed kernel: 256 % (C/8) == 0 (C = 64: 8 groups; C = 2048: 256 groups) or C/8 a multiple of 256
    "apply_fixed": ("apply_fixed_ff", A, dict(m=300, c=64)),
    "apply_fixed_relu_mask": ("apply_fixed_ff", A, dict(m=300, c=64, relu=True, mask=True)),
    "apply_fixed_resid": ("apply_fixed_tf", A, dict(m=300, c=64, resid="plain")),
    "apply_fixed_resid_relu_mask": ("apply_fixed_tf", A, dict(m=40, c=2048, resid="plain", relu=True, mask=True)),
    "apply_fixed_affine": ("apply_fixed_tt", A, dict(m=300, c=64, resid="affine")),
    "apply_fixed_affine_relu_mask": ("apply_fixed_tt", A, dict(m=20, c=4096, resid="affine", relu=True,
                                                               mask=True)),
    # generic kernel: C/8 neither divides 256 nor is a multiple of it, or an fp32 output is asked for
    "apply_generic_c96": ("apply_generic", A, dict(m=300, c=96, relu=True, mask=True)),
    "apply_generic_c200_resid": ("apply_generic", A, dict(m=300, c=200, resid="plain", relu=True, mask=True)),
    "apply_generic_c4800_affine": ("apply_generic", A, dict(m=24, c=4800, resid="affine", relu=True, mask=True)),
    "apply_generic_out_f32_only": ("apply_generic", A, dict(m=300, c=64, relu=True, out=False, out_f32=True)),
    "apply_generic_out_and_f32": ("apply_generic", A, dict(m=300, c=64, resid="affine", relu=True, mask=True,
                                                           out_f32=True)),
    "finalize_l1": ("finalize", FN, dict(c=200, lanes=1, count=4096)),
    "finalize_l2": ("finalize", FN, dict(c=64, lanes=2, count=37)),
    "finalize_l3": ("finalize", FN, dict(c=136, lanes=3, count=1)),
    "finalize_l4": ("finalize", FN, dict(c=4096, lanes=4, count=512)),
    "eval_coeffs": ("eval", eval_case, dict(c=200)),
    # max-pool: the ResNet stem pool on even and odd sizes, stride 1, and 2x2 / s2 without padding
    "maxpool_k3s2p1_even": ("maxpool", MP, dict(n=2, h=16, w=12, c=64, k=3, s=2, p=1, edges=True)),
    "maxpool_k3s2p1_odd": ("maxpool", MP, dict(n=2, h=15, w=13, c=64, k=3, s=2, p=1, edges=True)),
    "maxpool_k3s1p1": ("maxpool", MP, dict(n=2, h=9, w=10, c=64, k=3, s=1, p=1, edges=True)),
    "maxpool_k2s2p0": ("maxpool", MP, dict(n=2, h=10, w=9, c=64, k=2, s=2, p=0, edges=True)),
    "maxpool_f32_k3s2p1_even": ("maxpool_f32", MP, dict(n=2, h=16, w=12, c=24, k=3, s=2, p=1, edges=True,
                                                         fp32=True)),
    "maxpool_f32_k3s2p1_odd": ("maxpool_f32", MP, dict(n=2, h=15, w=13, c=24, k=3, s=2, p=1, edges=True,
                                                       fp32=True)),
    "maxpool_f32_k3s1p1": ("maxpool_f32", MP, dict(n=2, h=9, w=10, c=24, k=3, s=1, p=1, edges=True, fp32=True)),
    "maxpool_f32_k2s2p0": ("maxpool_f32", MP, dict(n=2, h=10, w=9, c=24, k=2, s=2, p=0, edges=True, fp32=True)),
    "maxpool_bwd_k3s2_56": ("pool_bwd_k3s2", PB, dict(n=2, h=56, w=56, c=64, k=3, s=2, p=1)),
    "maxpool_bwd_k3s2_16x10": ("pool_bwd_k3s2", PB, dict(n=2, h=16, w=10, c=64, k=3, s=2, p=1)),
    "maxpool_bwd_k3s2_odd": ("pool_bwd_generic", PB, dict(n=2, h=15, w=13, c=64, k=3, s=2, p=1)),
    "maxpool_bwd_k3s1p1": ("pool_bwd_generic", PB, dict(n=2, h=9, w=10, c=64, k=3, s=1, p=1)),
    "maxpool_bwd_k2s2p0": ("pool_bwd_generic", PB, dict(n=2, h=10, w=9, c=64, k=2, s=2, p=0)),
    "maxpool_bwd_f32_k3s2p1": ("maxpool_bwd_f32", PB, dict(n=2, h=16, w=12, c=24, k=3, s=2, p=1, fp32=True)),
    "maxpool_bwd_f32_k3s1p1": ("maxpool_bwd_f32", PB, dict(n=2, h=9, w=10, c=24, k=3, s=1, p=1, fp32=True)),
    "maxpool_bwd_f32_k2s2p0": ("maxpool_bwd_f32", PB, dict(n=2, h=10, w=9, c=24, k=2, s=2, p=0, fp32=True)),
    "avgpool_f32out_hw1": ("avgpool_fwd", avgpool_case, dict(n=3, h=1, w=1, c=64, want_bf16=False)),
    "avgpool_bf16out_hw16": ("avgpool_fwd", avgpool_case, dict(n=3, h=4, w=4, c=64, want_f32=False)),
    "avgpool_hw49": ("avgpool_fwd", avgpool_case, dict(n=3, h=7, w=7, c=64)),
    "avgpool_hw64": ("avgpool_fwd", avgpool_case, dict(n=3, h=8, w=8, c=2048)),
    "avgpool_hw144": ("avgpool_fwd", avgpool_case, dict(n=3, h=12, w=12, c=64)),
    "avgpool_bwd_a_hw1": ("avgpool_bwd", avgpool_bwd_case, dict(n=3, h=1, w=1, c=64, gb=False)),
    "avgpool_bwd_b_hw16": ("avgpool_bwd", avgpool_bwd_case, dict(n=3, h=4, w=4, c=64, ga=False)),
    "avgpool_bwd_ab_hw49": ("avgpool_bwd", avgpool_bwd_case, dict(n=3, h=7, w=7, c=64)),
    "avgpool_bwd_ab_hw64": ("avgpool_bwd", avgpool_bwd_case, dict(n=3, h=8, w=8, c=512)),
    "avgpool_bwd_ab_hw144": ("avgpool_bwd", avgpool_bwd_case, dict(n=3, h=12, w=12, c=64)),
    "avgpool_f32_hw1": ("avgpool_f32", avgpool_f32_case, dict(n=3, h=1, w=1, c=24)),
    "avgpool_f32_hw16": ("avgpool_f32", avgpool_f32_case, dict(n=3, h=4, w=4, c=24)),
    "avgpool_f32_hw49": ("avgpool_f32", avgpool_f32_case, dict(n=3, h=7, w=7, c=24)),
    "avgpool_f32_hw64": ("avgpool_f32", avgpool_f32_case, dict(n=3, h=8, w=8, c=24)),
    "avgpool_f32_hw144": ("avgpool_f32", avgpool_f32_case, dict(n=3, h=12, w=12, c=24)),
    "avgpool_bwd_f32_a_hw49": ("avgpool_bwd_f32", avgpool_bwd_f32_case, dict(n=3, h=7, w=7, c=24, gb=False)),
    "avgpool_bwd_f32_b_hw16": ("avgpool_bwd_f32", avgpool_bwd_f32_case, dict(n=3, h=4, w=4, c=24, ga=False)),
    "avgpool_bwd_f32_ab_hw144": ("avgpool_bwd_f32", avgpool_bwd_f32_case, dict(n=3, h=12, w=12, c=24)),
    "cast": ("cast", cast_case, dict(n=1001)),
    "cast2d_cout10": ("cast2d", cast2d_case, dict(rows=96, cols=10, ldx=10, ldy=16)),
    "cast2d_pitched": ("cast2d", cast2d_case, dict(rows=37, cols=13, ldx=29, ldy=24)),
    "subsample2": ("subsample2", subsample2_case, dict(n=2, h=14, w=10, c=72)),
    "stem4_cin3": ("stem4", stem4_case, dict(n=2, cin=3, h=20, w=18)),
    "stem4_cin1_w256": ("stem4", stem4_case, dict(n=1, cin=1, h=6, w=256)),
    "stem4_cin4": ("stem4", stem4_case, dict(n=1, cin=4, h=8, w=10)),
    "apply_f32_t3_all": ("apply_f32", apply_f32_case, dict(m=40, c=64, T=3, copy=True, mask=True, resid="affine")),
    "apply_f32_t6_all": ("apply_f32", apply_f32_case, dict(m=40, c=64, T=6, copy=True, mask=True, resid="plain")),
    "apply_f32_out32_only": ("apply_f32", apply_f32_case, dict(m=40, c=24, T=3, planes=False, relu=False)),
    "apply_f32_t6_planes_only": ("apply_f32", apply_f32_case, dict(m=40, c=24, T=6, out32=False)),
    "apply_f32_copy_mask": ("apply_f32", apply_f32_case, dict(m=40, c=24, T=6, out32=False, planes=False,
                                                              copy=True, mask=True, resid="affine")),
}
for _c in range(1, 9):
    ROWS["nhwc8_cin%d" % _c] = ("nhwc8", nhwc8_case, dict(n=2, cin=_c, h=5, w=7))
# fp32 path statistics -> coefficients: lanes 1 to 4, with and without running statistics, count 1 (unbiased =
# biased variance), and the var < 0 clamp
ROWS["finalize_f64_l1"] = ("finalize_f64", finalize_f64_case, dict(c=200, lanes=1, count=4096))
ROWS["finalize_f64_l2_no_running"] = ("finalize_f64", finalize_f64_case, dict(c=64, lanes=2, count=37, running=False))
ROWS["finalize_f64_l3_count1"] = ("finalize_f64", finalize_f64_case, dict(c=136, lanes=3, count=1))
ROWS["finalize_f64_l4_negvar"] = ("finalize_f64", finalize_f64_case, dict(c=264, lanes=4, count=512, negvar=True))
# fp32 path plane producers at T = 3 and 6
for _T in (3, 6):
    ROWS["split_planes_t%d" % _T] = ("split_planes", split_planes_case, dict(m=40, c=64, T=_T))
    ROWS["split_planes_cpad_ldx_copy_t%d" % _T] = ("split_planes", split_planes_case, dict(m=37, c=10, T=_T, cpad=16,
                                                                                          ldx=13, copy=True))
    ROWS["nchw_to_planes_cin3_t%d" % _T] = ("nchw_to_planes", nchw_to_planes_case, dict(n=2, cin=3, h=9, w=7, T=_T))
    for _taps, _cin, _cpad in ((1, 40, 40), (9, 24, 32), (49, 3, 8)):
        ROWS["prep_weight_planes_taps%d_cpad%d_t%d" % (_taps, _cpad, _T)] = (
            "prep_weight_planes", prep_weight_planes_case, dict(cout=16, cin=_cin, taps=_taps, T=_T, cpad=_cpad))
    ROWS["prep_weight_dgrad_planes_t%d" % _T] = ("prep_weight_dgrad_planes", prep_weight_dgrad_planes_case,
                                                  dict(cout=24, cin=16, taps=9, T=_T))
for _m in range(4):
    # fixed (C = 64, 2048) and generic (C = 96, 200) kernels, each mask mode with and without dz_out, and with the
    # parameter gradients of two lanes from rank-local sums
    ROWS["bwd_apply_fixed_m%d" % _m] = ("bwd_apply_fixed%d" % _m, BA, dict(m=300, c=64, mask_mode=_m))
    ROWS["bwd_apply_fixed_m%d_dz_grads" % _m] = ("bwd_apply_fixed%d" % _m, BA, dict(m=40, c=2048, mask_mode=_m,
                                                                                    dz_out=True, grads=True))
    ROWS["bwd_apply_generic_m%d" % _m] = ("bwd_apply_generic%d" % _m, BA, dict(m=300, c=96, mask_mode=_m))
    ROWS["bwd_apply_generic_m%d_dz_grads" % _m] = ("bwd_apply_generic%d" % _m, BA, dict(m=300, c=200, mask_mode=_m,
                                                                                        dz_out=True, grads=True))
for _m in (1, 3):
    ROWS["reduce_fixed_m%d" % _m] = ("reduce_fixed%d" % _m, R, dict(m=3000, c=64, mask_mode=_m))
    ROWS["reduce_fixed_m%d_c2048" % _m] = ("reduce_fixed%d" % _m, R, dict(m=50, c=2048, mask_mode=_m))
    ROWS["reduce_rows_m%d" % _m] = ("reduce_rows%d" % _m, R, dict(m=3000, c=96, mask_mode=_m))
    ROWS["reduce_rows_m%d_c200" % _m] = ("reduce_rows%d" % _m, R, dict(m=300, c=200, mask_mode=_m))
for _name, _kw in (("k3s2p1_even", dict(n=2, h=16, w=12, k=3, s=2, p=1)), ("k3s2p1_odd", dict(n=2, h=15, w=13, k=3,
                                                                                               s=2, p=1)),
                   ("k3s1p1", dict(n=2, h=9, w=10, k=3, s=1, p=1)), ("k2s2p0", dict(n=2, h=10, w=9, k=2, s=2, p=0))):
    ROWS["bnpool_idx_" + _name] = ("bnpool_idx", BP, dict(c=64, want_idx=True, **_kw))
    ROWS["bnpool_noidx_" + _name] = ("bnpool_noidx", BP, dict(c=64, want_idx=False, **_kw))
for _m, _T in ((0, 6), (1, 3), (3, 6)):
    ROWS["bwd_apply_f32_m%d_t%d" % (_m, _T)] = ("bwd_apply_f32_%d" % _m, bwd_apply_f32_case, dict(m=40, c=64,
                                                                                               mask_mode=_m, T=_T))
ROWS["bwd_apply_f32_planes_only"] = ("bwd_apply_f32_3", bwd_apply_f32_case, dict(m=40, c=24, mask_mode=3, T=3,
                                                                                 want_f32=False, want_dz=False))


def _build(dev, name):
    return row_case(dev, name, *ROWS[name][1:])


@pytest.mark.parametrize("name", list(ROWS))
def test_row_exact(cuda, name):
    run_and_check(_build(cuda, name))


def _check_launches():
    cases = {name: _build(torch.device("cuda:0"), name) for name in ROWS}

    def complaints(name, launched):
        case, want = cases[name], ROWS[name][0]
        wrong = []
        if case.route != want:
            wrong.append("%s: the restated host predicate gives %s, the row is meant for %s" % (name, case.route, want))
        if not any(re.search(ROUTE_KERNEL[want], k) for k in launched):
            wrong.append("%s: expected %s, launched %s" % (name, ROUTE_KERNEL[want], sorted(set(launched))))
        for fam in FAMILY:
            if re.search(fam, ROUTE_KERNEL[want].replace(_K, "")):
                other = [k for k in launched if re.search(fam, k) and not re.search(ROUTE_KERNEL[want], k)]
                if other:
                    wrong.append("%s: also launched %s" % (name, sorted(set(other))))
        return wrong
    check_row_launches({name: case.run for name, case in cases.items()}, complaints)


def test_rows_launch_their_kernels(cuda):
    """Each row runs the kernel named for it (the restated host predicate agrees), and no other variant of it.
    Checked in a fresh Python process: one that has already held many profiler sessions (the rest of the GPU suite)
    can drop CUDA kernel events."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# rounding records: the two average pools, and variance cancellation in bn_finalize
# ------------------------------------------------------------------------------------------------------------------
def test_avgpool_roundings_of_the_two_paths(cuda):
    """The bf16 path averages as RN(sum * RN(1/HW)), the fp32 path as RN(sum / HW): equal for power-of-two HW, at
    most 1 fp32 ulp apart otherwise (both outputs of the same integer sums)."""
    from byol_b200 import ops
    g = gen(cuda, 3)
    for hw in (1, 16, 49, 64, 144):
        x = acts((64, hw, 1, 256), cuda, g)
        a = ops.avgpool_fwd(x.to(BF), True, False)[0]
        b = ops.avgpool_f32(x.float())
        ulps = _ulps(a.cpu().numpy(), b.cpu().numpy().astype(np.float64))
        differ = int((a != b).sum())
        print("avgpool HW=%d: %d of %d averages differ between the bf16 and fp32 paths, by at most %.0f ulp"
              % (hw, differ, a.numel(), ulps.max()))
        if hw & (hw - 1) == 0:
            assert differ == 0
        assert ulps.max() <= 1.0


# Variance cancellation.  bn_finalize gets the sums as fp32 and takes var = E[x^2] - mean^2, so the relative invstd
# error grows as (mean/std)^2: <= 2^-24 * (2 (mean/std)^2 + 2) from the rounding of the two sums.  Measured on an
# H100 80GB HBM3 (700 W), 4096 bf16 rows x 64 channels: 1.9e-6 at |mean|/std = 10, 6.4e-5 at 51, 2.4e-4 at 103,
# 9.2e-4 at 197 (0.47 of half a bf16 ulp, 2^-9), 3.2e-3 at 452: half a bf16 ulp is first exceeded between 200 and
# 500.  The engine's BatchNorm inputs stay far below that (|mean| / sqrt(var + eps) <= 6.7 in the replayed steps).
CANCEL_RATIOS = (10, 20, 50, 100, 200, 500, 1000)


def test_finalize_variance_cancellation(cuda):
    from byol_b200 import ops
    g = gen(cuda, 11)
    m, c = 4096, 64
    first_over = None
    for r in CANCEL_RATIOS:
        x = (torch.randn((m, c), generator=g, device=cuda, dtype=F64) + r).to(BF)
        stats = torch.zeros(2 * c, device=cuda)
        ops.bn_stats(x, stats)
        co = torch.empty((1, 4, c), device=cuda)
        one, zero = torch.ones(c, device=cuda), torch.zeros(c, device=cuda)
        ops.bn_finalize_lanes(stats, m, [one], [zero], None, None, 0.1, 1e-5, co)
        x64 = x.to(F64)
        inv64 = 1.0 / torch.sqrt(x64.var(0, unbiased=False) + float(np.float32(1e-5)))
        ratio = float((x64.mean(0).abs() / x64.std(0, unbiased=False)).max())
        err = float((co[0, 3].double() / inv64 - 1).abs().max())
        print("|mean|/std %7.1f: max relative invstd error %.3e = %.3f bf16 half-ulps (bound %.3e)"
              % (ratio, err, err / 2 ** -9, 2 ** -24 * (2 * ratio ** 2 + 2)))
        assert err <= 2 ** -24 * (2 * ratio ** 2 + 2), "invstd error above the fp32-sum bound"
        if first_over is None and err > 2 ** -9:
            first_over = r
    print("invstd error first exceeds half a bf16 ulp at |mean|/std = %s" % first_over)
    assert first_over is None or first_over >= 50, "cancellation costs bf16 accuracy below |mean|/std = 50"


# ------------------------------------------------------------------------------------------------------------------
# replay of the engine's own calls
# ------------------------------------------------------------------------------------------------------------------
def _shape(t):
    return None if t is None else tuple(t.shape)


def _recorders(calls, ratios):
    """ops function name -> recorder noting the call's shapes and options (not its data)."""
    def bn_apply(x2d, scale, shift, relu, resid=None, rscale=None, rshift=None, out=None, out_f32=None, mask_out=None):
        kind = None if resid is None else "affine" if rscale is not None else "plain"
        calls.add(("bn_apply", x2d.shape[0], x2d.shape[1], kind, bool(relu), mask_out is not None,
                   out is not None or out_f32 is None, out_f32 is not None))

    def bn_bwd_apply(g, x, coeffs, gamma, s12, count, mask_mode, act=None, dy=None, dz_out=None, s12_local=None,
                     dgamma=None, dbeta=None):
        calls.add(("bn_bwd_apply", x.shape[0], x.shape[1], mask_mode, dz_out is not None, dgamma is not None))

    def bn_bwd_reduce(g, x, coeffs, s12, mask_mode, act=None):
        calls.add(("bn_bwd_reduce", x.shape[0], x.shape[1], mask_mode))

    def bn_finalize_lanes(stats, count, gammas, betas, running_mean, running_var, momentum, eps, coeffs):
        c = gammas[0].numel()
        calls.add(("bn_finalize_lanes", c, len(gammas), float(count)))
        # the invstd error of the fp32 sums is ~ 2^-24 mean^2 / (var + eps): eps bounds it for constant channels
        st = stats[:len(gammas) * 2 * c].view(-1, 2, c).double()
        mean = st[:, 0] / count
        ratios.append(float((mean.abs() / (st[:, 1] / count - mean * mean + eps).clamp_min(eps).sqrt()).max()))

    def bn_eval_coeffs(gamma, beta, running_mean, running_var, eps, coeffs):
        calls.add(("bn_eval_coeffs", gamma.numel()))

    def bn_relu_maxpool_fwd(x, scale, shift, k=3, s=2, p=1, want_idx=True):
        calls.add(("bn_relu_maxpool_fwd", _shape(x), k, s, p, bool(want_idx)))

    def maxpool_bwd(dy, idx, h, w, k=3, s=2, p=1):
        calls.add(("maxpool_bwd", dy.shape[0], h, w, dy.shape[3], k, s, p))

    def avgpool_bwd(g_bf16, g_f32, n, h, w, c):
        calls.add(("avgpool_bwd", n, h, w, c, g_bf16 is not None, g_f32 is not None))

    def subsample2(x):
        calls.add(("subsample2", _shape(x)))

    def cast_bf16(x, out=None):
        calls.add(("cast_bf16", x.numel()))

    def cast_bf16_pitched(x2d, ldy):
        calls.add(("cast_bf16_pitched", x2d.shape[0], x2d.shape[1], x2d.stride(0), ldy))

    def nchw_to_nhwc8(x, out=None):
        calls.add(("nchw_to_nhwc8", _shape(x)))

    def nchw_to_stem4(x, out=None):
        calls.add(("nchw_to_stem4", _shape(x)))

    def bn_apply_f32(y2d, scale, shift, relu, T, resid=None, rscale=None, rshift=None, want_out32=False,
                     want_planes=True, want_copy=False, want_mask=False):
        kind = None if resid is None else "affine" if rscale is not None else "plain"
        calls.add(("bn_apply_f32", y2d.shape[0], y2d.shape[1], T, kind, bool(relu), bool(want_out32),
                   bool(want_planes), bool(want_copy), bool(want_mask)))

    def bn_bwd_apply_f32(g, y, coeffs, gamma, s12, count, mask_mode, T, mask=None, want_planes=True, want_f32=False,
                         want_dz=False, s12_local=None, dgamma=None, dbeta=None):
        calls.add(("bn_bwd_apply_f32", y.shape[0], y.shape[1], mask_mode, T, bool(want_planes), bool(want_f32),
                   bool(want_dz)))

    def maxpool_f32(x, k=3, s=2, p=1, want_idx=True):
        calls.add(("maxpool_f32", _shape(x), k, s, p))

    def maxpool_bwd_f32(dy, idx, h, w, k=3, s=2, p=1):
        calls.add(("maxpool_bwd_f32", dy.shape[0], h, w, dy.shape[3], k, s, p))

    def avgpool_f32(x):
        calls.add(("avgpool_f32", _shape(x)))

    def avgpool_bwd_f32(ga, gb, n, h, w, c):
        calls.add(("avgpool_bwd_f32", n, h, w, c, ga is not None, gb is not None))

    def lib_avgpool_fwd(x, yf, yb, n, hw, c, stream):       # the engine calls the library entry directly
        calls.add(("avgpool_fwd", n, hw, c, bool(yf), bool(yb)))
    recs = {k: v for k, v in locals().items() if callable(v) and k not in ("calls", "ratios", "lib_avgpool_fwd")}
    recs["lib.byol_avgpool_fwd"] = lib_avgpool_fwd
    return recs


def _replay_case(dev, g, sig):
    """Case of one recorded call, replayed with exact operands of the same shapes and options."""
    op, a = sig[0], sig[1:]
    if op == "bn_apply":
        m, c, kind, relu, mask, out, out_f32 = a
        return bn_apply_case(dev, g, m, c, resid=kind, relu=relu, mask=mask, out=out, out_f32=out_f32)
    if op == "bn_bwd_apply":
        m, c, mode, dz, grads = a
        return bn_bwd_apply_case(dev, g, m, c, mode, dz_out=dz, grads=grads)
    if op == "bn_bwd_reduce":
        return bn_bwd_reduce_case(dev, g, *a)
    if op == "bn_finalize_lanes":
        c, lanes, count = a
        return finalize_case(dev, g, c, lanes, count)
    if op == "bn_eval_coeffs":
        return eval_case(dev, g, a[0])
    if op == "bn_relu_maxpool_fwd":
        (n, h, w, c), k, s, p, idx = a
        return bnpool_case(dev, g, n, h, w, c, k, s, p, idx)
    if op == "maxpool_bwd":
        return pool_bwd_case(dev, g, *a)
    if op == "avgpool_fwd":
        n, hw, c, yf, yb = a
        return avgpool_case(dev, g, n, hw, 1, c, want_f32=yf, want_bf16=yb)
    if op == "avgpool_bwd":
        n, h, w, c, ga, gb = a
        return avgpool_bwd_case(dev, g, n, h, w, c, ga=ga, gb=gb)
    if op == "subsample2":
        return subsample2_case(dev, g, *a[0])
    if op == "cast_bf16":
        return cast_case(dev, g, a[0])
    if op == "cast_bf16_pitched":
        return cast2d_case(dev, g, *a)
    if op == "nchw_to_nhwc8":
        n, cin, h, w = a[0]
        return nhwc8_case(dev, g, n, cin, h, w)
    if op == "nchw_to_stem4":
        n, cin, h, w = a[0]
        return stem4_case(dev, g, n, cin, h, w)
    if op == "bn_apply_f32":
        m, c, T, kind, relu, o32, planes, copy, mask = a
        return apply_f32_case(dev, g, m, c, T, out32=o32, planes=planes, copy=copy, mask=mask, resid=kind, relu=relu)
    if op == "bn_bwd_apply_f32":
        m, c, mode, T, planes, f32, dz = a
        return bwd_apply_f32_case(dev, g, m, c, mode, T, want_f32=f32, want_planes=planes, want_dz=dz)
    if op == "maxpool_f32":
        (n, h, w, c), k, s, p = a
        return maxpool_case(dev, g, n, h, w, c, k, s, p, fp32=True)
    if op == "maxpool_bwd_f32":
        return pool_bwd_case(dev, g, *a, fp32=True)
    if op == "avgpool_f32":
        n, h, w, c = a[0]
        return avgpool_f32_case(dev, g, n, h, w, c)
    if op == "avgpool_bwd_f32":
        n, h, w, c, ga, gb = a
        return avgpool_bwd_f32_case(dev, g, n, h, w, c, ga=ga, gb=gb)
    raise AssertionError("no replay for %s" % (sig,))


NETS = [("resnet18", 512, 8, 224, "bf16"), ("resnet:bottleneck:2,1,1,1", 2048, 8, 224, "bf16"),
        ("resnext:32x4:1,1,1,1", 2048, 2, 112, "bf16"), ("resnet18", 512, 4, 64, "fp32")]


def test_replay_engine_calls_exactly(cuda):
    calls, ratios = set(), []
    with recording(_recorders(calls, ratios)):
        for arch, rep, b, r, precision in NETS:
            byol_train_step(cuda, arch, rep, b, r, precision=precision, backward_precision=precision)
            torch.cuda.empty_cache()
    ops_seen = {sig[0] for sig in calls}
    pools = {sig[5] for sig in calls if sig[0] == "bn_relu_maxpool_fwd"}
    assert pools == {True, False}, "the stem pool with and without argmax must both be recorded, got %s" % pools
    assert "maxpool_bwd" in ops_seen and "avgpool_fwd" in ops_seen and "avgpool_bwd" in ops_seen
    modes = {sig[3] for sig in calls if sig[0] == "bn_bwd_apply"}
    assert {1, 3} <= modes, "bn_bwd_apply mask modes recorded: %s" % sorted(modes)
    for op in ("bn_apply_f32", "bn_bwd_apply_f32", "maxpool_f32", "maxpool_bwd_f32", "avgpool_f32"):
        assert op in ops_seen, "no %s call recorded from the fp32 path" % op
    print("largest |mean| / sqrt(var + eps) of a BatchNorm input in these steps: %.1f" % max(ratios))
    assert max(ratios) < 50, "a BatchNorm input approaches the variance-cancellation range of bn_finalize"
    replay(cuda, calls, _replay_case, 2000, " (%s)" % ", ".join(sorted(ops_seen)))
