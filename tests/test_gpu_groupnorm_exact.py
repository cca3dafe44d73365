"""GPU: the GroupNorm and weight-standardisation kernels (csrc/groupnorm.cu) bit for bit against float64, on every
kernel variant.

* Exact operands.  Activations and gradients are small integers, a few of them even integers in [256, 510] so that
  the bf16 outputs need the round-to-nearest-even; gamma, rstd and the residual's rgamma are signed powers of two,
  beta, the means and rbeta integers.  Every fp32 intermediate is then exact, so each output equals the float64
  reference rounded once (torch.equal, NaN == NaN).  The statistics are fed to the apply and backward kernels directly.
  gn_bwd_reduce adds into non-zero s12 / dgamma / dbeta: each must be fl32(init + fl32(exact sum)), fix_flush's single
  rounding of the exact fixed-point total.  gn_stats gets each (image, group) as mu +- a in equal halves (a a power
  of two, eps = 0), so its fp64 sums and (mean, rstd) are exact.
* Restatements.  Where the arithmetic is not dyadic (1/m for m = H*W*C/32 not a power of two, eps = 1e-5, the weight
  standardisation at any fan-in) the outputs are compared bit for bit with a restatement of the compiled order, and
  with float64 within a stated bound:
    - gn_finalize_kernel: q/count - mean*mean is contracted to one DFMA (tests/util.gn_finalize_restated);
    - gn_bwd_apply_kernel: fp32 FMUL / FADD only (every operation an explicit _rn intrinsic), inv_m = fl32(1.0/m);
    - ws_fwd_kernel: thread-strided fp64 sums, the xor butterfly, then the eight warp partials in warp order
      (block_sum_f64); the sum of squared deviations is a DFMA chain (q = fma(d, d, q)); w^ = fl32((w - mean) * rstd);
    - ws_bwd_kernel: s2 is a DFMA chain (b = fma(g, w^, b)); the update is DFMA(-w^, m2, g - m1) then DMUL by rstd,
      converted to fp32 and added with FADD.
* Route table.  One row per template instantiation and option at the edges of gn_geom (C/8 dividing 256 or not,
  C/8 > 256, H*W = 1, an image over several blocks with a short last chunk, N = 1 and N > 1); one test checks under
  torch.profiler, in a fresh process, that each row launches exactly its kernels.
* Non-finite inputs, batch independence per kernel, and a replay of the engine's own calls with exact operands.
"""
import re

import numpy as np
import pytest
import torch

from tests.exact import (Case, byol_model, byol_train_step, check_in_fresh_process, check_row_launches, expect,
                         expect_same, kernel_names, recording, replay, row_case, run_and_check, same)
from tests.test_gpu_elementwise_exact import acts, aten_pool, flat_index
from tests.util import fma32, fma64, gen, gn_finalize_restated, ints, pack_bits, pow2, unpack_bits

pytestmark = pytest.mark.gpu
BF, F32, F64, U8 = torch.bfloat16, torch.float32, torch.float64, torch.uint8
GROUPS = 32


# ------------------------------------------------------------------------------------------------------------------
# the host's geometry, restated (csrc/groupnorm.cu gn_geom / gn_grid)
# ------------------------------------------------------------------------------------------------------------------
def gn_geom(hw, c):
    """(vectors per image, vectors per block, blocks per image, C/8)"""
    cvecs = c // 8
    vecs = hw * cvecs
    per = 256 * 32
    blocks = -(-vecs // per)
    chunk = -(-vecs // blocks)
    chunk = -(-chunk // 256) * 256
    return vecs, chunk, -(-vecs // chunk), cvecs


# ------------------------------------------------------------------------------------------------------------------
# operands
# ------------------------------------------------------------------------------------------------------------------
def _grp(c, dev):
    return torch.arange(c, device=dev) // (c // GROUPS)


def _stats(n, dev, g):
    """fed statistics: integer means in [-3, 3], signed power-of-two rstd; fp64 [n, 32] each and fp32 [n, 32, 2]"""
    mean = ints((n, GROUPS), dev, g, 3)
    rstd = pow2(n * GROUPS, dev, g, signed=True).view(n, GROUPS)
    return mean, rstd, torch.stack([mean, rstd], -1).float().contiguous()


def _chan(t, c):
    """[n, 32] per-group values -> [n, 1, 1, c] per channel"""
    return t[:, _grp(c, t.device)].view(t.shape[0], 1, 1, c)


def _affine(gamma, beta, mean, rstd, c):
    """scale / shift [n, 1, 1, c] in fp64: sc = gamma*rstd, sh = beta - mean*sc (exact for these operands)"""
    sc = gamma.view(1, 1, 1, c) * _chan(rstd, c)
    return sc, beta.view(1, 1, 1, c) - _chan(mean, c) * sc


# ------------------------------------------------------------------------------------------------------------------
# statistics
# ------------------------------------------------------------------------------------------------------------------
def _pm_image(n, hw, c, dev, g):
    """y [n, hw, c] where every (image, group) is mu +- a in equal halves, shuffled; mu integer, a a power of two"""
    cpg = c // GROUPS
    cnt = hw * cpg
    assert cnt % 2 == 0, "mu +- a in equal halves needs an even group size"
    mu = ints((n, GROUPS, 1), dev, g, 8)
    a = torch.pow(2.0, torch.randint(0, 3, (n, GROUPS, 1), generator=g, device=dev).to(F64))
    sign = (torch.rand((n, GROUPS, cnt), generator=g, device=dev).argsort(-1) < cnt // 2).to(F64) * 2 - 1
    v = (mu + a * sign).view(n, GROUPS, hw, cpg).permute(0, 2, 1, 3).reshape(n, hw, c)
    return v, mu.view(n, GROUPS), a.view(n, GROUPS)


def _group_sums(y64, c):
    n = y64.shape[0]
    v = y64.reshape(n, -1, GROUPS, c // GROUPS)
    return torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1)


def stats_pm_case(dev, g, n, h, w, c):
    """mu +- a, eps = 0: sums64 equal the fp64 sums, mean = mu and rstd = 1/a exactly"""
    from byol_b200 import ops
    v, mu, a = _pm_image(n, h * w, c, dev, g)
    y = v.view(n, h, w, c)
    yd = y.to(BF)

    def run():
        sums = torch.full((n, GROUPS, 2), float("nan"), dtype=F64, device=dev)
        st = ops.gn_stats(yd, 0.0, sums64=sums)
        return [st, sums]

    def check(outs):
        st, sums = outs
        expect_same("sums64", sums, _group_sums(y, c))
        expect("stats", st, torch.stack([mu, 1.0 / a], -1))

    return Case(run, check, "stats")


def stats_rand_case(dev, g, n, h, w, c):
    """multiples of 2^-5 around an offset (the fp64 sums stay exact), eps = 1e-5: (mean, rstd) equal the restated
    gn_finalize_kernel bit for bit; mean and rstd within one fp32 ulp of float64"""
    from byol_b200 import ops
    off = ints((n, 1, 1, 1), dev, g, 6)
    y = ints((n, h, w, c), dev, g, 255) * 2.0 ** -5 + off
    yd = y.to(BF)
    y = yd.to(F64)                         # |y| may exceed bf16's 8 significant bits: use what the kernel reads

    def run():
        sums = torch.empty((n, GROUPS, 2), dtype=F64, device=dev)
        st = ops.gn_stats(yd, 1e-5, sums64=sums)
        return [st, sums]

    def check(outs):
        st, sums = outs
        want_sums = _group_sums(y, c)
        expect_same("sums64", sums, want_sums)
        cnt = h * w * (c // GROUPS)
        want = torch.from_numpy(gn_finalize_restated(want_sums.cpu().numpy(), float(cnt), 1e-5)).to(dev)
        expect_same("stats vs restated gn_finalize", st, want)
        s64 = want_sums.cpu()
        mean = s64[..., 0] / cnt
        var = (s64[..., 1] / cnt - mean * mean).clamp_min(0)
        rstd = 1.0 / torch.sqrt(var + float(np.float32(1e-5)))
        got = st.cpu().double()
        assert ((got[..., 0] - mean).abs() <= 2.0 ** -23 * mean.abs()).all(), "mean beyond one fp32 ulp"
        assert ((got[..., 1] - rstd).abs() <= 2.0 ** -23 * rstd).all(), "rstd beyond one fp32 ulp"

    return Case(run, check, "stats")


# ------------------------------------------------------------------------------------------------------------------
# apply and the fused stem
# ------------------------------------------------------------------------------------------------------------------
def apply_case(dev, g, n, h, w, c, resid=None, relu=False, mask=False):
    """y = act(x*scale + shift (+ r | + r*rscale + rshift)) and its mask bits; resid None / "plain" / "gn"."""
    from byol_b200 import ops
    x = acts((n, h, w, c), dev, g)
    gam, bet = pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    mean, rstd, st = _stats(n, dev, g)
    r = acts((n, h, w, c), dev, g) if resid else None
    rgn = None
    if resid == "gn":
        rgam, rbet = pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
        rmean, rrstd, rst = _stats(n, dev, g)
        rgn = (rgam.float(), rbet.float(), rst)
    xd, rd, gf, bf = x.to(BF), (r.to(BF) if resid else None), gam.float(), bet.float()

    def run():
        y = torch.empty((n, h, w, c), dtype=BF, device=dev)
        mo = torch.full((n * h * w * c // 8,), 0xA5, dtype=U8, device=dev) if mask else None
        ops.gn_apply(xd, gf, bf, st, relu, resid=rd, rgn=rgn, out=y, mask_out=mo)
        return [y, mo]

    def check(outs):
        y, mo = outs
        sc, sh = _affine(gam, bet, mean, rstd, c)
        ref = x * sc + sh
        if resid == "gn":
            rsc, rsh = _affine(rgam, rbet, rmean, rrstd, c)
            ref = ref + (r * rsc + rsh)
        elif resid:
            ref = ref + r
        if relu:
            ref = torch.relu(ref)
        expect("y", y, ref)
        if mask:
            assert torch.equal(unpack_bits(mo, ref.shape), ref > 0), "mask_out differs"

    return Case(run, check, "apply%d" % {None: 0, "plain": 1, "gn": 2}[resid])


def pool_case(dev, g, n, h, w, c, k=3, s=2, p=1, want_idx=True):
    """maxpool(relu(gn(x))): values against float64 rounded once, argmax against ATen's max_pool2d_with_indices (the
    first maximum in scan order).  Scales of both signs and one forced all-negative block give windows that are all
    zero after the ReLU (their argmax: the first in-image position)."""
    from byol_b200 import ops
    x = acts((n, h, w, c), dev, g)
    gam, bet = pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    mean, rstd, _ = _stats(n, dev, g)
    x[0, :, :, :8] = 0.0
    bet[:8] = -1.0
    mean[0, _grp(c, dev)[:8].unique()] = 0.0
    st = torch.stack([mean, rstd], -1).float().contiguous()
    xd, gf, bf = x.to(BF), gam.float(), bet.float()

    def run():
        return list(ops.gn_relu_maxpool_fwd(xd, gf, bf, st, k, s, p, want_idx=want_idx))

    def check(outs):
        y, idx = outs
        sc, sh = _affine(gam, bet, mean, rstd, c)
        a64 = torch.relu(x * sc + sh).float().to(BF).to(F64)
        ry, ri = aten_pool(a64, k, s, p)
        assert bool((ry[0, :, :, :8] == 0).all()), "the forced all-zero windows are missing"
        expect("y", y, ry)
        if want_idx:
            fi = flat_index(idx, w, k, s, p)
            bad = fi != ri
            assert not bad.any(), "argmax differs at %d of %d outputs (first %s: %d vs ATen %d)" % (
                int(bad.sum()), bad.numel(), bad.nonzero()[0].tolist(), int(fi[bad][0]), int(ri[bad][0]))
        else:
            assert idx is None

    return Case(run, check, "pool")


# ------------------------------------------------------------------------------------------------------------------
# backward
# ------------------------------------------------------------------------------------------------------------------
def _bwd_operands(dev, g, n, h, w, c, mask_mode):
    x, gr = acts((n, h, w, c), dev, g), acts((n, h, w, c), dev, g, 3)
    gam, bet = pow2(c, dev, g, signed=True), ints((c,), dev, g, 3)
    mean, rstd, st = _stats(n, dev, g)
    act, keep = None, None
    if mask_mode == 1:
        sc, sh = _affine(gam, bet, mean, rstd, c)
        keep = x * sc + sh > 0
    elif mask_mode == 2:
        a = acts((n, h, w, c), dev, g)
        keep, act = a > 0, a.to(BF)
    elif mask_mode == 3:
        keep = torch.rand((n, h, w, c), generator=g, device=dev) > 0.4
        act = pack_bits(keep)
    dz = gr * keep if keep is not None else gr
    xh = (x - _chan(mean, c)) * _chan(rstd, c)
    return dict(x=x, gr=gr, gam=gam, bet=bet, mean=mean, rstd=rstd, st=st, act=act, dz=dz, xh=xh)


def reduce_case(dev, g, n, h, w, c, mask_mode):
    """s12 / dgamma / dbeta from non-zero initial values: each fl32(init + fl32(exact sum))"""
    from byol_b200 import ops
    o = _bwd_operands(dev, g, n, h, w, c, mask_mode)
    xd, gd, gf, bf = o["x"].to(BF), o["gr"].to(BF), o["gam"].float(), o["bet"].float()
    s0 = torch.randn((n, GROUPS, 2), generator=g, device=dev)
    dg0, db0 = torch.randn(c, generator=g, device=dev), torch.randn(c, generator=g, device=dev)

    def run():
        s12, dg, db = s0.clone(), dg0.clone(), db0.clone()
        ops.gn_bwd_reduce(gd, xd, gf, bf, o["st"], s12, mask_mode, dgamma=dg, dbeta=db, act=o["act"])
        return [s12, dg, db]

    def check(outs):
        s12, dg, db = outs
        dz, xh, gam = o["dz"], o["xh"], o["gam"].view(1, 1, 1, c)
        db64, dg64 = dz.sum((0, 1, 2)), (dz * xh).sum((0, 1, 2))
        s1 = (gam * dz).reshape(n, -1, GROUPS, c // GROUPS).sum((1, 3))
        s2 = (gam * dz * xh).reshape(n, -1, GROUPS, c // GROUPS).sum((1, 3))
        for name, got, init, exact in (("s12", s12, s0, torch.stack([s1, s2], -1)), ("dgamma", dg, dg0, dg64),
                                       ("dbeta", db, db0, db64)):
            # fl32(init + fl32(exact)) with one rounding of the fp32 sum (an fp64 sum of the two could round twice)
            want = fma32(init.cpu().numpy(), np.float32(1), exact.float().cpu().numpy())
            expect_same(name, got, torch.from_numpy(want).to(dev).view(got.shape))

    return Case(run, check, "reduce%d" % mask_mode)


def bwd_apply_case(dev, g, n, h, w, c, mask_mode, dz_out=False):
    """dy = rstd*(gamma*dz - s1/m - xhat*s2/m).  m a power of two: s12 multiples of m, dy equals float64 rounded
    once.  Otherwise: dy equals the fp32 restatement (inv_m = fl32(1.0/m), m1 = fl32(s1*inv_m), every operation
    rounded) bit for bit, and that is within 2^-21 * |rstd| * (|gamma*dz| + |s1/m| + |xhat*s2/m|) of float64."""
    from byol_b200 import ops
    o = _bwd_operands(dev, g, n, h, w, c, mask_mode)
    m = h * w * (c // GROUPS)
    dyadic = m & (m - 1) == 0
    s12 = ints((n, GROUPS, 2), dev, g, 3) * m if dyadic else ints((n, GROUPS, 2), dev, g, 4000)
    s12f = s12.float().contiguous()
    xd, gd, gf, bf = o["x"].to(BF), o["gr"].to(BF), o["gam"].float(), o["bet"].float()

    def run():
        dy = torch.empty((n, h, w, c), dtype=BF, device=dev)
        dz = torch.empty((n, h, w, c), dtype=BF, device=dev) if dz_out else None
        ops.gn_bwd_apply(gd, xd, gf, bf, o["st"], s12f, mask_mode, act=o["act"], dy=dy, dz_out=dz)
        return [dy, dz]

    def check(outs):
        dy, dz = outs
        gam = o["gam"].view(1, 1, 1, c)
        s1, s2 = _chan(s12[..., 0], c), _chan(s12[..., 1], c)
        rs = _chan(o["rstd"], c)
        ref = rs * (gam * o["dz"] - s1 / m - o["xh"] * s2 / m)
        if dyadic:
            expect("dy", dy, ref)
        else:
            f = lambda t: t.float()
            inv_m = torch.tensor(float(np.float32(1.0 / m)), dtype=F32, device=dev)
            m1, m2 = f(s1) * inv_m, f(s2) * inv_m
            xh32 = (f(o["x"]) - f(_chan(o["mean"], c))) * f(rs)
            o32 = f(rs) * ((f(gam) * f(o["dz"]) - m1) - xh32 * m2)
            expect_same("dy vs the fp32 restatement", dy, o32.to(BF))
            bound = 2.0 ** -21 * rs.abs() * ((gam * o["dz"]).abs() + (s1 / m).abs() + (o["xh"] * s2 / m).abs())
            err = (o32.double() - ref).abs()
            assert bool((err <= bound).all()), "fp32 restatement beyond its bound by %g" % float((err - bound).max())
        if dz_out:
            expect("dz_out", dz, o["dz"])
        else:
            assert dz is None

    return Case(run, check, "bwd_apply%d" % mask_mode)


# ------------------------------------------------------------------------------------------------------------------
# weight standardisation: numpy restatement of the compiled order
# ------------------------------------------------------------------------------------------------------------------
def _ws_desc(units, dev):
    rows, off, row0 = [], 0, 0
    for cout, fan in units:
        rows.append([off, off, cout, fan, row0])
        off += cout * fan
        row0 += cout
    return torch.tensor(rows, dtype=torch.int64, device=dev), row0, off


def _block_sum(part):
    """block_sum_f64 of per-thread partials [rows, 256]: xor butterfly within each warp, then warp 0's partials added
    in warp order from 0.0"""
    v = part.copy()
    lane = np.arange(256)
    for o in (16, 8, 4, 2, 1):
        v = v + v[:, lane ^ o]
    t = np.zeros(v.shape[0])
    for wp in range(8):
        t = t + v[:, wp * 32]
    return t


def _strided(w, step):
    """per-thread partials [rows, 256]: thread t folds elements t, t + 256, ... in order with step(acc, column)"""
    rows, n = w.shape[0], w.shape[1]
    acc = np.zeros((rows, 256))
    for k in range(0, n, 256):
        cols = min(256, n - k)
        acc[:, :cols] = step(acc[:, :cols], k, cols)
    return acc


def _fma_rows(a, b, c):
    return fma64(a.reshape(-1), b.reshape(-1), c.reshape(-1)).reshape(a.shape)


def ws_fwd_restated(w):
    """w fp32 [rows, n] -> (w^ fp32, mean fp32, rstd fp32) as ws_fwd_kernel computes them"""
    w64 = w.astype(np.float64)
    n = w.shape[1]
    mean = _block_sum(_strided(w64, lambda acc, k, cols: acc + w64[:, k:k + cols])) / n
    d = w64 - mean[:, None]
    var = _block_sum(_strided(d, lambda acc, k, cols: _fma_rows(d[:, k:k + cols], d[:, k:k + cols], acc))) / n
    rstd = 1.0 / np.sqrt(var + 1e-5)
    return (d * rstd[:, None]).astype(np.float32), mean.astype(np.float32), rstd.astype(np.float32)


def ws_bwd_restated(dwh, wh, rstd32, grad0):
    """grad0 + fl32(rstd * fma(-w^, m2, g - m1)) with FADD, as ws_bwd_kernel computes it"""
    g64, w64 = dwh.astype(np.float64), wh.astype(np.float64)
    n = dwh.shape[1]
    m1 = _block_sum(_strided(g64, lambda acc, k, cols: acc + g64[:, k:k + cols])) / n
    m2 = _block_sum(_strided(g64, lambda acc, k, cols: _fma_rows(g64[:, k:k + cols], w64[:, k:k + cols], acc))) / n
    t = g64 - m1[:, None]
    u = _fma_rows(-w64, np.broadcast_to(m2[:, None], w64.shape), t)
    upd = (rstd32.astype(np.float64)[:, None] * u).astype(np.float32)
    return grad0 + upd, upd


def ws_case(dev, g, units, bwd=False, rows_checked=None):
    """ws_fwd (bwd=False) or ws_bwd of the weight rows of `units` [(cout, fan-in)], laid out back to back; against the
    restatement bit for bit, and against float64: w^, mean and rstd within one fp32 ulp, the gradient within
    2^-23 * (|update| + |grad|).  rows_checked: the rows of each unit compared (default all)."""
    from byol_b200 import ops
    desc, rows, numel = _ws_desc(units, dev)
    cpu = torch.Generator().manual_seed(int(torch.randint(0, 2 ** 30, (1,), generator=g, device=dev)))
    flat = (torch.randn(numel, generator=cpu) * 0.05 + 0.01)
    dwh = torch.randn(numel, generator=cpu)
    grad0 = torch.randn(numel, generator=cpu)
    stats_in = torch.stack([torch.randn(rows, generator=cpu), torch.rand(rows, generator=cpu) * 30 + 0.5], 1)
    fd, dd, g0d, sd = flat.to(dev), dwh.to(dev), grad0.to(dev), stats_in.to(dev).contiguous()

    def run():
        if not bwd:
            out, st = torch.empty(numel, device=dev), torch.empty((rows, 2), device=dev)
            ops.ws_fwd(fd, desc, rows, out, st)
            return [out, st]
        grad = g0d.clone()
        ops.ws_bwd(dd, fd, sd, desc, rows, grad)     # flat stands in for w^: any fp32 values
        return [grad]

    def check(outs):
        outs = [t.cpu().numpy() for t in outs]
        off, row0 = 0, 0
        for cout, fan in units:
            sel = np.arange(cout) if rows_checked is None else np.unique(np.clip(rows_checked, 0, cout - 1))
            idx = (off + sel[:, None] * fan + np.arange(fan)[None, :])
            w = flat.numpy()[idx]
            if not bwd:
                wh, mean, rstd = ws_fwd_restated(w)
                got_w, got_s = outs[0][idx], outs[1][row0 + sel]
                assert np.array_equal(got_w.view(np.int32), wh.view(np.int32)), "w^ differs (fan-in %d)" % fan
                assert np.array_equal(got_s[:, 0].view(np.int32), mean.view(np.int32)), "mean (fan-in %d)" % fan
                assert np.array_equal(got_s[:, 1].view(np.int32), rstd.view(np.int32)), "rstd (fan-in %d)" % fan
                w64 = w.astype(np.float64)
                m64 = w64.mean(1, keepdims=True)
                r64 = 1.0 / np.sqrt(((w64 - m64) ** 2).mean(1, keepdims=True) + 1e-5)
                wh64 = (w64 - m64) * r64
                assert (np.abs(got_w - wh64) <= 2.0 ** -23 * np.abs(wh64) + 1e-30).all(), fan
                assert (np.abs(got_s[:, 0] - m64[:, 0]) <= 2.0 ** -23 * np.abs(m64[:, 0])).all(), fan
                assert (np.abs(got_s[:, 1] - r64[:, 0]) <= 2.0 ** -23 * r64[:, 0]).all(), fan
            else:
                gr, wh = dwh.numpy()[idx], w
                r32 = stats_in.numpy()[row0 + sel, 1]
                want, upd = ws_bwd_restated(gr, wh, r32, grad0.numpy()[idx])
                got = outs[0][idx]
                assert np.array_equal(got.view(np.int32), want.view(np.int32)), "grad differs (fan-in %d)" % fan
                g64, w64 = gr.astype(np.float64), wh.astype(np.float64)
                u64 = r32.astype(np.float64)[:, None] * (g64 - g64.mean(1, keepdims=True)
                                                         - w64 * (g64 * w64).mean(1, keepdims=True))
                tot = grad0.numpy()[idx].astype(np.float64) + u64
                noise = 2.0 ** -50 * r32[:, None] * (np.abs(g64) + np.abs(g64).mean(1, keepdims=True)
                                                     + np.abs(w64) * np.abs(g64 * w64).mean(1, keepdims=True))
                assert (np.abs(got - tot) <= 2.0 ** -23 * (np.abs(u64) + np.abs(tot)) + noise).all(), fan
            off += cout * fan
            row0 += cout

    return Case(run, check, "ws_bwd" if bwd else "ws_fwd")


# ------------------------------------------------------------------------------------------------------------------
# route table
# ------------------------------------------------------------------------------------------------------------------
ROUTE_KERNELS = {
    "stats": ["gn_stats_kernel", "gn_finalize_kernel"],
    "pool": ["gn_relu_maxpool_fwd_kernel"],
    "ws_fwd": ["ws_fwd_kernel"],
    "ws_bwd": ["ws_bwd_kernel"],
}
for _m in range(3):
    ROUTE_KERNELS["apply%d" % _m] = ["gn_apply_kernel<%d>" % _m]
for _m in range(4):
    ROUTE_KERNELS["reduce%d" % _m] = ["gn_bwd_reduce_kernel<%d>" % _m] + ["fix_flush_kernel"] * 3
    ROUTE_KERNELS["bwd_apply%d" % _m] = ["gn_bwd_apply_kernel<%d>" % _m]

# (n, h, w, c) at the edges of gn_geom
SHAPES = {
    "c64": (2, 8, 8, 64),                # C/8 divides 256: a thread stays on one vector; m = 128
    "c64_hw1": (3, 1, 1, 64),            # H*W = 1: 8 vectors per image, most threads idle
    "c64_7x7": (1, 7, 7, 64),            # m = 98
    "c256": (2, 4, 4, 256),
    "c2048": (2, 2, 2, 2048),            # C/8 = 256: every thread on its own vector
    "c2048_7x7": (1, 7, 7, 2048),        # m = 3136
    "c96": (2, 6, 5, 96),                # C/8 = 12: groups straddle vectors, the vector changes every iteration
    "c160": (1, 4, 3, 160),              # C/8 = 20, 5 channels per group
    "c4096": (1, 2, 2, 4096),            # C/8 = 512 > 256 threads
    "c4096_hw1": (2, 1, 1, 4096),
    "stem224": (2, 112, 112, 64),        # 13 blocks per image, the last one short
}
GEOM_EDGE = {
    "c64": lambda v, ch, b, cv: 256 % cv == 0 and b == 1,
    "c64_hw1": lambda v, ch, b, cv: v == 8,
    "c2048": lambda v, ch, b, cv: cv == 256,
    "c96": lambda v, ch, b, cv: 256 % cv != 0,
    "c160": lambda v, ch, b, cv: 256 % cv != 0,
    "c4096": lambda v, ch, b, cv: cv > 256,
    "c4096_hw1": lambda v, ch, b, cv: cv > 256,
    "stem224": lambda v, ch, b, cv: b > 1 and v - (b - 1) * ch < ch,
}

ROWS = {}
for _s in ("c64", "c64_hw1", "c256", "c2048", "c96", "c160", "c4096", "stem224"):
    ROWS["stats_pm_" + _s] = ("stats", stats_pm_case, dict(zip("nhwc", SHAPES[_s])))
for _s in ("c64_7x7", "c96", "c2048_7x7", "stem224"):
    ROWS["stats_rand_" + _s] = ("stats", stats_rand_case, dict(zip("nhwc", SHAPES[_s])))
_APPLY_SHAPES = ["c64", "c96", "c4096", "stem224", "c64_hw1", "c160"]
for _i, (_r, _relu, _mask) in enumerate([(r, relu, mask) for r in (None, "plain", "gn") for relu in (False, True)
                                         for mask in (False, True)]):
    _s = _APPLY_SHAPES[_i % len(_APPLY_SHAPES)]
    ROWS["apply%d_relu%d_mask%d_%s" % ({None: 0, "plain": 1, "gn": 2}[_r], _relu, _mask, _s)] = (
        "apply%d" % {None: 0, "plain": 1, "gn": 2}[_r], apply_case,
        dict(zip("nhwc", SHAPES[_s]), resid=_r, relu=_relu, mask=_mask))
ROWS["apply2_relu1_mask1_c2048"] = ("apply2", apply_case, dict(zip("nhwc", SHAPES["c2048"]), resid="gn", relu=True,
                                                               mask=True))
for _name, _shape, _idx in (("pool_odd_idx", (2, 9, 7, 64), True), ("pool_odd_noidx", (2, 9, 7, 64), False),
                            ("pool_ho1_idx", (1, 2, 3, 64), True), ("pool_c96_idx", (2, 5, 5, 96), True),
                            ("pool_stem224_idx", (2, 112, 112, 64), True)):
    ROWS[_name] = ("pool", pool_case, dict(zip("nhwc", _shape), want_idx=_idx))
_BWD_SHAPES = ["c64", "c96", "c4096", "c64_hw1", "c160", "c2048", "c2048_7x7", "stem224", "c256", "c4096_hw1"]
for _m in range(4):
    for _j, _s in enumerate(_BWD_SHAPES[_m::2] if _m < 2 else _BWD_SHAPES[_m % 2::2]):
        ROWS["reduce%d_%s" % (_m, _s)] = ("reduce%d" % _m, reduce_case, dict(zip("nhwc", SHAPES[_s]), mask_mode=_m))
    for _dz in (False, True):
        for _s in (_BWD_SHAPES[(2 * _m + _dz) % len(_BWD_SHAPES)], _BWD_SHAPES[(2 * _m + _dz + 5) % len(_BWD_SHAPES)]):
            ROWS["bwd_apply%d_dz%d_%s" % (_m, _dz, _s)] = ("bwd_apply%d" % _m, bwd_apply_case,
                                                          dict(zip("nhwc", SHAPES[_s]), mask_mode=_m, dz_out=_dz))
WS_UNITS = [(6, 147), (4, 64), (3, 576), (5, 36), (4, 72), (2, 300), (3, 256), (1, 4608)]
ROWS["ws_fwd"] = ("ws_fwd", ws_case, dict(units=WS_UNITS))
ROWS["ws_bwd"] = ("ws_bwd", ws_case, dict(units=WS_UNITS, bwd=True))
ROWS["ws_fwd_one_unit"] = ("ws_fwd", ws_case, dict(units=[(3, 2048)]))
ROWS["ws_bwd_one_unit"] = ("ws_bwd", ws_case, dict(units=[(3, 2048)], bwd=True))


def _build(dev, name):
    return row_case(dev, name, *ROWS[name][1:])


def test_shapes_sit_at_their_geometry_edges():
    for name, edge in GEOM_EDGE.items():
        n, h, w, c = SHAPES[name]
        assert edge(*gn_geom(h * w, c)), "%s %s no longer sits at its gn_geom edge: %s" % (
            name, SHAPES[name], gn_geom(h * w, c))
    shapes = {(kw.get("n"), kw.get("c")) for _, _, kw in ROWS.values()}
    assert any(n == 1 for n, _ in shapes) and any(n is not None and n > 1 for n, _ in shapes)


@pytest.mark.parametrize("name", list(ROWS))
def test_row_exact(cuda, name):
    run_and_check(_build(cuda, name))


def _byol_kernels(run):
    """The sorted GroupNorm / WS / fix_flush kernels one run() launches, with their template argument."""
    names = []
    for k in kernel_names(run):
        m = re.search(r"\b((?:gn|ws)_\w+?_kernel|fix_flush_kernel)(<\d+>)?\(", k)
        if m:
            names.append(m.group(1) + (m.group(2) or ""))
    return sorted(names)


def _check_launches():
    cases = {name: _build(torch.device("cuda:0"), name) for name in ROWS}

    def complaints(name, launched):
        case, want = cases[name], ROWS[name][0]
        wrong = []
        if case.route != want:
            wrong.append("%s: the case says %s, the row is meant for %s" % (name, case.route, want))
        if launched != sorted(ROUTE_KERNELS[want]):
            wrong.append("%s: expected %s, launched %s" % (name, sorted(ROUTE_KERNELS[want]), launched))
        return wrong
    check_row_launches({name: case.run for name, case in cases.items()}, complaints, _byol_kernels)


def test_rows_launch_their_kernels(cuda):
    """Each row launches exactly its kernels: gn_stats_kernel + gn_finalize_kernel, the <MASK> / <RESID>
    instantiation named for it, gn_bwd_reduce with its three fix_flush_kernels (s12, dbeta, dgamma).  Checked in a
    fresh Python process (a process that has held many profiler sessions can drop CUDA kernel events)."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# non-finite inputs (the rules DESIGN.md records)
# ------------------------------------------------------------------------------------------------------------------
def test_non_finite_inputs(cuda):
    """A NaN or +-Inf in an image makes the statistics of its group NaN (rstd NaN; the mean NaN or +-Inf); the ReLU'd
    outputs of that group are 0 with mask bit 0 (fmaxf(NaN, 0) = 0, as BatchNorm's apply), without the ReLU they are
    NaN.  The image's other groups and the other images keep their bits.  Values near the bf16 maximum keep finite
    sums and statistics."""
    from byol_b200 import ops
    n, h, w, c = 3, 8, 8, 64
    g = gen(cuda, 71)
    x = (torch.randn((n, h, w, c), generator=g, device=cuda) * 2 + 0.5).to(BF)
    xs = x.clone()
    xs[1, 2, 3, 0] = float("nan")                  # group 0
    xs[1, 5, 5, 10] = float("inf")                 # group 5
    xs[1, 0, 7, 20] = float("-inf")                # group 10
    xs[1, 4, 4, 30], xs[1, 6, 1, 31] = float("inf"), float("-inf")      # group 15: Inf - Inf
    big = torch.finfo(BF).max
    xs[2, :, :, 40:42] = torch.where(torch.rand((h, w, 2), generator=g, device=cuda) < 0.5, big, -big).to(BF)
    gam = torch.rand(c, generator=g, device=cuda) + 0.5
    bet = torch.randn(c, generator=g, device=cuda)
    outs = []
    for t in (x, xs):
        sums = torch.empty((n, GROUPS, 2), dtype=F64, device=cuda)
        st = ops.gn_stats(t, 1e-5, sums64=sums)
        mo = torch.empty(t.numel() // 8, dtype=U8, device=cuda)
        y = ops.gn_apply(t, gam, bet, st, True, mask_out=mo)
        y_lin = ops.gn_apply(t, gam, bet, st, False)
        outs.append((st, sums, y, mo, y_lin))
    torch.cuda.synchronize()
    (st0, _, y0, m0, l0), (st, sums, y, mo, yl) = outs
    bad = [0, 5, 10, 15]
    good = [k for k in range(GROUPS) if k not in bad and k != 20]
    assert torch.isnan(st[1, bad, 1]).all(), "rstd of the groups holding NaN / Inf must be NaN"
    assert torch.isnan(st[1, [0, 15], 0]).all() and st[1, 5, 0] == float("inf") and st[1, 10, 0] == float("-inf")
    assert same(st[1, good], st0[1, good]) and same(st[0], st0[0]), "the statistics of finite groups changed"
    keep = unpack_bits(mo, y.shape)
    chans = torch.cat([torch.arange(k * 2, k * 2 + 2) for k in bad]).to(cuda)
    assert (y[1][..., chans] == 0).all() and not keep[1][..., chans].any()
    assert torch.isnan(yl[1][..., chans].float()).all()
    other = torch.tensor([ch for ch in range(c) if ch // 2 not in bad], device=cuda)
    assert same(y[1][..., other], y0[1][..., other]) and torch.equal(keep[1][..., other],
                                                                       unpack_bits(m0, y0.shape)[1][..., other])
    assert same(y[0], y0[0]) and same(yl[0], l0[0])
    assert torch.isfinite(sums[2]).all() and torch.isfinite(st[2]).all(), "sums near the bf16 maximum overflowed"
    assert float(sums[2, 20, 1]) == float(big) ** 2 * h * w * 2


# ------------------------------------------------------------------------------------------------------------------
# batch independence per kernel
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(5, 8, 8, 64), (5, 6, 5, 96), (5, 112, 112, 64)])
def test_batch_independence_per_kernel(cuda, shape):
    """stats (and their fp64 sums), apply, relu_maxpool, s12 and dy of each image have the same bits alone as inside
    the batch of 5.  The activations are scaled by 2^-20 and the gradients by 2^-40: their squares and products carry
    bits below the fixed point's 2^-50, so each block partial is rounded, and a partition of the image that depended
    on the batch would change the sums."""
    from byol_b200 import ops
    n, h, w, c = shape
    g = gen(cuda, 90 + c)
    x = ((torch.randn(shape, generator=g, device=cuda) * 1.5 + 0.3) * 2.0 ** -20).to(BF)
    gr = (torch.randn(shape, generator=g, device=cuda) * 2.0 ** -40).to(BF)
    gam, bet = torch.rand(c, generator=g, device=cuda) + 0.5, torch.randn(c, generator=g, device=cuda)

    def outs(xi, gi):
        sums = torch.empty((xi.shape[0], GROUPS, 2), dtype=F64, device=cuda)
        st = ops.gn_stats(xi, 1e-5, sums64=sums)
        mo = torch.empty(xi.numel() // 8, dtype=U8, device=cuda)
        y = ops.gn_apply(xi, gam, bet, st, True, mask_out=mo)
        p, idx = ops.gn_relu_maxpool_fwd(xi, gam, bet, st, 3, 2, 1) if c == 64 else (None, None)
        s12 = torch.zeros((xi.shape[0], GROUPS, 2), device=cuda)
        ops.gn_bwd_reduce(gi, xi, gam, bet, st, s12, 3, act=mo, dgamma=torch.zeros(c, device=cuda),
                          dbeta=torch.zeros(c, device=cuda))
        dy = ops.gn_bwd_apply(gi, xi, gam, bet, st, s12, 3, act=mo)
        return [st, sums, y, p, idx, s12, dy]

    full = outs(x, gr)
    for i in (0, 2, n - 1):
        alone = outs(x[i:i + 1].contiguous(), gr[i:i + 1].contiguous())
        torch.cuda.synchronize()
        for label, a, b in zip(("stats", "sums64", "y", "pool", "pool idx", "s12", "dy"), alone, full):
            if a is not None:
                assert same(a[0], b[i]), "%s of image %d differs alone and in the batch" % (label, i)


# ------------------------------------------------------------------------------------------------------------------
# argument checks
# ------------------------------------------------------------------------------------------------------------------
def _arg_cases(dev):
    from byol_b200 import ops
    n, h, w, c = 2, 4, 4, 64
    x = torch.zeros((n, h, w, c), dtype=BF, device=dev)
    gam, bet = torch.ones(c, device=dev), torch.zeros(c, device=dev)
    st = torch.ones((n, GROUPS, 2), device=dev)
    s12 = torch.zeros((n, GROUPS, 2), device=dev)
    dg, db = torch.zeros(c, device=dev), torch.zeros(c, device=dev)
    bits = torch.zeros(x.numel() // 8, dtype=U8, device=dev)
    desc = torch.tensor([[0, 0, 4, 16, 0]], dtype=torch.int64, device=dev)
    flat, wst = torch.zeros(64, device=dev), torch.zeros((4, 2), device=dev)
    strided = torch.ones(2 * c, device=dev)[::2]
    return {
        "gamma not contiguous": lambda: ops.gn_apply(x, strided, bet, st, True),
        "gamma on the CPU": lambda: ops.gn_relu_maxpool_fwd(x, gam.cpu(), bet, st),
        "beta fp64": lambda: ops.gn_apply(x, gam, bet.double(), st, True),
        "gamma of another C": lambda: ops.gn_bwd_apply(x, x, gam[:32], bet, st, s12, 0),
        "stats of a smaller batch": lambda: ops.gn_apply(x, gam, bet, st[:1], True),
        "rgamma of another C": lambda: ops.gn_apply(x, gam, bet, st, True, resid=x, rgn=(gam[:32], bet, st)),
        "rstats of a smaller batch": lambda: ops.gn_apply(x, gam, bet, st, True, resid=x, rgn=(gam, bet, st[:1])),
        "resid of another shape": lambda: ops.gn_apply(x, gam, bet, st, True, resid=x[:1]),
        "out of another shape": lambda: ops.gn_apply(x, gam, bet, st, True, out=x[:1]),
        "mask_out too short": lambda: ops.gn_apply(x, gam, bet, st, True, mask_out=bits[:-1]),
        "s12 fp64": lambda: ops.gn_bwd_reduce(x, x, gam, bet, st, s12.double(), 0, dgamma=dg, dbeta=db),
        "s12 of a smaller batch": lambda: ops.gn_bwd_apply(x, x, gam, bet, st, s12[:1], 0),
        "dgamma missing": lambda: ops.gn_bwd_reduce(x, x, gam, bet, st, s12, 0, dgamma=None, dbeta=db),
        "dbeta of another C": lambda: ops.gn_bwd_reduce(x, x, gam, bet, st, s12, 0, dgamma=dg, dbeta=db[:8]),
        "act bits too short": lambda: ops.gn_bwd_reduce(x, x, gam, bet, st, s12, 3, dgamma=dg, dbeta=db,
                                                        act=bits[:8]),
        "act of another shape": lambda: ops.gn_bwd_apply(x, x, gam, bet, st, s12, 2, act=x[:1]),
        "dy of another shape": lambda: ops.gn_bwd_apply(x, x, gam, bet, st, s12, 0, dy=x[:1]),
        "dz_out of another shape": lambda: ops.gn_bwd_apply(x, x, gam, bet, st, s12, 0, dz_out=x[:1]),
        "g of another shape": lambda: ops.gn_bwd_apply(x[:1], x, gam, bet, st, s12, 0),
        "sums64 of another shape": lambda: ops.gn_stats(x, 1e-5, sums64=torch.zeros((1, GROUPS, 2), dtype=F64,
                                                                                    device=dev)),
        "desc int32": lambda: ops.ws_fwd(flat, desc.int(), 4, flat.clone(), wst),
        "desc not [U, 5]": lambda: ops.ws_fwd(flat, desc[:, :4].contiguous(), 4, flat.clone(), wst),
        "desc not contiguous": lambda: ops.ws_bwd(flat, flat, wst, torch.cat([desc, desc], 1)[:, ::2], 4, flat),
        "ws stats of other rows": lambda: ops.ws_bwd(flat, flat, wst[:3], desc, 4, flat.clone()),
    }


ARG_CASES = ["gamma not contiguous", "gamma on the CPU", "beta fp64", "gamma of another C", "stats of a smaller batch",
             "rgamma of another C", "rstats of a smaller batch", "resid of another shape", "out of another shape",
             "mask_out too short", "s12 fp64", "s12 of a smaller batch", "dgamma missing", "dbeta of another C",
             "act bits too short", "act of another shape", "dy of another shape", "dz_out of another shape",
             "g of another shape", "sums64 of another shape", "desc int32", "desc not [U, 5]", "desc not contiguous",
             "ws stats of other rows"]


@pytest.mark.parametrize("label", ARG_CASES)
def test_argument_check(cuda, label):
    """The wrapper raises ValueError before any CUDA work (nothing is launched: the library's launch count stays)."""
    from byol_b200 import _lib
    call = _arg_cases(cuda)[label]
    before = _lib.launch_count[0]
    with pytest.raises(ValueError):
        call()
    assert _lib.launch_count[0] == before


# ------------------------------------------------------------------------------------------------------------------
# replay of the engine's own calls
# ------------------------------------------------------------------------------------------------------------------
def _recorders(calls, descs):
    """ops function name -> recorder noting the call's shapes and options (not its data)"""
    def _desc_key(desc, num_rows):
        descs.append(desc)                 # resolved after the step: reading it here would synchronise
        return len(descs) - 1, int(num_rows)

    def gn_stats(y, eps, out=None, sums64=None):
        calls.add(("gn_stats", tuple(y.shape), float(eps)))

    def gn_apply(x, gamma, beta, stats, relu, resid=None, rgn=None, out=None, mask_out=None):
        kind = 0 if resid is None else 2 if rgn is not None else 1
        calls.add(("gn_apply", tuple(x.shape), kind, bool(relu), mask_out is not None))

    def gn_relu_maxpool_fwd(x, gamma, beta, stats, k=3, s=2, p=1, want_idx=True):
        calls.add(("gn_relu_maxpool_fwd", tuple(x.shape), k, s, p, bool(want_idx)))

    def gn_bwd_reduce(g, x, gamma, beta, stats, s12, mask_mode, dgamma, dbeta, act=None):
        calls.add(("gn_bwd_reduce", tuple(x.shape), mask_mode))

    def gn_bwd_apply(g, x, gamma, beta, stats, s12, mask_mode, act=None, dy=None, dz_out=None):
        calls.add(("gn_bwd_apply", tuple(x.shape), mask_mode, dz_out is not None))

    def ws_fwd(flat, desc, num_rows, w_out, stats):
        calls.add(("ws_fwd",) + _desc_key(desc, num_rows))

    def ws_bwd(dwhat, what, stats, desc, num_rows, grad):
        calls.add(("ws_bwd",) + _desc_key(desc, num_rows))
    return {k: v for k, v in locals().items() if callable(v) and not k.startswith("_")}


def _record(dev, arch, b, r, what):
    """The signatures of one source's calls: a BYOL step, a fine-tune step or representations() of one image."""
    from byol_b200.finetune import FineTune
    calls, descs = set(), []
    model_kw = dict(classes=10, projection=64, head_latent_size=128, norm="group_ws")
    with recording(_recorders(calls, descs)):
        if what == "byol":
            byol_train_step(dev, arch, 512 if arch == "resnet18" else 2048, b, r, **model_kw)
        else:
            model, a1, _, lab = byol_model(dev, arch, 512 if arch == "resnet18" else 2048, b, r, **model_kw)
            if what == "finetune":
                FineTune(model, 5, 0.1, seed=2).step(a1, lab % 5, 1.0)
            else:
                model.representations(a1[:1])
            torch.cuda.synchronize()
    out = set()
    for sig in calls:
        if sig[0] in ("ws_fwd", "ws_bwd"):
            d = descs[sig[1]].cpu().tolist()
            sig = (sig[0], tuple((row[2], row[3]) for row in d), sig[2])
        out.add(sig)
    return out


def _replay_case(dev, g, sig):
    op, a = sig[0], sig[1:]
    if op == "gn_stats":
        (n, h, w, c), _ = a
        if h * w % 2 == 0:
            return stats_pm_case(dev, g, n, h, w, c)
        return stats_rand_case(dev, g, n, h, w, c)     # odd maps: the eps = 1e-5 route, against the restatement
    if op == "gn_apply":
        (n, h, w, c), kind, relu, mask = a
        return apply_case(dev, g, n, h, w, c, resid=[None, "plain", "gn"][kind], relu=relu, mask=mask)
    if op == "gn_relu_maxpool_fwd":
        (n, h, w, c), k, s, p, idx = a
        return pool_case(dev, g, n, h, w, c, k, s, p, want_idx=idx)
    if op == "gn_bwd_reduce":
        (n, h, w, c), mode = a
        return reduce_case(dev, g, n, h, w, c, mode)
    if op == "gn_bwd_apply":
        (n, h, w, c), mode, dz = a
        return bwd_apply_case(dev, g, n, h, w, c, mode, dz_out=dz)
    if op in ("ws_fwd", "ws_bwd"):
        units, rows = a
        assert rows == sum(u[0] for u in units)
        return ws_case(dev, g, list(units), bwd=op == "ws_bwd", rows_checked=np.array([0, 1, 10 ** 6]))
    raise AssertionError("no replay for %s" % (sig,))


SOURCES = [("resnet18", 4, 64, "byol"), ("resnet:bottleneck:1,1,1,1", 4, 64, "byol"),
           ("resnext:32x4:1,1,1,1", 4, 64, "byol"), ("resnet18", 2, 72, "byol"), ("resnet18", 4, 64, "finetune"),
           ("resnet:bottleneck:1,1,1,1", 1, 64, "representations")]


def test_replay_engine_calls_exactly(cuda):
    """Every distinct GroupNorm / weight-standardisation call of a BYOL step (ResNet-18, a bottleneck net and a
    ResNeXt net at 64 px, ResNet-18 at 72 px: maps of 36, 18, 9, 5 and 3), a fine-tune step and representations() of
    one image, replayed with exact operands (or against the restatement where m or the fan-in is not dyadic)."""
    calls = set()
    for arch, b, r, what in SOURCES:
        calls |= _record(cuda, arch, b, r, what)
        torch.cuda.empty_cache()
    modes = {sig[2] for sig in calls if sig[0] == "gn_bwd_apply"}
    assert {1, 3} <= modes, "gn_bwd_apply mask modes recorded: %s" % sorted(modes)
    kinds = {sig[2] for sig in calls if sig[0] == "gn_apply"}
    assert kinds == {0, 1, 2}, "gn_apply residual kinds recorded: %s" % sorted(kinds)
    assert any(sig[0] == "gn_relu_maxpool_fwd" for sig in calls), "the pooled stem was not recorded"
    assert any(sig[0] == "ws_bwd" for sig in calls) and any(sig[0] == "gn_bwd_reduce" for sig in calls)
    maps = {sig[1][1] for sig in calls if sig[0].startswith("gn_")}
    assert {36, 18, 9, 5, 3} <= maps, "map sizes recorded: %s" % sorted(maps)
    replay(cuda, calls, _replay_case, 3000)
