"""GPU: every cross-block reduction (the fixed-point accumulators of csrc/common.cuh, fix_scratch / fix_flush in
csrc/capi.cu) against an fp64 reference.

* Exact parity.  Small-integer inputs (or integers times a power of two) keep every fp32 partial sum and every
  tensor-core accumulator exact, so the fixed-point total is exact and the kernel's fp32 result must equal the fp64
  reference rounded once to fp32 (torch.equal), whatever order the blocks ran in: a dropped or doubled row, tile, tap,
  K chunk or column shows.  GEMM-epilogue statistics are checked against the kernel's own bf16 output.
* Run-to-run bits.  Random, non-exact inputs give the same bits on another stream, after a reduction of another size
  reused the stream's scratch, and replayed from a CUDA graph.
* Special values.  NaN / Inf propagate, cancellation is exact, huge addends and totals past 2^45 keep their value.
* Scratch lifecycle.  Growth, an early error return, a graph that outlives a grown scratch, two streams flushing into
  one destination.
"""
import contextlib
import gc
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64
REAL_M = 132 * 128 * 4      # conv / GEMM rows at which every CTA of a full H100 grid runs several 128-row tiles


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _vals(shape, exact, g, amp=2, density=1.0):
    """CPU fp32 values bf16 represents exactly: integers in [-amp, amp] (a fraction `density` of them non-zero) when
    `exact`, else bf16-rounded N(0, amp^2) samples."""
    if not exact:
        return (torch.randn(shape, generator=g) * amp).to(BF).float()
    v = torch.randint(-amp, amp + 1, shape, generator=g).float()
    if density < 1.0:
        v = v * (torch.rand(shape, generator=g) < density)
    return v


def _expect_equal(name, got, want64):
    got = got.detach().cpu()
    want = want64.to(got.dtype)
    if not torch.equal(got, want):
        d = (got.double() - want64.double()).abs()
        raise AssertionError("%s: %d of %d values differ from the fp64 reference; max |diff| %g at flat index %d" %
                             (name, int((got != want).sum()), got.numel(), float(d.max()), int(d.argmax())))


def _colstats(y2d):
    y = y2d.detach().cpu().double()
    return torch.cat([y.sum(0), (y * y).sum(0)])


def _nchw(t):
    return t.permute(0, 3, 1, 2).double()


# ------------------------------------------------------------------------------------------------------------------
# one builder per entry point: (device, exact, generator, **shape) -> (run, ref)
#   run() launches the reduction into freshly zeroed (or freshly copied) destinations and returns the device outputs;
#   ref(outs) -> [(label, kernel tensor, fp64 expectation)] (used with exact inputs)
# ------------------------------------------------------------------------------------------------------------------
def bn_stats_case(dev, exact, g, m, c):
    from byol_b200 import ops
    x = _vals((m, c), exact, g, 4)
    xd = x.to(dev, BF)

    def run():
        s = torch.zeros(2 * c, device=dev)
        ops.bn_stats(xd, s)
        return [s]
    return run, lambda o: [("stats", o[0], _colstats(x))]


def bn_bwd_reduce_case(dev, exact, g, m, c, mask_mode):
    from byol_b200 import ops
    gy, x = _vals((m, c), exact, g, 3), _vals((m, c), exact, g, 3)
    if exact:
        mean = torch.randint(-2, 3, (c,), generator=g).float()
        invstd = torch.pow(2.0, torch.randint(-1, 2, (c,), generator=g).float())
    else:
        mean, invstd = torch.randn(c, generator=g) * 0.1, torch.rand(c, generator=g) + 0.5
    act = _vals((m, c), exact, g, 2) if mask_mode == 2 else None
    coeffs = torch.stack([torch.ones(c), torch.zeros(c), mean, invstd]).to(dev)
    gd, xd = gy.to(dev, BF), x.to(dev, BF)
    actd = act.to(dev, BF) if act is not None else None

    def run():
        s12 = torch.zeros(2 * c, device=dev)
        ops.bn_bwd_reduce(gd, xd, coeffs, s12, mask_mode, act=actd)
        return [s12]

    def ref(o):
        dz = gy.double() * ((act > 0).double() if act is not None else 1.0)
        xhat = (x.double() - mean.double()) * invstd.double()
        return [("s12", o[0], torch.cat([dz.sum(0), (dz * xhat).sum(0)]))]
    return run, ref


def col_sum_case(dev, exact, g, m, c, ld, dtype):
    from byol_b200 import ops
    x = _vals((m, c), exact, g, 3)
    full = torch.full((m, ld), float("nan"))          # the pitch columns must never be read
    full[:, :c] = x
    xd = full.to(dev, dtype)[:, :c]

    def run():
        out = torch.zeros(c, device=dev)
        ops.col_sum(xd, out)
        return [out]
    return run, lambda o: [("col_sum", o[0], x.double().sum(0))]


def conv_stats_case(dev, exact, g, n, h, w, c, cout, k, s, p, gather):
    from byol_b200 import ops
    x = _vals((n, h, w, c), exact, g, 1, 0.25)
    wt = _vals((cout, c, k, k), exact, g, 1, 0.5) if exact else \
        (torch.randn(cout, c, k, k, generator=g) / (c * k * k) ** 0.5).to(BF).float()
    xd = x.to(dev, BF)
    w_f, _ = ops.prep_weight(wt.to(dev), cpad=c, want_dgrad=False)

    def run():
        st = torch.zeros(2 * cout, device=dev)
        y = ops.conv_fprop(xd, w_f, k, k, s, p, stats=st, force_gather=gather)
        return [st, y]

    def ref(o):
        y = torch.nn.functional.conv2d(_nchw(x), wt.double(), stride=s, padding=p).permute(0, 2, 3, 1)
        return [("y", o[1], y), ("stats", o[0], _colstats(o[1].reshape(-1, cout)))]
    return run, ref


def stem_stats_case(dev, exact, g, n, h, w):
    from byol_b200 import ops
    x = _vals((n, 3, h, w), exact, g, 1, 0.5)
    wt = _vals((64, 3, 7, 7), exact, g, 1, 0.5) if exact else (torch.randn(64, 3, 7, 7, generator=g) / 12).to(BF).float()
    xs4, ws = ops.nchw_to_stem4(x.to(dev)), ops.prep_weight_stem4(wt.to(dev))

    def run():
        st = torch.zeros(128, device=dev)
        y = ops.stem_conv_fprop(xs4, ws, h, w, stats=st)
        return [st, y]

    def ref(o):
        y = torch.nn.functional.conv2d(x.double(), wt.double(), stride=2, padding=3).permute(0, 2, 3, 1)
        return [("y", o[1], y), ("stats", o[0], _colstats(o[1].reshape(-1, 64)))]
    return run, ref


def wgrad_case(dev, exact, g, n, h, w, c, cout, k, s, p, gather):
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    x, dy = _vals((n, h, w, c), exact, g, 1, 0.25), _vals((n, ho, wo, cout), exact, g, 1, 0.25)
    dw0 = _vals((cout, c, k, k), exact, g, 3)                 # wgrad accumulates: start from a non-zero gradient
    xd, dyd, dw0d = x.to(dev, BF), dy.to(dev, BF), dw0.to(dev)

    def run():
        dw = dw0d.clone()
        ops.conv_wgrad(xd, dyd, dw, k, k, s, p, force_gather=gather)
        return [dw]

    def ref(o):
        dw = torch.nn.grad.conv2d_weight(_nchw(x), (cout, c, k, k), _nchw(dy), stride=s, padding=p)
        return [("dw", o[0], dw + dw0.double())]
    return run, ref


def stem_wgrad_case(dev, exact, g, n, h, w):
    from byol_b200 import ops
    x, dy = _vals((n, 3, h, w), exact, g, 1, 0.5), _vals((n, h // 2, w // 2, 64), exact, g, 1, 0.25)
    dw0 = _vals((64, 3, 7, 7), exact, g, 3)
    xs4, dyd, dw0d = ops.nchw_to_stem4(x.to(dev)), dy.to(dev, BF), dw0.to(dev)

    def run():
        dw = dw0d.clone()
        ops.stem_conv_wgrad(xs4, dyd, dw, h, w)
        return [dw]

    def ref(o):
        dw = torch.nn.grad.conv2d_weight(x.double(), (64, 3, 7, 7), _nchw(dy), stride=2, padding=3)
        return [("dw", o[0], dw + dw0.double())]
    return run, ref


def mlp_case(dev, exact, g, b, k1, h, o):
    from byol_b200 import ops
    if not ops.mlp_fused_supported(b, k1, h, o):
        pytest.skip("shape not supported by the cooperative kernel on this device")
    x = _vals((b, k1), exact, g, 1, 1.0 / 16)
    w1, w2 = _vals((h, k1), exact, g, 1, 0.5), _vals((o, h), exact, g, 1, 0.25)
    if exact:
        # gamma = 0: the BatchNorm output is relu(beta), small integers, so the second GEMM (split-K, fp32 output
        # through the fixed-point accumulators) is exact as well
        b1, b2 = torch.randint(-2, 3, (h,), generator=g).float(), torch.randint(-2, 3, (o,), generator=g).float()
        gamma, beta = torch.zeros(h), torch.randint(-1, 3, (h,), generator=g).float()
    else:
        w1, w2 = (w1 / k1 ** 0.5).to(BF).float(), (w2 / h ** 0.5).to(BF).float()
        b1, b2 = torch.randn(h, generator=g) * 0.1, torch.randn(o, generator=g) * 0.1
        gamma, beta = torch.rand(h, generator=g) + 0.5, torch.randn(h, generator=g) * 0.1
    xd, w1d, w2d = x.to(dev, BF), w1.to(dev, BF), w2.to(dev, BF)
    b1d, b2d, gd, bd = b1.to(dev), b2.to(dev), gamma.to(dev), beta.to(dev)
    rm, rv = torch.zeros(h, device=dev), torch.ones(h, device=dev)
    coeffs = torch.empty(4, h, device=dev)
    bar = torch.zeros(2, dtype=torch.int32, device=dev)

    def run():
        stats = torch.zeros(2 * h, device=dev)
        out, hs, as_ = ops.mlp_fused_fwd(xd, w1d, b1d, gd, bd, w2d, b2d, stats, rm, rv, 0.1, 1e-5, b, coeffs, bar,
                                         True, True)
        return [stats, out, hs, as_]

    def ref(outs):
        hid = x.double() @ w1.double().t() + b1.double()
        a = torch.relu(beta.double()).expand(b, h)
        return [("h", outs[2], hid), ("a", outs[3], a), ("stats", outs[0], _colstats(outs[2])),
                ("out", outs[1], outs[3].cpu().double() @ w2.double().t() + b2.double())]
    return run, ref


def loss_case(dev, exact, g, rows, dim):
    from byol_b200 import ops
    q1, q2, z1, z2 = [_vals((rows, dim), True, g, 3) if exact else torch.randn(rows, dim, generator=g)
                      for _ in range(4)]
    d = [t.to(dev) for t in (q1, q2, z1, z2)]

    def run():
        ws, loss, saved = torch.zeros(6, dtype=F64, device=dev), torch.zeros(1, device=dev), torch.zeros(6, device=dev)
        ops.loss_fwd(*d, ws, loss, saved)
        return [saved, loss]

    def ref(o):
        q1d, q2d, z1d, z2d = [t.double() for t in (q1, q2, z1, z2)]
        sums = torch.stack([(q1d * q1d).sum(), (q2d * q2d).sum(), (z1d * z1d).sum(), (z2d * z2d).sum(),
                            (q1d * z2d).sum(), (q2d * z1d).sum()])
        # saved = the four norms (fp32 sqrt of the fp32 sums, correctly rounded) and the two inner products
        want = torch.cat([torch.sqrt(sums[:4].float()).double(), sums[4:]])
        return [("saved", o[0], want)]
    return run, ref


def stats_f32_case(dev, exact, g, m, c):
    from byol_b200 import ops
    y = _vals((m, c), True, g, 40) * 0.0625 if exact else torch.randn(m, c, generator=g) * 0.3 + 5.0
    yd = y.to(dev)

    def run():
        st = torch.zeros(2 * c, dtype=F64, device=dev)
        ops.stats_f32(yd, st)
        return [st]
    return run, lambda o: [("stats64", o[0], _colstats(y))]


def bn_bwd_reduce_f32_case(dev, exact, g, m, c, mask_mode):
    """The fp32 path's BatchNorm-backward sums (fp64 partials per row block): dz = g, or g where y*scale + shift > 0
    (mask_mode 1), or where the mask bits are set (3); s12 += [sum dz, sum dz * (y - mean) * invstd]."""
    from byol_b200 import ops
    from tests.util import pack_bits
    gy, y = _vals((m, c), exact, g, 3) * 0.5, _vals((m, c), exact, g, 3)
    mean = torch.randint(-2, 3, (c,), generator=g).float()
    invstd = torch.pow(2.0, torch.randint(-1, 2, (c,), generator=g).float())
    scale = torch.pow(2.0, torch.randint(-1, 2, (c,), generator=g).float())
    scale = scale * (torch.randint(0, 2, (c,), generator=g) * 2 - 1)
    shift = torch.randint(-2, 3, (c,), generator=g).float()
    keep = None
    if mask_mode == 1:
        keep = y * scale + shift > 0
    elif mask_mode == 3:
        keep = torch.rand((m, c), generator=g) > 0.4
    mk = pack_bits(keep).to(dev) if mask_mode == 3 else None
    coeffs = torch.stack([scale, shift, mean, invstd]).to(dev)
    gd, yd = gy.to(dev), y.to(dev)

    def run():
        s12 = torch.zeros(2 * c, dtype=F64, device=dev)
        ops.bn_bwd_reduce_f32(gd, yd, coeffs, s12, mask_mode, mask=mk)
        return [s12]

    def ref(o):
        dz = gy.double() * (keep.double() if keep is not None else 1.0)
        xhat = (y.double() - mean.double()) * invstd.double()
        return [("s12", o[0], torch.cat([dz.sum(0), (dz * xhat).sum(0)]))]
    return run, ref


def gn_stats_case(dev, exact, g, n, h, w, c, big=False):
    """GroupNorm statistics: fp64 (sum, sum of squares) per (image, group) in sums64 and (mean, rstd); big: every
    value +-8192, so the sums of squares pass 2^45 (2^26 per value)"""
    from byol_b200 import ops
    from tests.util import gn_finalize_restated
    y = _vals((n, h, w, c), exact, g, 3)
    if big:
        y = torch.where(torch.rand((n, h, w, c), generator=g) < 0.5, 8192.0, -8192.0)
    yd = y.to(dev, BF)
    cnt = h * w * (c // 32)

    def run():
        sums = torch.zeros((n, 32, 2), dtype=F64, device=dev)
        st = ops.gn_stats(yd, 1e-5, sums64=sums)
        return [st, sums]

    def ref(o):
        v = y.double().reshape(n, -1, 32, c // 32)
        sums = torch.stack([v.sum((1, 3)), (v * v).sum((1, 3))], -1)
        st = torch.from_numpy(gn_finalize_restated(sums.numpy(), float(cnt), 1e-5)).double()
        return [("sums64", o[1], sums), ("stats", o[0], st)]
    return run, ref


def gn_bwd_reduce_case(dev, exact, g, n, h, w, c, mask_mode, big=False):
    """GroupNorm-backward sums: s12 [n, 32, 2] += (sum gamma*dz, sum gamma*dz*xhat) per (image, group), dbeta / dgamma
    [c] += sum dz / sum dz*xhat per channel; big: dz = xhat = +-8192, so the channel sums pass 2^45"""
    from byol_b200 import ops
    gy, x = _vals((n, h, w, c), exact, g, 3), _vals((n, h, w, c), exact, g, 3)
    if big:
        gy = torch.full((n, h, w, c), 8192.0)
        x = torch.where(torch.rand((n, h, w, c), generator=g) < 0.95, 8192.0, -8192.0)
    if exact:
        gamma = torch.pow(2.0, torch.randint(-1, 2, (c,), generator=g).float())
        mean = torch.randint(-2, 3, (n, 32), generator=g).float() * (not big)
        rstd = torch.pow(2.0, torch.randint(-1, 2, (n, 32), generator=g).float()) if not big else torch.ones(n, 32)
    else:
        gamma, mean, rstd = torch.rand(c, generator=g) + 0.5, torch.randn(n, 32, generator=g) * 0.1, \
            torch.rand(n, 32, generator=g) + 0.5
    act = _vals((n, h, w, c), exact, g, 2) if mask_mode == 2 else None
    st = torch.stack([mean, rstd], -1).to(dev)
    gd, xd, gmd, bd = gy.to(dev, BF), x.to(dev, BF), gamma.to(dev), torch.zeros(c, device=dev)
    actd = act.to(dev, BF) if act is not None else None

    def run():
        s12, dg, db = torch.zeros((n, 32, 2), device=dev), torch.zeros(c, device=dev), torch.zeros(c, device=dev)
        ops.gn_bwd_reduce(gd, xd, gmd, bd, st, s12, mask_mode, dgamma=dg, dbeta=db, act=actd)
        return [s12, dg, db]

    def ref(o):
        grp = torch.arange(c) // (c // 32)
        dz = gy.double() * ((act > 0).double() if act is not None else 1.0)
        xh = (x.double() - mean.double()[:, grp].view(n, 1, 1, c)) * rstd.double()[:, grp].view(n, 1, 1, c)
        gdz = gamma.double() * dz
        s1 = gdz.reshape(n, -1, 32, c // 32).sum((1, 3))
        s2 = (gdz * xh).reshape(n, -1, 32, c // 32).sum((1, 3))
        return [("s12", o[0], torch.stack([s1, s2], -1)), ("dgamma", o[1], (dz * xh).sum((0, 1, 2))),
                ("dbeta", o[2], dz.sum((0, 1, 2)))]
    return run, ref


def augment_case(dev, exact, g, n, hs, ws, r):
    from byol_b200.augment import TwoViewAugment
    imgs = torch.rand(n, 3, hs, ws, generator=g).to(dev)
    aug = TwoViewAugment(image_size=r, seed=5)
    params = aug.sample_params(n, hs, ws, dev)

    def run():
        return list(aug.apply(imgs, params))
    return run, None


# (builder, shape): real sizes for the exact checks
EXACT = {
    "bn_stats_2^20x64": (bn_stats_case, dict(m=1 << 20, c=64)),
    "bn_stats_4096ch": (bn_stats_case, dict(m=512, c=4096)),
    "bn_bwd_reduce_fixed_grid_2^20x64": (bn_bwd_reduce_case, dict(m=1 << 20, c=64, mask_mode=0)),
    "bn_bwd_reduce_row_blocks_c96": (bn_bwd_reduce_case, dict(m=300000, c=96, mask_mode=2)),
    "bn_bwd_reduce_wide_c4096": (bn_bwd_reduce_case, dict(m=512, c=4096, mask_mode=0)),
    "bn_bwd_reduce_wide_row_blocks_c4800": (bn_bwd_reduce_case, dict(m=200, c=4800, mask_mode=2)),
    "col_sum_bf16_pitched": (col_sum_case, dict(m=60000, c=1000, ld=1032, dtype=BF)),
    "col_sum_f32_pitched": (col_sum_case, dict(m=60000, c=1000, ld=1032, dtype=torch.float32)),
    "conv1x1_tma_real": (conv_stats_case, dict(n=22, h=56, w=56, c=64, cout=256, k=1, s=1, p=0, gather=False)),
    "conv1x1_gather_real": (conv_stats_case, dict(n=22, h=56, w=56, c=64, cout=256, k=1, s=1, p=0, gather=True)),
    "conv1x1_s2": (conv_stats_case, dict(n=4, h=28, w=28, c=256, cout=512, k=1, s=2, p=0, gather=False)),
    "conv3x3_s2_gather": (conv_stats_case, dict(n=4, h=28, w=28, c=128, cout=128, k=3, s=2, p=1, gather=False)),
    "conv3x3_gather_14": (conv_stats_case, dict(n=8, h=14, w=14, c=128, cout=128, k=3, s=1, p=1, gather=False)),
    "conv3x3_patch_real": (conv_stats_case, dict(n=22, h=56, w=56, c=64, cout=64, k=3, s=1, p=1, gather=False)),
    "conv3x3_patch_24": (conv_stats_case, dict(n=3, h=24, w=24, c=128, cout=128, k=3, s=1, p=1, gather=False)),
    "conv3x3_patch_30x26": (conv_stats_case, dict(n=3, h=30, w=26, c=64, cout=256, k=3, s=1, p=1, gather=False)),
    "stem_30x26": (stem_stats_case, dict(n=3, h=30, w=26)),
    "stem_real": (stem_stats_case, dict(n=6, h=224, w=224)),
    "wgrad1x1_tma_real": (wgrad_case, dict(n=22, h=56, w=56, c=64, cout=256, k=1, s=1, p=0, gather=False)),
    "wgrad1x1_gather_real": (wgrad_case, dict(n=22, h=56, w=56, c=64, cout=256, k=1, s=1, p=0, gather=True)),
    "wgrad3x3_gather": (wgrad_case, dict(n=4, h=14, w=14, c=128, cout=128, k=3, s=1, p=1, gather=True)),
    "wgrad3x3_s2": (wgrad_case, dict(n=4, h=28, w=28, c=128, cout=128, k=3, s=2, p=1, gather=False)),
    "wgrad3x3_patch_real": (wgrad_case, dict(n=22, h=56, w=56, c=64, cout=64, k=3, s=1, p=1, gather=False)),
    "wgrad3x3_patch_30x26": (wgrad_case, dict(n=3, h=30, w=26, c=64, cout=256, k=3, s=1, p=1, gather=False)),
    "stem_wgrad_30x26": (stem_wgrad_case, dict(n=3, h=30, w=26)),
    "stem_wgrad_real": (stem_wgrad_case, dict(n=6, h=224, w=224)),
    "mlp_fused_512": (mlp_case, dict(b=512, k1=2048, h=4096, o=256)),
    "mlp_fused_24": (mlp_case, dict(b=24, k1=256, h=4096, o=256)),
    "loss_fwd": (loss_case, dict(rows=512, dim=256)),
    "stats_f32": (stats_f32_case, dict(m=1 << 18, c=64)),
    # the fp32 path's backward sums: C below and above 256 (a second, partial column tile), row counts that leave the
    # last row block short
    "bn_bwd_reduce_f32_m0_c96": (bn_bwd_reduce_f32_case, dict(m=3001, c=96, mask_mode=0)),
    "bn_bwd_reduce_f32_m1_c300": (bn_bwd_reduce_f32_case, dict(m=2999, c=300, mask_mode=1)),
    "bn_bwd_reduce_f32_m3_c264": (bn_bwd_reduce_f32_case, dict(m=5003, c=264, mask_mode=3)),
    "bn_bwd_reduce_f32_m3_c64": (bn_bwd_reduce_f32_case, dict(m=REAL_M + 37 * 8, c=64, mask_mode=3)),
    # GroupNorm: C/8 dividing 256 (a thread stays on one vector) and not (it changes vector every iteration), the
    # 224 px stem map (13 blocks per image, the last one short), and totals past 2^45
    "gn_stats_stem224": (gn_stats_case, dict(n=3, h=112, w=112, c=64)),
    "gn_stats_c96": (gn_stats_case, dict(n=3, h=30, w=26, c=96)),
    "gn_stats_past_2^45": (gn_stats_case, dict(n=1, h=1024, w=512, c=64, big=True)),
    "gn_bwd_reduce_stem224": (gn_bwd_reduce_case, dict(n=3, h=112, w=112, c=64, mask_mode=0)),
    "gn_bwd_reduce_c96": (gn_bwd_reduce_case, dict(n=3, h=30, w=26, c=96, mask_mode=2)),
    "gn_bwd_reduce_past_2^45": (gn_bwd_reduce_case, dict(n=3, h=512, w=512, c=64, mask_mode=0, big=True)),
}

# smaller shapes for the run-to-run checks (four launches each, plus a graph capture)
BITS = {
    "bn_stats": (bn_stats_case, dict(m=200000, c=64)),
    "bn_bwd_reduce_fixed_grid": (bn_bwd_reduce_case, dict(m=100000, c=64, mask_mode=0)),
    "bn_bwd_reduce_row_blocks": (bn_bwd_reduce_case, dict(m=100000, c=96, mask_mode=2)),
    "bn_bwd_reduce_wide": (bn_bwd_reduce_case, dict(m=512, c=4096, mask_mode=0)),
    "col_sum_bf16": (col_sum_case, dict(m=20000, c=1000, ld=1032, dtype=BF)),
    "col_sum_f32": (col_sum_case, dict(m=20000, c=1000, ld=1032, dtype=torch.float32)),
    "conv1x1_tma": (conv_stats_case, dict(n=8, h=28, w=28, c=64, cout=256, k=1, s=1, p=0, gather=False)),
    "conv1x1_gather": (conv_stats_case, dict(n=8, h=28, w=28, c=64, cout=256, k=1, s=1, p=0, gather=True)),
    "conv3x3_patch": (conv_stats_case, dict(n=3, h=30, w=26, c=64, cout=256, k=3, s=1, p=1, gather=False)),
    "stem": (stem_stats_case, dict(n=3, h=64, w=64)),
    "wgrad1x1_tma": (wgrad_case, dict(n=8, h=28, w=28, c=64, cout=256, k=1, s=1, p=0, gather=False)),
    "wgrad1x1_gather": (wgrad_case, dict(n=8, h=28, w=28, c=64, cout=256, k=1, s=1, p=0, gather=True)),
    "wgrad3x3_patch": (wgrad_case, dict(n=3, h=30, w=26, c=64, cout=64, k=3, s=1, p=1, gather=False)),
    "stem_wgrad": (stem_wgrad_case, dict(n=3, h=64, w=64)),
    "mlp_fused": (mlp_case, dict(b=24, k1=256, h=4096, o=256)),
    "loss_fwd": (loss_case, dict(rows=512, dim=256)),
    "stats_f32": (stats_f32_case, dict(m=50000, c=64)),
    "augment": (augment_case, dict(n=8, hs=96, ws=128, r=64)),
    "gn_stats": (gn_stats_case, dict(n=3, h=112, w=112, c=64)),
    "gn_stats_c96": (gn_stats_case, dict(n=3, h=30, w=26, c=96)),
    "gn_bwd_reduce": (gn_bwd_reduce_case, dict(n=3, h=112, w=112, c=64, mask_mode=0)),
    "gn_bwd_reduce_c96": (gn_bwd_reduce_case, dict(n=3, h=30, w=26, c=96, mask_mode=2)),
}


@pytest.mark.parametrize("name", list(EXACT))
def test_exact_parity_with_fp64(cuda, name):
    build, shape = EXACT[name]
    run, ref = build(cuda, True, _gen(sum(map(ord, name))), **shape)
    outs = run()
    torch.cuda.synchronize()
    for label, got, want in ref(outs):
        _expect_equal("%s %s" % (name, label), got, want)


def _other_reduction(dev):
    from byol_b200 import ops
    ops.bn_stats(torch.ones(3000, 200, dtype=BF, device=dev), torch.zeros(400, device=dev))


@contextlib.contextmanager
def _capture(g, stream):
    """torch.cuda.graph with Python's cycle collector off: a dead model of an earlier test that still owns captured
    graphs must not be finalized (cudaGraphExecDestroy) in the middle of this capture."""
    gc.collect()
    gc.disable()
    try:
        with torch.cuda.graph(g, stream=stream):
            yield
    finally:
        gc.enable()


def _graph_outputs(run):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run()                                  # the capture stream's scratch exists before the capture
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with _capture(g, side):
        outs = run()
    g.replay()
    g.replay()                                 # a replay leaves the scratch zeroed for the next one
    torch.cuda.synchronize()
    return [o.clone() for o in outs], g


@pytest.mark.parametrize("name", list(BITS))
def test_run_to_run_bits(cuda, name):
    build, shape = BITS[name]
    run, _ = build(cuda, False, _gen(sum(map(ord, name))), **shape)
    base = [o.clone() for o in run()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        on_new_stream = [o.clone() for o in run()]
    torch.cuda.current_stream().wait_stream(s)
    _other_reduction(cuda)
    after_other = [o.clone() for o in run()]
    from_graph, _ = _graph_outputs(run)
    torch.cuda.synchronize()
    for label, outs in (("new stream", on_new_stream), ("scratch reused", after_other), ("CUDA graph", from_graph)):
        for i, (a, b) in enumerate(zip(base, outs)):
            assert torch.equal(a, b), "%s output %d: %s launch differs in %d values" % (
                name, i, label, int((a != b).sum()))


# ------------------------------------------------------------------------------------------------------------------
# special values
# ------------------------------------------------------------------------------------------------------------------
NAN, INF = float("nan"), float("inf")


def test_special_values_bn_stats(cuda):
    """One special case per column of a 2^20-row bn_stats (1 056 blocks); columns 8.. are untouched random data and
    must keep the bits of the run without the special columns."""
    from byol_b200 import ops
    m, c = 1 << 20, 16
    x = (torch.randn(m, c, generator=_gen(31)) * 3).to(BF).float()
    xs = x.clone()
    xs[5, 0] = NAN
    xs[7, 1] = INF
    xs[3, 2], xs[m - 3, 2] = INF, -INF
    xs[:, 3] = 0.0
    xs[0, 3], xs[m - 1, 3] = 3.0, -3.0                   # first and last block: the sum cancels exactly
    xs[:, 4] = 0.0
    xs[1, 4], xs[m - 2, 4] = 2.0 ** 37, -2.0 ** 37        # huge addends (fp64 side sum), cancelling exactly
    xs[m // 2, 5] = 1.5 * 2.0 ** 40                      # one huge addend among ordinary ones
    xs[:, 6] = 8192.0                                     # sum of squares 2^46: past the 2^45 range of the hi word
    xs[:, 7] = -8192.0
    outs = []
    for t in (x, xs):
        st = torch.zeros(2 * c, device=cuda)
        ops.bn_stats(t.to(cuda, BF), st)
        outs.append(st.cpu())
    base, got = outs
    s, q = got[:c], got[c:]
    assert torch.equal(got.view(2, c)[:, 8:], base.view(2, c)[:, 8:])
    assert math.isnan(s[0]) and math.isnan(q[0])
    assert s[1] == INF and q[1] == INF
    assert math.isnan(s[2]) and q[2] == INF
    assert s[3] == 0.0 and q[3] == 18.0
    assert s[4] == 0.0 and q[4] == 2.0 ** 75
    ref = _colstats(xs[:, 5:6])
    assert abs(float(s[5]) - float(ref[0])) <= 1e-6 * abs(float(ref[0]))
    assert abs(float(q[5]) - float(ref[1])) <= 1e-6 * abs(float(ref[1]))
    assert s[6] == 2.0 ** 33 and q[6] == 2.0 ** 46, (float(s[6]), float(q[6]))
    assert s[7] == -2.0 ** 33 and q[7] == 2.0 ** 46, (float(s[7]), float(q[7]))


@pytest.mark.parametrize("c", [64, 96])
def test_special_values_bn_bwd_reduce(cuda, c):
    """NaN / Inf in the gradient, and sums of dz*xhat past +2^45 and below -2^45 (fixed-grid and row-block paths)."""
    from byol_b200 import ops
    m = 1 << 20
    gen = _gen(37 + c)
    gy = (torch.randn(m, c, generator=gen)).to(BF).float()
    x = (torch.randn(m, c, generator=gen)).to(BF).float()
    coeffs = torch.stack([torch.ones(c), torch.zeros(c), torch.zeros(c), torch.ones(c)]).to(cuda)
    gs, xs = gy.clone(), x.clone()
    gs[11, 0] = NAN
    gs[13, 1], xs[13, 1] = INF, 1.0
    gs[:, 2], xs[:, 2] = 8192.0, 8192.0
    gs[:, 3], xs[:, 3] = -8192.0, 8192.0
    outs = []
    for a, b in ((gy, x), (gs, xs)):
        s12 = torch.zeros(2 * c, device=cuda)
        ops.bn_bwd_reduce(a.to(cuda, BF), b.to(cuda, BF), coeffs, s12, 0)
        outs.append(s12.cpu().view(2, c))
    base, got = outs
    assert torch.equal(got[:, 4:], base[:, 4:])
    assert math.isnan(got[0, 0]) and math.isnan(got[1, 0])
    assert got[0, 1] == INF and got[1, 1] == INF
    assert got[0, 2] == 2.0 ** 33 and got[1, 2] == 2.0 ** 46, got[:, 2]
    assert got[0, 3] == -2.0 ** 33 and got[1, 3] == -2.0 ** 46, got[:, 3]


def test_special_values_gemm_epilogue_total_past_2_45(cuda):
    """2^18 rows of y = 2^14 give a sum of squares of 2^46 through the implicit-GEMM epilogue.  It sums a warp's rows
    in fp32 registers until it moves to other columns, so each addend here is far above 2^20 and mostly lands in the
    fp64 side sum: the total must still equal fp64 exactly."""
    from byol_b200 import ops
    m, k, n = 1 << 18, 64, 128
    gen = _gen(41)
    x = _vals((m, k), True, gen, 1, 0.25)
    w = _vals((n, k), True, gen, 1, 0.5)
    x[:, 0] = 128.0
    w[:, 0] = 0.0
    w[0, :], w[0, 0] = 0.0, 128.0                        # column 0 of y is 2^14 in every row
    xd, wd = x.to(cuda, BF), w.to(cuda, BF)
    st_ig = torch.zeros(2 * n, device=cuda)
    y_ig = ops.linear_fprop(xd, ops.prep_weight(w.to(cuda), want_dgrad=False)[0], stats=st_ig)
    torch.cuda.synchronize()
    _expect_equal("implicit-GEMM stats", st_ig, _colstats(y_ig))
    assert float(st_ig[n]) == 2.0 ** 46


def test_special_values_col_sum_f32(cuda):
    """fp32 column sums: NaN, Inf, cancellation across blocks, a huge addend, and sub-resolution values (the fixed point
    rounds each block's partial to 2^-50)."""
    from byol_b200 import ops
    m, c = 60000, 16
    gen = _gen(43)
    x = torch.randn(m, c, generator=gen)
    xs = x.clone()
    xs[9, 0] = NAN
    xs[9, 1] = -INF
    xs[2, 2], xs[m - 2, 2] = INF, -INF
    xs[:, 3] = 0.0
    xs[0, 3], xs[m - 1, 3] = 0.75, -0.75
    xs[m // 3, 4] = 3.0 * 2.0 ** 40
    xs[:, 5] = torch.randint(1, 1001, (m,), generator=gen).float() * 2.0 ** -60    # ~1e-15 .. 1e-12, exact partials
    outs = []
    for t in (x, xs):
        out = torch.zeros(c, device=cuda)
        ops.col_sum(t.to(cuda), out)
        outs.append(out.cpu())
    base, got = outs
    assert torch.equal(got[6:], base[6:])
    assert math.isnan(got[0]) and got[1] == -INF and math.isnan(got[2]) and got[3] == 0.0
    ref4 = float(xs[:, 4].double().sum())
    assert abs(float(got[4]) - ref4) <= 1e-6 * abs(ref4)
    # col_sum splits the rows over at most 64 blocks: at most 64 roundings of 2^-51 each, then one fp32 rounding
    ref5 = float(xs[:, 5].double().sum())
    ulp = math.ulp(float(got[5]))
    ulp32 = ulp * 2.0 ** 29                                # fp32 has 29 fewer mantissa bits than fp64
    assert abs(float(got[5]) - ref5) <= 64 * 2.0 ** -51 + ulp32 / 2, (float(got[5]), ref5)


# ------------------------------------------------------------------------------------------------------------------
# scratch lifecycle
# ------------------------------------------------------------------------------------------------------------------
def _exact_col_sum(dev, m, c, seed):
    from byol_b200 import ops
    x = torch.randint(-3, 4, (m, c), generator=_gen(seed)).float()
    out = torch.zeros(c, device=dev)
    ops.col_sum(x.to(dev), out)
    return out, x.double().sum(0)


def test_scratch_growth(cuda):
    """small reduction, one that grows the stream's scratch past every other reduction of this file, small again"""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        runs = [_exact_col_sum(cuda, 500, 24, 1), _exact_col_sum(cuda, 8, 300000, 2), _exact_col_sum(cuda, 500, 24, 1)]
    torch.cuda.synchronize()
    for i, (got, want) in enumerate(runs):
        _expect_equal("growth run %d" % i, got, want)


def test_error_return_after_taking_the_scratch(cuda):
    """bn_bwd_reduce takes the scratch before it rejects a channel count whose accumulators do not fit in shared
    memory: it raises, and the next reductions on that stream are still exact."""
    from byol_b200 import ops
    from byol_b200._lib import ByolLibraryError
    m, c = 16, 4824
    z = torch.zeros(m, c, dtype=BF, device=cuda)
    coeffs = torch.ones(4, c, device=cuda)
    with pytest.raises(ByolLibraryError, match="too wide"):
        ops.bn_bwd_reduce(z, z, coeffs, torch.zeros(2 * c, device=cuda), 0)
    run, ref = bn_stats_case(cuda, True, _gen(3), m=5000, c=64)
    got = run()
    run2, ref2 = bn_bwd_reduce_case(cuda, True, _gen(4), m=5000, c=64, mask_mode=0)
    got2 = run2()
    torch.cuda.synchronize()
    for label, a, b in ref(got) + ref2(got2):
        _expect_equal("after the error: " + label, a, b)


def test_graph_replay_after_scratch_growth(cuda):
    """A captured reduction keeps its (old) scratch buffer when an eager reduction on the same stream grows the
    scratch: replaying it afterwards gives the same bits."""
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    run, _ = bn_stats_case(cuda, False, _gen(5), m=100000, c=64)
    with torch.cuda.stream(s):
        run()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with _capture(g, s):
        outs = run()
    g.replay()
    torch.cuda.synchronize()
    first = outs[0].clone()
    with torch.cuda.stream(s):
        big, want = _exact_col_sum(cuda, 4, 1000000, 6)          # grows the stream's scratch
    torch.cuda.synchronize()
    _expect_equal("growing reduction", big, want)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(outs[0], first)
    with torch.cuda.stream(s):
        again = run()[0]
    torch.cuda.synchronize()
    assert torch.equal(again, first)


def test_two_streams_flush_into_one_destination(cuda):
    """The two backward views flush dgamma / dbeta / wgrad sums into one zeroed gradient from two streams: the result
    equals either sequential order bit for bit."""
    from byol_b200 import ops
    gen = _gen(7)
    xa, xb = [(torch.randn(100000, 64, generator=gen) * 2).to(cuda, BF) for _ in range(2)]
    ya, yb = [(torch.randn(4, 28, 28, 64, generator=gen)).to(cuda, BF) for _ in range(2)]
    da, db = [(torch.randn(4, 28, 28, 128, generator=gen)).to(cuda, BF) for _ in range(2)]

    def seq(order):
        st, dw = torch.zeros(128, device=cuda), torch.zeros(128, 64, 1, 1, device=cuda)
        for i in order:
            ops.bn_stats((xa, xb)[i], st)
            ops.conv_wgrad((ya, yb)[i], (da, db)[i], dw, 1, 1, 1, 0)
        return st, dw
    ab, ba = seq((0, 1)), seq((1, 0))
    st, dw = torch.zeros(128, device=cuda), torch.zeros(128, 64, 1, 1, device=cuda)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for i, s in enumerate(streams):
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            ops.bn_stats((xa, xb)[i], st)
            ops.conv_wgrad((ya, yb)[i], (da, db)[i], dw, 1, 1, 1, 0)
    for s in streams:
        torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    assert torch.equal(ab[0], ba[0]) and torch.equal(ab[1], ba[1])
    assert torch.equal(st, ab[0]) and torch.equal(dw, ab[1])


def test_gradient_less_gn_bwd_reduce_cannot_dirty_a_captured_scratch(cuda):
    """gn_bwd_reduce always accumulates its per-channel sums in the stream's scratch; only their flush into dgamma /
    dbeta leaves those slots at zero.  A graph captured earlier on the stream holds no memset (its scratch was clean
    and large enough at capture), so a call that left the channel sums behind would corrupt the replay of a captured
    gn_stats.  The C entry point refuses a call without dgamma / dbeta before it takes the scratch: the replay keeps
    the eager bits."""
    from byol_b200 import ops
    gen = _gen(11)
    n, h, w, c = 4, 8, 8, 64
    y = (torch.randn((n, h, w, c), generator=gen) * 2 + 0.5).to(cuda, BF)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.gn_stats(y, 1e-5)                          # the stream's scratch exists and is clean before the capture
    torch.cuda.synchronize()
    sums = torch.zeros((n, 32, 2), dtype=F64, device=cuda)
    g = torch.cuda.CUDAGraph()
    with _capture(g, s):
        st = ops.gn_stats(y, 1e-5, sums64=sums)
    with torch.cuda.stream(s):
        eager_sums = torch.zeros_like(sums)
        eager = ops.gn_stats(y, 1e-5, sums64=eager_sums)
        x1, g1 = y[:1], (torch.randn((1, h, w, c), generator=gen)).to(cuda, BF)
        gamma, beta = torch.ones(c, device=cuda), torch.zeros(c, device=cuda)
        st1, s12 = eager[:1].contiguous(), torch.zeros((1, 32, 2), device=cuda)
        rc = ops.lib.byol_gn_bwd_reduce(g1.data_ptr(), x1.data_ptr(), None, gamma.data_ptr(), beta.data_ptr(),
                                        st1.data_ptr(), s12.data_ptr(), None, None, 1, h * w, c, 0, s.cuda_stream)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    bad = int((sums != eager_sums).any(-1).sum())
    assert torch.equal(sums, eager_sums) and torch.equal(st, eager), \
        "the replayed gn_stats read leftover sums in %d of %d (image, group) slots" % (bad, n * 32)
    assert rc != 0, "byol_gn_bwd_reduce without dgamma / dbeta must be refused"
