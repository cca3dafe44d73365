"""GPU: the split-operand ("plane") convolutions bit for bit against float64, with plane-tagged operands.

* Plane-tagged operands.  The fp32-accurate path feeds the bf16 kernels T planes per channel (csrc/split.cu): channel
  j*C + c of an activation (or dY) holds plane A_PAT[j] of channel c, and the weight side holds plane B_PAT[j] at the
  same term j.  Here every element gets three INDEPENDENT planes (p0, p1, p2): small integers in units of 1, 2^-3 and
  2^-6.  They are deliberately not a valid split, so the float64 reference, the sum over the term set of
  conv(activation plane a, weight plane b), changes when a term is dropped, doubled, paired with the wrong plane or
  read at the wrong offset; with real splits such a mistake hides below 1e-5.
* Exactness.  Every product is a multiple of 2^-6, and each row asserts that the sum of the magnitudes of an output's
  products (with its residual or starting dW) stays below 2^24 such units, so every fp32 partial sum is exact in any
  order and on any split: the output must equal the float64 reference rounded once to fp32 (NaN matches NaN).
* Route table and launch check.  One row per (op, route) at the edges of the host predicates (conv_igemm_impl and
  conv_wgrad_impl in csrc/conv_igemm.cu, restated); one test checks under torch.profiler that each row launches the
  conv_igemm_kernel / conv_wgrad_kernel variant the restated predicate names.
* Replay.  One eager step each of ResNet-18 and a bottleneck net at precision = backward_precision = "fp32", and of
  ResNet-18 at precision "bf16x2", records the split path's calls, and every distinct call is replayed.
"""
import re

import pytest
import torch

from tests.exact import (Case, byol_train_step, check_in_fresh_process, check_row_launches, conv64, dgrad64, expect,
                         recording, replay, row_case, run_and_check, wgrad64)
from tests.test_gpu_conv_exact import igemm_route
from tests.test_gpu_elementwise_exact import (nchw_to_planes_case, prep_weight_dgrad_planes_case,
                                              prep_weight_planes_case, split_planes_case)
from tests.util import ints

pytestmark = pytest.mark.gpu
BF, F32, F64 = torch.bfloat16, torch.float32, torch.float64

# the plane patterns of csrc/split.cu (make_pattern), restated: term j pairs activation plane A_PAT[j] with weight plane
# B_PAT[j]
A_PAT = {3: (0, 0, 1), 6: (0, 0, 1, 1, 0, 2)}
B_PAT = {3: (0, 1, 0), 6: (0, 1, 0, 1, 2, 0)}
UNITS = (1.0, 2.0 ** -3, 2.0 ** -6)     # plane p holds integers times UNITS[p]
UNIT = 2.0 ** -6                        # every product of two planes is a multiple of this
WG_KROWS = 64                           # wgrad k-block rows (csrc/conv_igemm.cu)


# ------------------------------------------------------------------------------------------------------------------
# operands, layouts and the exactness bound
# ------------------------------------------------------------------------------------------------------------------
def _density(k):
    """About 16 non-zero products per output and plane pair for a reduction length k."""
    return min(1.0, (16.0 / k) ** 0.5)


def _tagged(shape, dev, g, density=1.0):
    """Three independent planes: integers in [-2, 2] / [-3, 3] / [-3, 3] times 1 / 2^-3 / 2^-6 (all exact in bf16)."""
    return [ints(shape, dev, g, amp, density) * u for amp, u in zip((2, 3, 3), UNITS)]


def _lay_act(planes, T):
    """[..., C] planes -> [..., T*C]: channel j*C + c = plane A_PAT[j] of channel c."""
    return torch.cat([planes[a] for a in A_PAT[T]], -1)


def _lay_w(planes, T):
    """[Cout, Cin, KH, KW] planes -> the fprop layout [Cout, taps*T*Cin]: column (tap*T + j)*Cin + c = plane B_PAT[j]
    of w[co, c, tap] (byol_prep_weight_planes)."""
    cout, cin = planes[0].shape[:2]
    return torch.stack([planes[b].reshape(cout, cin, -1).permute(0, 2, 1) for b in B_PAT[T]], 2).reshape(cout, -1)


def _lay_wd(planes, T):
    """[Cout, Cin, KH, KW] planes -> the dgrad layout [Cin, taps*T*Cout]: column (tap*T + j)*Cout + co = plane B_PAT[j]
    of w[co, ci, tap] (byol_prep_weight_dgrad_planes)."""
    cout, cin = planes[0].shape[:2]
    return torch.stack([planes[b].reshape(cout, cin, -1).permute(1, 2, 0) for b in B_PAT[T]], 2).reshape(cin, -1)


def _terms(T, f):
    """Sum over the term set of f(activation plane, weight plane): {00, 01, 10, 11, 02, 20} (T = 6), {00, 01, 10}."""
    return sum(f(a, b) for a, b in zip(A_PAT[T], B_PAT[T]))


def _fin_abs(t):
    return torch.where(torch.isfinite(t), t.abs(), torch.zeros_like(t))


def _assert_exact(name, mag):
    """mag: per output, the sum of |products| (+ |residual| or |dW start|).  Below 2^24 units of 2^-6 (2^18), every
    fp32 partial sum is exact, and so is wgrad's fixed-point sum (2^-50 resolution, words exact below 2^20)."""
    top = float(mag.max()) / UNIT
    assert top < 2 ** 24, "%s: operands not exact: a sum of |products| reaches %.3g units of 2^-6" % (name, top)


def _nan_counts(got, want):
    return " | NaN: %d got, %d expected" % (int(torch.isnan(got).sum()), int(torch.isnan(want).sum()))


def _expect(name, got, ref64):
    expect(name, got, ref64, note=_nan_counts)


def _poison(planes):
    """One NaN and one inf in plane 1, at elements that reach several outputs."""
    p = planes[1]
    p.view(-1)[p.numel() // 3] = float("nan")
    p.view(-1)[(2 * p.numel()) // 3 + 5] = float("inf")


# ------------------------------------------------------------------------------------------------------------------
# the host's kernel choice, restated (conv_igemm_impl / conv_wgrad_impl in csrc/conv_igemm.cu)
# ------------------------------------------------------------------------------------------------------------------
def igemm_kernel(route, ndim):
    """conv_igemm_kernel<BN, STAGES, A_TMA, GROUPED, H16> of an fp32-output call: BN 128 when Ndim > 64."""
    bn = 128 if ndim > 64 else 64
    if route == "tma":
        return r"conv_igemm_kernel<%d,3,true,false,false>" % bn
    assert route == "gather", route
    return r"conv_igemm_kernel<%d,%d,false,false,false>" % (bn, 3 if bn == 128 else 4)


def wgrad_plan(sm, T, n, ho, wo, c, cout, k, s, p):
    """(kernel regex, splits, k-blocks per split, k-blocks per term) of byol_conv_wgrad_planes."""
    fold = c == 8 and 1 < k <= 8
    ncols = k * 64 if fold else k * k * c
    bn = 128 if ncols > 64 else 64
    kb_per_term = -(-(n * ho * wo) // WG_KROWS)
    total = T * kb_per_term
    base = -(-cout // 128) * -(-ncols // bn)
    splits = max(1, min(sm // base, max(1, -(-total // 8))))
    kbs = -(-total // splits)
    splits = -(-total // kbs)
    b_tma = k == 1 and s == 1 and p == 0
    return r"conv_wgrad_kernel<%d,4,%s,false>" % (bn, "true" if b_tma else "false"), splits, kbs, kb_per_term


def _sm_count(dev):
    return torch.cuda.get_device_properties(dev).multi_processor_count


# ------------------------------------------------------------------------------------------------------------------
# builders: (device, generator, T, **shape / options) -> Case whose route is the kernel regex
# ------------------------------------------------------------------------------------------------------------------
def fprop_case(dev, g, T, n, h, w, c, cout, k, s, p, bias=False, linear=False, nonfinite=False):
    """y fp32 = conv(x planes [n, h, w, T*c], weight planes [cout, taps*T*c]) (+ bias)."""
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    d = _density(k * k * c)
    xp, wq = _tagged((n, h, w, c), dev, g, d), _tagged((cout, c, k, k), dev, g, d)
    if nonfinite:
        _poison(xp)
    b = ints((cout,), dev, g, 3) if bias else None
    xd, wf, bf = _lay_act(xp, T).to(BF), _lay_w(wq, T).to(BF), (b.float() if bias else None)

    def run():
        if linear:
            return [ops.linear_fprop(xd.view(n, T * c), wf, bias=bf, out_fp32=True)]
        return [ops.conv_fprop(xd, wf, k, k, s, p, bias=bf, out_fp32=True)]

    def check(outs):
        ref = _terms(T, lambda a, bb: conv64(xp[a], wq[bb], s, p))
        mag = _terms(T, lambda a, bb: conv64(_fin_abs(xp[a]), wq[bb].abs(), s, p))
        if bias:
            ref, mag = ref + b, mag + b.abs()
        _assert_exact("y", mag)
        _expect("y", outs[0], ref)

    route, _ = igemm_route(False, n, h, w, T * c, ho, wo, cout, k, s, p, bias=bias, out_fp32=True)
    return Case(run, check, igemm_kernel(route, cout))


def dgrad_case(dev, g, T, n, h, w, cin, cout, k, s, p, resid=False, linear=False, cout_real=None, nonfinite=False):
    """dx fp32 [n, h, w, cin] = conv_transpose(dY planes [n, ho, wo, T*cout], dgrad weight planes) (+ fp32 resid);
    cout_real < cout: the gradient columns past cout_real are +0 in every plane (a padded classifier gradient)."""
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    d = _density(k * k * cout)
    dyp, wq = _tagged((n, ho, wo, cout), dev, g, d), _tagged((cout, cin, k, k), dev, g, d)
    if cout_real:
        for t in dyp:
            t[..., cout_real:] = 0.0
    if nonfinite:
        _poison(dyp)
    r = ints((n, h, w, cin), dev, g, 100) * UNIT if resid else None
    dyd, wd, rf = _lay_act(dyp, T).to(BF), _lay_wd(wq, T).to(BF), (r.float() if resid else None)

    def run():
        if linear:
            return [ops.linear_dgrad_planes(dyd.view(n, T * cout), wd, T)]
        return [ops.conv_dgrad_planes(dyd, wd, h, w, k, k, s, p, T, resid=rf)]

    def check(outs):
        ref = _terms(T, lambda a, b: dgrad64(dyp[a], wq[b], h, w, s, p))
        mag = _terms(T, lambda a, b: dgrad64(_fin_abs(dyp[a]), wq[b].abs(), h, w, s, p))
        if resid:
            ref, mag = ref + r, mag + r.abs()
        _assert_exact("dx", mag)
        _expect("dx", outs[0], ref)

    route, _ = igemm_route(True, n, ho, wo, T * cout, h, w, cin, k, s, p, resid=resid, out_fp32=True)
    return Case(run, check, igemm_kernel(route, cin))


def wgrad_case(dev, g, T, n, h, w, c, cin_real, cout, k, s, p, ldy=None, nonfinite=False, splits=None, guard=1024):
    """dW [cout, cin_real, k, k] += sum over the terms of dY plane a^T im2col(x plane b), with dW a view into a buffer
    whose margins must keep their value; ldy > cout: pitched dY planes whose padding columns hold NaN;
    splits: "straddle" (a split runs across a term boundary) or "single", asserted from the restated host formula."""
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    ldy = ldy or cout
    d = _density(n * ho * wo)
    xp, dyp = _tagged((n, h, w, c), dev, g, d), _tagged((n, ho, wo, cout), dev, g, d)
    if nonfinite:
        _poison(xp)
    padded = []
    for t in dyp:
        tp = torch.full((n, ho, wo, ldy), float("nan"), dtype=F64, device=dev)
        tp[..., :cout] = t
        padded.append(tp)
    dw0 = ints((cout, cin_real, k, k), dev, g, 3)
    numel = dw0.numel()
    xd, dyd = _lay_act(xp, T).to(BF), _lay_act(padded, T).to(BF)
    kernel, nsplit, kbs, kb_term = wgrad_plan(_sm_count(dev), T, n, ho, wo, c, cout, k, s, p)
    if splits == "straddle":
        assert nsplit > 1 and kb_term % kbs != 0, "no split crosses a term boundary (%d splits of %d k-blocks, %d " \
            "k-blocks per term)" % (nsplit, kbs, kb_term)
    elif splits == "single":
        assert nsplit == 1, "%d splits" % nsplit

    def run():
        buf = torch.full((guard + numel + guard,), 7.0, device=dev)
        dw = buf[guard:guard + numel].view(dw0.shape)
        dw.copy_(dw0)
        ops.conv_wgrad_planes(xd, dyd, dw, k, k, s, p, T)
        return [buf]

    def check(outs):
        buf = outs[0]
        ref = _terms(T, lambda a, b: wgrad64(xp[b][..., :cin_real], dyp[a], dw0.shape, s, p)) + dw0
        mag = _terms(T, lambda a, b: wgrad64(_fin_abs(xp[b][..., :cin_real]), dyp[a].abs(), dw0.shape, s, p))
        _assert_exact("dw", mag + dw0.abs())
        _expect("dw", buf[guard:guard + numel].view(dw0.shape), ref)
        margins = torch.cat([buf[:guard], buf[guard + numel:]])
        assert bool((margins == 7.0).all()), "wgrad wrote outside dw"

    return Case(run, check, kernel)


def near_max_case(dev, g, m, k, n):
    """A linear layer on planes that split_planes / prep_weight_planes made from fp32 values at and past 0x7F7F8000
    (they round to inf in bf16): the outputs must be finite and within the T = 6 error bound of float64."""
    from byol_b200 import ops
    big = torch.tensor([0x7F7F8000, 0x7F7F7FFF, 0x7F7FFFFF, 0x7F7FC000], dtype=torch.int32).view(F32).to(dev)
    x = torch.randn((m, k), generator=g, device=dev)
    wt = torch.randn((n, k), generator=g, device=dev) * 2.0 ** -10
    x[0, :4] = big
    x[1, :4] = -big
    x[:, 5] *= 2.0 ** -20          # a weight column with FLT_MAX meets small activations only
    wt[3, 5] = float(big[2])
    wt[4, 5] = -float(big[1])
    wp = torch.empty((n, 6 * k), dtype=BF, device=dev)
    ops.prep_weight_planes(wt, 6, k, wp)

    def run():
        return [ops.linear_fprop(ops.split_planes(x, 6)[0], wp, out_fp32=True)]

    def check(outs):
        y = outs[0].double()
        ref = x.double() @ wt.double().t()
        mag = x.double().abs() @ wt.double().abs().t()
        assert bool(torch.isfinite(y).all()), "non-finite outputs from finite operands"
        # dropped terms x1w2 + x2w1 + x2w2 <= 2^-23 |xw| per product, fp32 accumulation of 6k terms
        bound = (2.0 ** -23 + 6 * k * 2.0 ** -24) * mag
        err = (y - ref).abs()
        assert bool((err <= bound).all()), "max error %.3g of a bound %.3g" % (float((err / bound).max()), 1.0)

    return Case(run, check, igemm_kernel("tma", n))


# ------------------------------------------------------------------------------------------------------------------
# the row table
# ------------------------------------------------------------------------------------------------------------------
FP, D, W = fprop_case, dgrad_case, wgrad_case
ROWS = {}
for _T in (6, 3):
    _rows = {
        # fprop on planes: the 7x7 / 2 stem over 8 padded channels (6*8 = 48, 3*8 = 24), 3x3 and 1x1 bodies at T*64
        "fprop_stem": (FP, dict(n=2, h=32, w=32, c=8, cout=64, k=7, s=2, p=3)),
        "fprop_3x3": (FP, dict(n=2, h=14, w=14, c=64, cout=64, k=3, s=1, p=1)),
        "fprop_1x1": (FP, dict(n=2, h=14, w=14, c=64, cout=256, k=1, s=1, p=0)),
        "fprop_linear_bias_n1000": (FP, dict(n=96, h=1, w=1, c=512, cout=1000, k=1, s=1, p=0, bias=True,
                                             linear=True)),
        # dgrad on planes: 1x1 / 3x3, stride 1 / 2, with and without the fp32 residual
        "dgrad_1x1": (D, dict(n=2, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0)),
        "dgrad_1x1_resid": (D, dict(n=2, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0, resid=True)),
        "dgrad_1x1s2_resid": (D, dict(n=2, h=16, w=16, cin=64, cout=128, k=1, s=2, p=0, resid=True)),
        "dgrad_3x3": (D, dict(n=2, h=14, w=14, cin=64, cout=64, k=3, s=1, p=1)),
        "dgrad_3x3_resid": (D, dict(n=2, h=14, w=14, cin=64, cout=64, k=3, s=1, p=1, resid=True)),
        "dgrad_3x3s2_resid": (D, dict(n=2, h=16, w=16, cin=64, cout=128, k=3, s=2, p=1, resid=True)),
        # Cin past the last full column tile: 200 of 256 (BN 128), 40 of 64
        "dgrad_cin200_resid": (D, dict(n=1, h=9, w=9, cin=200, cout=64, k=1, s=1, p=0, resid=True)),
        "dgrad_cin40_3x3": (D, dict(n=2, h=8, w=8, cin=40, cout=64, k=3, s=1, p=1)),
        # linear_dgrad_planes: the 4096-wide MLP layers, the 1000-class and the 10-class (padded to 16) classifier
        "linear_dgrad_mlp_out": (D, dict(n=64, h=1, w=1, cin=4096, cout=256, k=1, s=1, p=0, linear=True)),
        "linear_dgrad_mlp_in": (D, dict(n=64, h=1, w=1, cin=2048, cout=4096, k=1, s=1, p=0, linear=True)),
        "linear_dgrad_cls1000": (D, dict(n=96, h=1, w=1, cin=512, cout=1000, k=1, s=1, p=0, linear=True)),
        "linear_dgrad_cls10_pad16": (D, dict(n=96, h=1, w=1, cin=512, cout=16, k=1, s=1, p=0, linear=True,
                                             cout_real=10)),
        # wgrad on planes: TMA 1x1 (M = 392: every term ends in a partial k-block), gathered 3x3, stride 2, the
        # folded stem, a pitched 10-class classifier gradient with NaN padding columns, splits across term
        # boundaries (M = 5157) and a single split (the MLP output layer at 64 rows)
        "wgrad_1x1_tma": (W, dict(n=2, h=14, w=14, c=64, cin_real=64, cout=256, k=1, s=1, p=0)),
        "wgrad_3x3": (W, dict(n=2, h=10, w=10, c=64, cin_real=64, cout=128, k=3, s=1, p=1)),
        "wgrad_3x3s2": (W, dict(n=2, h=16, w=16, c=64, cin_real=64, cout=128, k=3, s=2, p=1)),
        "wgrad_1x1s2": (W, dict(n=2, h=16, w=16, c=64, cin_real=64, cout=256, k=1, s=2, p=0)),
        "wgrad_stem": (W, dict(n=2, h=32, w=32, c=8, cin_real=3, cout=64, k=7, s=2, p=3)),
        "wgrad_cls10_ldy16": (W, dict(n=96, h=1, w=1, c=512, cin_real=512, cout=10, ldy=16, k=1, s=1, p=0)),
        "wgrad_m81": (W, dict(n=1, h=9, w=9, c=64, cin_real=64, cout=64, k=1, s=1, p=0)),
        "wgrad_straddle": (W, dict(n=5157, h=1, w=1, c=64, cin_real=64, cout=128, k=1, s=1, p=0,
                                   splits="straddle")),
        "wgrad_single_split": (W, dict(n=64, h=1, w=1, c=4096, cin_real=4096, cout=256, k=1, s=1, p=0,
                                       splits="single")),
    }
    for _name, (_b, _kw) in _rows.items():
        ROWS["%s_t%d" % (_name, _T)] = (_b, dict(T=_T, **_kw))
# non-finite operands: a NaN and an inf in plane 1; the outputs they reach are NaN (or inf), all others exact
ROWS["fprop_nonfinite_t6"] = (FP, dict(T=6, n=2, h=10, w=10, c=64, cout=64, k=3, s=1, p=1, nonfinite=True))
ROWS["dgrad_nonfinite_t6"] = (D, dict(T=6, n=2, h=10, w=10, cin=64, cout=64, k=3, s=1, p=1, resid=True,
                                      nonfinite=True))
ROWS["wgrad_nonfinite_t6"] = (W, dict(T=6, n=2, h=10, w=10, c=64, cin_real=64, cout=128, k=3, s=1, p=1,
                                      nonfinite=True))
ROWS["near_flt_max_t6"] = (near_max_case, dict(m=64, k=64, n=64))


def _build(dev, name):
    return row_case(dev, name, *ROWS[name])


@pytest.mark.parametrize("name", list(ROWS))
def test_plane_row_exact(cuda, name):
    run_and_check(_build(cuda, name))


def _check_launches():
    cases = {name: _build(torch.device("cuda:0"), name) for name in ROWS}

    def complaints(name, launched):
        convs = sorted({k for k in launched if re.search(r"conv_(igemm|wgrad)_kernel|conv3x3|gemm_fused|stem_", k)})
        if not convs or not all(re.search(cases[name].route, k) for k in convs):
            return ["%s: expected %s, launched %s" % (name, cases[name].route, convs)]
        return []
    check_row_launches({name: case.run for name, case in cases.items()}, complaints)


def test_plane_rows_launch_their_kernels(cuda):
    """Each row launches the conv_igemm_kernel / conv_wgrad_kernel variant its restated host predicate names, and no
    other variant of either.  Checked in a fresh Python process: one that has already held many profiler sessions
    (the rest of the GPU suite) can drop CUDA kernel events."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# replay of the engine's split-path calls
# ------------------------------------------------------------------------------------------------------------------
def _shape(t):
    return None if t is None else tuple(t.shape)


def _recorders(calls, T):
    """ops function name -> recorder that notes the call's shapes, options and T (not its data)."""
    def conv_fprop(x, w_f, kh, kw, stride, pad, bias=None, resid=None, stats=None, relu=False, out_fp32=False,
                   out=None, force_gather=False):
        calls.add(("conv_fprop", T, _shape(x), _shape(w_f), kh, kw, stride, pad, bias is not None, _shape(resid),
                   stats is not None, bool(relu), bool(out_fp32), bool(force_gather)))

    def conv_dgrad_planes(dyp, wdp, h, w, kh, kw, stride, pad, T_, resid=None):
        calls.add(("conv_dgrad_planes", T_, _shape(dyp), _shape(wdp), h, w, kh, kw, stride, pad, resid is not None))

    def conv_wgrad_planes(xp, dyp, dw, kh, kw, stride, pad, T_):
        calls.add(("conv_wgrad_planes", T_, _shape(xp), _shape(dyp), _shape(dw), kh, kw, stride, pad))

    def split_planes(x2d, T_, cpad=None, want_copy=False, copy_out=None):
        calls.add(("split_planes", T_, x2d.shape[0], x2d.shape[1], cpad or x2d.shape[1], x2d.stride(0),
                   bool(want_copy) or copy_out is not None))

    def nchw_to_planes(x, T_, cpad=8, out=None):
        calls.add(("nchw_to_planes", T_, _shape(x), cpad))

    def prep_weight_planes(w, T_, cpad, out):
        calls.add(("prep_weight_planes", T_, w.shape[0], w.shape[1], w.numel() // (w.shape[0] * w.shape[1]), cpad))

    def prep_weight_dgrad_planes(w, T_, out):
        calls.add(("prep_weight_dgrad_planes", T_, w.shape[0], w.shape[1], w.numel() // (w.shape[0] * w.shape[1])))
    return {k: v for k, v in locals().items() if callable(v)}


def _replay_case(dev, g, sig):
    """Case of one recorded call, replayed with plane-tagged operands of the same shapes and options."""
    op, T = sig[0], sig[1]
    if op == "conv_fprop":
        _, _, (n, h, w, tc), ws, kh, kw, s, p, bias, resid, stats, relu, out_fp32, gather = sig
        assert tc % T == 0 and kh == kw and ws[1] == kh * kw * tc and out_fp32 and resid is None and not stats \
            and not relu and not gather, "not a plane-fed fprop: %s" % (sig,)
        return fprop_case(dev, g, T, n, h, w, tc // T, ws[0], kh, s, p, bias=bias)
    if op == "conv_dgrad_planes":
        _, _, (n, _, _, tc), wds, h, w, kh, kw, s, p, resid = sig
        assert kh == kw and wds[1] == kh * kw * tc
        return dgrad_case(dev, g, T, n, h, w, wds[0], tc // T, kh, s, p, resid=resid)
    if op == "conv_wgrad_planes":
        _, _, (n, h, w, tc), dys, dws, kh, kw, s, p = sig
        return wgrad_case(dev, g, T, n, h, w, tc // T, dws[1], dws[0], kh, s, p, ldy=dys[3] // T)
    if op == "split_planes":
        _, _, m, c, cpad, ldx, copy = sig
        return split_planes_case(dev, g, m, c, T, cpad=cpad, ldx=ldx, copy=copy)
    if op == "nchw_to_planes":
        (n, cin, h, w), cpad = sig[2], sig[3]
        return nchw_to_planes_case(dev, g, n, cin, h, w, T, cpad=cpad)
    if op == "prep_weight_planes":
        _, _, cout, cin, taps, cpad = sig
        return prep_weight_planes_case(dev, g, cout, cin, taps, T, cpad=cpad)
    if op == "prep_weight_dgrad_planes":
        _, _, cout, cin, taps = sig
        return prep_weight_dgrad_planes_case(dev, g, cout, cin, taps, T)
    raise AssertionError("no replay for %s" % (sig,))


# (arch, representation size, classes, batch, resolution, precision, backward_precision); grouped nets cannot run
# the split path (check_grouped_convs)
NETS = [("resnet18", 512, 10, 4, 64, "fp32", "fp32"), ("resnet:bottleneck:2,1,1,1", 2048, 1000, 4, 64, "fp32", "fp32"),
        ("resnet18", 512, 1000, 4, 64, "bf16x2", "bf16")]


def test_replay_split_calls_exactly(cuda):
    calls = set()
    for arch, rep, classes, b, r, precision, bwd in NETS:
        with recording(_recorders(calls, {"bf16x2": 3, "fp32": 6}[precision])):
            byol_train_step(cuda, arch, rep, b, r, classes, precision=precision, backward_precision=bwd)
        torch.cuda.empty_cache()
    by_op = {}
    for sig in calls:
        by_op.setdefault(sig[0], []).append(sig)
    for op in ("conv_fprop", "conv_dgrad_planes", "conv_wgrad_planes", "split_planes", "nchw_to_planes",
               "prep_weight_planes", "prep_weight_dgrad_planes"):
        assert op in by_op, "no %s call recorded" % op
    assert any(sig[10] for sig in by_op["conv_dgrad_planes"]), "no plane dgrad with a residual recorded"
    assert any(sig[2][3] == 8 * sig[1] and sig[5] == 7 for sig in by_op["conv_wgrad_planes"]), \
        "no folded stem wgrad recorded"
    assert any(sig[3][3] // sig[1] > sig[4][0] for sig in by_op["conv_wgrad_planes"]), \
        "no pitched classifier wgrad recorded"
    assert {sig[1] for sig in calls} == {3, 6}, "T values recorded: %s" % sorted({sig[1] for sig in calls})
    replay(cuda, calls, _replay_case, 3000,
           " (%s)" % ", ".join("%s %d" % (op, len(v)) for op, v in sorted(by_op.items())))
