"""GPU: every convolution kernel route and epilogue bit for bit against float64.

* Exact operands.  Activations, gradients and residuals are integers in [-2, 2], weights integers in [-1, 1] (sparse
  where K is large) and biases integers.  Every product and every fp32 partial sum is then an exact integer far below
  2^24, in any order and on any tile split, so a kernel output must equal the float64 reference rounded once to its
  dtype (torch.equal): a dropped channel, tap or residual, or a residual added to the wrong pixel, shows.  The
  references run in float64 on the device with cuDNN off (im2col + GEMM, exact on integers).
* Route table.  One row per (op, route, epilogue) at the edge of its host predicate (conv_igemm_impl and
  conv_wgrad_impl in csrc/conv_igemm.cu); one test checks under torch.profiler that each row launches the kernel it is
  meant for, so a row cannot drift to another route unnoticed.
* Replay.  One eager training step of a few small nets records the engine's own ops calls (shapes and options only)
  and replays every distinct call with exact operands, so the routes the product actually takes are covered too.
"""
import re

import pytest
import torch
import torch.nn.functional as F

from tests.exact import (Case, byol_train_step, check_in_fresh_process, check_row_launches, conv64, dgrad64, expect,
                         nchw, nhwc, recording, replay, rounded_like, row_case, run_and_check, wgrad64)
from tests.util import ints as _ints, pack_bits as _pack

pytestmark = pytest.mark.gpu
BF = torch.bfloat16
F64 = torch.float64


# ------------------------------------------------------------------------------------------------------------------
# operands and comparison
# ------------------------------------------------------------------------------------------------------------------
def _density(k, stats):
    """Density of both GEMM operands for a reduction length k: about 8 (with statistics: 4) non-zero products per
    output, so outputs stay small and the statistics' fp32 partial sums of squares stay exact."""
    return min(1.0, ((4.0 if stats else 8.0) / k) ** 0.5)


def _colstats(y2d):
    y = y2d.to(F64)
    return torch.cat([y.sum(0), (y * y).sum(0)])


def _bad_parities(got, want):
    """NHWC: which (h, w) parities hold the bad pixels."""
    if got.dim() != 4:
        return ""
    bad = (got.float() != want.float()).any(-1)
    hh = torch.arange(bad.shape[1], device=bad.device).view(1, -1, 1) % 2
    ww = torch.arange(bad.shape[2], device=bad.device).view(1, 1, -1) % 2
    per = {"%d%d" % (a, b): int((bad & (hh == a) & (ww == b)).sum()) for a in (0, 1) for b in (0, 1)}
    return " | bad pixels by (h %% 2, w %% 2): %s of %d each" % (per, bad.numel() // 4)


def _expect(name, got, ref64):
    """torch.equal: a NaN output fails even where the reference is NaN."""
    expect(name, got, ref64, equal=torch.equal, note=_bad_parities)


# ------------------------------------------------------------------------------------------------------------------
# the host's route choice, restated (conv_igemm_impl / conv_wgrad_impl in csrc/conv_igemm.cu)
# ------------------------------------------------------------------------------------------------------------------
def _patch_ok(w, c, ndim, k, s, p):
    # patch_conv_applicable: 3x3 / stride 1 / pad 1, C % 64 == 0, and the halo patch of a 128-row tile fits its
    # 32 KB slot: 12 <= W <= 61
    return k == 3 and s == 1 and p == 1 and c % 64 == 0 and ndim % 8 == 0 and 12 <= w <= 61


def _tap_classes(k, p):
    return sum(1 for ph in (0, 1) for pw in (0, 1)
               if (k - ((ph + p) & 1) + 1) >> 1 > 0 and (k - ((pw + p) & 1) + 1) >> 1 > 0)


def igemm_route(dgrad, n, hs, ws, c, ho, wo, ndim, k, s, p, resid=False, mask=False, up=False, bias=False,
                stats=False, relu=False, out_fp32=False, gather=False, grouped=False):
    """(route, parity) of one byol_conv_igemm call: src [n, hs, ws, c] -> out [n, ho, wo, ndim]."""
    if (not gather and resid and not up and k == 1 and s == 1 and p == 0 and not out_fp32 and not stats
            and ndim > 64):
        return "gemm_fused", False
    if (not gather and not mask and not up and hs == ho and ws == wo and not out_fp32 and not bias
            and _patch_ok(ws, c, ndim, k, s, p)):
        return "patch", False
    parity = (dgrad and s == 2 and ho % 2 == 0 and wo % 2 == 0 and c % 64 == 0 and k <= 3 and not out_fp32
              and (n * (ho // 2) * (wo // 2)) % 128 == 0 and (not resid or _tap_classes(k, p) == 4))
    if grouped:
        return "grouped", parity
    a_tma = not gather and k == 1 and s == 1 and p == 0
    if a_tma and not out_fp32 and not bias and not resid and not relu:
        return "h16", parity
    return ("tma" if a_tma else "gather"), parity


def wgrad_route(n, h, w, c, cin_real, cout, ldy, k, s, p, gather=False, grouped=False):
    same = (h + 2 * p - k) // s + 1 == h and (w + 2 * p - k) // s + 1 == w
    if (not gather and same and (grouped or ldy == cout) and k == 3 and s == 1 and p == 1 and c % 64 == 0
            and (grouped or c == cin_real) and cout % 8 == 0 and 12 <= w <= 61):
        return "wgrad_patch"
    return "wgrad"


ROUTE_KERNEL = {
    "gemm_fused": r"gemm_fused_kernel",
    "patch": r"conv3x3_patch_kernel",
    "h16": r"conv_igemm_kernel<\d+,3,true,false,true>",
    "tma": r"conv_igemm_kernel<\d+,3,true,false,false>",
    "gather": r"conv_igemm_kernel<\d+,\d,false,false,false>",     # also parity mode: same kernel, other tile map
    "grouped": r"conv_igemm_kernel<64,4,false,true,false>",
    "wgrad_patch": r"conv3x3_wgrad_patch_kernel",
    "wgrad": r"conv_wgrad_kernel",
}


# ------------------------------------------------------------------------------------------------------------------
# builders: (device, generator, **shape / options) -> Case
# ------------------------------------------------------------------------------------------------------------------
def fprop_case(dev, g, n, h, w, c, cout, k, s, p, bias=False, resid=False, stats=False, relu=False, out_fp32=False,
               gather=False, cg=None, linear=False, fold=False):
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    cin = cg if cg else c
    d = _density(cin * k * k, stats)
    x = _ints((n, h, w, c), dev, g, 1 if stats else 2, d)
    wt = _ints((cout, cin, k, k), dev, g, 1, d)
    b = _ints((cout,), dev, g, 3) if bias else None
    r = _ints((n, ho, wo, cout), dev, g, 2) if resid else None
    if cg:
        w_f, _ = ops.prep_weight_grouped(wt.float(), want_dgrad=False)
    elif fold:
        w_f = ops.prep_weight_fold(wt.float())
    else:
        w_f, _ = ops.prep_weight(wt.float(), cpad=c, want_dgrad=False)
    xd = x.to(BF)
    bd = b.float() if bias else None
    rd = r.to(BF) if resid else None

    def run():
        st = torch.zeros(2 * cout, device=dev) if stats else None
        if linear:
            y = ops.linear_fprop(xd.view(n, c), w_f, bias=bd, stats=st, relu=relu, out_fp32=out_fp32)
        else:
            y = ops.conv_fprop(xd, w_f, k, k, s, p, bias=bd, resid=rd, stats=st, relu=relu, out_fp32=out_fp32,
                               force_gather=gather)
        return [y, st]

    def check(outs):
        y, st = outs
        ref = conv64(x, wt, s, p, c // cin)
        if bias:
            ref = ref + b
        if resid:
            ref = ref + r
        if relu:
            ref = torch.relu(ref)
        _expect("y", y, ref.reshape(y.shape))
        if stats:
            _expect("stats", st, _colstats(rounded_like(y, ref).reshape(-1, cout)))

    route, parity = igemm_route(False, n, h, w, c, ho, wo, cout, k, s, p, resid=resid, bias=bias, stats=stats,
                                relu=relu, out_fp32=out_fp32, gather=gather, grouped=bool(cg))
    return Case(run, check, route, parity)


def dgrad_case(dev, g, n, h, w, cin, cout, k, s, p, resid=None, gather=False, cg=None, linear=False):
    """dx [n, h, w, cin] of a conv with weight [cout, cin, k, k] (grouped: cin = cout = C, cg channels per group);
    resid: None, "plain", "mask" (only where the ReLU bits are set) or "up" (compact, scattered to even pixels)."""
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    wcin = cg if cg else cin
    d = _density((cg if cg else cout) * k * k, False)
    dy = _ints((n, ho, wo, cout), dev, g, 2, d)
    wt = _ints((cout, wcin, k, k), dev, g, 1, d)
    if cg:
        _, w_d = ops.prep_weight_grouped(wt.float())
    else:
        _, w_d = ops.prep_weight(wt.float())
    r = keep = None
    if resid == "up":
        r = _ints((n, h // 2, w // 2, cin), dev, g, 2)
    elif resid:
        r = _ints((n, h, w, cin), dev, g, 2)
    if resid == "mask":
        keep = torch.rand(n, h, w, cin, generator=g, device=dev) > 0.4
    dyd, rd = dy.to(BF), (r.to(BF) if r is not None else None)
    bits = _pack(keep) if keep is not None else None

    def run():
        if linear:
            return [ops.linear_dgrad(dyd.view(n, cout), w_d)]
        return [ops.conv_dgrad(dyd, w_d, h, w, k, k, s, p, resid=rd, force_gather=gather, resid_mask=bits,
                               resid_up=resid == "up")]

    def check(outs):
        ref = dgrad64(dy, wt, h, w, s, p, cout // wcin if cg else 1)
        if resid == "up":
            ref[:, ::2, ::2, :] += r
        elif resid == "mask":
            ref = ref + r * keep
        elif resid:
            ref = ref + r
        _expect("dx", outs[0], ref.reshape(outs[0].shape))

    route, parity = igemm_route(True, n, ho, wo, cout, h, w, cin, k, s, p, resid=resid is not None,
                                mask=resid == "mask", up=resid == "up", gather=gather, grouped=bool(cg))
    return Case(run, check, route, parity)


def wgrad_case(dev, g, n, h, w, c, cin_real, cout, k, s, p, ldy=None, gather=False, grouped=False, guard=1024):
    """dw [cout, cin_real, k, k] += dy^T im2col(x), dw a view into a buffer whose margins must keep their value;
    grouped: cin_real channels per group; ldy > cout: pitched dy rows whose padding columns hold NaN."""
    from byol_b200 import ops
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    ldy = ldy or cout
    x = _ints((n, h, w, c), dev, g, 2, 0.5)
    dy = _ints((n, ho, wo, cout), dev, g, 2, 0.5)
    dyp = torch.full((n, ho, wo, ldy), float("nan"), dtype=F64, device=dev)
    dyp[..., :cout] = dy
    dw0 = _ints((cout, cin_real, k, k), dev, g, 3)            # wgrad accumulates: start from a non-zero gradient
    numel = dw0.numel()
    xd, dyd = x.to(BF), dyp.to(BF)

    def run():
        buf = torch.full((guard + numel + guard,), 7.0, device=dev)
        dw = buf[guard:guard + numel].view(dw0.shape)
        dw.copy_(dw0)
        ops.conv_wgrad(xd, dyd, dw, k, k, s, p, force_gather=gather)
        return [buf]

    def check(outs):
        buf = outs[0]
        if grouped:
            ref = wgrad64(x, dy, dw0.shape, s, p, c // cin_real)
        else:
            ref = wgrad64(x[..., :cin_real], dy, dw0.shape, s, p)
        _expect("dw", buf[guard:guard + numel].view(dw0.shape), ref + dw0)
        margins = torch.cat([buf[:guard], buf[guard + numel:]])
        assert bool((margins == 7.0).all()), "wgrad wrote outside dw"

    return Case(run, check, wgrad_route(n, h, w, c, cin_real, cout, ldy, k, s, p, gather, grouped))


def stem_fprop_case(dev, g, n, h, w, stats=False):
    from byol_b200 import ops
    x = _ints((n, 3, h, w), dev, g, 1 if stats else 2, 0.5)
    wt = _ints((64, 3, 7, 7), dev, g, 1, 0.5)
    xs4, ws = ops.nchw_to_stem4(x.float()), ops.prep_weight_stem4(wt.float())

    def run():
        st = torch.zeros(128, device=dev) if stats else None
        return [ops.stem_conv_fprop(xs4, ws, h, w, stats=st), st]

    def check(outs):
        with torch.backends.cudnn.flags(enabled=False):
            ref = nhwc(F.conv2d(x, wt, None, 2, 3))
        _expect("y", outs[0], ref)
        if stats:
            _expect("stats", outs[1], _colstats(rounded_like(outs[0], ref).reshape(-1, 64)))
    return Case(run, check, "stem")


def stem_wgrad_case(dev, g, n, h, w, cin):
    from byol_b200 import ops
    x = _ints((n, cin, h, w), dev, g, 2, 0.5)
    dy = _ints((n, h // 2, w // 2, 64), dev, g, 2, 0.5)
    dw0 = _ints((64, cin, 7, 7), dev, g, 3)
    xs4, dyd = ops.nchw_to_stem4(x.float()), dy.to(BF)

    def run():
        dw = dw0.float()
        ops.stem_conv_wgrad(xs4, dyd, dw, h, w)
        return [dw]

    def check(outs):
        with torch.backends.cudnn.flags(enabled=False):
            ref = torch.nn.grad.conv2d_weight(x, dw0.shape, nchw(dy), 2, 3)
        _expect("dw", outs[0], ref + dw0)
    return Case(run, check, "stem")


# ------------------------------------------------------------------------------------------------------------------
# the route table: one row per (op, route, epilogue), at the edge of its predicate
# ------------------------------------------------------------------------------------------------------------------
D, FP, W = dgrad_case, fprop_case, wgrad_case
ROWS = {
    # dgrad: 1x1 bf16 hand-off (partial column tiles, M = 81)
    "dgrad_h16_n40": ("h16", D, dict(n=1, h=9, w=9, cin=40, cout=64, k=1, s=1, p=0)),
    "dgrad_h16_n200": ("h16", D, dict(n=1, h=9, w=9, cin=200, cout=128, k=1, s=1, p=0)),
    # dgrad + residual on gemm_fused_kernel (Ndim 136: the mask bytes of a row are not 16-byte aligned); M = 588
    "dgrad_fused_n256": ("gemm_fused", D, dict(n=3, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0, resid="plain")),
    "dgrad_fused_n256_mask": ("gemm_fused", D, dict(n=3, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0, resid="mask")),
    "dgrad_fused_n136": ("gemm_fused", D, dict(n=3, h=14, w=14, cin=136, cout=128, k=1, s=1, p=0, resid="plain")),
    "dgrad_fused_n136_mask": ("gemm_fused", D, dict(n=3, h=14, w=14, cin=136, cout=128, k=1, s=1, p=0,
                                                    resid="mask")),
    # Ndim 64: not gemm_fused, the TMA-operand implicit GEMM with the residual in its epilogue
    "dgrad_tma_n64": ("tma", D, dict(n=3, h=14, w=14, cin=64, cout=256, k=1, s=1, p=0, resid="plain")),
    "dgrad_tma_n64_mask": ("tma", D, dict(n=3, h=14, w=14, cin=64, cout=256, k=1, s=1, p=0, resid="mask")),
    # compact stride-2 branch gradient scattered to the even pixels
    "dgrad_up": ("tma", D, dict(n=3, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0, resid="up")),
    "dgrad_up_gather": ("gather", D, dict(n=3, h=14, w=14, cin=256, cout=64, k=1, s=1, p=0, resid="up",
                                          gather=True)),
    "dgrad_up_tail": ("tma", D, dict(n=3, h=10, w=10, cin=64, cout=128, k=1, s=1, p=0, resid="up")),
    # 3x3 patch kernel + residual: both width edges, ragged H with an odd number of M-tiles, three 64-channel chunks
    "dgrad_patch_w12": ("patch", D, dict(n=5, h=12, w=12, cin=64, cout=64, k=3, s=1, p=1, resid="plain")),
    "dgrad_patch_w61": ("patch", D, dict(n=1, h=61, w=61, cin=64, cout=64, k=3, s=1, p=1, resid="plain")),
    "dgrad_patch_30x26": ("patch", D, dict(n=3, h=30, w=26, cin=128, cout=64, k=3, s=1, p=1, resid="plain")),
    "dgrad_patch_26x30_odd_tiles": ("patch", D, dict(n=3, h=26, w=30, cin=64, cout=64, k=3, s=1, p=1,
                                                     resid="plain")),
    "dgrad_patch_c192": ("patch", D, dict(n=2, h=14, w=14, cin=64, cout=192, k=3, s=1, p=1, resid="plain")),
    "dgrad_patch_n40": ("patch", D, dict(n=2, h=16, w=16, cin=40, cout=64, k=3, s=1, p=1, resid="plain")),
    # just outside the patch kernel's widths: the gathered operand
    "dgrad_gather_w11": ("gather", D, dict(n=2, h=11, w=11, cin=64, cout=64, k=3, s=1, p=1, resid="plain")),
    "dgrad_gather_w62": ("gather", D, dict(n=1, h=62, w=62, cin=64, cout=64, k=3, s=1, p=1, resid="plain")),
    "dgrad_gather_w7": ("gather", D, dict(n=4, h=7, w=7, cin=128, cout=256, k=3, s=1, p=1, resid="plain")),
    # stride-2 3x3 in parity mode (N * H/2 * W/2 a multiple of 128)
    "dgrad_parity_16": ("parity", D, dict(n=2, h=16, w=16, cin=64, cout=128, k=3, s=2, p=1, resid="plain")),
    "dgrad_parity_16_mask": ("parity", D, dict(n=2, h=16, w=16, cin=64, cout=128, k=3, s=2, p=1, resid="mask")),
    "dgrad_parity_56": ("parity", D, dict(n=8, h=56, w=56, cin=64, cout=128, k=3, s=2, p=1, resid="plain")),
    "dgrad_parity_56_mask": ("parity", D, dict(n=8, h=56, w=56, cin=64, cout=128, k=3, s=2, p=1, resid="mask")),
    # stride-2 1x1: only class (0, 0) has a tap
    "dgrad_1x1s2_16": ("parity", D, dict(n=2, h=16, w=16, cin=64, cout=128, k=1, s=2, p=0)),
    "dgrad_1x1s2_16_resid": ("gather", D, dict(n=2, h=16, w=16, cin=64, cout=128, k=1, s=2, p=0, resid="plain")),
    "dgrad_1x1s2_28": ("gather", D, dict(n=1, h=28, w=28, cin=64, cout=128, k=1, s=2, p=0)),
    "dgrad_1x1s2_28_resid": ("gather", D, dict(n=1, h=28, w=28, cin=64, cout=128, k=1, s=2, p=0, resid="plain")),
    # grouped 3x3: patch (W >= 12), gather (7x7, stride 2), stride 2 in parity mode
    "dgrad_grouped_patch_cg4": ("patch", D, dict(n=2, h=14, w=14, cin=128, cout=128, k=3, s=1, p=1, cg=4)),
    "dgrad_grouped_patch_cg64": ("patch", D, dict(n=2, h=14, w=14, cin=128, cout=128, k=3, s=1, p=1, cg=64)),
    "dgrad_grouped_7_cg4": ("grouped", D, dict(n=4, h=7, w=7, cin=128, cout=128, k=3, s=1, p=1, cg=4)),
    "dgrad_grouped_7_cg64": ("grouped", D, dict(n=4, h=7, w=7, cin=128, cout=128, k=3, s=1, p=1, cg=64)),
    "dgrad_grouped_s2_cg4": ("grouped", D, dict(n=2, h=14, w=14, cin=128, cout=128, k=3, s=2, p=1, cg=4)),
    "dgrad_grouped_s2_cg64": ("grouped", D, dict(n=2, h=14, w=14, cin=128, cout=128, k=3, s=2, p=1, cg=64)),
    "dgrad_grouped_s2_parity_cg32": ("grouped_parity", D, dict(n=8, h=16, w=16, cin=128, cout=128, k=3, s=2, p=1,
                                                               cg=32)),
    "linear_dgrad_m200": ("h16", D, dict(n=200, h=1, w=1, cin=512, cout=256, k=1, s=1, p=0, linear=True)),
    # fprop: TMA 1x1 with bias + ReLU + residual (BN 64 and 128; fp32 and bf16 outputs)
    "fprop_tma_f32_n64": ("tma", FP, dict(n=3, h=14, w=14, c=128, cout=64, k=1, s=1, p=0, bias=True, resid=True,
                                          relu=True, out_fp32=True)),
    "fprop_tma_f32_n192": ("tma", FP, dict(n=3, h=14, w=14, c=128, cout=192, k=1, s=1, p=0, bias=True, resid=True,
                                           relu=True, out_fp32=True)),
    "fprop_tma_bf16_n64": ("tma", FP, dict(n=3, h=14, w=14, c=128, cout=64, k=1, s=1, p=0, bias=True, resid=True,
                                           relu=True)),
    "fprop_tma_bf16_n192_bias_relu": ("tma", FP, dict(n=3, h=14, w=14, c=128, cout=192, k=1, s=1, p=0, bias=True,
                                                      relu=True)),
    # fp32 outputs of any width (the classifier)
    "fprop_f32_n10": ("tma", FP, dict(n=96, h=1, w=1, c=512, cout=10, k=1, s=1, p=0, bias=True, out_fp32=True,
                                      linear=True)),
    "fprop_f32_n1000": ("tma", FP, dict(n=96, h=1, w=1, c=512, cout=1000, k=1, s=1, p=0, bias=True, out_fp32=True,
                                        linear=True)),
    # residual + ReLU without statistics: gemm_fused_kernel
    "fprop_fused_resid_relu": ("gemm_fused", FP, dict(n=3, h=14, w=14, c=64, cout=256, k=1, s=1, p=0, resid=True,
                                                      relu=True)),
    # 3x3 patch + residual + ReLU + statistics at the width edges, and the gathers just outside
    "fprop_patch_w12": ("patch", FP, dict(n=5, h=12, w=12, c=64, cout=64, k=3, s=1, p=1, resid=True, relu=True,
                                          stats=True)),
    "fprop_patch_w61": ("patch", FP, dict(n=1, h=61, w=61, c=64, cout=128, k=3, s=1, p=1, resid=True, relu=True,
                                          stats=True)),
    "fprop_gather_w11": ("gather", FP, dict(n=2, h=11, w=11, c=64, cout=64, k=3, s=1, p=1, resid=True, relu=True,
                                            stats=True)),
    "fprop_gather_w62": ("gather", FP, dict(n=1, h=62, w=62, c=64, cout=128, k=3, s=1, p=1, resid=True, relu=True,
                                            stats=True)),
    "fprop_gather_bias": ("gather", FP, dict(n=2, h=16, w=16, c=64, cout=64, k=3, s=1, p=1, bias=True, relu=True)),
    # grouped + statistics on both routes
    "fprop_grouped_patch_stats": ("patch", FP, dict(n=2, h=14, w=14, c=128, cout=128, k=3, s=1, p=1, cg=8,
                                                    stats=True)),
    "fprop_grouped_7_stats": ("grouped", FP, dict(n=4, h=7, w=7, c=128, cout=128, k=3, s=1, p=1, cg=64,
                                                  stats=True)),
    "fprop_grouped_s2_stats": ("grouped", FP, dict(n=2, h=14, w=14, c=128, cout=128, k=3, s=2, p=1, cg=4,
                                                   stats=True)),
    # wgrad cases test_gpu_reductions does not have
    "wgrad_grouped_patch_cg4": ("wgrad_patch", W, dict(n=2, h=14, w=14, c=128, cin_real=4, cout=128, k=3, s=1, p=1,
                                                       grouped=True)),
    "wgrad_grouped_patch_cg64": ("wgrad_patch", W, dict(n=2, h=14, w=14, c=128, cin_real=64, cout=128, k=3, s=1,
                                                        p=1, grouped=True)),
    "wgrad_grouped_7_cg4": ("wgrad", W, dict(n=4, h=7, w=7, c=128, cin_real=4, cout=128, k=3, s=1, p=1,
                                             grouped=True)),
    "wgrad_grouped_s2_cg64": ("wgrad", W, dict(n=2, h=14, w=14, c=128, cin_real=64, cout=128, k=3, s=2, p=1,
                                               grouped=True)),
    "wgrad_pitched_cout10": ("wgrad", W, dict(n=96, h=1, w=1, c=512, cin_real=512, cout=10, ldy=16, k=1, s=1, p=0)),
    "wgrad_cout200": ("wgrad", W, dict(n=2, h=14, w=14, c=64, cin_real=64, cout=200, k=1, s=1, p=0)),
    "wgrad_cout200_3x3": ("wgrad", W, dict(n=2, h=10, w=10, c=64, cin_real=64, cout=200, k=3, s=1, p=1)),
    "wgrad_cin_real_stem": ("wgrad", W, dict(n=2, h=32, w=32, c=8, cin_real=3, cout=64, k=7, s=2, p=3)),
    "wgrad_cin_real_1x1": ("wgrad", W, dict(n=2, h=14, w=14, c=40, cin_real=36, cout=64, k=1, s=1, p=0)),
    # 5157 rows: 81 k-blocks in 11 splits of 8, the last one a single k-block of 37 rows
    "wgrad_short_last_split": ("wgrad", W, dict(n=5157, h=1, w=1, c=64, cin_real=64, cout=128, k=1, s=1, p=0)),
}


def _build(dev, name):
    return row_case(dev, name, *ROWS[name][1:])


@pytest.mark.parametrize("name", list(ROWS))
def test_route_exact(cuda, name):
    run_and_check(_build(cuda, name))


def _check_launches():
    cases = {name: _build(torch.device("cuda:0"), name) for name in ROWS}

    def complaints(name, launched):
        case, want = cases[name], ROWS[name][0]
        parity = want == "parity" or want.endswith("_parity")
        route = "gather" if want == "parity" else want[:-len("_parity")] if parity else want
        wrong = []
        if (case.route, case.parity) != (route, parity):
            wrong.append("%s: the host predicate gives %s%s, the row is meant for %s" % (
                name, case.route, " (parity)" if case.parity else "", want))
        if not any(re.search(ROUTE_KERNEL[route], k) for k in launched):
            wrong.append("%s: expected %s, launched %s" % (name, ROUTE_KERNEL[route], sorted(set(launched))))
        return wrong
    check_row_launches({name: case.run for name, case in cases.items()}, complaints)


def test_routes_launch_their_kernels(cuda):
    """Each row runs the kernel it is meant for.  Parity mode and the gathered operand share conv_igemm_kernel: for
    those rows the restated host predicate (igemm_route, after conv_igemm_impl) decides.  Checked in a fresh Python
    process: one that has already held many profiler sessions (the rest of the GPU suite) can drop CUDA kernel
    events."""
    check_in_fresh_process(__name__)


# ------------------------------------------------------------------------------------------------------------------
# replay of the engine's own calls
# ------------------------------------------------------------------------------------------------------------------
def _shape(t):
    return None if t is None else tuple(t.shape)


def _recorders(calls):
    """ops function name -> recorder that notes the call's shapes and options (not its data) and runs it."""
    def conv_fprop(x, w_f, kh, kw, stride, pad, bias=None, resid=None, stats=None, relu=False, out_fp32=False,
                   out=None, force_gather=False):
        calls.add(("conv_fprop", _shape(x), _shape(w_f), kh, kw, stride, pad, bias is not None, _shape(resid),
                   stats is not None, bool(relu), bool(out_fp32), bool(force_gather)))

    def conv_dgrad(dy, w_d, h, w, kh, kw, stride, pad, resid=None, out=None, force_gather=False, resid_mask=None,
                   resid_up=False):
        calls.add(("conv_dgrad", _shape(dy), _shape(w_d), h, w, kh, kw, stride, pad, _shape(resid),
                   bool(force_gather), resid_mask is not None, bool(resid_up)))

    def conv_wgrad(x, dy, dw, kh, kw, stride, pad, force_gather=False):
        calls.add(("conv_wgrad", _shape(x), _shape(dy), _shape(dw), kh, kw, stride, pad, bool(force_gather)))

    def stem_conv_fprop(xs4, w_stem4, h, w, stats=None):
        calls.add(("stem_conv_fprop", xs4.shape[0], h, w, stats is not None))

    def stem_conv_wgrad(xs4, dy, dw, h, w):
        calls.add(("stem_conv_wgrad", xs4.shape[0], h, w, dw.shape[1]))
    return dict(conv_fprop=conv_fprop, conv_dgrad=conv_dgrad, conv_wgrad=conv_wgrad,
                stem_conv_fprop=stem_conv_fprop, stem_conv_wgrad=stem_conv_wgrad)


def _replay_case(dev, g, sig, cg_by_c):
    """Case of one recorded call, replayed with exact operands of the same shapes and options."""
    op = sig[0]
    if op == "conv_fprop":
        _, xs, ws, kh, kw, s, p, bias, resid, stats, relu, out_fp32, gather = sig
        n, h, w, c = xs
        assert kh == kw
        if len(ws) == 3:
            return fprop_case(dev, g, n, h, w, c, c, kh, s, p, stats=stats, cg=cg_by_c.get(c, 64))
        fold = ws[1] == kh * 64 and c == 8 and kh > 1
        assert fold or ws[1] == kh * kw * c, "unknown fprop weight layout %s" % (ws,)
        return fprop_case(dev, g, n, h, w, c, ws[0], kh, s, p, bias=bias, resid=resid is not None, stats=stats,
                          relu=relu, out_fp32=out_fp32, gather=gather, fold=fold)
    if op == "conv_dgrad":
        _, dys, ws, h, w, kh, kw, s, p, resid, gather, mask, up = sig
        n, _, _, cout = dys
        kind = None if resid is None else "up" if up else "mask" if mask else "plain"
        if len(ws) == 3:
            return dgrad_case(dev, g, n, h, w, cout, cout, kh, s, p, cg=cg_by_c.get(cout, 64))
        assert ws[1] == kh * kw * cout, "unknown dgrad weight layout %s" % (ws,)
        return dgrad_case(dev, g, n, h, w, ws[0], cout, kh, s, p, resid=kind, gather=gather)
    if op == "conv_wgrad":
        _, xs, dys, dws, kh, kw, s, p, gather = sig
        n, h, w, c = xs
        grouped = dws[1] < c and c % 64 == 0
        return wgrad_case(dev, g, n, h, w, c, dws[1], dws[0], kh, s, p, ldy=dys[3], gather=gather, grouped=grouped)
    if op == "stem_conv_fprop":
        return stem_fprop_case(dev, g, sig[1], sig[2], sig[3], stats=sig[4])
    return stem_wgrad_case(dev, g, sig[1], sig[2], sig[3], sig[4])


NETS = [("resnet18", 512, 8, 224), ("resnet:bottleneck:2,1,1,1", 2048, 8, 224), ("resnext:32x4:1,1,1,1", 2048, 2, 112)]


def _dgrad_sig_route(sig):
    _, dys, ws, h, w, kh, kw, s, p, resid, gather, mask, up = sig
    n, ho, wo, cout = dys
    return igemm_route(True, n, ho, wo, cout, h, w, ws[0] if len(ws) == 2 else cout, kh, s, p,
                       resid=resid is not None, mask=mask, up=up, gather=gather, grouped=len(ws) == 3)


def test_replay_engine_calls_exactly(cuda):
    calls = set()
    with recording(_recorders(calls)):
        for arch, rep, b, r in NETS:
            byol_train_step(cuda, arch, rep, b, r)
            torch.cuda.empty_cache()
    dgrads = [sig for sig in calls if sig[0] == "conv_dgrad"]
    resid_routes = {_dgrad_sig_route(sig) for sig in dgrads if sig[9] is not None}
    # the replay must keep covering the residual epilogues where the backward pass joins its branches
    assert ("gather", True) in resid_routes, "no parity-mode dgrad with a residual recorded"
    assert ("patch", False) in resid_routes, "no patch-kernel dgrad with a residual recorded"
    assert any(sig[9] is not None and sig[11] and _dgrad_sig_route(sig)[0] == "gemm_fused" for sig in dgrads), \
        "no gemm_fused dgrad with a masked residual recorded"
    assert any(sig[12] for sig in dgrads), "no resid_up dgrad recorded"
    cg_by_c = {sig[1][3]: sig[3][1] for sig in calls
               if sig[0] == "conv_wgrad" and sig[3][1] < sig[1][3] and sig[1][3] % 64 == 0}
    replay(cuda, calls, lambda dev, g, sig: _replay_case(dev, g, sig, cg_by_c), 1000)
