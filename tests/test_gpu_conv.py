"""GPU parity: wgmma implicit-GEMM conv / linear (fprop, dgrad, wgrad) vs the CPU oracle (oracle/ops_ref.py).

Inputs are bf16-representable, the oracle runs in fp32 on the same values, so the only differences are fp32
accumulation order (tolerance 2e-3 relative to the output scale, stated per test) and, where the kernel
stores bf16, one bf16 rounding (2^-8 relative).
"""
import pytest
import torch

from oracle import ops_ref as R
from tests.util import assert_close

pytestmark = pytest.mark.gpu

# (name, N, H, W, Cin_real, Cpad, Cout, k, stride, pad)
CONV_CASES = [
    ("1x1_64_64", 2, 8, 8, 64, 64, 64, 1, 1, 0),
    ("1x1_256_128", 2, 8, 8, 256, 256, 128, 1, 1, 0),
    ("1x1_64_256", 2, 8, 8, 64, 64, 256, 1, 1, 0),
    ("1x1_tailM", 3, 7, 7, 128, 128, 64, 1, 1, 0),
    ("3x3_64_64", 2, 8, 8, 64, 64, 64, 3, 1, 1),
    ("3x3_128_128", 2, 14, 14, 128, 128, 128, 3, 1, 1),
    ("3x3_patch_28", 2, 28, 28, 128, 128, 128, 3, 1, 1),        # auto -> patch-reuse kernel (W >= 24)
    ("3x3_patch_56_64", 1, 56, 56, 64, 64, 64, 3, 1, 1),
    ("3x3_patch_30x26", 3, 30, 26, 64, 64, 256, 3, 1, 1),       # ragged: H not a multiple of the tile rows
    ("3x3_patch_48", 1, 48, 48, 64, 64, 64, 3, 1, 1),           # 384x384 input geometries (ResNet stages 2-4)
    ("3x3_patch_24", 3, 24, 24, 128, 128, 128, 3, 1, 1),
    ("3x3_patch_12", 5, 12, 12, 256, 256, 256, 3, 1, 1),
    ("3x3s2_128_128", 1, 28, 28, 128, 128, 128, 3, 2, 1),
    ("1x1s2_256_512", 1, 28, 28, 256, 256, 512, 1, 2, 0),
    ("3x3_512_512_7", 3, 7, 7, 512, 512, 512, 3, 1, 1),
    ("3x3s2_parity", 2, 16, 16, 128, 128, 128, 3, 2, 1),     # dgrad runs in output-parity mode (Mc % 128 == 0)
    ("1x1s2_parity", 2, 16, 16, 256, 256, 512, 1, 2, 0),
    ("3x3s2_parity_64", 4, 16, 16, 64, 64, 128, 3, 2, 1),
    ("stem7x7", 2, 32, 32, 3, 8, 64, 7, 2, 3),
]


def _mk(case, dev, seed=0):
    name, n, h, w, cin, cpad, cout, k, s, p = case
    g = torch.Generator().manual_seed(seed)
    x = R.bf16_round(torch.randn(n, h, w, cin, generator=g))
    wt = R.bf16_round(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5)
    xp = torch.zeros(n, h, w, cpad)
    xp[..., :cin] = x
    return x, wt, xp.to(dev, torch.bfloat16)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize("force_gather", [False, True], ids=["auto", "gather"])
def test_conv_fprop(cuda, case, force_gather):
    from byol_b200 import ops
    name, n, h, w, cin, cpad, cout, k, s, p = case
    x, wt, xd = _mk(case, cuda)
    w_f, _ = ops.prep_weight(wt.to(cuda), cpad=cpad, want_dgrad=False)
    ref = R.conv_fprop_ref(x, wt, s, p)
    y32 = ops.conv_fprop(xd, w_f, k, k, s, p, out_fp32=True, force_gather=force_gather)
    torch.cuda.synchronize()
    scale = float(ref.abs().max())
    assert_close("fprop_f32[%s]" % name, y32, ref, atol=2e-3 * scale, rtol=0)
    stats = torch.zeros(2 * cout, device=cuda)
    y16 = ops.conv_fprop(xd, w_f, k, k, s, p, stats=stats, force_gather=force_gather)
    torch.cuda.synchronize()
    assert_close("fprop_bf16[%s]" % name, y16, ref, atol=1e-2 * scale, rtol=0)
    yr = y16.float().cpu().reshape(-1, cout)
    assert_close("fprop_stats_sum[%s]" % name, stats[:cout], yr.sum(0), atol=1e-3 * yr.abs().sum(0).max().item(), rtol=0)
    assert_close("fprop_stats_sq[%s]" % name, stats[cout:], (yr * yr).sum(0), atol=0, rtol=1e-3)


def test_conv_fprop_epilogue(cuda):
    from byol_b200 import ops
    case = ("3x3_64_64", 2, 8, 8, 64, 64, 64, 3, 1, 1)
    name, n, h, w, cin, cpad, cout, k, s, p = case
    x, wt, xd = _mk(case, cuda, seed=3)
    g = torch.Generator().manual_seed(5)
    bias = torch.randn(cout, generator=g)
    resid = R.bf16_round(torch.randn(n, h, w, cout, generator=g))
    w_f, _ = ops.prep_weight(wt.to(cuda), cpad=cpad, want_dgrad=False)
    ref = R.conv_fprop_ref(x, wt, s, p, bias=bias, resid_nhwc=resid, relu=True)
    y = ops.conv_fprop(xd, w_f, k, k, s, p, bias=bias.to(cuda), resid=resid.to(cuda, torch.bfloat16), relu=True,
                       out_fp32=True)
    torch.cuda.synchronize()
    assert_close("fprop_epilogue", y, ref, atol=2e-3 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("case", CONV_CASES[:-1], ids=[c[0] for c in CONV_CASES[:-1]])
@pytest.mark.parametrize("force_gather", [False, True], ids=["auto", "gather"])
def test_conv_dgrad(cuda, case, force_gather):
    from byol_b200 import ops
    name, n, h, w, cin, cpad, cout, k, s, p = case
    _, wt, _ = _mk(case, cuda)
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    g = torch.Generator().manual_seed(11)
    dy = R.bf16_round(torch.randn(n, ho, wo, cout, generator=g))
    _, w_d = ops.prep_weight(wt.to(cuda), cpad=cpad, want_dgrad=True)
    ref = R.conv_dgrad_ref(dy, wt, (h, w), s, p)
    dx = ops.conv_dgrad(dy.to(cuda, torch.bfloat16), w_d, h, w, k, k, s, p, force_gather=force_gather)
    torch.cuda.synchronize()
    assert_close("dgrad[%s]" % name, dx, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("case", CONV_CASES, ids=[c[0] for c in CONV_CASES])
@pytest.mark.parametrize("force_gather", [False, True], ids=["auto", "gather"])
def test_conv_wgrad(cuda, case, force_gather):
    from byol_b200 import ops
    name, n, h, w, cin, cpad, cout, k, s, p = case
    x, wt, xd = _mk(case, cuda)
    ho, wo = ops.conv_out_size(h, k, s, p), ops.conv_out_size(w, k, s, p)
    g = torch.Generator().manual_seed(13)
    dy = R.bf16_round(torch.randn(n, ho, wo, cout, generator=g))
    ref = R.conv_wgrad_ref(x, dy, wt.shape, s, p)
    dw = torch.zeros(cout, cin, k, k, device=cuda)
    ops.conv_wgrad(xd, dy.to(cuda, torch.bfloat16), dw, k, k, s, p, force_gather=force_gather)
    torch.cuda.synchronize()
    assert_close("wgrad[%s]" % name, dw, ref, atol=2e-3 * float(ref.abs().max()), rtol=0)
    # accumulate semantics: a second call doubles the result
    ops.conv_wgrad(xd, dy.to(cuda, torch.bfloat16), dw, k, k, s, p, force_gather=force_gather)
    torch.cuda.synchronize()
    assert_close("wgrad_acc[%s]" % name, dw, 2 * ref, atol=4e-3 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("shape", [(2, 32, 32), (3, 30, 26), (1, 224, 224)])
def test_stem_folded_layout(cuda, shape):
    """7x7/2 stem with the folded weight layout (one k-block per kh, contiguous 128-byte gathers)."""
    from byol_b200 import ops
    n, h, w = shape
    g = torch.Generator().manual_seed(23)
    x = R.bf16_round(torch.rand(n, h, w, 3, generator=g))
    wt = R.bf16_round(torch.randn(64, 3, 7, 7, generator=g) / 12.0)
    xp = torch.zeros(n, h, w, 8)
    xp[..., :3] = x
    wf = ops.prep_weight_fold(wt.to(cuda))
    assert wf.shape == (64, 448)
    ref = R.conv_fprop_ref(x, wt, 2, 3)
    stats = torch.zeros(128, device=cuda)
    y = ops.conv_fprop(xp.to(cuda, torch.bfloat16), wf, 7, 7, 2, 3, stats=stats)
    torch.cuda.synchronize()
    assert_close("stem_fold", y, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)
    yr = y.float().cpu().reshape(-1, 64)
    assert_close("stem_fold_stats", stats[:64], yr.sum(0), atol=1e-3 * yr.abs().sum(0).max().item(), rtol=0)


@pytest.mark.parametrize("shape", [(2, 32, 32), (3, 30, 26), (2, 224, 224), (5, 64, 64), (1, 256, 256)])
def test_stem4_fprop(cuda, shape):
    """Dedicated stem kernel: padded NHWC4 input, im2col formed by overlapping no-swizzle wgmma descriptors."""
    from byol_b200 import ops
    n, h, w = shape
    assert ops.stem4_supported(3, 64, h, w, 7, 2, 3)
    g = torch.Generator().manual_seed(29)
    x = R.bf16_round(torch.rand(n, 3, h, w, generator=g) - 0.3)        # NCHW fp32 (values exactly bf16)
    wt = R.bf16_round(torch.randn(64, 3, 7, 7, generator=g) / 12.0)
    xs4 = ops.nchw_to_stem4(x.to(cuda))
    ws = ops.prep_weight_stem4(wt.to(cuda))
    ref = R.conv_fprop_ref(x.permute(0, 2, 3, 1).contiguous(), wt, 2, 3)
    stats = torch.zeros(128, device=cuda)
    y = ops.stem_conv_fprop(xs4, ws, h, w, stats=stats)
    y2 = ops.stem_conv_fprop(xs4, ws, h, w)
    torch.cuda.synchronize()
    assert y.shape == (n, h // 2, w // 2, 64) and torch.equal(y, y2)
    assert_close("stem4", y, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)
    yr = y.float().cpu().reshape(-1, 64)
    assert_close("stem4_sum", stats[:64], yr.sum(0), atol=1e-3 * yr.abs().sum(0).max().item(), rtol=0)
    assert_close("stem4_sqsum", stats[64:], (yr * yr).sum(0), atol=1e-3 * (yr * yr).sum(0).max().item(), rtol=0)
    # same weights through the generic implicit-GEMM path (NHWC8 input, folded layout): both round the same products
    x8 = ops.nchw_to_nhwc8(x.to(cuda))
    y_ig = ops.conv_fprop(x8, ops.prep_weight_fold(wt.to(cuda)), 7, 7, 2, 3)
    torch.cuda.synchronize()
    assert_close("stem4_vs_igemm", y, y_ig.float().cpu(), atol=2e-2 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("shape", [(2, 32, 32), (3, 30, 26), (2, 224, 224), (301, 64, 64), (1, 256, 256)])
def test_stem4_wgrad(cuda, shape):
    """Dedicated stem weight-gradient kernel (dY row pairs x input row, overlapping no-swizzle B operand)."""
    from byol_b200 import ops
    n, h, w = shape
    g = torch.Generator().manual_seed(31)
    x = R.bf16_round(torch.rand(n, 3, h, w, generator=g) - 0.3)
    dy = R.bf16_round(torch.randn(n, h // 2, w // 2, 64, generator=g))
    xs4 = ops.nchw_to_stem4(x.to(cuda))
    ref = R.conv_wgrad_ref(x.permute(0, 2, 3, 1).contiguous(), dy, (64, 3, 7, 7), 2, 3)
    dw = torch.zeros(64, 3, 7, 7, device=cuda)
    ops.stem_conv_wgrad(xs4, dy.to(cuda, torch.bfloat16), dw, h, w)
    torch.cuda.synchronize()
    assert_close("stem4_wgrad", dw, ref, atol=2e-3 * float(ref.abs().max()), rtol=0)
    ops.stem_conv_wgrad(xs4, dy.to(cuda, torch.bfloat16), dw, h, w)
    torch.cuda.synchronize()
    assert_close("stem4_wgrad_acc", dw, 2 * ref, atol=4e-3 * float(ref.abs().max()), rtol=0)


def test_conv_dgrad_parity_with_residual(cuda):
    """BasicBlock-style strided 3x3 dgrad with the residual gradient added in the epilogue (parity mode)."""
    from byol_b200 import ops
    case = ("3x3s2_parity", 2, 16, 16, 128, 128, 128, 3, 2, 1)
    name, n, h, w, cin, cpad, cout, k, s, p = case
    _, wt, _ = _mk(case, cuda)
    g = torch.Generator().manual_seed(19)
    dy = R.bf16_round(torch.randn(n, 8, 8, cout, generator=g))
    resid = R.bf16_round(torch.randn(n, h, w, cin, generator=g))
    _, w_d = ops.prep_weight(wt.to(cuda), cpad=cpad, want_dgrad=True)
    ref = R.conv_dgrad_ref(dy, wt, (h, w), s, p) + resid
    dx = ops.conv_dgrad(dy.to(cuda, torch.bfloat16), w_d, h, w, k, k, s, p, resid=resid.to(cuda, torch.bfloat16))
    torch.cuda.synchronize()
    assert_close("dgrad_parity_resid", dx, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("hw,cin,cout", [(14, 256, 64), (9, 64, 128), (8, 512, 2048)])
def test_conv_dgrad_masked_residual(cuda, hw, cin, cout):
    """Bottleneck identity block: 1x1 dgrad + (gradient of the residual branch where the ReLU-mask bit is set)."""
    from byol_b200 import ops
    n, k, s, p = 3, 1, 1, 0
    g = torch.Generator().manual_seed(23)
    wt = R.bf16_round(torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5)
    dy = R.bf16_round(torch.randn(n, hw, hw, cout, generator=g))
    resid = R.bf16_round(torch.randn(n, hw, hw, cin, generator=g))
    keep = torch.rand(n, hw, hw, cin, generator=g) > 0.4
    bits = ((keep.view(-1, 8).to(torch.int32) * (2 ** torch.arange(8, dtype=torch.int32))).sum(1)).to(torch.uint8)
    _, w_d = ops.prep_weight(wt.to(cuda), cpad=cin, want_dgrad=True)
    ref = R.conv_dgrad_ref(dy, wt, (hw, hw), s, p) + resid * keep
    dx = ops.conv_dgrad(dy.to(cuda, torch.bfloat16), w_d, hw, hw, k, k, s, p, resid=resid.to(cuda, torch.bfloat16),
                        resid_mask=bits.to(cuda))
    torch.cuda.synchronize()
    assert_close("dgrad_masked_resid", dx, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)


@pytest.mark.parametrize("hw,cin,cout", [(14, 256, 64), (10, 64, 128), (8, 512, 256)])
def test_conv_dgrad_upsampled_residual(cuda, hw, cin, cout):
    """Down block: 1x1 dgrad + the COMPACT gradient of the stride-2 branch scattered to the even pixels."""
    from byol_b200 import ops
    n, k, s, p = 3, 1, 1, 0
    g = torch.Generator().manual_seed(27)
    wt = R.bf16_round(torch.randn(cout, cin, 1, 1, generator=g) / cin ** 0.5)
    dy = R.bf16_round(torch.randn(n, hw, hw, cout, generator=g))
    rc = R.bf16_round(torch.randn(n, hw // 2, hw // 2, cin, generator=g))
    _, w_d = ops.prep_weight(wt.to(cuda), cpad=cin, want_dgrad=True)
    up = torch.zeros(n, hw, hw, cin)
    up[:, ::2, ::2, :] = rc
    ref = R.conv_dgrad_ref(dy, wt, (hw, hw), s, p) + up
    dx = ops.conv_dgrad(dy.to(cuda, torch.bfloat16), w_d, hw, hw, k, k, s, p, resid=rc.to(cuda, torch.bfloat16),
                        resid_up=True)
    torch.cuda.synchronize()
    assert_close("dgrad_up_resid", dx, ref, atol=1e-2 * float(ref.abs().max()), rtol=0)


LINEAR_CASES = [("head1", 64, 2048, 4096), ("head2", 64, 4096, 256), ("cls", 96, 2048, 1000), ("pred1", 200, 256, 4096)]


@pytest.mark.parametrize("case", LINEAR_CASES, ids=[c[0] for c in LINEAR_CASES])
def test_linear(cuda, case):
    from byol_b200 import ops
    name, m, k, n = case
    g = torch.Generator().manual_seed(17)
    x = R.bf16_round(torch.randn(m, k, generator=g))
    w = R.bf16_round(torch.randn(n, k, generator=g) / k ** 0.5)
    b = torch.randn(n, generator=g)
    dy = R.bf16_round(torch.randn(m, n, generator=g))
    w_f, w_d = ops.prep_weight(w.to(cuda), want_dgrad=(n % 8 == 0))
    y = ops.linear_fprop(x.to(cuda, torch.bfloat16), w_f, bias=b.to(cuda), out_fp32=True)
    torch.cuda.synchronize()
    ref = x @ w.t() + b
    assert_close("linear_fprop[%s]" % name, y, ref, atol=2e-3 * float(ref.abs().max()), rtol=0)
    dx = ops.linear_dgrad(dy.to(cuda, torch.bfloat16), w_d)
    torch.cuda.synchronize()
    refdx = dy @ w
    assert_close("linear_dgrad[%s]" % name, dx, refdx, atol=1e-2 * float(refdx.abs().max()), rtol=0)
    dw = torch.zeros(n, k, device=cuda)
    ops.linear_wgrad(x.to(cuda, torch.bfloat16), dy.to(cuda, torch.bfloat16), dw)
    torch.cuda.synchronize()
    refdw = dy.t() @ x
    assert_close("linear_wgrad[%s]" % name, dw, refdw, atol=2e-3 * float(refdw.abs().max()), rtol=0)
