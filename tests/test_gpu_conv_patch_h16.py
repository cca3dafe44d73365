"""GPU: the bf16 hand-off variant of conv3x3_patch_kernel (3x3 / stride 1 fprop with BatchNorm statistics and dgrad
without residual or ReLU), bit for bit against float64 with the exact small-integer operands of test_gpu_conv_exact:
both tile widths (64 columns over pairs of M-tiles, 128 columns over one M-tile), ragged output widths, the image
widths at and between the edges of the patch route, ragged H with an odd number of M-tiles, 1, 2 and 4 input-channel
chunks; plus run-to-run equality of the statistics and the variant each kind of call launches."""
import re

import pytest
import torch

from tests.exact import check_in_fresh_process, check_row_launches, row_case, run_and_check
from tests.test_gpu_conv_exact import dgrad_case, fprop_case
from tests.util import gen

pytestmark = pytest.mark.gpu

# name: (fprop (True) or dgrad, image n, h, w, input channels C, output channels Ndim)
CASES = {
    # 64-column tiles over pairs of M-tiles; 14 M-tiles / 13 M-tiles (odd: the last pair has one M-tile)
    "n64_c64_w56": (True, 1, 56, 56, 64, 64),
    "n64_c64_w56_dgrad": (False, 1, 56, 56, 64, 64),
    "n64_c64_h27_w28_odd": (True, 1, 27, 28, 64, 64),
    "n40_c64_w12": (True, 5, 12, 12, 64, 40),
    "n40_c128_w61_dgrad": (False, 1, 61, 61, 128, 40),
    # 128-column tiles: one and two column tiles, 1 / 2 / 4 channel chunks
    "n128_c128_w28": (True, 3, 28, 28, 128, 128),
    "n128_c128_w28_dgrad": (False, 3, 28, 28, 128, 128),
    "n256_c256_w14": (True, 5, 14, 14, 256, 256),
    "n256_c256_w14_dgrad": (False, 5, 14, 14, 256, 256),
    "n192_c64_w12": (True, 3, 12, 12, 64, 192),
    "n192_c256_h19_w14_dgrad": (False, 3, 19, 14, 256, 192),
    "n320_c128_w61": (True, 1, 61, 61, 128, 320),
    "n320_c64_h25_w30_dgrad": (False, 3, 25, 30, 64, 320),
    "n136_c128_h13_w56": (True, 1, 13, 56, 128, 136),
}


def _case(dev, name):
    fprop, n, h, w, c, ndim = CASES[name]
    if fprop:
        return row_case(dev, name, fprop_case, dict(n=n, h=h, w=w, c=c, cout=ndim, k=3, s=1, p=1, stats=True))
    return row_case(dev, name, dgrad_case, dict(n=n, h=h, w=w, cin=ndim, cout=c, k=3, s=1, p=1))


@pytest.mark.parametrize("name", list(CASES))
def test_patch_h16_exact(cuda, name):
    case = _case(cuda, name)
    assert case.route == "patch"
    run_and_check(case)


@pytest.mark.parametrize("c, ndim, hw", [(64, 64, 56), (128, 128, 28), (256, 256, 14), (64, 192, 30)])
def test_patch_h16_stats_run_to_run(cuda, c, ndim, hw):
    """Statistics of real-valued data (inexact fp32 partial sums) are the same bits on every run."""
    from byol_b200 import ops
    g = gen(cuda, c + ndim + hw)
    x = torch.randn(6, hw, hw, c, device=cuda, generator=g).to(torch.bfloat16)
    w_f, _ = ops.prep_weight(torch.randn(ndim, c, 3, 3, device=cuda, generator=g) / (3 * c ** 0.5), want_dgrad=False)
    runs = []
    for _ in range(2):
        st = torch.zeros(2 * ndim, device=cuda)
        y = ops.conv_fprop(x, w_f, 3, 3, 1, 1, stats=st)
        runs.append((y, st))
    torch.cuda.synchronize()
    assert torch.equal(runs[0][0], runs[1][0])
    assert torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("c, ndim, h, w", [(128, 128, 28, 28), (256, 256, 14, 14), (128, 136, 14, 14),
                                           (64, 192, 30, 26), (256, 320, 15, 14)])
def test_patch_h16_matches_fp32_tile_kernel(cuda, c, ndim, h, w):
    """On real-valued data (inexact fp32 partial sums) the bf16 hand-off gives the bits of the fp32-tile kernel with
    64-column pair tiles, reached here through an all-zero residual: the same outputs, and the same statistics,
    which the 128-column tiles sum in the pair kernel's grouping."""
    from byol_b200 import ops
    g = gen(cuda, c + ndim + h)
    x = torch.randn(23, h, w, c, device=cuda, generator=g).to(torch.bfloat16)
    w_f, _ = ops.prep_weight(torch.randn(ndim, c, 3, 3, device=cuda, generator=g) / (3 * c ** 0.5), want_dgrad=False)
    zero = torch.zeros(23, h, w, ndim, device=cuda, dtype=torch.bfloat16)
    st_h16, st_f32 = torch.zeros(2 * ndim, device=cuda), torch.zeros(2 * ndim, device=cuda)
    y_h16 = ops.conv_fprop(x, w_f, 3, 3, 1, 1, stats=st_h16)
    y_f32 = ops.conv_fprop(x, w_f, 3, 3, 1, 1, resid=zero, stats=st_f32)
    torch.cuda.synchronize()
    assert torch.equal(y_h16.float(), y_f32.float())   # + 0 residual: -0 becomes +0, nothing else changes
    assert torch.equal(st_h16, st_f32)


# the kernel each call launches: <BN, GROUPED, H16>
H16_64 = r"conv3x3_patch_kernel<64,false,true>"
H16_128 = r"conv3x3_patch_kernel<128,false,true>"
F32_TILE = r"conv3x3_patch_kernel<64,false,false>"
GROUPED = r"conv3x3_patch_kernel<64,true,false>"
LAUNCHES = {
    # the stride-1 3x3 layers of ResNet-50 (conv2 of the bottleneck), fprop with statistics and dgrad
    "rn50_56_fprop": (H16_64, dict(fprop=True, n=2, h=56, w=56, c=64, ndim=64, stats=True)),
    "rn50_56_dgrad": (H16_64, dict(fprop=False, n=2, h=56, w=56, c=64, ndim=64)),
    "rn50_28_fprop": (H16_128, dict(fprop=True, n=2, h=28, w=28, c=128, ndim=128, stats=True)),
    "rn50_28_dgrad": (H16_128, dict(fprop=False, n=2, h=28, w=28, c=128, ndim=128)),
    "rn50_14_fprop": (H16_128, dict(fprop=True, n=2, h=14, w=14, c=256, ndim=256, stats=True)),
    "rn50_14_dgrad": (H16_128, dict(fprop=False, n=2, h=14, w=14, c=256, ndim=256)),
    # epilogues the bf16 hand-off does not take
    "resid_fprop": (F32_TILE, dict(fprop=True, n=2, h=28, w=28, c=128, ndim=128, resid=True)),
    "relu_fprop": (F32_TILE, dict(fprop=True, n=2, h=28, w=28, c=128, ndim=128, relu=True)),
    "resid_dgrad": (F32_TILE, dict(fprop=False, n=2, h=14, w=14, c=256, ndim=256, resid=True)),
    "grouped_fprop": (GROUPED, dict(fprop=True, n=2, h=14, w=14, c=128, ndim=128, cg=4)),
}


def _launch(dev, fprop, n, h, w, c, ndim, stats=False, resid=False, relu=False, cg=None):
    from byol_b200 import ops
    x = torch.randn(n, h, w, c if fprop else ndim, device=dev).to(torch.bfloat16)
    if cg:
        wf, wd = ops.prep_weight_grouped(torch.randn(c, cg, 3, 3, device=dev))
    else:
        wf, wd = ops.prep_weight(torch.randn(ndim, c, 3, 3, device=dev))
    r = torch.randn(n, h, w, ndim if fprop else c, device=dev).to(torch.bfloat16) if resid else None
    st = torch.zeros(2 * ndim, device=dev) if stats else None
    if fprop:
        return lambda: ops.conv_fprop(x, wf, 3, 3, 1, 1, resid=r, stats=st, relu=relu)
    return lambda: ops.conv_dgrad(x, wd, h, w, 3, 3, 1, 1, resid=r)


def _check_launches():
    dev = torch.device("cuda:0")

    def complaints(name, launched):
        want = LAUNCHES[name][0]
        names = [k for k in launched if "conv3x3_patch_kernel" in k]
        if not any(re.search(re.escape(want), k) for k in names):
            return ["%s: expected %s, launched %s" % (name, want, sorted(set(names)))]
        return []
    check_row_launches({name: _launch(dev, **kw) for name, (_, kw) in LAUNCHES.items()}, complaints)


def test_patch_variant_launched(cuda):
    """Each kind of call launches its variant.  Checked in a fresh Python process: one that has already held many
    profiler sessions (the rest of the GPU suite) can drop CUDA kernel events."""
    check_in_fresh_process(__name__)
