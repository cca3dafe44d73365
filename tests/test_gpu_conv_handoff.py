"""GPU: the bf16 hand-off of conv_igemm_kernel (plain 1x1 GEMMs whose epilogue only stores bf16 values and sums their
statistics) on shapes that hit its edges: a last tile whose third row quarter is partial and whose fourth is empty,
partial column tiles (Ndim 40 with BN = 64, 200 with BN = 128), a partial k-block (C = 96), and more tiles than SMs,
so that a CTA moves to another column tile and flushes its statistics between tiles, into block-local fixed-point
words in shared memory or, for an Ndim too wide for them, into the global accumulators.

* The stored output is bit-equal to the gathered-operand path of the same kernel (force_gather=True: the same K loop,
  BN and tile order, the fp32 hand-off).
* The fused statistics are checked bit for bit with small-integer inputs, where every partial sum is exact, so they
  must equal the fp64 column sums of the stored output rounded once to fp32.  (With random inputs the gathered path
  is no bitwise reference for the statistics: it differs from the TMA-operand path in the last bit of a few column
  sums with either hand-off.)
"""
import pytest
import torch

pytestmark = pytest.mark.gpu
BF = torch.bfloat16

# (name, images, h, w, C): rows = images * h * w
GEOMS = [
    ("rows17500", 7, 50, 50, 256),   # 137 row tiles (> 132 SMs); the last has 92 rows: quarter 2 has 28, quarter 3 none
    ("rows81", 1, 9, 9, 96),         # one row tile of 81 rows (quarter 2: 17 rows); K = 96 is one and a half k-blocks
]
# 2048: 16 column tiles, so a CTA changes column tile after every tile and sums its statistics in shared memory;
# 2176: too wide for the block-local statistic words, the flushes go to the global accumulators directly
NDIMS = [40, 64, 128, 200, 2048, 2176]


def _operands(dev, geom, ndim, seed, exact):
    _, n, h, w, c = geom
    g = torch.Generator().manual_seed(seed)
    if exact:   # integers in [-1, 1], mostly zero: |y| <= C is exact in bf16 and every fp32 partial sum is exact
        src = torch.randint(-1, 2, (n, h, w, c), generator=g).float() * (torch.rand(n, h, w, c, generator=g) < 0.25)
        wt = torch.randint(-1, 2, (ndim, c), generator=g).float() * (torch.rand(ndim, c, generator=g) < 0.5)
    else:
        src = torch.randn(n, h, w, c, generator=g)
        wt = torch.randn(ndim, c, generator=g) / c ** 0.5
    return src.to(BF).to(dev), wt.to(BF).to(dev)   # wt: [Ndim][K], the fprop and dgrad layout of a 1x1


@pytest.mark.parametrize("exact", [False, True], ids=["random", "integer"])
@pytest.mark.parametrize("ndim", NDIMS)
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_fprop_stats_handoff(cuda, geom, ndim, exact):
    from byol_b200 import ops
    src, wt = _operands(cuda, geom, ndim, 100 + ndim, exact)
    st = torch.zeros(2 * ndim, device=cuda)
    y = ops.conv_fprop(src, wt, 1, 1, 1, 0, stats=st)
    yg = ops.conv_fprop(src, wt, 1, 1, 1, 0, force_gather=True)
    torch.cuda.synchronize()
    assert torch.equal(y, yg), "y: %d values differ from the gathered path" % int((y != yg).sum())
    yr = y.double().reshape(-1, ndim)
    want = torch.cat([yr.sum(0), (yr * yr).sum(0)])
    if exact:
        bad = st != want.float()
        assert not bad.any(), "statistics: %d of %d differ from the fp64 sums" % (int(bad.sum()), 2 * ndim)
    else:
        torch.testing.assert_close(st[:ndim].double(), want[:ndim], atol=1e-3 * float(yr.abs().sum(0).max()), rtol=0)
        torch.testing.assert_close(st[ndim:].double(), want[ndim:], atol=0, rtol=1e-4)


@pytest.mark.parametrize("ndim", NDIMS)
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_dgrad_handoff(cuda, geom, ndim):
    from byol_b200 import ops
    _, n, h, w, c = geom
    dy, wd = _operands(cuda, geom, ndim, 200 + ndim, False)
    dx = ops.conv_dgrad(dy, wd, h, w, 1, 1, 1, 0)
    dxg = ops.conv_dgrad(dy, wd, h, w, 1, 1, 1, 0, force_gather=True)
    torch.cuda.synchronize()
    assert dx.shape == (n, h, w, ndim)
    assert torch.equal(dx, dxg), "dx: %d values differ from the gathered path" % int((dx != dxg).sum())
