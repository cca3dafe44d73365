"""CPU: the arithmetic behind the fp32-accurate path (csrc/split.cu), restated with torch on the host.

* the 3-way bf16 split is EXACT: x0 + x1 + x2 == x for every finite fp32 |x| >= 2^-110 up to FLT_MAX (below, x2 can
  fall under bf16's subnormal spacing 2^-133), with x0 clamped to the largest finite bf16 where x rounds to inf;
* the plane patterns of the kernels (activation side A, weight side B) enumerate exactly the product terms
  x0w0, x0w1, x1w0, x1w1, x0w2, x2w0 (T = 6) / x0w0, x0w1, x1w0 (T = 3);
* a dot product over those terms with fp32 accumulation matches float64 to ~1e-7 (T = 6) / ~1e-5 (T = 3), where
  plain bf16 operands are at ~1e-3 and TF32 operands at ~1e-4 — the per-layer numbers behind DESIGN.md §4's table.
"""
import torch

A6, B6 = (0, 0, 1, 1, 0, 2), (0, 1, 0, 1, 2, 0)
A3, B3 = (0, 0, 1), (0, 1, 0)


BF16_MAX = torch.finfo(torch.bfloat16).max


def _planes(x):
    """split3 (csrc/split.cu): a finite x that rounds to inf in bf16 takes x0 = the largest finite bf16 of its sign."""
    p0 = x.to(torch.bfloat16).float()
    p0 = torch.where(torch.isinf(p0) & torch.isfinite(x), torch.sign(x) * BF16_MAX, p0)
    r1 = x - p0
    p1 = r1.to(torch.bfloat16).float()
    r2 = r1 - p1
    p2 = r2.to(torch.bfloat16).float()
    return [p0, p1, p2], r1, r2


def test_three_way_split_is_exact():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(1 << 16, generator=g) * torch.logspace(-6, 6, 1 << 16)
    (p0, p1, p2), r1, r2 = _planes(x)
    # residuals are exactly representable: the subtraction commits no rounding error
    assert torch.equal((x.double() - p0.double()).float().double(), x.double() - p0.double())
    assert torch.equal((r1.double() - p1.double()).float().double(), r1.double() - p1.double())
    recon = p0.double() + p1.double() + p2.double()
    rel = ((recon - x.double()).abs() / x.double().abs()).max().item()
    assert rel <= 2.0 ** -24, rel
    two = p0.double() + p1.double()
    assert ((two - x.double()).abs() / x.double().abs()).max().item() <= 2.0 ** -16


def _bits(v):
    return torch.tensor(v, dtype=torch.int64).to(torch.int32).view(torch.float32)


def test_three_way_split_is_exact_over_the_finite_range():
    g = torch.Generator().manual_seed(2)
    n = 1 << 18
    # every exponent from the fp32 subnormals to FLT_MAX, random mantissas and signs, plus the edges of the bf16
    # overflow: 0x7F7F8000 is the smallest finite value that rounds to inf
    bits = torch.randint(0, 0x7F800000, (n,), generator=g, dtype=torch.int64)
    edges = [0x7F7F7FFF, 0x7F7F8000, 0x7F7F8001, 0x7F7FC000, 0x7F7FFFFF, 0x7F000000, 0x00800000, 0x007FFFFF, 1,
             0x0A800000, 0x0A800001, 0x0A7FFFFF, 0x0A000001]
    bits[:len(edges)] = torch.tensor(edges)
    x = _bits(bits.tolist())
    x = torch.where(torch.rand(n, generator=g) < 0.5, -x, x)
    (p0, p1, p2), r1, r2 = _planes(x)
    for p in (p0, p1, p2):
        assert bool(torch.isfinite(p).all()), "a finite value split into a non-finite plane"
    assert torch.equal(p0[1:5].abs(), torch.full((4,), BF16_MAX)), "x0 of values past 0x7F7F8000 is not clamped"
    assert torch.equal(p0[0], torch.tensor(BF16_MAX).copysign(x[0])), "0x7F7F7FFF rounds down to the largest bf16"
    # exact for |x| >= 2^-110: the residual r2 is then a multiple of 2^-133, bf16's subnormal spacing
    exact_from = 2.0 ** -110
    back = p0.double() + p1.double() + p2.double()
    big = x.abs() >= exact_from
    assert torch.equal(back[big], x.double()[big])
    # below 2^-110 the split loses at most 2^-134 (half of bf16's subnormal spacing), and it does lose bits there:
    # 2^-111 (1 + 2^-23) = 0x08000001 splits into (2^-111, 0, 0)
    assert float((back[~big] - x.double()[~big]).abs().max()) <= 2.0 ** -134
    tiny = _bits([0x08000001])
    (q0, q1, q2), _, _ = _planes(tiny)
    assert float(tiny) < exact_from and float(q0 + q1 + q2) == 2.0 ** -111 != float(tiny)
    # just above: 0x0A000001 = 2^-107 (1 + 2^-23) still splits exactly
    assert float(x[12].abs()) >= exact_from and float(back[12]) == float(x[12])
    # non-finite operands: +-inf splits into (+-inf, NaN, NaN), NaN into NaNs, so every product they reach is NaN
    (i0, i1, i2), _, _ = _planes(torch.tensor([float("inf"), float("-inf"), float("nan")]))
    assert torch.equal(i0[:2], torch.tensor([float("inf"), float("-inf")])) and bool(torch.isnan(i0[2]))
    assert bool(torch.isnan(i1).all() and torch.isnan(i2).all())


def test_plane_patterns_enumerate_the_product_terms():
    assert sorted(zip(A6, B6)) == sorted([(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)])
    assert sorted(zip(A3, B3)) == sorted([(0, 0), (0, 1), (1, 0)])
    # every dropped term (a, b) has a + b >= 3 (T = 6: <= 2^-24 relative) / a + b >= 2 (T = 3: <= 2^-16)
    assert all(a + b >= 3 for a in range(3) for b in range(3) if (a, b) not in set(zip(A6, B6)))
    assert all(a + b >= 2 for a in range(3) for b in range(3) if (a, b) not in set(zip(A3, B3)))


def _split_dot(x, w, pa, pb):
    xp, wp = _planes(x)[0], _planes(w)[0]
    # the kernels run ONE GEMM over the concatenated planes: products of bf16 values are exact in fp32, accumulation fp32
    xa = torch.cat([xp[a] for a in pa], 1)
    wb = torch.cat([wp[b] for b in pb], 1)
    return xa @ wb.t()


def test_split_dot_products_reach_fp32_accuracy():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(64, 1152, generator=g) * 2 + 0.7          # 3x3 x 128 channels, large mean like pre-BN activations
    w = torch.randn(32, 1152, generator=g) * 0.05
    ref = x.double() @ w.double().t()
    scale = ref.abs().max()
    err = lambda y: ((y.double() - ref).abs().max() / scale).item()
    e6, e3 = err(_split_dot(x, w, A6, B6)), err(_split_dot(x, w, A3, B3))
    ebf = err(x.to(torch.bfloat16).float() @ w.to(torch.bfloat16).float().t())
    tf32 = lambda t: ((t.view(torch.int32) + 0x1000) & ~0x1FFF).view(torch.float32)
    etf = err(tf32(x.clone()) @ tf32(w.clone()).t())
    efp = err(x @ w.t())
    print("dot-product errors: fp32 %.1e  T=6 %.1e  T=3 %.1e  tf32 %.1e  bf16 %.1e" % (efp, e6, e3, etf, ebf))
    assert e6 < 5e-7 and e6 < 4 * efp + 1e-7          # the 6-term split is as good as fp32 itself
    assert e3 < 3e-5 and etf < 2e-3 and ebf < 2e-2
    assert e6 < e3 < etf < ebf
