"""GPU: the weight-gradient kernels give the same bits as the build that recorded tests/golden/wgrad_bits_h100_rn50.json.

Every wgrad shape tools/bench_wgrad.py times (ResNet-50 @224 at 512 images: the stem, the 1x1, patch and gather 3x3
convolutions, the head and classifier linears), the split-operand planes (T = 3 and 6) and the grouped routes at small
sizes run once on seeded bf16 operands at the magnitudes of real data (ReLU activations, gradients around 1e-3) into a
non-zero fp32 dw, and the SHA-256 of dw must match the fixture.  A kernel change that keeps every dW element's fp32
partials and their fixed-point sum gives the same digests; one that regroups the pixels or changes a split does not.
The split counts depend on the SM count, so the test skips on a GPU with another count than the fixture's.

The special-value cases check the split-K reduction against float64: partials of 2^20 and more (the fp64 side sum of
the fixed-point accumulators), NaN, and +Inf / -Inf in different splits, on a many-split 1x1 GEMM (several threads per
element in wgrad_reduce_kernel), a one-split linear (added from the accumulators) and the 3x3 patch route.

Regenerate (on the build whose bits are the reference):  python tests/test_gpu_wgrad_bits.py --write
"""
import hashlib
import json
import math
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

FIXTURE = os.path.join(ROOT, "tests", "golden", "wgrad_bits_h100_rn50.json")
BF = torch.bfloat16
BATCH = 512

pytestmark = pytest.mark.gpu


def _cases():
    """name -> dict(op, shapes...).  The bench_wgrad rows at full size, then the planes and grouped routes."""
    from bench_wgrad import shape_rows
    cases = {}
    for r in shape_rows(BATCH, 224):
        k = r["k"]
        pad = (k - 1) // 2
        if r["kind"] == "linear":
            n, hw = r["M"], 1
        else:
            hw = r["hw"]
            ho = (hw + 2 * pad - k) // r["stride"] + 1
            n = r["M"] // (ho * ho)
        cases[r["name"]] = dict(op=r["kind"], n=n, hw=hw, cin=r["Cin"], cout=r["Cout"], k=k, s=r["stride"], p=pad)
    for T in (3, 6):
        cases["planes%d_1x1_256_512_14" % T] = dict(op="planes", T=T, n=16, hw=14, cin=256, cout=512, k=1, s=1, p=0)
        cases["planes%d_3x3_64_64_s2_28" % T] = dict(op="planes", T=T, n=8, hw=28, cin=64, cout=64, k=3, s=2, p=1)
        cases["planes%d_linear_2048_256" % T] = dict(op="planes", T=T, n=64, hw=1, cin=2048, cout=256, k=1, s=1, p=0)
    for s in (1, 2):
        cases["grouped_3x3_256_g32_s%d_28" % s] = dict(op="grouped", n=8, hw=28, cin=256, cout=256, cg=8, k=3, s=s, p=1)
    cases["gather_forced_3x3_128_128_28"] = dict(op="gather", n=8, hw=28, cin=128, cout=128, k=3, s=1, p=1)
    return cases


def _digest(name, c, dev):
    from byol_b200 import ops
    g = torch.Generator(device=dev).manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:15], 16))
    n, hw, cin, cout, k, s, p = c["n"], c["hw"], c["cin"], c["cout"], c["k"], c["s"], c["p"]
    ho = (hw + 2 * p - k) // s + 1
    T = c.get("T", 1)
    cin_w = c.get("cg", cin)
    dw = torch.randn(cout, cin_w, k, k, device=dev, generator=g) * 0.05     # wgrad accumulates into dw
    if c["op"] == "stem":
        img = torch.rand(n, 3, hw, hw, device=dev, generator=g)
        dy = (torch.randn(n, ho, ho, cout, device=dev, generator=g) * 1e-3).to(BF)
        ops.stem_conv_wgrad(ops.nchw_to_stem4(img), dy, dw, hw, hw)
    else:
        x = torch.randn(n, hw, hw, T * cin, device=dev, generator=g).relu_().to(BF)
        dy = (torch.randn(n, ho, ho, T * cout, device=dev, generator=g) * 1e-3).to(BF)
        if c["op"] == "planes":
            ops.conv_wgrad_planes(x, dy, dw, k, k, s, p, T)
        else:
            ops.conv_wgrad(x, dy, dw, k, k, s, p, force_gather=c["op"] == "gather")
    torch.cuda.synchronize()
    return hashlib.sha256(dw.cpu().numpy().tobytes()).hexdigest()


def _sm_count():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def golden(cuda):
    fx = _fixture()
    if fx["sm_count"] != _sm_count():
        pytest.skip("fixture recorded with %d SMs, this GPU has %d: the split counts differ"
                    % (fx["sm_count"], _sm_count()))
    return fx["digests"]


def test_fixture_covers_every_case():
    assert sorted(_fixture()["digests"]) == sorted(_cases())


@pytest.mark.parametrize("name", sorted(_cases()))
def test_wgrad_bits(cuda, golden, name):
    assert _digest(name, _cases()[name], cuda) == golden[name]


def _special_operands(n, hw, c, cout, k, specials):
    """Integer operands (exact products and fp32 partials): x in [-2, 2] with channel 0 = 2^12 and channel 1 = -2^12,
    dy in [-2, 2] with output channel 0 = 2, so dW[0, 0] and dW[0, 1] get partials of 2^20 and more per split.
    specials: x[pixel 0, 2] = +Inf and x[last pixel, 2] = -Inf (NaN after the sum), x[pixel 0, 3] = +Inf,
    x[pixel 5, 4] = NaN; dy is 1 at those pixels."""
    g = torch.Generator().manual_seed(11)
    ho = (hw + 2 * ((k - 1) // 2) - k) + 1
    x = torch.randint(-2, 3, (n, hw, hw, c), generator=g).double()
    dy = torch.randint(-2, 3, (n, ho, ho, cout), generator=g).double()
    x[..., 0], x[..., 1], dy[..., 0] = 4096.0, -4096.0, 2.0
    if specials:
        xf, dyf = x.view(-1, c), dy.view(-1, cout)
        xf[0, 2], xf[-1, 2], xf[0, 3], xf[5, 4] = math.inf, -math.inf, math.inf, math.nan
        dyf[0], dyf[-1], dyf[5] = 1.0, 1.0, 1.0
    dw0 = torch.randint(-3, 4, (cout, c, k, k), generator=g).double()
    return x, dy, dw0


def _expect_same(got, want):
    nan = torch.isnan(want)
    assert torch.equal(torch.isnan(got), nan), "NaN positions differ"
    assert torch.equal(got[~nan], want[~nan]), "max |diff| %g" % (got[~nan] - want[~nan]).abs().max().item()


@pytest.mark.parametrize("n,hw,k,specials", [(8, 28, 1, True), (512, 1, 1, True), (8, 28, 3, False)],
                         ids=["gemm1x1_many_splits", "linear_one_split", "patch3x3_many_splits"])
def test_reduction_special_values_match_float64(cuda, n, hw, k, specials):
    from byol_b200 import ops
    c = cout = 64 if hw > 1 else 256
    x, dy, dw0 = _special_operands(n, hw, c, cout, k, specials)
    dw = dw0.float().to(cuda)
    ops.conv_wgrad(x.to(cuda, BF), dy.to(cuda, BF), dw, k, k, 1, (k - 1) // 2)
    torch.cuda.synchronize()
    if k == 1:
        s64 = (dy.reshape(-1, cout).t() @ x.reshape(-1, c)).view(cout, c, 1, 1)
    else:
        s64 = torch.nn.grad.conv2d_weight(x.permute(0, 3, 1, 2), dw0.shape, dy.permute(0, 3, 1, 2), 1, 1)
    assert s64[0, 0].abs().max() >= 2 ** 20
    # the kernels add each element's exact total, rounded once to fp32, to dW with one fp32 addition
    _expect_same(dw.cpu(), s64.float() + dw0.float())


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        raise SystemExit("usage: python tests/test_gpu_wgrad_bits.py --write")
    dev = torch.device("cuda", 0)
    out = {"sm_count": _sm_count(), "device": torch.cuda.get_device_name(0),
           "digests": {name: _digest(name, c, dev) for name, c in sorted(_cases().items())}}
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d digests to %s" % (len(out["digests"]), FIXTURE))
