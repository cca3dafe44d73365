"""GPU: the fixed-route BatchNorm kernels give the same bits as the build that recorded
tests/golden/bn_bits_h100_rn50.json.

Every shape tools/bench_bn.py times (ResNet-50 @224 at 512 images: the forward apply with no residual, an identity
residual and a downsample-BN residual, the backward reduction and apply with the ReLU mask recomputed from x and with
the forward's mask bits, the stem and the heads' BatchNorm1d at 4096 x 512) runs once on seeded operands at the
magnitudes of real data: activations around N(0, 1) in bf16, gradients around 1e-3, random mask bits and coefficients
that are not powers of two.  The SHA-256 of every output must match the fixture: y and the mask bits of the forward
apply, the fp32 sums s12 of the reduction, dy of the backward apply.

The apply kernels are elementwise, so any schedule gives their bits.  The reduction's result is defined by its
S = fixed_grid(M*C/8, C/8) * 256 fp32 partial sums per channel (partial t sums the 8-channel vectors t, t+S, t+2S, ...
in that order) and their fixed-point total; S is computed with the constant 132 of fixed_grid, not from the device.
The operands are drawn with a CPU generator and copied to the GPU (torch's CUDA sampling kernels size their grids
from the SM count, which would change the values).  So neither the operands nor the digests depend on the SM count,
and the test runs on any GPU.

Regenerate (on the build whose bits are the reference):  python tests/test_gpu_bn_bits.py --write
"""
import hashlib
import json
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

FIXTURE = os.path.join(ROOT, "tests", "golden", "bn_bits_h100_rn50.json")
BATCH = 512

pytestmark = pytest.mark.gpu


def _cases():
    from bench_bn import shape_rows
    return {r["name"]: (r["kind"], r["M"], r["C"]) for r in shape_rows(BATCH, 224)}


def _digests(name, dev):
    from bench_bn import operands
    kind, m, c = _cases()[name]
    # a CPU generator: the same operands on every GPU (see the docstring)
    g = torch.Generator().manual_seed(int(hashlib.sha256(name.encode()).hexdigest()[:15], 16))
    run, outs = operands(kind, m, c, dev, g)
    run()
    torch.cuda.synchronize()
    d = {"%s/%s" % (name, k): hashlib.sha256(v.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()
         for k, v in outs.items()}
    del run, outs
    torch.cuda.empty_cache()
    return d


def _fixture():
    with open(FIXTURE) as f:
        return json.load(f)


def test_fixture_covers_every_case():
    names = sorted({k.split("/")[0] for k in _fixture()["digests"]})
    assert names == sorted(_cases())


@pytest.mark.parametrize("name", sorted(_cases()))
def test_bn_bits(cuda, name):
    want = {k: v for k, v in _fixture()["digests"].items() if k.split("/")[0] == name}
    assert _digests(name, cuda) == want


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        raise SystemExit("usage: python tests/test_gpu_bn_bits.py --write")
    dev = torch.device("cuda", 0)
    digests = {}
    for name in sorted(_cases()):
        digests.update(_digests(name, dev))
    out = {"device": torch.cuda.get_device_name(0), "digests": digests}
    with open(FIXTURE, "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote %d digests to %s" % (len(digests), FIXTURE))
