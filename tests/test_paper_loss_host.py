"""CPU: the torch restatement of the BYOL paper's loss (tests/paper_loss_oracle.py) against float64
numpy of the definition and against float64 autograd of F.normalize, and the variant checks of the public entry
points.

Definition: r(x) = max(sum x^2, 1e-12)^(-1/2), x^ = r(x) x, L = mean_i |q1^_i - z2^_i|^2 + |q2^_i - z1^_i|^2, the
targets constant.  F.normalize clamps the norm at 1e-12 instead of the sum of squares; the two agree on rows with
|x| >= 1e-6.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import byol_oracle
from tests import paper_loss_oracle as O


def _rows(seed, b, d, tiny=False):
    g = torch.Generator().manual_seed(seed)
    xs = [torch.randn(b, d, generator=g, dtype=torch.float64) for _ in range(4)]
    xs[3] = xs[0] * 0.6 + xs[3] * 0.4          # correlated targets, as in training
    xs[2] = xs[1] * 0.6 + xs[2] * 0.4
    if tiny:
        xs[0][0] = 0.0                          # a zero row
        xs[1][1] = 0.0
        xs[1][1, 0] = 3e-7                      # sum of squares 9e-14 <= 1e-12: clamped
        xs[2][2] *= 1e-5                        # small but not clamped
    return xs


def _numpy_definition(q1, q2, z1, z2):
    def nrm(x):
        return x / np.sqrt(np.maximum((x * x).sum(1, keepdims=True), 1e-12))
    return float((((nrm(q1) - nrm(z2)) ** 2).sum(1) + ((nrm(q2) - nrm(z1)) ** 2).sum(1)).mean())


@pytest.mark.parametrize("b,d,tiny", [(1, 8, False), (7, 256, True), (64, 2048, True), (512, 256, False)])
def test_oracle_paper_loss_matches_numpy_definition(b, d, tiny):
    xs = _rows(b + d, b, d, tiny)
    got = float(O.paper_loss_function(*xs))
    want = _numpy_definition(*[x.numpy() for x in xs])
    assert abs(got - want) <= 1e-13 * max(1.0, abs(want)), (got, want)
    assert 0.0 <= got <= 8.0
    # no row clamped: 4 - 2 cos - 2 cos
    if not tiny:
        c12 = F.cosine_similarity(xs[0], xs[3], dim=1, eps=0.0)
        c21 = F.cosine_similarity(xs[1], xs[2], dim=1, eps=0.0)
        assert abs(got - float((4 - 2 * c12 - 2 * c21).mean())) < 1e-12


@pytest.mark.parametrize("b,d", [(7, 8), (64, 256), (16, 2048)])
def test_oracle_paper_loss_matches_normalize_autograd(b, d):
    """Rows with |x| >= 1e-6: the oracle's loss and gradients equal float64 autograd of F.normalize."""
    xs = _rows(3 * b + d, b, d)
    xs[0][1] *= 2e-6 / float(xs[0][1].norm())   # a row of norm 2e-6
    q1, q2 = (x.clone().requires_grad_(True) for x in xs[:2])
    q1r, q2r = (x.clone().requires_grad_(True) for x in xs[:2])
    got = O.paper_loss_function(q1, q2, xs[2], xs[3])
    ref = (((F.normalize(q1r, dim=1) - F.normalize(xs[3], dim=1)) ** 2).sum(1) +
           ((F.normalize(q2r, dim=1) - F.normalize(xs[2], dim=1)) ** 2).sum(1)).mean()
    go = torch.tensor(0.75, dtype=torch.float64)
    got.backward(go)
    ref.backward(go)
    assert abs(got.item() - ref.item()) < 1e-13
    for a, r in ((q1.grad, q1r.grad), (q2.grad, q2r.grad)):
        assert float((a - r).abs().max()) <= 1e-11 * float(r.abs().max())


def test_oracle_train_step_selects_the_loss():
    """OracleBYOL.train_step(loss=...) optimises the selected loss and leaves the pinned oracle's loss in place."""
    params, buffers = byol_oracle.init_reference_state("resnet:basic:1,1,1,1", 3, head_latent=64, num_classes=10)
    oracle = O.OracleBYOL("resnet:basic:1,1,1,1", params, buffers, 10)
    g = torch.Generator().manual_seed(4)
    a1, a2 = torch.rand(4, 3, 32, 32, generator=g), torch.rand(4, 3, 32, 32, generator=g)
    lab = torch.randint(0, 10, (4,), generator=g)
    for name, fn in (("byol", O.paper_loss_function), ("reference", byol_oracle.loss_function)):
        res = oracle.train_step(a1, a2, lab, 0.1, loss=name)
        want = fn(res["online_prediction1"], res["online_prediction2"], res["target_projection1"],
                  res["target_projection2"])
        assert torch.equal(res["byol_loss"], want), name
        assert byol_oracle.loss_function is O.LOSSES["reference"]


def test_bad_variant_raises_before_cuda_work():
    from byol_b200.objective import loss_function
    from byol_b200 import wiring
    x = torch.zeros(4, 8)
    for bad in ("BYOL", "paper", None, ""):
        with pytest.raises(ValueError, match="variant"):
            loss_function(x, x, x, x, variant=bad)
        # the step checks its variant before it calls the model
        with pytest.raises(ValueError, match="variant"):
            wiring.train_step(None, None, x, x, None, loss_variant=bad)
    with pytest.raises(RuntimeError, match="CUDA"):
        loss_function(x, x, x, x, variant="byol")
