"""GPU: checkpoint / resume of the flat buffers (SURVEY.md §8(f)3): state_dict keys are the reference's, a restored
model + optimizer continue exactly like the original, and CosEMA.step is NOT part of the checkpoint (Q13)."""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu


def _make(seed):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    torch.manual_seed(seed)
    m = BYOL(512, 256, 1000, 20, arch="resnet:basic:1,1,1,1").cuda().train()
    opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(m, 1e-6), lr=0.3, momentum=0.9), eps=0.0)
    return m, opt


def test_checkpoint_round_trip(cuda):
    from byol_b200 import wiring
    g = torch.Generator().manual_seed(1)
    batches = [(torch.rand(8, 3, 64, 64, generator=g).cuda(), torch.rand(8, 3, 64, 64, generator=g).cuda(),
                torch.randint(0, 1000, (8,), generator=g).cuda()) for _ in range(3)]
    m1, o1 = _make(0)
    for b in batches[:2]:
        wiring.train_step(m1, o1, *b)
    sd_m = {k: v.clone() for k, v in m1.state_dict().items()}
    sd_o = copy.deepcopy(o1.state_dict())   # state_dict() returns references; a real checkpoint serialises them
    assert "target_network.mean" in sd_m and not any("step" in k for k in sd_m if k.startswith("target_network"))
    assert all(k.split(".")[0] in ("base_network", "head", "predictor", "linear_classifier", "target_network")
               for k in sd_m)
    m2, o2 = _make(123)                                   # different init: everything must come from the checkpoint
    m2.load_state_dict(sd_m)
    o2.load_state_dict(sd_o)
    m2.target_network.step = m1.target_network.step        # Q13: the reference's saver does not restore it either
    assert torch.equal(torch.nn.utils.parameters_to_vector(m2.parameters()),
                       torch.nn.utils.parameters_to_vector(m1.parameters()))
    assert torch.equal(m2.target_network.mean, m1.target_network.mean)
    r1 = wiring.train_step(m1, o1, *batches[2])
    r2 = wiring.train_step(m2, o2, *batches[2])
    torch.cuda.synchronize()
    # every cross-block sum is order-independent (fixed point, csrc/common.cuh): the restored model continues with
    # the same bits as the original
    assert torch.equal(r1["loss_mean"], r2["loss_mean"])
    t0 = torch.cat([sd_m[k].reshape(-1).float() for k, _ in m1.named_parameters()])
    t1 = torch.nn.utils.parameters_to_vector(m1.parameters()).detach()
    t2 = torch.nn.utils.parameters_to_vector(m2.parameters()).detach()
    assert float((t1 - t0).norm()) > 0 and torch.equal(t1, t2)          # incl. the restored momentum
    mom = [torch.cat([s["momentum_buffer"].reshape(-1) for s in o.state_dict()["state"].values()]) for o in (o1, o2)]
    assert torch.equal(mom[0], mom[1])
    assert torch.equal(m1.target_network.mean, m2.target_network.mean)
    assert all(torch.equal(a, b) for a, b in zip(m1.buffers(), m2.buffers()))
    for p in m2.parameters():                              # still views of the flat buffer after load_state_dict
        assert p.data_ptr() >= m2._engine.theta.data_ptr()
    assert m2._engine.is_flat()
