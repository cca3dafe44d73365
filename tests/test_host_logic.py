"""CPU: host-side logic of the drop-in API — parameter order, state_dict keys, EMA schedule, LARS proxy behaviour,
optimizer wiring — and the guarantee that no CPU compute fallback exists."""
import numpy as np
import pytest
import torch

from oracle import byol_oracle as O


def test_byol_container_matches_reference_layout():
    from byol_b200.model import BYOL
    torch.manual_seed(7)
    m = BYOL(512, 256, 1000, 100, arch="resnet18")
    params, buffers = O.init_reference_state("resnet18", 7)
    names = [k for k, _ in m.named_parameters()]
    assert names == list(params.keys())                       # flat order = registration order (Q3)
    for (k, p) in m.named_parameters():
        assert torch.equal(p.detach(), params[k]), k           # same init as main.py:190-208 under the same seed
    sd = m.state_dict()
    assert "target_network.mean" in sd and sd["target_network.mean"].numel() == sum(p.numel() for p in m.parameters())
    assert "target_network.step" not in sd                     # Q13: step is not checkpointed
    for k in buffers:
        assert k in sd
    assert m.target_network.total_steps == 100 and m.target_network.base_decay == 0.996


def test_cos_ema_schedule_is_float64_numpy():
    from byol_b200.model import CosEMA
    ema = CosEMA(1000, 0.996)
    for step in (0, 1, 17, 500, 1000):
        assert ema.decay_at(step) == O.cos_ema_decay(step, 1000, 0.996)
    assert isinstance(ema.decay_at(3), (float, np.floating))


def test_no_cpu_fallback():
    from byol_b200.model import BYOL
    from byol_b200.objective import loss_function
    from byol_b200 import ops
    m = BYOL(512, 256, 1000, 10, arch="resnet18")
    x = torch.rand(2, 3, 32, 32)
    with pytest.raises(RuntimeError):
        m(x, x)
    with pytest.raises(RuntimeError):
        loss_function(torch.randn(4, 8), torch.randn(4, 8), torch.randn(4, 8), torch.randn(4, 8))
    with pytest.raises(ValueError):
        ops.bn_stats(torch.zeros(8, 8, dtype=torch.bfloat16), torch.zeros(16))


def test_lars_wrapper_api():
    from byol_b200.lars import LARS
    from byol_b200.wiring import add_weight_decay, build_optimizer
    net = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.BatchNorm1d(4))
    groups = add_weight_decay(net, 1e-6)
    assert [g["ignore"] for g in groups] == [True, False]
    assert len(groups[0]["params"]) == 3 and len(groups[1]["params"]) == 1   # bias + BN params vs the weight matrix
    assert groups[0]["weight_decay"] == 0.0 and groups[1]["weight_decay"] == 1e-6
    sgd = torch.optim.SGD(groups, lr=0.1, momentum=0.9)
    opt = LARS(sgd, eps=0.0)
    assert opt.param_groups is sgd.param_groups and opt.state is sgd.state
    assert opt.state_dict().keys() == sgd.state_dict().keys()
    with pytest.raises(ValueError):
        LARS(sgd, eps=-1.0)
    with pytest.raises(ValueError):
        LARS(sgd, trust_coef=-1.0)
    with pytest.raises(NotImplementedError):
        LARS(torch.optim.Adam(net.parameters()))
    # LR schedulers accept it (main.py:288-297 wraps it in LambdaLR / CosineAnnealingLR)
    sched = torch.optim.lr_scheduler.LambdaLR(opt, lambda e: 0.5)
    assert opt.param_groups[0]["lr"] == 0.05
    # lr scaling of main.py:334
    o2 = build_optimizer(net, base_lr=0.2, global_batch_size=4096)
    assert abs(o2.param_groups[0]["lr"] - 3.2) < 1e-12 and isinstance(o2, LARS)
    with pytest.raises(RuntimeError):   # parameters live on the CPU here: the fused step refuses to run
        for p in net.parameters():
            p.grad = torch.zeros_like(p)
        opt.step()


def test_bn_statistic_combination_matches_global_batch():
    """SyncBN restated on the host: summing per-rank (sum, sum of squares) and finalising with the global count
    equals BatchNorm over the concatenated batch (what byol_bn_finalize does after the all-reduce)."""
    g = torch.Generator().manual_seed(0)
    shards = [torch.randn(6, 5, generator=g) * 2 + 1 for _ in range(4)]
    s = sum(x.sum(0) for x in shards)
    q = sum((x * x).sum(0) for x in shards)
    n = 24
    mean, var = s / n, q / n - (s / n) ** 2
    full = torch.cat(shards)
    np.testing.assert_allclose(mean.numpy(), full.mean(0).numpy(), rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(var.numpy(), full.var(0, unbiased=False).numpy(), rtol=1e-4, atol=1e-6)


def test_lr_schedule_matches_reference_wiring():
    """f2: the closed-form per-epoch schedule reproduces the learning rates of the reference's own wiring
    (main.build_lr_schedule + optimizers/scheduler.py, recorded by tests/golden/make_golden.py) — including Q11:
    lr = 0.2 * 4096/256 = 3.2, linear warm-up over 10 epochs starting AT 0, then cosine."""
    import os
    from byol_b200.wiring import build_optimizer
    from byol_b200.schedule import EpochSchedule
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "lr_schedule.npz"))
    for tag, kind in (("cosine_w10_e40", "cosine"), ("fixed_w3_e12", "fixed"), ("cosine_w0_e8", "cosine")):
        epochs, warmup = [int(v) for v in z[tag + "_cfg"]]
        p = torch.nn.Parameter(torch.zeros(4))
        opt = torch.optim.SGD([p], lr=0.2, momentum=0.9)
        sched = EpochSchedule(opt, epochs, warmup, kind)
        lrs = []
        for _ in range(epochs):
            lrs.append(opt.param_groups[0]["lr"])
            sched.step()
        np.testing.assert_allclose(lrs, z[tag], rtol=1e-12, atol=1e-15, err_msg=tag)
    net = torch.nn.Sequential(torch.nn.Linear(4, 4), torch.nn.BatchNorm1d(4))
    opt = build_optimizer(net, base_lr=0.2, global_batch_size=4096)       # wraps SGD in byol_b200.LARS
    sched = EpochSchedule(opt, epochs=100, warmup=10)
    lrs = []
    for _ in range(14):
        lrs.append(opt.param_groups[0]["lr"])
        sched.step()
    assert lrs[0] == 0.0                                        # the whole first epoch trains with lr = 0
    np.testing.assert_allclose(lrs[1:11], [0.32 * i for i in range(1, 11)], rtol=1e-12)
    assert abs(lrs[10] - 3.2) < 1e-12 and lrs[12] < lrs[11] <= 3.2   # then cosine decay
    st = sched.state_dict()
    sched2 = EpochSchedule(opt, epochs=100, warmup=10)
    sched2.load_state_dict(st)
    assert sched2.get_last_lr() == sched.get_last_lr()


def test_vectorised_fma32_rounds_once():
    """tests.util.fma32 (the fused multiply-add of the numpy kernel restatements) equals the exact rational a*b + c
    rounded once to fp32, on random operands, on sums that cancel and on ties."""
    from tests.util import _fma32, fma32
    rng = np.random.default_rng(3)
    a = (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)).astype(np.float32)
    b = (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)).astype(np.float32)
    c = np.concatenate([(rng.standard_normal(2000) * 2.0 ** rng.integers(-60, 60, 2000)).astype(np.float32),
                        -(a[2000:].astype(np.float64) * b[2000:]).astype(np.float32)])   # near-total cancellation
    one = np.float32(1.0)
    ties = np.array([1 + 2.0 ** -23, 1 + 2.0 ** -22], dtype=np.float32)          # 1 * x + 2^-24: ties to even
    a = np.concatenate([a, ties, ties, [one, np.float32(np.inf), np.float32(np.nan)]])
    b = np.concatenate([b, [one, one], [one, one], [np.float32(0), one, one]])
    c = np.concatenate([c, np.float32([2.0 ** -24] * 2), np.float32([2.0 ** -24 + 2.0 ** -48] * 2),
                        [np.float32(-0.0), np.float32(-np.inf), one]])
    got, want = fma32(a, b, c), _fma32(a[:-2], b[:-2], c[:-2])
    assert np.array_equal(got[:-2].view(np.uint32), want.view(np.uint32))
    assert np.isnan(got[-2]) and np.isnan(got[-1])
