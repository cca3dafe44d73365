"""CPU: argument checks and host-side rules of the linear evaluation (byol_b200.linear_eval): the head grid, the cosine
factor, the hold-out split, the head selection; and the numpy oracle the GPU tests compare against
(tests/linear_oracle.py)."""
import math
import types

import numpy as np
import pytest
import torch

from tests import linear_oracle as O


def _feats(n=32, d=64, dtype=torch.bfloat16):
    return torch.zeros(n, d, dtype=dtype), torch.zeros(n, dtype=torch.int64)


@pytest.mark.parametrize("kw, match", [
    (dict(lrs=()), "lrs"),
    (dict(lrs=(0.1, float("nan"))), "lrs"),
    (dict(lrs=(0.1, -0.1)), "lrs"),
    (dict(lrs=(float("inf"),)), "lrs"),
    (dict(weight_decays=(-1e-4,)), "weight_decays"),
    (dict(weight_decays=(float("nan"),)), "weight_decays"),
    (dict(weight_decays=()), "weight_decays"),
    (dict(momentum=1.0), "momentum"),
    (dict(momentum=-0.1), "momentum"),
    (dict(momentum=float("nan")), "momentum"),
    (dict(epochs=0), "epochs"),
    (dict(epochs=2.0), "epochs"),
    (dict(batch_size=0), "batch_size"),
    (dict(batch_size=33), "fill one batch"),
    (dict(num_classes=1), "num_classes"),
])
def test_train_linear_heads_rejects_bad_arguments(kw, match):
    from byol_b200.linear_eval import train_linear_heads
    f, l = _feats()
    args = dict(num_classes=10, epochs=1, batch_size=8)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        train_linear_heads(f, l, f, l, **args)


def test_train_linear_heads_rejects_bad_features():
    from byol_b200.linear_eval import train_linear_heads
    f, l = _feats()
    with pytest.raises(ValueError, match="multiple of 64"):
        train_linear_heads(torch.zeros(32, 96, dtype=torch.bfloat16), l, f, l, 10, batch_size=8)
    with pytest.raises(ValueError, match="width"):
        train_linear_heads(f, l, torch.zeros(4, 128, dtype=torch.bfloat16), l[:4], 10, batch_size=8)
    with pytest.raises(ValueError, match="bf16 or fp32"):
        train_linear_heads(f.half(), l, f, l, 10, batch_size=8)
    with pytest.raises(ValueError, match="labels"):
        train_linear_heads(f, l.int(), f, l, 10, batch_size=8)
    with pytest.raises(ValueError, match="labels"):
        train_linear_heads(f, l[:5], f, l, 10, batch_size=8)
    with pytest.raises(ValueError, match="validation split is empty"):
        train_linear_heads(f, l, f[:0], l[:0], 10, batch_size=8)
    with pytest.raises(TypeError):
        train_linear_heads([1], l, f, l, 10)


def test_cpu_tensors_raise_runtime_error():
    from byol_b200 import linear_eval as L
    f, l = _feats()
    with pytest.raises(RuntimeError, match="CUDA"):
        L.train_linear_heads(f, l, f, l, 10, epochs=1, batch_size=8)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.train_linear_heads(f.float(), l, f.float(), l, 10, epochs=1, batch_size=8)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.multihead_ce(torch.zeros(4, 16), torch.zeros(4, dtype=torch.int64), 1, 10, hits=torch.zeros(1, 2))
    with pytest.raises(RuntimeError, match="CUDA"):
        L.LinearHeads(64, 10, (0.1,), (0.0,), device="cpu")


def _loader(n_train, n_test=3, n_valid=None, classes=3, batch=4):
    def split(n):
        return types.SimpleNamespace(samples=[("img%d.JPEG" % i, i % classes) for i in range(n)], batch_size=batch,
                                     augment=None, workers=2)
    return types.SimpleNamespace(output_size=classes, train_loader=split(n_train), test_loader=split(n_test),
                                 valid_loader=None if n_valid is None else split(n_valid))


@pytest.mark.parametrize("kw, match", [
    (dict(lrs=()), "lrs"),
    (dict(weight_decays=(-1.0,)), "weight_decays"),
    (dict(momentum=1.5), "momentum"),
    (dict(epochs=0), "epochs"),
    (dict(batch_size=0), "batch_size"),
    (dict(network="both"), "network"),
])
def test_linear_accuracy_rejects_bad_arguments(kw, match):
    from byol_b200.linear_eval import linear_accuracy
    model = types.SimpleNamespace(base_network_output_size=512)
    with pytest.raises(ValueError, match=match):
        linear_accuracy(model, _loader(20), **kw)


def test_linear_accuracy_checks_splits_before_device_work():
    """The model below would fail on any call: every error must come from the checks."""
    from byol_b200.linear_eval import linear_accuracy
    model = types.SimpleNamespace(base_network_output_size=512)
    with pytest.raises(ValueError, match="test split is empty"):
        linear_accuracy(model, _loader(20, n_test=0), batch_size=4)
    with pytest.raises(ValueError, match="fill one batch"):      # 20 images, 2 held out: 18 < 19
        linear_accuracy(model, _loader(20), batch_size=19)
    with pytest.raises(ValueError, match="fill one batch"):      # a valid split: all 20 train
        linear_accuracy(model, _loader(20, n_valid=5), batch_size=21)
    with pytest.raises(ValueError, match="multiple of 64"):
        linear_accuracy(types.SimpleNamespace(base_network_output_size=100), _loader(20), batch_size=4)
    with pytest.raises(ValueError, match="2 classes"):
        linear_accuracy(model, _loader(20, classes=1), batch_size=4)


def test_head_grid_is_lr_major():
    from byol_b200.linear_eval import head_grid
    assert head_grid((0.4, 0.1), (0.0, 1e-4, 1e-3)) == [(0.4, 0.0), (0.4, 1e-4), (0.4, 1e-3), (0.1, 0.0),
                                                        (0.1, 1e-4), (0.1, 1e-3)]
    assert head_grid((0.3,), (0.0,)) == [(0.3, 0.0)]


def test_cosine_factor():
    from byol_b200.linear_eval import cosine_factor
    total = 1000
    f = [cosine_factor(t, total) for t in range(total)]
    assert all(isinstance(v, np.float32) for v in f)
    assert f[0] == 1.0 and f[total // 2] == np.float32(0.5)
    assert all(a >= b for a, b in zip(f, f[1:])) and f[-1] > 0
    for t in (1, 137, 999):      # fp64 formula rounded once to fp32
        assert f[t] == np.float32(0.5 * (1.0 + math.cos(math.pi * t / total)))
    assert cosine_factor(0, 1) == 1.0


@pytest.mark.parametrize("n", [1, 9, 10, 57, 1000, 123457])
def test_holdout_split(n):
    from byol_b200.linear_eval import holdout_split
    fit, val = holdout_split(n, seed=3)
    assert len(val) == max(1, min(10000, n // 10)) and len(fit) == n - len(val)
    assert not np.intersect1d(fit, val).size
    assert np.array_equal(np.sort(np.concatenate([fit, val])), np.arange(n))
    assert (np.diff(fit) > 0).all() and (np.diff(val) > 0).all()
    fit2, val2 = holdout_split(n, seed=3)
    assert np.array_equal(fit, fit2) and np.array_equal(val, val2)
    if n >= 57:
        assert not np.array_equal(val, holdout_split(n, seed=4)[1])
    with pytest.raises(ValueError):
        holdout_split(0, 0)


def test_select_head_ties_go_to_the_earlier_head():
    from byol_b200.linear_eval import select_head
    assert select_head([3, 7, 7, 2]) == 1
    assert select_head(np.array([5, 5, 5])) == 0
    assert select_head([0, 0, 1]) == 2
    with pytest.raises(ValueError):
        select_head([])


def test_select_head_skips_diverged_heads():
    from byol_b200.linear_eval import select_head
    assert select_head([9, 7, 7, 2], finite=[False, True, True, True]) == 1
    assert select_head([100.0, 0.0], finite=[False, True]) == 1
    assert select_head(np.array([0, 0, 0]), finite=np.array([False, False, True])) == 2
    with pytest.raises(ValueError, match="diverged"):
        select_head([5, 6], finite=[False, False])


# ---- the oracle ----
def test_oracle_bf16_rounds_to_nearest_even():
    x = np.array([1.0, 1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8, 1.0 + 2.0 ** -9, -3.14159], dtype=np.float32)
    got = O.bf16(x)
    assert got[0] == 1.0 and got[1] == 1.0 and got[2] == 1.0 + 2.0 ** -6 and got[3] == 1.0
    assert np.array_equal(got, torch.from_numpy(x).bfloat16().float().numpy())


def test_oracle_cross_entropy():
    z = np.array([[1.0, 2.0, 2.0, 0.0, 9.0, 9.0, 9.0, 9.0,     # head 0: C = 3 of Cp = 8, padding ignored
                   0.5, 0.5, -1.0, 0.0, 0.0, 0.0, 0.0, 0.0]])
    loss, rank, grad = O.cross_entropy(z, np.array([1]), 2, 3)
    p = np.exp([1.0, 2.0, 2.0]) / np.exp([1.0, 2.0, 2.0]).sum()
    assert np.isclose(loss[0, 0], -np.log(p[1])) and rank.tolist() == [[0, 0]]    # ties do not count
    assert np.allclose(grad[0, :3], p - [0, 1, 0]) and not grad[0, 3:8].any()
    assert np.allclose(grad.reshape(2, 8).sum(1), 0)


def test_oracle_rank_counts_nan_above_and_misses_nan_labels():
    nan, inf = np.nan, np.inf
    s = np.array([[1.0, 2.0, 2.0, 0.0],
                  [1.0, nan, 0.5, 0.0],       # a NaN elsewhere ranks above the label
                  [nan, 1.0, 2.0, 0.0],       # the label's value is NaN: a miss
                  [inf, 1.0, inf, 0.0],       # ties with +inf do not count
                  [1.0, 2.0, 3.0, 4.0],       # label out of range
                  [1.0, 2.0, 3.0, 4.0]])
    r = O.rank(s, np.array([1, 0, 0, 0, 4, -1]))
    assert r.tolist() == [0, 1, O.MISS, 0, O.MISS, O.MISS]
    loss, ranks, grad = O.cross_entropy(s, np.array([1, 0, 0, 0, 4, -1]), 1, 4)
    assert ranks[:, 0].tolist() == r.tolist()
    assert not loss[4:].any() and not grad[4:].any()


def test_oracle_sgd_first_step_is_plain_momentum_sgd():
    w = np.float32([1.0, -2.0])
    g = np.float32([0.5, 0.25])
    w1, buf = O.sgd(w, np.zeros(2, np.float32), g, np.float32(0.1), np.float32(0.0), 0.9)
    assert np.array_equal(buf, g)
    assert np.array_equal(w1, w - np.float32(0.1) * (g + np.float32(0.9) * g))
