"""CPU: the host side of semi-supervised evaluation (byol_b200.finetune) and the lane-aware memory planner.

* The labelled subset: per-class counts max(1, floor(f n_c + 0.5)), seeded and reproducible, every class present;
  file-name subsets matched by base name, unknown and ambiguous names rejected.
* The selection hold-out: disjoint from the subset, of size max(1, min(10 000, M // 10)), ValueError when nothing is
  left.
* Every bad argument raises before any device work.
* Engine.memory_model / step_need: the BYOL defaults give the numbers of the two-lane formula; one lane without target
  pair or MLPs saves one lane's bytes and has no target term.
"""
import math
import types

import numpy as np
import pytest

from byol_b200 import finetune as F


def _samples(counts):
    out = []
    for c, n in enumerate(counts):
        out += [("/data/train/class%d/img_%d_%d.JPEG" % (c, c, i), c) for i in range(n)]
    return out


@pytest.mark.parametrize("f", [0.01, 0.1, 0.37, 1.0])
def test_subset_per_class_counts(f):
    counts = [1300, 732, 5, 1, 40]
    s = _samples(counts)
    idx = F.label_subset(s, len(counts), label_fraction=f, seed=3)
    assert np.all(np.diff(idx) > 0)
    got = np.bincount([s[i][1] for i in idx], minlength=len(counts))
    want = [max(1, int(math.floor(f * n + 0.5))) for n in counts]
    assert got.tolist() == want
    assert (got > 0).all()                                          # every class present


def test_subset_is_seeded_and_reproducible():
    s = _samples([200, 300, 100])
    a = F.label_subset(s, 3, label_fraction=0.1, seed=0)
    assert np.array_equal(a, F.label_subset(s, 3, label_fraction=0.1, seed=0))
    assert not np.array_equal(a, F.label_subset(s, 3, label_fraction=0.1, seed=1))


def test_subset_by_file_names():
    s = _samples([4, 4])
    names = ["img_0_2.JPEG", "  img_1_3.JPEG\n", "", "img_0_2.JPEG"]      # white space, blank lines, repeats
    assert F.label_subset(s, 2, subset=names).tolist() == [2, 7]
    with pytest.raises(ValueError, match="matches no training image"):
        F.label_subset(s, 2, subset=["img_0_9.JPEG"])
    s2 = s + [("/data/train/class1/sub/img_0_2.JPEG", 1)]                  # the same base name twice
    with pytest.raises(ValueError, match="matches 2 training images"):
        F.label_subset(s2, 2, subset=["img_0_2.JPEG"])
    with pytest.raises(ValueError, match="names no image"):
        F.label_subset(s, 2, subset=["", " "])
    with pytest.raises(ValueError, match="single string"):
        F.label_subset(s, 2, subset="img_0_2.JPEG")


@pytest.mark.parametrize("kw", [dict(), dict(label_fraction=0.1, subset=["a.JPEG"])])
def test_exactly_one_of_fraction_and_subset(kw):
    with pytest.raises(ValueError, match="exactly one"):
        F.label_subset(_samples([4]), 1, **kw)


@pytest.mark.parametrize("f", [0.0, -0.1, 1.5, float("nan"), True, "0.1"])
def test_bad_fraction(f):
    with pytest.raises(ValueError, match="label_fraction"):
        F.label_subset(_samples([4]), 1, label_fraction=f)


@pytest.mark.parametrize("n,n_lab", [(50, 6), (1000, 10), (200000, 2000), (12, 11)])
def test_holdout(n, n_lab):
    labelled = np.sort(np.random.default_rng(0).permutation(n)[:n_lab])
    h = F.holdout_indices(n, labelled, seed=4)
    m = n - n_lab
    assert h.size == max(1, min(10000, m // 10))
    assert not set(h.tolist()) & set(labelled.tolist())
    assert np.all(np.diff(h) > 0) and h.min() >= 0 and h.max() < n
    assert np.array_equal(h, F.holdout_indices(n, labelled, seed=4))


def test_holdout_needs_an_unlabelled_image():
    with pytest.raises(ValueError, match="no image is left"):
        F.holdout_indices(5, np.arange(5), seed=0)


# ---- argument validation (nothing here may touch a device) ----
def _loader(n_train, n_test=3, n_valid=None, classes=3, batch=4):
    def split(n):
        return types.SimpleNamespace(samples=[("/d/c%d/img%d.JPEG" % (i % classes, i), i % classes) for i in range(n)],
                                     batch_size=batch, augment=types.SimpleNamespace(R=64), workers=2)
    return types.SimpleNamespace(output_size=classes, train_loader=split(n_train), test_loader=split(n_test),
                                 valid_loader=None if n_valid is None else split(n_valid))


def _model(d=512):
    """Any attribute access beyond base_network_output_size fails: the checks must come first."""
    return types.SimpleNamespace(base_network_output_size=d)


@pytest.mark.parametrize("kw, match", [
    (dict(label_fraction=0.5, lrs=()), "lrs"),
    (dict(label_fraction=0.5, weight_decays=(-1.0,)), "weight_decays"),
    (dict(label_fraction=0.5, momentum=1.0), "momentum"),
    (dict(label_fraction=0.5, epochs=0), "epochs"),
    (dict(label_fraction=0.5, batch_size=0), "batch_size"),
    (dict(label_fraction=0.5, network="both"), "network"),
    (dict(), "exactly one"),
    (dict(label_fraction=0.5, subset=["img1.JPEG"]), "exactly one"),
    (dict(label_fraction=2.0), "label_fraction"),
    (dict(subset=["nope.JPEG"]), "matches no training image"),
    (dict(label_fraction=0.2, batch_size=5), "fill one batch"),            # 4 of 20 labelled
])
def test_finetune_accuracy_rejects_bad_arguments(kw, match):
    with pytest.raises(ValueError, match=match):
        F.finetune_accuracy(_model(), _loader(20), **dict(dict(batch_size=4), **kw))


def test_finetune_accuracy_checks_splits_before_device_work():
    with pytest.raises(ValueError, match="test split is empty"):
        F.finetune_accuracy(_model(), _loader(20, n_test=0), label_fraction=0.5, batch_size=4)
    with pytest.raises(ValueError, match="no image is left"):                 # all labelled, no valid/
        F.finetune_accuracy(_model(), _loader(20), label_fraction=1.0, batch_size=4)
    with pytest.raises(ValueError, match="multiple of 64"):
        F.finetune_accuracy(_model(100), _loader(20), label_fraction=0.5, batch_size=4)
    with pytest.raises(ValueError, match="2 classes"):
        F.finetune_accuracy(_model(), _loader(20, classes=1), label_fraction=0.5, batch_size=4)


def test_valid_split_allows_a_fully_labelled_training_split():
    """With valid/ images nothing is held out, so label_fraction=1 passes the checks and fails only at the model."""
    with pytest.raises(AttributeError):
        F.finetune_accuracy(_model(), _loader(20, n_valid=4), label_fraction=1.0, batch_size=4)


def test_cpu_model_raises_runtime_error():
    import torch
    from byol_b200.model import BYOL
    model = BYOL(512, 64, 3, 10, arch="resnet18", head_latent_size=128)
    with pytest.raises(RuntimeError, match="CUDA"):
        F.FineTune(model, 3, 0.1)
    with pytest.raises(RuntimeError, match="CUDA"):
        F.finetune_accuracy(model, _loader(20), label_fraction=0.5, batch_size=4)
    with pytest.raises(ValueError, match="num_classes"):
        F.FineTune(model, 1, 0.1)
    with pytest.raises(ValueError, match="lrs"):
        F.FineTune(model, 3, -0.1)
    del torch


# ---- the lane-aware planner ----
def _engine(arch):
    from byol_b200.model import BYOL
    eng = BYOL(2048, 256, 1000, 10, arch=arch)._engine
    eng.walk_layers()
    return eng


def _old_need(eng, mm, plan):
    """The two-lane BYOL step's need, written out as before the planner took lanes."""
    blocks = mm["blocks"]
    saved = 2 * eng.lane_bytes(mm, plan)
    fwd = saved + 2 * max(blk["stored"] for blk in blocks)
    bwd = saved + sum(blk["dy"] for i, blk in enumerate(blocks) if i not in plan) + \
        max(blk["work"] + (blk["stored"] - blk["kept"] if i in plan else 0) for i, blk in enumerate(blocks))
    return int(eng.RESERVE_FACTOR * (max(fwd, bwd) + mm["fixed"])) + eng.MARGIN


@pytest.mark.parametrize("arch,n,r", [("resnet50", 512, 224), ("resnet:basic:2,2,2,2", 256, 160)])
def test_planner_defaults_are_the_byol_step(arch, n, r):
    eng = _engine(arch)
    mm = eng.memory_model(n, r, r)
    assert mm == eng.memory_model(n, r, r, lanes=2, target=True, mlps=True)
    first_block = eng.memory_model(n, r, r)["blocks"]
    e0 = n * (r // 2) * (r // 2) * 64
    mlp = sum(2 * n * (l1.cin + 2 * l1.cout) for l1, _ in eng.mlps)
    assert mm["fixed"] == 2 * (2 * e0 + mm["first_input"] // 2 + mlp) + 2 * (2 * n * r * r * 8)
    for plan in (frozenset(), frozenset([0, 2]), frozenset(range(len(first_block)))):
        assert eng.step_need(mm, plan) == _old_need(eng, mm, plan)


def test_planner_one_lane_without_target_or_mlps():
    eng = _engine("resnet50")
    n, r = 1024, 224
    two = eng.memory_model(n, r, r)
    one = eng.memory_model(n, r, r, lanes=1, target=False, mlps=False)
    assert one["blocks"] == two["blocks"] and one["first_input"] == two["first_input"]
    e0 = n * (r // 2) * (r // 2) * 64
    assert one["fixed"] == 2 * e0 + one["first_input"] // 2 + 2 * n * r * r * 8
    for plan in (frozenset(), frozenset(range(len(one["blocks"])))):
        blocks = one["blocks"]
        saved = eng.lane_bytes(one, plan)                       # one lane's saved bytes, no target term
        bwd = saved + sum(b["dy"] for i, b in enumerate(blocks) if i not in plan) + \
            max(b["work"] + (b["stored"] - b["kept"] if i in plan else 0) for i, b in enumerate(blocks))
        assert eng.step_need(one, plan) == int(eng.RESERVE_FACTOR * (bwd + one["fixed"])) + eng.MARGIN
        assert eng.step_need(one, plan) < eng.step_need(two, plan)
    # a budget that the stored one-lane step fits but the two-lane step does not
    budget = eng.step_need(one, frozenset())
    eng._mem_budget = budget
    assert eng.recompute_plan(n, r, r, 1, False, False) == frozenset()
    assert eng.recompute_plan(n, r, r) != frozenset()
