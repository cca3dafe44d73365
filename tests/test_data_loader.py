"""CPU: byol_b200.data's image-folder listing, counts, sharding, per-epoch order and argument checks (no decoding)."""
import os

import numpy as np
import pytest

from tests.image_folder import CLASSES, loader_kwargs, make_image_folder


@pytest.fixture
def folder(tmp_path):
    made = make_image_folder(tmp_path, seed=11)
    return tmp_path, made


def test_classes_and_global_counts(folder):
    from byol_b200.data import get_loader
    root, made = folder
    ld = get_loader(**loader_kwargs(root))
    assert ld.classes == CLASSES and ld.output_size == 3 and ld.input_shape == [3, 64, 64]
    train = sorted((os.path.relpath(p, root), c) for p, c in ld.train_loader.samples)
    assert train == sorted((rel, c) for rel, (c, _) in made.items() if rel.startswith("train"))
    assert ld.num_train_samples == 12 and ld.num_test_samples == 5 and ld.num_valid_samples == 0
    assert ld.valid_loader is None
    os.makedirs(os.path.join(root, "valid", CLASSES[0]))
    os.rename(os.path.join(root, "test", CLASSES[0], "t0.JPEG"), os.path.join(root, "valid", CLASSES[0], "v.JPEG"))
    ld = get_loader(**loader_kwargs(root))
    assert ld.num_valid_samples == 1 and ld.num_test_samples == 4 and len(ld.valid_loader) == 1


@pytest.mark.parametrize("replicas,batch", [(1, 4), (2, 2), (3, 1), (2, 5), (5, 2)])
def test_shards_are_disjoint_and_cover(folder, replicas, batch):
    from byol_b200.data import get_loader
    root, _ = folder
    parts = []
    for rank in range(replicas):
        ld = get_loader(**loader_kwargs(root, num_replicas=replicas, distributed_rank=rank, batch_size=batch))
        ld.set_all_epochs(3)
        tl = ld.train_loader
        # main.py:421-424: num_train_samples // num_replicas, then // batch_size steps per epoch
        assert len(tl) == ld.num_train_samples // replicas // batch
        idx = tl.indices()
        assert len(idx) == len(tl) * batch
        parts.append(idx)
    flat = np.concatenate(parts)
    assert len(set(flat.tolist())) == len(flat)                          # disjoint
    per = 12 // replicas
    if per % batch == 0:                                                 # no per-rank remainder: all of the shard
        perm = np.random.default_rng([5, 3]).permutation(12)
        assert sorted(flat.tolist()) == sorted(perm[:replicas * per].tolist())
    # the test split: every image, in order, on every rank; the last batch may be short
    assert ld.test_loader.indices().tolist() == list(range(5))
    assert len(ld.test_loader) == (5 + batch - 1) // batch


def test_covering_without_remainder(folder):
    """12 images over 3 ranks of batch 2: the ranks' epochs together are a permutation of the whole split."""
    from byol_b200.data import get_loader
    root, _ = folder
    idx = []
    for rank in range(3):
        ld = get_loader(**loader_kwargs(root, num_replicas=3, distributed_rank=rank, batch_size=2))
        idx += ld.train_loader.indices().tolist()
    assert sorted(idx) == list(range(12))


def test_epoch_order(folder):
    from byol_b200.data import get_loader
    root, _ = folder
    a = get_loader(**loader_kwargs(root)).train_loader
    b = get_loader(**loader_kwargs(root)).train_loader
    a.set_epoch(4)
    b.set_epoch(4)
    assert np.array_equal(a.indices(), b.indices())
    first = a.indices()
    a.set_epoch(5)
    assert not np.array_equal(a.indices(), first)
    c = get_loader(**loader_kwargs(root, seed=6)).train_loader
    c.set_epoch(4)
    assert not np.array_equal(c.indices(), first)


def test_gpu_decoder_routing(folder):
    """3-component JPEGs go to nvJPEG; the grayscale JPEG and the PNG named .JPEG are decoded on the host."""
    from byol_b200.data import _nvjpeg_decodable, _read
    root, made = folder
    for rel, (_, kind) in made.items():
        assert _nvjpeg_decodable(_read(os.path.join(root, rel))) == (kind == "rgb"), rel
    assert not _nvjpeg_decodable(bytearray(b"\xff\xd8"))


def test_rejected_tasks_and_directories(folder, tmp_path_factory):
    from byol_b200.data import get_loader
    root, _ = folder
    for task in ("dali_multi_augment_image_folder", "multi_augment_dali_image_folder", "cifar10", "image_folder"):
        with pytest.raises(ValueError, match="task"):
            get_loader(**loader_kwargs(root, task=task))
    with pytest.raises(FileNotFoundError, match="does not exist"):
        get_loader(**loader_kwargs(os.path.join(root, "missing")))
    empty = tmp_path_factory.mktemp("no_test_split")
    os.makedirs(os.path.join(empty, "train", "x"))
    with pytest.raises(FileNotFoundError, match="test/"):
        get_loader(**loader_kwargs(empty))
    with pytest.raises(ValueError, match="cannot fill one batch"):
        get_loader(**loader_kwargs(root, batch_size=7, num_replicas=2))
