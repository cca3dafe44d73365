"""CPU: argument checks of the k-NN evaluation (byol_b200.knn, BYOL.representations) and the float64 oracle the GPU
tests compare against (tests/knn_oracle.py)."""
import numpy as np
import pytest
import torch

from tests import knn_oracle as O


def _args(n=10, q=3, d=64, dtype=torch.bfloat16):
    return torch.zeros(n, d, dtype=dtype), torch.zeros(n, dtype=torch.int64), torch.zeros(q, d, dtype=dtype)


@pytest.mark.parametrize("k", [0, 257, -1, 2.0, True])
def test_k_out_of_range(k):
    from byol_b200.knn import knn_classify
    b, l, q = _args()
    with pytest.raises(ValueError, match="k must be"):
        knn_classify(b, l, q, 10, k=k)


@pytest.mark.parametrize("kw, match", [
    (dict(num_classes=0), "num_classes"),
    (dict(temperature=0.0), "temperature"),
    (dict(temperature=float("inf")), "temperature"),
    (dict(query_chunk=0), "query_chunk"),
    (dict(bank_chunk=-5), "bank_chunk"),
])
def test_bad_scalars(kw, match):
    from byol_b200.knn import knn_classify
    b, l, q = _args()
    args = dict(num_classes=10)
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        knn_classify(b, l, q, **args)


def test_bad_shapes_and_dtypes():
    from byol_b200.knn import knn_classify
    b, l, q = _args(d=96)
    with pytest.raises(ValueError, match="multiple of 64"):
        knn_classify(b, l, q, 10)
    b, l, q = _args()
    with pytest.raises(ValueError, match="differ in width"):
        knn_classify(b, l, torch.zeros(3, 128, dtype=torch.bfloat16), 10)
    with pytest.raises(ValueError, match="bf16 or fp32"):
        knn_classify(b.half(), l, q, 10)
    with pytest.raises(ValueError, match="bank_labels"):
        knn_classify(b, l.int(), q, 10)
    with pytest.raises(ValueError, match="bank_labels"):
        knn_classify(b, l[:5], q, 10)
    with pytest.raises(TypeError):
        knn_classify([1, 2], l, q, 10)


def test_cpu_tensors_raise_runtime_error():
    from byol_b200 import knn
    b, l, q = _args()
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.knn_classify(b, l, q, 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.knn_classify(b.float(), l, q.float(), 10)
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.l2_normalize_rows(torch.zeros(4, 64))
    vals, idx = torch.zeros(3, 5), torch.zeros(3, 5, dtype=torch.int32)
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.topk_update(torch.zeros(3, 7), 0, vals, idx, False)
    with pytest.raises(RuntimeError, match="CUDA"):
        knn.vote(vals, idx, l, 10)


def test_representations_arguments():
    from byol_b200.model import BYOL
    m = BYOL(512, 64, 10, 10, arch="resnet18", head_latent_size=64)
    with pytest.raises(ValueError, match="network"):
        m.representations(torch.zeros(1, 3, 32, 32), network="ema")
    with pytest.raises(RuntimeError, match="CUDA"):
        m.representations(torch.zeros(1, 3, 32, 32))


def test_knn_accuracy_arguments():
    from byol_b200.knn import knn_accuracy
    with pytest.raises(ValueError, match="k must be"):
        knn_accuracy(None, None, k=300)
    with pytest.raises(ValueError, match="network"):
        knn_accuracy(None, None, network="both")
    with pytest.raises(ValueError, match="temperature"):
        knn_accuracy(None, None, temperature=-1.0)


# ---- the oracle ----
def test_oracle_topk_order_and_ties():
    sim = np.array([[0.5, 0.9, 0.5, -0.0, 0.0, 0.9]], dtype=np.float32)
    vals, idx = O.topk(sim, 6, n0=10)
    assert idx.tolist() == [[11, 15, 10, 12, 13, 14]]    # ties: lower bank index first; -0 == +0
    assert vals[0, :2].tolist() == [np.float32(0.9)] * 2


def test_oracle_topk_is_chunk_independent():
    rng = np.random.default_rng(0)
    sim = rng.integers(-4, 5, size=(7, 300)).astype(np.float32) / 4      # many ties
    k = 20
    full_v, full_i = O.topk(sim, k)
    for chunk in (1, 17, 64, 300):
        run_v, run_i = None, None
        for n0 in range(0, 300, chunk):
            v, i = O.topk(sim[:, n0:n0 + chunk], k, n0)
            if run_v is not None:
                v, i = np.concatenate([run_v, v], 1), np.concatenate([run_i, i], 1)
                order = [np.lexsort((i[r], -v[r].astype(np.float64)))[:k] for r in range(7)]
                v = np.stack([v[r, o] for r, o in enumerate(order)])
                i = np.stack([i[r, o] for r, o in enumerate(order)])
            run_v, run_i = v, i
        assert np.array_equal(run_v, full_v) and np.array_equal(run_i, full_i), chunk


def test_oracle_vote():
    labels = np.array([2, 0, 2, 1, 0])
    vals = np.array([[0.7, 0.7, 0.1, -1.0]], dtype=np.float32)
    idx = np.array([[1, 4, 2, -1]])                 # classes 0, 0, 2, empty slot
    T = 0.07
    s = O.class_scores(vals, idx, labels, 4, T)
    w = O.weights(vals, T)
    assert s[0, 0] == w[0, 0] + w[0, 1] and s[0, 2] == w[0, 2] and s[0, 1] == 0 and s[0, 3] == 0
    assert O.rank_classes(s).tolist() == [[0, 2, 1, 3]]              # zero scores: class index order
    assert O.rank_classes(np.array([[1.0, 2.0, 2.0, 0.5, 3.0, 0.0]])).tolist() == [[4, 1, 2, 0, 3]]


def test_oracle_weights_round_the_quotient_to_fp32():
    s = np.float32(0.123456789)
    assert O.weights(np.array([s]), 0.07)[0] == np.exp(np.float64(s / np.float32(0.07)))
