"""GPU: k-NN evaluation (byol_b200.knn over csrc/knn.cu) and the encoder-only forward BYOL.representations.

* byol_knn_topk returns exactly the float64 oracle's neighbours (indices and similarity bits) on random fp32
  similarity matrices with ragged shapes and many ties, for every chunking, run after run.
* knn_search's neighbours are as good as fp32 accumulation of the bf16 features allows, and exactly the oracle's
  where the similarities are exact; the vote's scores match the oracle's given the GPU's neighbours.
* representations is the eval forward's representation bit for bit, close to torch's fp32 encoder, and leaves
  training (graphed steps, running statistics, EMA) untouched.
"""
import copy

import numpy as np
import pytest
import torch

from tests import knn_oracle as O
from tests.image_folder import loader_kwargs, make_image_folder
from tests.util import assert_close

pytestmark = pytest.mark.gpu


def _bits(x):
    return np.ascontiguousarray(np.asarray(x, dtype=np.float32)).view(np.int32)


def _run_topk(sim, k, chunk):
    from byol_b200.knn import topk_update
    q, n = sim.shape
    vals = torch.empty((q, k), dtype=torch.float32, device=sim.device)
    idx = torch.empty((q, k), dtype=torch.int32, device=sim.device)
    for n0 in range(0, n, chunk):
        topk_update(sim[:, n0:n0 + chunk].contiguous(), n0, vals, idx, merge=n0 > 0)
    torch.cuda.synchronize()
    return vals.cpu().numpy(), idx.cpu().numpy()


def _expect(sim_np, k):
    """Oracle lists padded to k slots as the kernel leaves them (-inf / -1); -0 reads as +0."""
    v, i = O.topk(sim_np, k)
    q, m = v.shape
    vals = np.full((q, k), -np.inf, dtype=np.float32)
    idx = np.full((q, k), -1, dtype=np.int64)
    vals[:, :m] = v + np.float32(0.0)
    idx[:, :m] = i
    return vals, idx


@pytest.mark.parametrize("kind", ["random", "ties", "constant"])
@pytest.mark.parametrize("k", [1, 20, 200])
def test_topk_selection_is_exact(cuda, kind, k):
    rng = np.random.default_rng(k)
    q, n = 37, 5003
    if kind == "random":
        sim = rng.standard_normal((q, n)).astype(np.float32)
    elif kind == "ties":       # a handful of values (signed zeros included): ties everywhere, broken by bank index
        sim = rng.choice(np.array([-0.5, -0.0, 0.0, 0.25, 0.5, 0.75, 1.0], dtype=np.float32), size=(q, n))
    else:                      # one value: the radix selection runs down to the index digits
        sim = np.full((q, n), 0.375, dtype=np.float32)
    ev, ei = _expect(sim, k)
    g = torch.from_numpy(sim).to(cuda)
    first = None
    for chunk in (n, 4096, 1000, 257, 64):       # 64 < k = 200: the list is mostly the earlier chunks'
        v, i = _run_topk(g, k, chunk)
        assert np.array_equal(i, ei), (kind, k, chunk, np.argwhere(i != ei)[:5])
        assert np.array_equal(_bits(v), _bits(ev)), (kind, k, chunk)
        if first is None:
            first = (v, i)
        assert np.array_equal(_bits(v), _bits(first[0])) and np.array_equal(i, first[1])
    v2, i2 = _run_topk(g, k, 257)
    assert np.array_equal(_bits(v2), _bits(first[0])) and np.array_equal(i2, first[1])


def test_topk_short_bank_and_padded_rows(cuda):
    """Fewer bank rows than k leave -inf / -1 slots; columns past Nc of a pitched chunk are never read."""
    from byol_b200 import ops
    from byol_b200._lib import check, lib
    rng = np.random.default_rng(5)
    q, n, k, ld = 9, 13, 20, 32
    sim = rng.standard_normal((q, ld)).astype(np.float32)
    sim[:, n:] = 1e30                                   # padding that must not enter
    g = torch.from_numpy(sim).to(cuda)
    vals = torch.empty((q, k), dtype=torch.float32, device=cuda)
    idx = torch.empty((q, k), dtype=torch.int32, device=cuda)
    check(lib.byol_knn_topk(g.data_ptr(), q, n, ld, 100, k, 0, vals.data_ptr(), idx.data_ptr(), ops._stream()),
          "byol_knn_topk")
    ev, ei = _expect(sim[:, :n], k)
    ei[ei >= 0] += 100
    assert np.array_equal(idx.cpu().numpy(), ei)
    assert np.array_equal(_bits(vals.cpu().numpy()), _bits(ev))


def test_l2_normalize_rows(cuda):
    from byol_b200.knn import l2_normalize_rows
    rng = np.random.default_rng(1)
    x = rng.standard_normal((300, 2048)).astype(np.float32) * rng.uniform(0.01, 100, (300, 1)).astype(np.float32)
    x[7] = 0.0
    g = torch.from_numpy(x).to(cuda)
    y = l2_normalize_rows(g)
    y2 = l2_normalize_rows(g)
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16))
    got = y.float().cpu().numpy().astype(np.float64)
    assert not got[7].any()
    ref = x.astype(np.float64) / np.maximum(np.linalg.norm(x.astype(np.float64), axis=1, keepdims=True), 1e-300)
    err = np.abs(got - ref)
    assert (err <= 2.0 ** -8 * np.abs(ref) + 1e-30).all(), float(err.max())   # within one bf16 rounding
    assert np.abs(np.linalg.norm(got, axis=1)[np.arange(300) != 7] - 1).max() < 1e-2


def _features(rng, rows, d, cuda):
    from byol_b200.knn import l2_normalize_rows
    return l2_normalize_rows(torch.from_numpy(rng.standard_normal((rows, d)).astype(np.float32)).to(cuda))


@pytest.mark.parametrize("chunks", [(None, None), (64, 1000), (300, 777)])
def test_search_within_fp32_accumulation_bound(cuda, chunks):
    from byol_b200.knn import knn_search
    rng = np.random.default_rng(2)
    n, q, d, k = 6001, 301, 256, 20
    bank, queries = _features(rng, n, d, cuda), _features(rng, q, d, cuda)
    vals, idx = knn_search(bank, queries, k, query_chunk=chunks[0], bank_chunk=chunks[1])
    vals, idx = vals.cpu().numpy(), idx.cpu().numpy().astype(np.int64)
    b64, q64 = bank.float().cpu().numpy().astype(np.float64), queries.float().cpu().numpy().astype(np.float64)
    s64 = q64 @ b64.T
    bound = d * 2.0 ** -23 * (np.abs(q64) @ np.abs(b64).T).max()
    kth = np.sort(s64, axis=1)[:, -k]
    got = np.take_along_axis(s64, idx, 1)
    assert (got >= kth[:, None] - bound).all(), float((kth[:, None] - got).max())
    assert np.abs(vals - got).max() <= bound
    assert (np.diff(vals, axis=1) <= 0).all()
    v0, i0 = knn_search(bank, queries, k)
    assert np.array_equal(i0.cpu().numpy(), idx) and np.array_equal(_bits(v0.cpu().numpy()), _bits(vals))


def test_search_exact_on_exact_similarities(cuda):
    """Unit rows of +-1/8 on 64 of 128 dimensions: every similarity is a multiple of 1/64 and exact in fp32 in any
    summation order, so the GPU must return the oracle's lists exactly, ties included."""
    from byol_b200.knn import knn_search
    rng = np.random.default_rng(3)

    def rows(m):
        x = np.zeros((m, 128), dtype=np.float32)
        for r in range(m):
            x[r, rng.choice(128, 64, replace=False)] = rng.choice([-0.125, 0.125], 64)
        return x

    bank, queries = rows(3000), rows(200)
    for k in (1, 20, 200):
        vals, idx = knn_search(torch.from_numpy(bank).to(cuda).bfloat16(), torch.from_numpy(queries).to(cuda).bfloat16(),
                               k, bank_chunk=1024)
        ev, ei = _expect(queries.astype(np.float64) @ bank.astype(np.float64).T, k)
        assert np.array_equal(idx.cpu().numpy(), ei), k
        assert np.array_equal(vals.cpu().numpy(), ev.astype(np.float32)), k


@pytest.mark.parametrize("classes", [3, 10, 1000])
@pytest.mark.parametrize("k", [1, 20, 200])
def test_vote_matches_oracle(cuda, classes, k):
    from byol_b200.knn import knn_search, vote
    rng = np.random.default_rng(classes + k)
    n, q, d = 4000, 257, 128
    bank, queries = _features(rng, n, d, cuda), _features(rng, q, d, cuda)
    labels = torch.from_numpy(rng.integers(0, classes, n)).to(cuda)
    vals, idx = knn_search(bank, queries, k)
    pred, scores = vote(vals, idx, labels, classes, 0.07, want_scores=True)
    pred, scores = pred.cpu().numpy(), scores.cpu().numpy().astype(np.float64)
    ref = O.class_scores(vals.cpu().numpy(), idx.cpu().numpy(), labels.cpu().numpy(), classes, 0.07)
    top = O.rank_classes(ref)
    m = top.shape[1]
    assert (pred[:, m:] == -1).all()
    got_ref = np.take_along_axis(ref, pred[:, :m].astype(np.int64), 1)
    rel = np.abs(scores[:, :m] - got_ref) / np.maximum(got_ref, 1e-300)
    assert (np.abs(scores[:, :m] - got_ref) <= 1e-6 * got_ref).all(), float(rel.max())
    top_s = np.take_along_axis(ref, top, 1)
    for r in np.argwhere((pred[:, :m] != top).any(1)).ravel():
        # a different order only among classes whose oracle scores are within 1e-5 relative of each other
        assert np.allclose(got_ref[r], top_s[r], rtol=1e-5, atol=0), (r, pred[r], top[r], got_ref[r], top_s[r])


def test_classify_end_to_end_against_oracle(cuda):
    from byol_b200.knn import knn_classify
    rng = np.random.default_rng(4)
    n, q, d, classes = 2000, 100, 64, 7
    bank = torch.from_numpy(rng.standard_normal((n, d)).astype(np.float32)).to(cuda)
    queries = torch.from_numpy(rng.standard_normal((q, d)).astype(np.float32)).to(cuda)
    labels = torch.from_numpy(rng.integers(0, classes, n)).to(cuda)
    pred = knn_classify(bank, labels, queries, classes, k=20).cpu().numpy()
    pred2 = knn_classify(bank, labels, queries, classes, k=20, query_chunk=33, bank_chunk=300).cpu().numpy()
    assert np.array_equal(pred, pred2)
    from byol_b200.knn import l2_normalize_rows
    b64 = l2_normalize_rows(bank).float().cpu().numpy().astype(np.float64)
    q64 = l2_normalize_rows(queries).float().cpu().numpy().astype(np.float64)
    ref = O.classify(q64 @ b64.T, labels.cpu().numpy(), classes, 20, 0.07)
    assert (pred[:, 0] == ref[:, 0]).mean() > 0.95


def test_classify_validates_on_device(cuda):
    from byol_b200.knn import knn_classify
    b = torch.zeros(10, 64, dtype=torch.bfloat16, device=cuda)
    with pytest.raises(ValueError, match="labels span"):
        knn_classify(b, torch.full((10,), 5, dtype=torch.int64, device=cuda), b[:2], 5)
    with pytest.raises(ValueError, match="labels span"):
        knn_classify(b, torch.full((10,), -1, dtype=torch.int64, device=cuda), b[:2], 5)


# ---- representations ----
def _model(arch, precision, cuda, rep=512):
    from byol_b200.model import BYOL
    torch.manual_seed(8)
    model = BYOL(rep, 64, 10, 10, arch=arch, head_latent_size=128, precision=precision)
    g = torch.Generator().manual_seed(9)
    with torch.no_grad():              # non-trivial BatchNorm: eval mode reads these
        for m in model.base_network.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.running_mean.copy_(torch.randn(m.num_features, generator=g) * 0.1)
                m.running_var.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.weight.copy_(torch.rand(m.num_features, generator=g) + 0.5)
                m.bias.copy_(torch.randn(m.num_features, generator=g) * 0.1)
        model.target_network.mean.copy_(torch.nn.utils.parameters_to_vector(model.parameters()) * 0.9)
    return model.cuda()


@pytest.mark.parametrize("arch, precision, rep", [("resnet18", "bf16", 512), ("resnet18", "fp32", 512),
                                                  ("resnext:32x4:1,1,1,1", "bf16", 2048)])
def test_representations_equal_eval_forward(cuda, arch, precision, rep):
    model = _model(arch, precision, cuda, rep)
    g = torch.Generator().manual_seed(10)
    x = torch.rand(6, 3, 64, 64, generator=g).to(cuda)
    model.train()                      # representations runs eval BatchNorm whatever the module mode
    online, target = model.representations(x), model.representations(x, network="target")
    assert online.dtype == torch.float32 and online.shape == (6, rep) and not online.requires_grad
    model.eval()
    with torch.no_grad():
        out = model(x, x)
    assert torch.equal(online, out["online_representation1"])
    assert torch.equal(target, out["target_representation1"])
    assert not torch.equal(online, target)
    if precision == "fp32":
        net = copy.deepcopy(model.base_network).cpu().eval()
        with torch.no_grad():
            ref = net(x.cpu()).flatten(1)
        assert_close("representations vs torch fp32", online, ref, atol=1e-3 * float(ref.abs().max()), rtol=1e-3)


def _bn_state(model):
    return [t.clone() for n, t in model.state_dict().items() if "running_" in n or "num_batches" in n]


def _step(model, opt, a1, a2, lab, hook=None):
    from byol_b200.objective import cross_entropy_topk, loss_function
    out = model(a1, a2)
    loss = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                         target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
    loss = loss + cross_entropy_topk(out["linear_preds"], lab)[0]
    if hook is not None:
        hook()
    opt.zero_grad()
    loss.backward()
    opt.step()
    return loss.detach().clone()


def test_training_is_undisturbed(cuda, tmp_path):
    """Graphed training steps give the same bits with representations / knn_accuracy calls between steps and between
    a step's forward and backward; the calls change no running statistic, num_batches_tracked or EMA step."""
    from byol_b200 import wiring
    from byol_b200.data import get_loader
    from byol_b200.knn import knn_accuracy
    from byol_b200.model import BYOL
    make_image_folder(tmp_path, seed=2)
    loader = get_loader(**loader_kwargs(tmp_path))
    arch, b, r = "resnet:bottleneck:1,1,1,1", 8, 64
    g = torch.Generator().manual_seed(3)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 10, (b,), generator=g).cuda()) for _ in range(4)]
    probe = torch.rand(5, 3, 48, 48, generator=g).cuda()
    res = {}
    for mode in ("plain", "probed"):
        torch.manual_seed(11)
        model = BYOL(2048, 64, 10, 20, arch=arch, head_latent_size=128).cuda().train()
        opt = wiring.build_optimizer(model, global_batch_size=256)
        calls = []

        def probe_calls():
            before, step = _bn_state(model), model.target_network.step
            calls.append((model.representations(probe).clone(), model.representations(probe, "target").clone()))
            acc = knn_accuracy(model, loader, k=3)
            assert 0.0 <= acc["knn_top1"] <= acc["knn_top5"] <= 100.0
            after = _bn_state(model)
            assert all(torch.equal(x, y) for x, y in zip(before, after)) and model.target_network.step == step

        hook = probe_calls if mode == "probed" else None
        losses = []
        for bt in batches:
            losses.append(_step(model, opt, *bt, hook=hook))
            if hook is not None:
                hook()
        torch.cuda.synchronize()
        assert len([v for v in model._engine.graphs.values() if v != "warm"]) == 1     # steps 2-4 were graphed
        res[mode] = {"loss": torch.stack(losses), "theta": model._engine.theta.clone(),
                     "target": model.target_network.mean.clone(), "bn": _bn_state(model),
                     "step": model.target_network.step}
        model = opt = None
    for key in ("loss", "theta", "target"):
        assert torch.equal(res["plain"][key], res["probed"][key]), key
    assert all(torch.equal(x, y) for x, y in zip(res["plain"]["bn"], res["probed"]["bn"]))
    assert res["plain"]["step"] == res["probed"]["step"]


def test_knn_accuracy_finds_each_image_itself(cuda, tmp_path):
    """With the test split pointed at the training images, each query's nearest neighbour is its own bank entry."""
    from byol_b200.data import ImageFolderLoader, get_loader
    from byol_b200.knn import knn_accuracy
    from byol_b200.model import BYOL
    make_image_folder(tmp_path, seed=4)
    loader = get_loader(**loader_kwargs(tmp_path))
    loader.test_loader = ImageFolderLoader(loader.train_loader.samples, 4, loader.test_loader.augment, train=False)
    torch.manual_seed(12)
    model = BYOL(512, 64, loader.output_size, 10, arch="resnet18", head_latent_size=128)
    with torch.no_grad():              # the EMA weights at construction are 0.004 x theta: give them the online ones
        model.target_network.mean.copy_(torch.nn.utils.parameters_to_vector(model.parameters()))
    model = model.cuda()
    for network in ("online", "target"):
        acc = knn_accuracy(model, loader, k=1, network=network)
        assert acc == {"knn_top1": 100.0, "knn_top5": 100.0}, (network, acc)
    acc = knn_accuracy(model, loader, k=20, batch_size=3)
    assert 0.0 <= acc["knn_top1"] <= acc["knn_top5"] <= 100.0
