"""GPU: linear evaluation (byol_b200.linear_eval over csrc/linear_eval.cu).

* byol_linprobe_ce matches float64 on random, tie-heavy and non-finite logits of 1, 3 and 25 heads of 2, 10 and 1000
  classes: loss sums within fp32 rounding, hit counts exactly (a NaN is never a hit), the bf16 gradient within one
  bf16 ulp, padding exactly 0, and the same bits on every launch; rows labelled outside [0, C) count for nothing.
* byol_linprobe_sgd is bit-exact against the fp32 restatement of its operation order over 20 steps, and close to
  torch.optim.SGD(nesterov=True).
* A whole step matches tests/linear_oracle.py within the fp32 accumulation bound, and a head's logits do not depend
  on the heads sharing its GEMM.
* Non-finite features score no hit, a diverged head is never selected, and training on non-finite features raises.
* Training on cached features separates Gaussian clusters and is reproducible; linear_accuracy runs both modes on an
  image folder, reuses the test transform's features bit for bit, and leaves graphed training untouched.
"""
import numpy as np
import pytest
import torch

from tests import linear_oracle as O
from tests.image_folder import loader_kwargs, make_image_folder

pytestmark = pytest.mark.gpu


def _bits(t):
    return t.contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16).cpu()


def _bf16_ulp(x):
    a = np.abs(np.asarray(x, dtype=np.float64))
    return np.where(a > 0, 2.0 ** (np.floor(np.log2(np.maximum(a, 1e-300))) - 7), 2.0 ** -133)


# ---- the cross-entropy kernel ----
@pytest.mark.parametrize("kind", ["random", "ties", "nonfinite"])
@pytest.mark.parametrize("classes", [2, 10, 1000])
@pytest.mark.parametrize("heads", [1, 3, 25])
def test_ce_kernel_against_fp64(cuda, heads, classes, kind):
    from byol_b200.linear_eval import multihead_ce
    rng = np.random.default_rng(heads * 1000 + classes)
    b, cp = 67, O.padded(classes)
    ld = heads * cp + 8                                  # pitched rows
    labels = rng.integers(0, classes, b)
    if kind != "ties":
        z = (rng.standard_normal((b, ld)) * 3).astype(np.float32)
    else:                                                # few values: ties everywhere, also with the label
        z = rng.integers(-2, 3, size=(b, ld)).astype(np.float32)
    bad = np.zeros(b, dtype=bool)                        # rows holding a non-finite logit
    if kind == "nonfinite":                              # diverged features / weights: no NaN may count as a hit
        other = (labels + 1) % classes
        for h in range(heads):
            z[0, h * cp:(h + 1) * cp] = np.nan                          # the whole row
            z[1, h * cp + labels[1]] = np.nan                           # the label's logit only
            z[2, h * cp + other[2]] = np.nan                            # another column
            z[3, h * cp + labels[3]] = np.inf
            z[4, h * cp + other[4]] = -np.inf
            z[5, h * cp + other[5]] = np.inf
        bad[:6] = True
    for h in range(heads):                               # padding columns must never enter
        z[:, h * cp + classes:(h + 1) * cp] = 1e30
    z[:, heads * cp:] = np.nan
    lg = torch.from_numpy(z).to(cuda)
    lab = torch.from_numpy(labels).to(cuda)

    def run():
        dl = torch.full((b, heads * cp), 7.0, dtype=torch.bfloat16, device=cuda)
        loss = torch.zeros(heads, dtype=torch.float32, device=cuda)
        hits = torch.zeros((heads, 2), dtype=torch.int64, device=cuda)
        multihead_ce(lg, lab, heads, classes, dlogits=dl, loss_sum=loss, hits=hits)
        torch.cuda.synchronize()
        return dl, loss, hits

    dl, loss, hits = run()
    zm = z.astype(np.float64)
    for h in range(heads):
        zm[:, h * cp + classes:(h + 1) * cp] = 0.0
    ref_loss, rank, ref_grad = O.cross_entropy(zm, labels, heads, classes)
    got_loss = loss.cpu().numpy().astype(np.float64)
    if kind == "nonfinite":
        assert np.isnan(got_loss).all()                  # a NaN row makes every head's loss NaN: divergence shows
        assert (rank[:2] == O.MISS).all() and (rank[2] >= 1).all()
    else:
        tol = 1e-6 * (np.abs(ref_loss) + 1).sum(0)
        assert (np.abs(got_loss - ref_loss.sum(0)) <= tol).all(), (got_loss, ref_loss.sum(0))
    assert np.array_equal(hits.cpu().numpy(), np.stack([(rank < 1).sum(0), (rank < 5).sum(0)], 1))
    g = dl.float().cpu().numpy().astype(np.float64).reshape(b, heads, cp)[~bad]
    rg = ref_grad.reshape(b, heads, cp)[~bad]
    assert (g[:, :, classes:] == 0).all() and not np.signbit(g[:, :, classes:]).any()
    err = np.abs(g[:, :, :classes] - rg[:, :, :classes])
    assert (err <= _bf16_ulp(rg[:, :, :classes])).all(), float((err / _bf16_ulp(rg[:, :, :classes])).max())
    dl2, loss2, hits2 = run()
    assert torch.equal(_bits(dl), _bits(dl2)) and torch.equal(_bits(loss), _bits(loss2)) and torch.equal(hits, hits2)


def test_ce_kernel_ignores_rows_with_out_of_range_labels(cuda):
    """A label outside [0, C) is never used as an index: its row adds no loss and no hit and gets a zero gradient."""
    from byol_b200.linear_eval import multihead_ce
    rng = np.random.default_rng(8)
    b, h, c = 40, 2, 10
    cp = O.padded(c)
    z = (rng.standard_normal((b, h * cp)) * 2).astype(np.float32)
    labels = rng.integers(0, c, b)
    labels[[3, 7, 11, 12]] = [-1, c, 2 ** 40, -(2 ** 40)]
    dl = torch.full((b, h * cp), 7.0, dtype=torch.bfloat16, device=cuda)
    loss = torch.zeros(h, dtype=torch.float32, device=cuda)
    hits = torch.zeros((h, 2), dtype=torch.int64, device=cuda)
    multihead_ce(torch.from_numpy(z).to(cuda), torch.from_numpy(labels).to(cuda), h, c, dlogits=dl, loss_sum=loss,
                 hits=hits)
    ref_loss, rank, ref_grad = O.cross_entropy(z, labels, h, c)
    assert (rank[[3, 7, 11, 12]] == O.MISS).all()
    assert np.array_equal(hits.cpu().numpy(), np.stack([(rank < 1).sum(0), (rank < 5).sum(0)], 1))
    assert np.allclose(loss.cpu().numpy(), ref_loss.sum(0), rtol=1e-6, atol=1e-5)
    g = dl.float().cpu().numpy()
    assert not g[[3, 7, 11, 12]].any() and not np.signbit(g[[3, 7, 11, 12]]).any()
    assert (np.abs(g - ref_grad) <= _bf16_ulp(ref_grad)).all()


def test_ce_kernel_accumulates_hits_only(cuda):
    from byol_b200.linear_eval import multihead_ce
    rng = np.random.default_rng(7)
    z = torch.from_numpy(rng.standard_normal((50, 32)).astype(np.float32)).to(cuda)
    lab = torch.from_numpy(rng.integers(0, 10, 50)).to(cuda)
    hits = torch.zeros((2, 2), dtype=torch.int64, device=cuda)
    multihead_ce(z, lab, 2, 10, hits=hits)
    once = hits.clone()
    multihead_ce(z, lab, 2, 10, hits=hits)
    assert torch.equal(hits, 2 * once) and (once[:, 0] <= once[:, 1]).all()


# ---- the update kernel ----
def test_sgd_kernel_bit_exact_over_20_steps(cuda):
    from byol_b200.linear_eval import LinearHeads, cosine_factor
    lrs, wds, mu = (0.4, 0.0, 0.05), (0.0, 1e-3), 0.9
    C, D = 10, 128
    heads = LinearHeads(D, C, lrs, wds, momentum=mu, seed=3, device=cuda)
    H, Cp = heads.H, heads.Cp
    nw = H * Cp * D
    rng = np.random.default_rng(0)
    pad = np.zeros((H, Cp), dtype=bool)
    pad[:, C:] = True
    pad_w = np.repeat(pad[:, :, None], D, 2).reshape(-1)
    pad_all = np.concatenate([pad_w, pad.reshape(-1)])
    # sentinels in the padding rows of every buffer: the kernel must leave them alone
    for t in (heads.params, heads.momentum_buf):
        v = t.cpu().numpy()
        v[pad_all] = rng.standard_normal(int(pad_all.sum())).astype(np.float32)
        t.copy_(torch.from_numpy(v))
    w = heads.params.cpu().numpy().copy()
    buf = heads.momentum_buf.cpu().numpy().copy()
    w_init = w.copy()
    wb_pad = heads.weight_bf16.cpu()[torch.from_numpy(pad.reshape(-1))].clone()
    lr_e = np.array([lr for lr, _ in heads.grid], dtype=np.float32)
    wd_e = np.array([wd for _, wd in heads.grid], dtype=np.float32)
    per = np.concatenate([np.repeat(np.arange(H), Cp * D), np.repeat(np.arange(H), Cp)])
    torch.manual_seed(1)
    tw = [torch.nn.Parameter(torch.from_numpy(w[:nw].reshape(H, Cp, D)[h, :C].copy()).to(cuda)) for h in range(H)]
    tb = [torch.nn.Parameter(torch.from_numpy(w[nw:].reshape(H, Cp)[h, :C].copy()).to(cuda)) for h in range(H)]
    opt = torch.optim.SGD([{"params": [tw[h], tb[h]], "lr": 0.0, "weight_decay": float(wds[h % 2])} for h in range(H)],
                          lr=0.0, momentum=mu, nesterov=True)
    # momentum buffers of torch start from its first step (buf = g); ours from the zero buffer: same thing, as long as
    # ours starts at zero in the rows torch sees
    assert not buf[~pad_all].any()
    for step in range(20):
        scale = cosine_factor(step, 20)
        g = (rng.standard_normal(w.shape) * 0.01).astype(np.float32)
        heads.grads.copy_(torch.from_numpy(g))
        heads.apply_gradients(scale)
        lr_step = (lr_e * scale).astype(np.float32)
        w_ref, buf_ref = O.sgd(w, buf, g, lr_step[per], wd_e[per], mu)
        w = np.where(pad_all, w, w_ref)
        buf = np.where(pad_all, buf, buf_ref)
        got_w, got_m, got_g = heads.params.cpu().numpy(), heads.momentum_buf.cpu().numpy(), heads.grads.cpu().numpy()
        assert np.array_equal(got_w.view(np.int32), w.view(np.int32)), step
        assert np.array_equal(got_m.view(np.int32), buf.view(np.int32)), step
        assert not got_g[~pad_all].any() and np.array_equal(got_g[pad_all], g[pad_all]), step
        wb = heads.weight_bf16.cpu()
        assert torch.equal(wb[torch.from_numpy(~pad.reshape(-1))],
                           torch.from_numpy(w[:nw].reshape(H * Cp, D)[~pad.reshape(-1)]).to(torch.bfloat16))
        assert torch.equal(wb[torch.from_numpy(pad.reshape(-1))], wb_pad)
        for h in range(H):
            opt.param_groups[h]["lr"] = float(lr_step[h])
            tw[h].grad = torch.from_numpy(g[:nw].reshape(H, Cp, D)[h, :C].copy()).to(cuda)
            tb[h].grad = torch.from_numpy(g[nw:].reshape(H, Cp)[h, :C].copy()).to(cuda)
        opt.step()
    for h in (2, 3):                                     # lr = 0: the init, exactly
        assert lrs[h // 2] == 0.0
        assert np.array_equal(w[per == h], w_init[per == h])
    for h in range(H):
        ours_w = w[:nw].reshape(H, Cp, D)[h, :C]
        ours_b = w[nw:].reshape(H, Cp)[h, :C]
        for ours, theirs in ((ours_w, tw[h]), (ours_b, tb[h])):
            theirs = theirs.detach().cpu().numpy()
            assert np.abs(ours - theirs).max() <= 1e-6 * max(np.abs(theirs).max(), 1e-3), h


# ---- one whole step ----
def _setup(cuda, heads_args, b, seed):
    from byol_b200.linear_eval import LinearHeads
    heads = LinearHeads(*heads_args, seed=seed, device=cuda)
    rng = np.random.default_rng(seed)
    feats = torch.from_numpy(rng.standard_normal((b, heads.D)).astype(np.float32)).to(cuda).bfloat16()
    labels = torch.from_numpy(rng.integers(0, heads.C, b)).to(cuda)
    return heads, feats, labels


def test_full_step_against_oracle(cuda):
    from byol_b200 import ops
    from byol_b200.linear_eval import multihead_ce
    lrs, wds = (0.4, 0.3, 0.2, 0.1, 0.05), (0.0, 1e-5, 1e-4, 1e-3, 1e-2)
    C, D, B = 100, 256, 200
    heads, feats, labels = _setup(cuda, (D, C, lrs, wds, 0.9), B, 5)
    H, Cp = heads.H, heads.Cp
    nw = H * Cp * D
    heads.step(feats, labels, 1.0)                      # a first step: non-zero bias and momentum from here on
    w0, buf0 = heads.params.cpu().numpy().copy(), heads.momentum_buf.cpu().numpy().copy()
    x = feats.float().cpu().numpy().astype(np.float64)
    lab = labels.cpu().numpy()
    # the pieces of the step, one by one
    logits = heads.logits(feats)
    dl = torch.empty((B, H * Cp), dtype=torch.bfloat16, device=cuda)
    loss = torch.zeros(H, dtype=torch.float32, device=cuda)
    multihead_ce(logits, labels, H, C, dlogits=dl, loss_sum=loss)
    dw = torch.zeros((H * Cp, D), dtype=torch.float32, device=cuda)
    db = torch.zeros(H * Cp, dtype=torch.float32, device=cuda)
    ops.linear_wgrad(feats, dl, dw)
    ops.col_sum(dl, db)
    torch.cuda.synchronize()
    wq = O.bf16(w0[:nw]).astype(np.float64).reshape(H * Cp, D)
    ref_logits = O.logits(feats.float().cpu().numpy(), w0[:nw].reshape(H, Cp, D), w0[nw:])
    bound = D * 2.0 ** -23 * (np.abs(x) @ np.abs(wq).T) + 2.0 ** -23 * np.abs(w0[nw:])
    assert (np.abs(logits.cpu().numpy() - ref_logits) <= bound).all()
    ref_loss, _, ref_grad = O.cross_entropy(ref_logits, lab, H, C)
    g = dl.float().cpu().numpy().astype(np.float64)
    valid = np.tile(np.arange(Cp) < C, H)
    assert (np.abs(g - ref_grad)[:, valid] <= 2 * _bf16_ulp(ref_grad[:, valid])).all()
    assert not g[:, ~valid].any()
    assert np.allclose(loss.cpu().numpy() / B, ref_loss.mean(0), rtol=1e-4, atol=0)
    gw_bound = B * 2.0 ** -23 * (np.abs(g).T @ np.abs(x))
    assert (np.abs(dw.cpu().numpy() - g.T @ x) <= gw_bound).all()
    assert (np.abs(db.cpu().numpy() - g.sum(0)) <= B * 2.0 ** -23 * np.abs(g).sum(0)).all()
    # the step itself: the same logits / gradient bits, then the update in its exact fp32 order
    mean_loss = heads.step(feats, labels, 0.75)
    assert torch.equal(_bits(mean_loss), _bits(loss / B))
    grads = np.concatenate([dw.cpu().numpy().reshape(-1), db.cpu().numpy()])
    per = np.concatenate([np.repeat(np.arange(H), Cp * D), np.repeat(np.arange(H), Cp)])
    lr_e = (np.array([lr for lr, _ in heads.grid], np.float32) * np.float32(0.75)).astype(np.float32)
    wd_e = np.array([wd for _, wd in heads.grid], np.float32)
    w1, buf1 = O.sgd(w0, buf0, grads, lr_e[per], wd_e[per], 0.9)
    pad = ~np.concatenate([np.repeat(valid, D), valid])
    w1[pad], buf1[pad] = 0.0, 0.0
    assert np.array_equal(heads.params.cpu().numpy().view(np.int32), w1.view(np.int32))
    assert np.array_equal(heads.momentum_buf.cpu().numpy().view(np.int32), buf1.view(np.int32))
    assert not heads.grads.cpu().numpy().any()


def test_head_logits_do_not_depend_on_the_shared_gemm(cuda):
    """The logit GEMM has no split-K (every CTA runs the whole K loop), so a head's logits are the same bits whether it
    shares the GEMM with 24 other heads or runs alone."""
    from byol_b200.linear_eval import LinearHeads
    lrs, wds = (0.4, 0.3, 0.2, 0.1, 0.05), (0.0, 1e-5, 1e-4, 1e-3, 1e-2)
    C, D, B = 100, 512, 300
    heads, feats, _ = _setup(cuda, (D, C, lrs, wds), B, 9)
    bias = torch.randn(C, generator=torch.Generator().manual_seed(2)).to(cuda)
    heads.bias[:, :C] = bias
    full = heads.logits(feats)
    for k in (0, 7, 24):
        one = LinearHeads(D, C, (heads.grid[k][0],), (heads.grid[k][1],), seed=9, device=cuda)
        one.bias[0, :C] = bias
        assert torch.equal(one.weight_bf16, heads.weight_bf16[k * heads.Cp:(k + 1) * heads.Cp])
        alone = one.logits(feats)
        assert torch.equal(_bits(alone), _bits(full[:, k * heads.Cp:(k + 1) * heads.Cp])), k


def test_nonfinite_features_are_misses(cuda):
    """Feature rows with a NaN, or all infinite (NaN logits), score no hit in evaluate; the other rows count as without
    them."""
    heads, feats, labels = _setup(cuda, (128, 10, (0.1, 0.05), (0.0,)), 300, 13)
    for _ in range(5):
        heads.step(feats, labels, 1.0)
    poisoned = feats.clone()
    rows = torch.tensor([0, 5, 6, 299], device=cuda)
    poisoned[0] = float("nan")
    poisoned[5, 3] = float("nan")
    poisoned[6, :] = float("inf")
    poisoned[299, 7] = float("nan")
    keep = torch.ones(300, dtype=torch.bool, device=cuda)
    keep[rows] = False
    got = heads.evaluate(poisoned, labels)
    ref = heads.evaluate(feats[keep].contiguous(), labels[keep].contiguous())
    assert torch.equal(got, ref), (got, ref)
    assert heads.finite_heads().all()


def test_diverged_heads_are_never_selected(cuda):
    from byol_b200.linear_eval import select_heads, train_linear_heads
    rng = np.random.default_rng(14)
    centers = rng.standard_normal((5, 64)).astype(np.float32)
    (tf, tl), (vf, vl) = [(torch.from_numpy(x).to(cuda), torch.from_numpy(y).to(cuda))
                          for x, y in (_clusters(rng, 600, centers), _clusters(rng, 200, centers))]
    heads, rep = train_linear_heads(tf, tl, vf, vl, 5, epochs=3, batch_size=100, lrs=(0.2, 0.1, 0.05), seed=1)
    assert all(h["finite"] for h in rep["heads"])
    best = rep["best"]
    heads.weight[best, 1, 2] = float("nan")              # the best head diverges: a NaN in one weight, in the fp32
    heads.weight_bf16[best * heads.Cp + 1, 2] = float("nan")     # master and in the GEMM copy a step would write
    again = select_heads(heads, vf.bfloat16(), vl)
    assert not again["heads"][best]["finite"] and again["best"] != best
    assert again["heads"][best]["val_top1"] == 0.0          # its class-1 logits are NaN: no row is a top-1 hit
    heads.bias[:, 0] = float("inf")                     # every head: no selection at all
    with pytest.raises(ValueError, match="diverged"):
        select_heads(heads, vf.bfloat16(), vl)
    # non-finite training features make every head diverge: an error, not a number
    tf_bad = tf.clone()
    tf_bad[17, 5] = float("nan")
    with pytest.raises(ValueError, match="diverged"):
        train_linear_heads(tf_bad, tl, vf, vl, 5, epochs=1, batch_size=100, lrs=(0.1,), seed=1)


# ---- training on cached features ----
def _clusters(rng, n, centers):
    lab = rng.integers(0, centers.shape[0], n)
    x = centers[lab] + rng.standard_normal((n, centers.shape[1])).astype(np.float32) * 0.5
    return x.astype(np.float32), lab


def test_cached_training_separates_clusters(cuda):
    from byol_b200.linear_eval import train_linear_heads
    rng = np.random.default_rng(11)
    C, D = 10, 128
    centers = rng.standard_normal((C, D)).astype(np.float32) * 0.5
    xs = [_clusters(rng, n, centers) for n in (4000, 500, 1000)]
    (tf, tl), (vf, vl), (sf, sl) = [(torch.from_numpy(x).to(cuda), torch.from_numpy(y).to(cuda)) for x, y in xs]
    runs = []
    for _ in range(2):
        heads, rep = train_linear_heads(tf, tl, vf, vl, C, epochs=5, batch_size=256, lrs=(0.4, 0.1, 0.01, 0.0),
                                        weight_decays=(0.0, 1e-4), seed=4)
        runs.append((heads.params.clone(), rep, heads.evaluate(sf.bfloat16(), sl).cpu()))
    (p0, r0, e0), (p1, r1, e1) = runs
    assert torch.equal(_bits(p0), _bits(p1)) and r0 == r1 and torch.equal(e0, e1)
    assert len(r0["heads"]) == 8 and r0["heads"][6]["lr"] == 0.0 and r0["heads"][6]["weight_decay"] == 0.0
    best = r0["best"]
    assert r0["heads"][best]["val_top1"] == max(h["val_top1"] for h in r0["heads"])
    assert 100.0 * float(e0[best, 0]) / 1000 >= 99.0, (r0, e0)
    assert r0["heads"][6]["val_top1"] < 50.0                # lr = 0: the random init


# ---- linear_accuracy on an image folder ----
def _model(loader, cuda):
    from byol_b200.model import BYOL
    torch.manual_seed(12)
    model = BYOL(512, 64, loader.output_size, 10, arch="resnet18", head_latent_size=128)
    return model.cuda()


@pytest.mark.parametrize("augment", [False, True])
def test_linear_accuracy_on_image_folder(cuda, tmp_path, augment):
    from byol_b200.data import get_loader
    from byol_b200.linear_eval import linear_accuracy
    make_image_folder(tmp_path, seed=6)
    loader = get_loader(**loader_kwargs(tmp_path))
    model = _model(loader, cuda)
    kw = dict(epochs=2, batch_size=4, lrs=(0.3, 0.1, 0.0), weight_decays=(0.0, 1e-4), augment=augment)
    acc = linear_accuracy(model, loader, **kw)
    assert set(acc) == {"linear_top1", "linear_top5", "lr", "weight_decay", "heads"}
    assert len(acc["heads"]) == 6
    assert [(h["lr"], h["weight_decay"]) for h in acc["heads"]] == [(0.3, 0.0), (0.3, 1e-4), (0.1, 0.0), (0.1, 1e-4),
                                                                     (0.0, 0.0), (0.0, 1e-4)]
    for h in acc["heads"]:
        assert 0.0 <= h["val_top1"] <= h["val_top5"] <= 100.0
        assert 0.0 <= h["test_top1"] <= h["test_top5"] <= 100.0
    assert 0.0 <= acc["linear_top1"] <= acc["linear_top5"] <= 100.0
    assert acc == linear_accuracy(model, loader, **kw)
    target = linear_accuracy(model, loader, network="target", **kw)
    assert 0.0 <= target["linear_top1"] <= target["linear_top5"] <= 100.0 and len(target["heads"]) == 6


def test_cached_training_features_equal_test_features(cuda, tmp_path, monkeypatch):
    """With the test split pointed at the training images, every cached training feature is bit-equal to the test
    feature of the same image (same transform, whatever the batch it came in)."""
    from byol_b200 import linear_eval
    from byol_b200.data import ImageFolderLoader, get_loader
    make_image_folder(tmp_path, seed=7)
    loader = get_loader(**loader_kwargs(tmp_path))
    loader.test_loader = ImageFolderLoader(loader.train_loader.samples, 3, loader.test_loader.augment, train=False)
    model = _model(loader, cuda)
    seen = []
    real = linear_eval._extract

    def spy(model, samples, batch_size, augment, network):
        out = real(model, samples, batch_size, augment, network)
        seen.append((list(samples), out[0].clone(), out[1].clone()))
        return out

    monkeypatch.setattr(linear_eval, "_extract", spy)
    linear_eval.linear_accuracy(model, loader, epochs=1, batch_size=4)
    assert len(seen) == 3                                   # validation (hold-out), test, training
    (val_s, _, _), (test_s, test_f, test_l), (fit_s, fit_f, fit_l) = seen
    assert test_s == list(loader.train_loader.samples) and len(val_s) == 1 and len(fit_s) == len(test_s) - 1
    assert not set(val_s) & set(fit_s)
    rows = [test_s.index(s) for s in fit_s]
    assert torch.equal(_bits(fit_f), _bits(test_f[rows])) and torch.equal(fit_l, test_l[rows])


def test_training_is_undisturbed(cuda, tmp_path):
    """Graphed training steps give the same bits with linear_accuracy calls between steps and between a step's forward
    and backward; the calls change no running statistic, num_batches_tracked or EMA step."""
    from byol_b200 import wiring
    from byol_b200.data import get_loader
    from byol_b200.linear_eval import linear_accuracy
    from byol_b200.model import BYOL
    from tests.test_gpu_knn import _bn_state, _step
    make_image_folder(tmp_path, seed=2)
    loader = get_loader(**loader_kwargs(tmp_path))
    arch, b, r = "resnet:bottleneck:1,1,1,1", 8, 64
    g = torch.Generator().manual_seed(3)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 10, (b,), generator=g).cuda()) for _ in range(4)]
    res = {}
    for mode in ("plain", "probed"):
        torch.manual_seed(11)
        model = BYOL(2048, 64, 10, 20, arch=arch, head_latent_size=128).cuda().train()
        opt = wiring.build_optimizer(model, global_batch_size=256)

        def probe_calls():
            before, step = _bn_state(model), model.target_network.step
            for augment in (False, True):
                acc = linear_accuracy(model, loader, epochs=1, batch_size=4, lrs=(0.1,), augment=augment)
                assert 0.0 <= acc["linear_top1"] <= acc["linear_top5"] <= 100.0
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
