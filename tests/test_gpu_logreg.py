"""GPU: transfer linear evaluation (byol_b200.logreg, csrc/logreg.cu).

* one function evaluation: f_h and grad f_h (W and b) of several heads at random (W, b), on features bf16 cannot
  represent, against float64 autograd; the plane gradient's padding columns are zero
* the vector kernels against a float64 numpy restatement; a head's dot products are the same bits alone and beside
  other heads
* the batched L-BFGS reaches scipy's float64 optimum (L-BFGS-B to gtol 1e-12) within 1e-6 max(1, f*), every head
  converged, alone or beside other heads; a stopped head is never written again; two runs give the same bits
* transfer_accuracy end to end on a synthetic image folder, with and without valid/
* the "byol_transfer" window records against torchvision
"""
import types

import numpy as np
import pytest
import torch

from tests.image_folder import loader_kwargs, make_image_folder
from tests.test_eval_transform_host import SIZES

pytestmark = pytest.mark.gpu


def _problem(n, d, c, seed):
    """fp32 features with full 24-bit mantissas and labels from a noisy linear teacher (every class present)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n, d, generator=g, dtype=torch.float64).float()
    teacher = torch.randn(c, d, generator=g, dtype=torch.float64) / d ** 0.5
    y = (x.double() @ teacher.T + torch.randn(n, c, generator=g, dtype=torch.float64)).argmax(1)
    y[:c] = torch.arange(c)
    return x, y


def _objective64(x, y, w, b, l2):
    """f(W, b) in float64 (numpy): mean cross-entropy + l2 / 2 ||W||^2."""
    z = x @ w.T + b
    z = z - z.max(1, keepdims=True)
    lse = np.log(np.exp(z).sum(1))
    return float(np.mean(lse - z[np.arange(len(y)), y]) + 0.5 * l2 * np.sum(w * w))


def _solver(x, y, c, l2s):
    from byol_b200 import logreg, ops
    planes, _ = ops.split_planes(x.cuda().contiguous(), logreg.T_PLANES)
    return logreg._Solver(planes, y.cuda(), x.shape[0], x.shape[1], c, l2s, torch.device("cuda"))


def test_objective_and_gradient_against_float64(cuda):
    from byol_b200 import logreg
    n, d, c, l2s = 9000, 128, 10, (0.0, 1e-3, 0.5)        # two row chunks
    x, y = _problem(n, d, c, 1)
    s = _solver(x, y, c, l2s)
    H, Cp = s.H, s.Cp
    g = torch.Generator().manual_seed(2)
    w0 = torch.randn(H, c, d, generator=g, dtype=torch.float64).float() * 0.05
    b0 = torch.randn(H, c, generator=g, dtype=torch.float64).float()
    s.xt[:s.nw].view(H, Cp, d)[:, :c] = w0.cuda()
    s.xt[s.nw:].view(H, Cp)[:, :c] = b0.cuda()
    s.set_modes(np.full(H, logreg._SEARCH), np.ones(H))
    s.evaluate(logreg._bit(logreg._SEARCH))
    sc = s.scalars.cpu().numpy()
    gw = s.gt[:s.nw].view(H, Cp, d).cpu()
    gb = s.gt[s.nw:].view(H, Cp).cpu()
    assert not gw[:, c:].any() and not gb[:, c:].any()
    # the last chunk's plane gradient: zero in every padding column of every plane
    rows = n - 8192
    dp = s.dplanes[:rows].view(rows, logreg.T_PLANES, H, Cp)
    assert not dp[..., c:].float().any()
    xd, yd = x.double(), y
    for h in range(H):
        w = w0[h].double().requires_grad_()
        b = b0[h].double().requires_grad_()
        f = torch.nn.functional.cross_entropy(xd @ w.T + b, yd) + 0.5 * l2s[h] * (w * w).sum()
        f.backward()
        f_dev = sc[h, 0] / n + 0.5 * l2s[h] * sc[h, 2]
        assert abs(f_dev - f.item()) <= 1e-6 * abs(f.item()), (h, f_dev, f.item())
        for got, ref in ((gw[h, :c].double(), w.grad), (gb[h, :c].double(), b.grad)):
            err = float((got - ref).norm() / ref.norm())
            assert err <= 1e-6, (h, err)
        ginf = max(float(w.grad.abs().max()), float(b.grad.abs().max()))
        assert abs(sc[h, 1] - ginf) <= 1e-6 * ginf


def _heads(H, c, d, seed):
    """A stand-in for the solver (mode, part, shape) and H heads' parameter-shaped random vectors."""
    from byol_b200 import logreg
    cp = logreg._padded(c)
    size = H * cp * d + H * cp
    ns = types.SimpleNamespace(H=H, C=c, Cp=cp, D=d, mode=torch.full((H,), logreg._ACCEPT, dtype=torch.int32).cuda(),
                               part=torch.zeros(8 * H * logreg.vec_blocks(c, d), dtype=torch.float64).cuda())
    g = torch.Generator().manual_seed(seed)
    return ns, [torch.randn(size, generator=g) for _ in range(4)]


def _head_view(v, H, cp, d, h):
    nw = H * cp * d
    return torch.cat([v[:nw].view(H, cp * d)[h], v[nw:].view(H, cp)[h]])


def _place(vs_alone, H, cp, d, h, seed):
    """Embeds one head's vectors as head h of H heads (the other heads random)."""
    g = torch.Generator().manual_seed(seed)
    out = []
    for v in vs_alone:
        full = torch.randn(H * cp * d + H * cp, generator=g)
        full[:H * cp * d].view(H, cp * d)[h] = v[:cp * d]
        full[H * cp * d:].view(H, cp)[h] = v[cp * d:]
        out.append(full)
    return out


@pytest.mark.parametrize("c,d", [(10, 128), (100, 2048)])
def test_dots_against_float64_and_alone(cuda, c, d):
    from byol_b200 import logreg
    ns1, v1 = _heads(1, c, d, 3)
    pairs = [(0, 1), (1, 1), (2, 3), (0, 3)]
    out1 = torch.zeros((1, 8), dtype=torch.float64).cuda()
    logreg.dots(ns1, [(v1[a].cuda(), v1[b].cuda()) for a, b in pairs], logreg._bit(logreg._ACCEPT), out1)
    ref = [float(v1[a].double() @ v1[b].double()) for a, b in pairs]
    np.testing.assert_allclose(out1[0, :4].cpu().numpy(), ref, rtol=1e-12)
    for H, h in ((3, 1), (7, 6)):
        ns, _ = _heads(H, c, d, 0)
        vh = [t.cuda() for t in _place(v1, H, ns.Cp, d, h, H)]
        out = torch.zeros((H, 8), dtype=torch.float64).cuda()
        logreg.dots(ns, [(vh[a], vh[b]) for a, b in pairs], logreg._bit(logreg._ACCEPT), out)
        assert torch.equal(out[h, :4], out1[0, :4]), (H, h)


def _two_loop64(g, S, Y):
    """float64 L-BFGS direction from pairs oldest first."""
    q = g.copy()
    alphas = []
    for s, y in reversed(list(zip(S, Y))):
        a = (s @ q) / (s @ y)
        q -= a * y
        alphas.append(a)
    if S:
        q *= (S[-1] @ Y[-1]) / (Y[-1] @ Y[-1])
    else:
        q /= np.linalg.norm(g)
    for (s, y), a in zip(zip(S, Y), reversed(alphas)):
        beta = (y @ q) / (s @ y)
        q += (a - beta) * s
    return -q


def test_accept_twoloop_trial_against_float64(cuda):
    """Feeds 13 accepted steps (more than the history holds) through accept / commit / two-loop / trial and compares
    every direction and trial point with the float64 restatement."""
    from byol_b200 import logreg
    H, c, d = 3, 10, 64
    x, y = _problem(64, d, c, 0)
    s = _solver(x, y, c, (0.0,) * H)
    rng = np.random.default_rng(4)
    size = s.x.numel()
    S, Y = [[] for _ in range(H)], [[] for _ in range(H)]
    gs = rng.standard_normal(size).astype(np.float32)
    s.gt.copy_(torch.from_numpy(gs))
    s.set_modes(np.full(H, logreg._START), np.ones(H))
    s.step()
    for it in range(13):
        g_all = s.g.cpu().numpy()
        d_all = s.d.cpu().numpy()
        for h in range(H):
            gh = _head_view(torch.from_numpy(g_all), H, s.Cp, d, h).double().numpy()
            dh = _head_view(torch.from_numpy(d_all), H, s.Cp, d, h).double().numpy()
            ref = _two_loop64(gh, S[h][-logreg.HISTORY:], Y[h][-logreg.HISTORY:])
            assert np.linalg.norm(dh - ref) <= 1e-5 * np.linalg.norm(ref), (it, h)
            gtd = float(s.scalars[h, 3])
            assert abs(gtd - gh @ dh) <= 1e-9 * abs(gh @ dh)
        t = np.array([1.0, 0.5, 0.25])
        s.set_modes(np.full(H, logreg._SEARCH), t)
        s.step()
        np.testing.assert_array_equal(s.xt.cpu().numpy(), s.x.cpu().numpy() +
                                      _scaled(s.d.cpu().numpy(), t, H, s.Cp, d))
        # a new gradient: a convex-looking change so that s.y > 0
        xt_all, x_all = s.xt.cpu().numpy(), s.x.cpu().numpy()
        g_new = (g_all + 0.3 * (xt_all - x_all) + 0.01 * rng.standard_normal(size)).astype(np.float32)
        s.gt.copy_(torch.from_numpy(g_new))
        for h in range(H):
            sh = _head_view(torch.from_numpy(xt_all - x_all), H, s.Cp, d, h).double().numpy()
            yh = _head_view(torch.from_numpy(g_new - g_all), H, s.Cp, d, h).double().numpy()
            if sh @ yh > 1e-10 * (yh @ yh):
                S[h].append(sh); Y[h].append(yh)
        s.set_modes(np.full(H, logreg._ACCEPT), np.ones(H))
        s.step()
    assert (s.hist[:, 1].cpu() == logreg.HISTORY).all()


def _scaled(dv, t, H, cp, d):
    out = np.empty_like(dv)
    nw = H * cp * d
    for h in range(H):
        tf = np.float32(t[h])
        out[h * cp * d:(h + 1) * cp * d] = tf * dv[h * cp * d:(h + 1) * cp * d]
        out[nw + h * cp:nw + (h + 1) * cp] = tf * dv[nw + h * cp:nw + (h + 1) * cp]
    return out


def _scipy_optimum(x, y, c, l2):
    from scipy.optimize import minimize
    n, d = x.shape

    def fun(p):
        w, b = p[:c * d].reshape(c, d), p[c * d:]
        z = x @ w.T + b
        z = z - z.max(1, keepdims=True)
        e = np.exp(z)
        s = e.sum(1, keepdims=True)
        f = np.mean(np.log(s[:, 0]) - z[np.arange(n), y]) + 0.5 * l2 * np.sum(w * w)
        gz = e / s
        gz[np.arange(n), y] -= 1.0
        gz /= n
        return f, np.concatenate([(gz.T @ x + l2 * w).ravel(), gz.sum(0)])

    r = minimize(fun, np.zeros(c * d + c), jac=True, method="L-BFGS-B",
                 options=dict(gtol=1e-12, ftol=0.0, maxiter=50000, maxfun=100000, maxcor=20))
    return r.fun


def _check_optimum(fit, x, y, l2s, ref):
    for h, l2 in enumerate(l2s):
        e = fit.heads[h]
        assert e["converged"] and e["finite"], (h, e)
        w = fit.weight[h].double().cpu().numpy()
        b = fit.bias[h].double().cpu().numpy()
        gap = _objective64(x, y, w, b, l2) - ref[h]
        assert gap <= 1e-6 * max(1.0, ref[h]), (h, l2, gap, ref[h], e)


@pytest.mark.parametrize("c,d", [(10, 128), (3, 64)])
def test_fit_reaches_scipy_optimum(cuda, c, d):
    from byol_b200.logreg import fit_logistic_regression
    n = 2048
    l2s = tuple(np.logspace(-4, 1, 6)) if c == 10 else (1e-3, 1e-1)
    x, y = _problem(n, d, c, 5 + c)
    x64, y64 = x.double().numpy(), y.numpy()
    ref = [_scipy_optimum(x64, y64, c, l2) for l2 in l2s]
    fit = fit_logistic_regression(x.cuda(), y.cuda(), c, l2s)
    print("heads:", fit.heads, "evaluations:", fit.evaluations)
    _check_optimum(fit, x64, y64, l2s, ref)
    # each head alone reaches the same optimum
    for h in (0, len(l2s) - 1):
        alone = fit_logistic_regression(x.cuda(), y.cuda(), c, (l2s[h],))
        _check_optimum(alone, x64, y64, (l2s[h],), [ref[h]])


def test_stopped_heads_are_frozen_and_runs_reproduce(cuda, monkeypatch):
    from byol_b200 import logreg
    c, d, n = 10, 128, 2048
    x, y = _problem(n, d, c, 9)
    l2s = (1e-4, 1e-2, 1.0, 100.0)
    real = logreg._Solver.step
    frozen, checks = {}, [0]

    def spy(self):
        real(self)
        mode = self.mode.cpu().numpy()
        for h in range(self.H):
            cur = _head_view(self.x, self.H, self.Cp, self.D, h).clone()
            if h in frozen:
                assert torch.equal(frozen[h], cur), h
                checks[0] += 1
            elif mode[h] in (logreg._STOPPED, logreg._FINAL):
                frozen[h] = cur

    monkeypatch.setattr(logreg._Solver, "step", spy)
    a = logreg.fit_logistic_regression(x.cuda(), y.cuda(), c, l2s)
    assert len(frozen) == len(l2s) and checks[0] > 0
    iters = [e["iterations"] for e in a.heads]
    assert len(set(iters)) > 1, iters                        # the heads stopped at different times
    monkeypatch.setattr(logreg._Solver, "step", real)
    b = logreg.fit_logistic_regression(x.cuda(), y.cuda(), c, l2s)
    assert torch.equal(a.params.view(torch.int32), b.params.view(torch.int32))
    assert a.heads == b.heads and a.evaluations == b.evaluations


def test_fit_rejects_missing_class(cuda):
    from byol_b200.logreg import fit_logistic_regression
    x, y = _problem(256, 64, 4, 1)
    y[y == 2] = 1
    with pytest.raises(ValueError, match="no training image"):
        fit_logistic_regression(x.cuda(), y.cuda(), 4)
    with pytest.raises(ValueError, match="outside"):
        fit_logistic_regression(x.cuda(), y.cuda(), 2)


# ---- transfer_accuracy on an image folder ----
@pytest.mark.parametrize("valid", [False, True])
def test_transfer_accuracy_on_image_folder(cuda, tmp_path, monkeypatch, valid):
    import shutil
    from byol_b200 import logreg
    from byol_b200.data import get_loader
    from byol_b200.model import BYOL
    from tests.test_gpu_knn import _bn_state
    make_image_folder(tmp_path, seed=6)
    if valid:
        shutil.copytree(tmp_path / "test", tmp_path / "valid")
    loader = get_loader(**loader_kwargs(tmp_path, eval_transform="byol_transfer"))
    torch.manual_seed(12)
    model = BYOL(512, 64, loader.output_size, 10, arch="resnet18", head_latent_size=128).cuda()
    before = ([t.clone() for t in _bn_state(model)], {k: v.clone() for k, v in model.state_dict().items()},
              model.target_network.step)
    fits, feats = [], []
    real_fit, real_extract = logreg.fit_logistic_regression, logreg._extract

    def fit_spy(*a, **k):
        fits.append(real_fit(*a, **k))
        return fits[-1]

    def extract_spy(*a, **k):
        feats.append(real_extract(*a, **k))
        return feats[-1]

    monkeypatch.setattr(logreg, "fit_logistic_regression", fit_spy)
    monkeypatch.setattr(logreg, "_extract", extract_spy)
    l2s = (1e-3, 1e-1, 10.0)
    acc = logreg.transfer_accuracy(model, loader, l2s=l2s, max_iter=300)
    assert set(acc) == {"transfer_accuracy", "metric", "l2", "refit", "heads"}
    assert set(acc["refit"]) >= {"iterations", "objective", "converged"}
    assert acc["metric"] == "top1" and acc["l2"] in l2s and len(acc["heads"]) == 3
    for e in acc["heads"]:
        assert set(e) == {"l2", "val_metric", "finite", "iterations", "objective", "converged"}
        assert 0.0 <= e["val_metric"] <= 100.0
    n_train = len(loader.train_loader.samples)
    n_val = len(loader.valid_loader.samples) if valid else 0
    assert fits[0].rows == (n_train if valid else n_train - 1)
    assert fits[1].rows == n_train + n_val and fits[1].l2s == (acc["l2"],)     # the refit: train + valid
    after = _bn_state(model)
    assert all(torch.equal(a, b) for a, b in zip(before[0], after))
    state = model.state_dict()
    assert set(state) == set(before[1]) and all(torch.equal(before[1][k], state[k]) for k in state)
    assert before[2] == model.target_network.step
    test_x, test_y = feats[-1]
    assert test_x.dtype == torch.float32
    w, b = fits[1].weight[0].double().cpu(), fits[1].bias[0].double().cpu()
    pred = (test_x.double().cpu() @ w.T + b).argmax(1)
    assert acc["transfer_accuracy"] == pytest.approx(100.0 * float((pred == test_y.cpu()).double().mean()), abs=1e-9)
    mpc = logreg.transfer_accuracy(model, loader, l2s=l2s, max_iter=300, metric="mean_per_class")
    assert mpc["metric"] == "mean_per_class" and 0.0 <= mpc["transfer_accuracy"] <= 100.0


# ---- the "byol_transfer" window records ----
def _transfer_oracle(img, R):
    import torchvision.transforms.v2.functional as F
    x = F.resize(img, R, interpolation=F.InterpolationMode.BICUBIC, antialias=True).clamp(0.0, 1.0)
    return F.center_crop(x, [R, R])


@pytest.mark.parametrize("R", [64, 224])
def test_transfer_records_match_torchvision(cuda, R):
    from byol_b200.augment import TwoViewAugment
    aug = TwoViewAugment(image_size=R, seed=1, eval_transform="byol_transfer")
    g = torch.Generator().manual_seed(R)
    u8 = [torch.randint(0, 256, (3, h, w), dtype=torch.uint8, generator=g) for h, w in SIZES]
    p = aug.eval_params(SIZES, cuda)
    v1, v2 = aug.apply_ragged([t.to(cuda) for t in u8], p)
    lut = torch.from_numpy(np.arange(256, dtype=np.float32) / np.float32(255))
    worst = 0.0
    for i, t in enumerate(u8):
        ref = _transfer_oracle(lut[t.long()], R)
        for v in (v1, v2):
            err = float((v[i].cpu() - ref).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, (i, tuple(t.shape), err)
    # dense fp32 sources
    for hs, ws in SIZES[::3]:
        imgs = torch.rand(2, 3, hs, ws, generator=g)
        p = aug.eval_params([(hs, ws)] * 2, cuda)
        o1, _ = aug.apply(imgs.cuda(), p)
        for i in range(2):
            err = float((o1[i].cpu() - _transfer_oracle(imgs[i], R)).abs().max())
            worst = max(worst, err)
            assert err < 2e-4, ((hs, ws), err)
    print("byol_transfer records at R %d vs torchvision: worst abs error %.2e" % (R, worst))
