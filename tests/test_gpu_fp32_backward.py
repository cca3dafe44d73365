"""The fp32-accurate backward pass (BYOL(precision="fp32", backward_precision="fp32")): exact 3-way bf16 splits on every
backward GEMM (T = 6 product terms), fp32 gradients between layers, fp64 BatchNorm-backward sums.

* single kernels against float64 torch on the CPU (inputs that bf16 cannot represent): 1e-5 relative
* every parameter gradient of bottleneck and basic-block nets against float64 autograd given the same ReLU decisions
* the UNMODIFIED reference's gradient norm and updated parameters (tests/golden/*.npz), its 20-step loss curve, an
  unusual gradient pattern against float64 autograd, bit reproducibility
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_oracle_golden import _batches, _sample_index, load_case

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
T = 6


def _rel(got, ref):
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    return float((got - ref).abs().max() / ref.abs().max())


def _planes_nhwc(x_nhwc, cuda):
    from byol_b200 import ops
    c = x_nhwc.shape[-1]
    return ops.split_planes(x_nhwc.reshape(-1, c).to(cuda), T)[0].view(tuple(x_nhwc.shape[:-1]) + (T * c,))


CONVS = [(64, 64, 1, 1, 14), (64, 128, 3, 1, 10), (128, 128, 3, 2, 12), (256, 512, 1, 2, 8), (3, 64, 7, 2, 32)]


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,k,stride,hw", CONVS)
def test_split_dgrad_wgrad_match_fp64(cuda, cin, cout, k, stride, hw):
    """dX = dY * W^T and dW = dY^T * im2col(X) through the tensor cores with split operands equal float64 torch."""
    from byol_b200 import ops
    g = torch.Generator().manual_seed(21)
    n, pad = 3, k // 2
    x = torch.randn(n, cin, hw, hw, generator=g) * 2 + 0.7
    w = torch.randn(cout, cin, k, k, generator=g) * 0.1
    ho = (hw + 2 * pad - k) // stride + 1
    dy = torch.randn(n, cout, ho, ho, generator=g) * 0.37 + 0.01
    dy_nhwc = dy.permute(0, 2, 3, 1).contiguous()
    dyp = _planes_nhwc(dy_nhwc, cuda)
    # wgrad
    xp = ops.nchw_to_planes(x.to(cuda), T, 8) if cin < 8 else _planes_nhwc(x.permute(0, 2, 3, 1).contiguous(), cuda)
    dw = torch.zeros(cout, cin, k, k, device=cuda)
    ops.conv_wgrad_planes(xp, dyp, dw, k, k, stride, pad, T)
    ref_dw = torch.nn.grad.conv2d_weight(x.double(), w.shape, dy.double(), stride, pad)
    # dgrad (the stem's 3 input channels padded to 8 with zero weights)
    cpad = (cin + 7) // 8 * 8
    wpad = torch.zeros(cout, cpad, k, k)
    wpad[:, :cin] = w
    wd = torch.empty(cpad, k * k * T * cout, dtype=torch.bfloat16, device=cuda)
    ops.prep_weight_dgrad_planes(wpad.to(cuda), T, wd)
    resid = torch.randn(n, hw, hw, cpad, generator=g)
    dx = ops.conv_dgrad_planes(dyp, wd, hw, hw, k, k, stride, pad, T, resid=resid.to(cuda))
    ref_dx = torch.nn.grad.conv2d_input(x.shape, w.double(), dy.double(), stride, pad).permute(0, 2, 3, 1)
    torch.cuda.synchronize()
    e_dx = _rel(dx[..., :cin].cpu() - resid[..., :cin], ref_dx)
    e_dw = _rel(dw, ref_dw)
    print("split backward %dx%d/%d %d->%d: dgrad %.2e wgrad %.2e" % (k, k, stride, cin, cout, e_dx, e_dw))
    assert e_dx < 1e-5 and e_dw < 1e-5, (e_dx, e_dw)
    if cpad > cin:        # zero weights: the padding channels hold the residual only
        assert torch.equal(dx[..., cin:].cpu(), resid[..., cin:])


@pytest.mark.gpu
@pytest.mark.parametrize("m,k_in,n_out", [(64, 2048, 1000), (64, 2048, 4096), (64, 4096, 256), (32, 2048, 10)])
def test_split_linear_backward_matches_fp64(cuda, m, k_in, n_out):
    """The classifier (2048 -> 1000, and a 10-class head with a pitched gradient) and the 4096-wide MLP linears."""
    from byol_b200 import ops
    g = torch.Generator().manual_seed(22)
    x = torch.randn(m, k_in, generator=g).abs() * 1.3
    w = torch.randn(n_out, k_in, generator=g) * 0.02
    d = torch.randn(m, n_out, generator=g) * 0.11
    npad = (n_out + 7) // 8 * 8
    dp = ops.split_planes(d.to(cuda), T, cpad=npad)[0]
    xp = ops.split_planes(x.to(cuda), T)[0]
    dw = torch.zeros(n_out, k_in, device=cuda)
    ops.conv_wgrad_planes(xp.view(m, 1, 1, -1), dp.view(m, 1, 1, -1), dw.view(n_out, k_in, 1, 1), 1, 1, 1, 0, T)
    e_dw = _rel(dw, d.double().t() @ x.double())
    # dgrad sums up to T * 4096 products of both signs in the fp32 tensor-core accumulator: 1e-5 plus sqrt(K) x 2^-24
    tol_dx = 1e-5 + (T * n_out) ** 0.5 * 2.0 ** -24 * 4
    e_dx = 0.0
    if n_out % 8 == 0:
        wd = torch.empty(k_in, T * n_out, dtype=torch.bfloat16, device=cuda)
        ops.prep_weight_dgrad_planes(w.to(cuda), T, wd)
        dx = ops.linear_dgrad_planes(dp, wd, T)
        e_dx = _rel(dx, d.double() @ w.double())
    torch.cuda.synchronize()
    print("split linear backward %d -> %d: dgrad %.2e wgrad %.2e" % (k_in, n_out, e_dx, e_dw))
    assert e_dx < tol_dx and e_dw < 1e-5, (e_dx, tol_dx, e_dw)


def _bn_fixture(cuda, m, c, seed):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(seed)
    y = torch.randn(m, c, generator=g) * 0.3 + 5.0
    gamma, beta = torch.rand(c, generator=g) + 0.5, torch.randn(c, generator=g) * 0.2
    stats = torch.zeros(2 * c, dtype=torch.float64, device=cuda)
    ops.stats_f32(y.to(cuda), stats)
    co = torch.empty(1, 4, c, device=cuda)
    ops.bn_finalize_lanes_f64(stats, m, [gamma.to(cuda)], [beta.to(cuda)], None, None, 0.1, 1e-5, co)
    return g, y, gamma, beta, co[0]


@pytest.mark.gpu
@pytest.mark.parametrize("mask_mode", [1, 3])
def test_fp32_bn_backward_matches_fp64(cuda, mask_mode):
    """fp32 BatchNorm backward (ReLU recomputed from y / ReLU mask bits of a block output with a residual) against
    float64 autograd: dy, dz, dgamma, dbeta, and the planes of dy reconstruct the fp32 dy."""
    from byol_b200 import ops
    m, c = 3000, 64
    g, y, gamma, beta, co = _bn_fixture(cuda, m, c, 23)
    grad = torch.randn(m, c, generator=g)
    resid = torch.randn(m, c, generator=g)
    mask = None
    if mask_mode == 3:
        _, _, _, mask = ops.bn_apply_f32(y.to(cuda), co[0], co[1], True, T, resid=resid.to(cuda), want_planes=False,
                                         want_out32=True, want_mask=True)
    gd = grad.to(cuda)
    s12 = torch.zeros(2 * c, dtype=torch.float64, device=cuda)
    ops.bn_bwd_reduce_f32(gd, y.to(cuda), co, s12, mask_mode, mask=mask)
    dgamma, dbeta = torch.zeros(c, device=cuda), torch.zeros(c, device=cuda)
    pl, dy, dz = ops.bn_bwd_apply_f32(gd, y.to(cuda), co, gamma.to(cuda), s12, m, mask_mode, T, mask=mask,
                                      want_f32=True, want_dz=True, dgamma=dgamma, dbeta=dbeta)
    torch.cuda.synchronize()
    y64 = y.double().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    xhat = (y64 - y64.mean(0)) / torch.sqrt(y64.var(0, unbiased=False) + 1e-5)
    o = xhat * g64 + b64
    if mask_mode == 1:
        dz_ref = grad.double() * (torch.relu(o) > 0).double()
    else:
        bits = np.unpackbits(mask.cpu().numpy(), bitorder="little").reshape(m, c)
        dz_ref = grad.double() * torch.from_numpy(bits).double()
    (o * dz_ref.detach()).sum().backward()
    errs = {"dy": _rel(dy, y64.grad), "dz": _rel(dz, dz_ref), "dgamma": _rel(dgamma, g64.grad),
            "dbeta": _rel(dbeta, b64.grad)}
    planes = pl.float().cpu().view(m, T, c).double()
    errs["planes"] = _rel(planes[:, 0] + planes[:, 2] + planes[:, 5], dy.cpu())
    print("fp32 BN backward mask %d: %s" % (mask_mode, {k: "%.2e" % v for k, v in errs.items()}))
    assert max(errs.values()) < 1e-5, errs


@pytest.mark.gpu
def test_fp32_pool_backward_matches_fp64(cuda):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(24)
    n, h, c = 2, 20, 64
    x = torch.randn(n, h, h, c, generator=g)
    _, idx = ops.maxpool_f32(x.to(cuda), 3, 2, 1, want_idx=True)
    ho = (h + 2 - 3) // 2 + 1
    dy = torch.randn(n, ho, ho, c, generator=g)
    dx = ops.maxpool_bwd_f32(dy.to(cuda), idx, h, h, 3, 2, 1)
    x64 = x.double().permute(0, 3, 1, 2).requires_grad_(True)
    (F.max_pool2d(x64, 3, 2, 1) * dy.double().permute(0, 3, 1, 2)).sum().backward()
    e_max = _rel(dx, x64.grad.permute(0, 2, 3, 1))
    ga, gb = torch.randn(n, c, generator=g), torch.randn(n, c, generator=g)
    da = ops.avgpool_bwd_f32(ga.to(cuda), gb.to(cuda), n, 7, 7, c)
    x64 = torch.zeros(n, c, 7, 7, dtype=torch.float64, requires_grad=True)
    (F.adaptive_avg_pool2d(x64, 1).flatten(1) * (ga + gb).double()).sum().backward()
    e_avg = _rel(da, x64.grad.permute(0, 2, 3, 1))
    torch.cuda.synchronize()
    print("fp32 pool backward: max %.2e avg %.2e" % (e_max, e_avg))
    assert e_max < 1e-6 and e_avg < 1e-6


def _momentum_flat(model, opt):
    return torch.cat([opt.state[p]["momentum_buffer"].reshape(-1) for p in model.parameters()])


GOLDEN_CASES = ["rn18_b8_r64", "rn18_b32_r224", "rn50_b8_r64", "rn50_b16_r224"]


@pytest.mark.gpu
@pytest.mark.parametrize("bwd", ["fp32", "bf16"])
@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_fp32_backward_matches_reference_golden(cuda, name, bwd):
    """Every step the golden file holds: the sampled flat gradient, its norm, the LARS momentum and the updated
    parameters against the UNMODIFIED reference, for both backward precisions (the errors are printed).
    The sampled entries (and the LARS momentum, which rescales every tensor's gradient) are dominated by ReLU inputs
    near zero that the reference's forward and ours decide differently (test_fp32_backward_matches_fp64_per_tensor,
    DESIGN.md §4), so they are printed, not held to 1e-3.
    Held: at the first step the fp32 backward's gradient norm within 1e-3 and its updated parameters within 1e-4 of
    their largest entry (1e-2 / 1e-3 at later steps, which start from chaotically diverged parameters); the bf16
    backward's norm within 10 %."""
    from byol_b200.model import BYOL
    from byol_b200.objective import loss_function
    from byol_b200 import wiring
    z, arch, rep, b, r, steps, seed, lr, total = load_case(name)
    torch.manual_seed(seed)
    model = BYOL(rep, 256, 1000, total, arch=arch, precision="fp32", backward_precision=bwd).cuda().train()
    opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(model, 1e-6), lr=lr, momentum=0.9), eps=0.0)
    idx = _sample_index(int(z["numel"]))
    for s, (a1, a2, lab) in enumerate(_batches(seed, steps, b, r)):
        pre = "s%d_" % s
        out = model(a1.cuda(), a2.cuda())
        byol = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                             target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
        loss = byol + F.cross_entropy(out["linear_preds"], torch.cat([lab, lab]).cuda())
        opt.zero_grad()
        loss.backward()
        torch.cuda.synchronize()
        gflat = model._engine.grad.detach().cpu()
        ref = torch.from_numpy(z[pre + "grad_sample"]).double()
        got = gflat[idx].double()
        e_max = float((got - ref).abs().max() / ref.abs().max())
        e_l2 = float((got - ref).norm() / ref.norm())
        e_norm = abs(float(gflat.double().norm()) / float(z[pre + "grad_norm"]) - 1.0)
        opt.step()
        torch.cuda.synchronize()
        mref = torch.from_numpy(z[pre + "momentum_sample"]).double()
        e_mom = float((_momentum_flat(model, opt).cpu()[idx].double() - mref).abs().max() / mref.abs().max())
        theta = model._engine.theta.cpu()[idx].numpy()
        e_theta = float(np.abs(theta - z[pre + "theta_sample"]).max() / np.abs(z[pre + "theta_sample"]).max())
        print("%s step %d backward %s: grad max %.2e l2 %.2e norm %.2e momentum %.2e theta %.2e" %
              (name, s, bwd, e_max, e_l2, e_norm, e_mom, e_theta))
        if bwd == "fp32" and s == 0:
            assert e_norm < 1e-3 and e_theta < 1e-4, (s, e_norm, e_theta)
        elif bwd == "fp32":         # later steps start from diverged parameters (the small cases are chaotic)
            assert e_norm < 1e-2 and e_theta < 1e-3, (s, e_norm, e_theta)
        else:
            assert e_norm < 0.1


class _ForcedRelu(torch.nn.Module):
    """Stands in for an nn.ReLU module: the k-th call multiplies by the k-th given 0/1 mask (torchvision blocks call
    their one `relu` module two or three times)."""

    def __init__(self, masks):
        super(_ForcedRelu, self).__init__()
        self.masks, self.i = masks, 0

    def forward(self, x):
        m = self.masks[self.i]
        self.i += 1
        return x * m.to(x.dtype)


def _relu_masks(S, kind):
    """The ReLU decisions the fp32 forward made for one online lane, in the reference modules' NCHW layout."""
    def bn_mask(y, c):     # relu(y*scale + shift) > 0, evaluated exactly (the kernels round that value once)
        return ((y.double() * c[0].double() + c[1].double()) > 0).cpu()

    def nchw(t):
        return t.permute(0, 3, 1, 2) if t.dim() == 4 else t
    stem = nchw(bn_mask(S["y0"], S["c0"]))
    blocks = []
    for B in S["blocks"]:
        n, h, w, c = B["y3" if kind == "bottleneck" else "y2"].shape
        bits = np.unpackbits(B["mask"].cpu().numpy(), bitorder="little").reshape(n, h, w, c)
        ms = [nchw(bn_mask(B["y1"], B["c1"]))]
        if kind == "bottleneck":
            ms.append(nchw(bn_mask(B["y2"], B["c2"])))
        ms.append(torch.from_numpy(bits).bool().permute(0, 3, 1, 2))
        blocks.append(ms)
    return stem, blocks, bn_mask(S["head"]["h"], S["head"]["c"]), bn_mask(S["pred"]["h"], S["pred"]["c"])


@pytest.mark.gpu
@pytest.mark.parametrize("arch,rep,b,r", [("resnet:bottleneck:1,1,1,1", 2048, 8, 96), ("resnet18", 512, 8, 64)])
def test_fp32_backward_matches_fp64_per_tensor(cuda, arch, rep, b, r):
    """Every parameter gradient of both online views (loss on the predictions) against float64 autograd of the same
    torchvision modules, tensor by tensor, on bottleneck nets with stride-2 and downsample blocks (c3 under the
    block-output mask, the downsample dgrad feeding the residual gradient, 1x1/s2 and 3x3/s2 gather dgrads) and on
    basic blocks.

    The reference takes the ReLU decisions of our fp32 forward (each of its ReLUs multiplies by our mask).  The fp32
    forward is accurate to ~1e-5 relative at the representation; at these batch sizes that still puts a few ReLU
    inputs on the other side of zero than float64 does, and each such flip moves a BatchNorm channel's gradient by a
    whole sample's share -- a property of the forward, which both backward precisions inherit.  With the decisions
    shared, what is left is the backward's arithmetic plus the forward's error in the saved conv outputs: each
    tensor must be within 2x the error of plain fp32 autograd given the same decisions, or 3e-4 of its largest entry
    (measured on an H100: at most 0.33x / 0.46x of max(fp32 autograd error, 3e-4)).  On the 16 blocks of a full
    ResNet-50 the forward's error (~10x fp32 autograd's) compounds: single BatchNorm biases reach 5-6x there
    (DESIGN.md §4), so ResNet-50 is not in this list."""
    from byol_b200.model import BYOL
    torch.manual_seed(31)
    g = torch.Generator().manual_seed(32)
    views = [torch.rand(b, 3, r, r, generator=g) for _ in range(2)]
    Rs = [torch.randn(b, 256, generator=g) for _ in range(2)]
    model = BYOL(rep, 256, 1000, 10, arch=arch, precision="fp32", backward_precision="fp32").cuda().train()
    sd = {k: v.cpu().clone() for k, v in model.state_dict().items()}
    eng = model._engine
    with torch.no_grad():
        model(views[0].cuda(), views[1].cuda())          # plan and weight layouts
    eng.prep_step(model.target_network.mean, True)
    saved = [{}, {}]
    eng.forward_lanes([v.cuda() for v in views], [(eng.theta, eng.w_online, s) for s in saved], True)
    eng.grad.zero_()
    eng._backward_group_split(saved, [None, None], [None, None], [R.cuda() for R in Rs])
    torch.cuda.synchronize()
    ours = {n: eng.grad[eng.offsets[id(p)]:eng.offsets[id(p)] + p.numel()].view(p.shape).double().cpu()
            for n, p in model.named_parameters()}
    kind = eng.blocks[0].kind
    masks = [_relu_masks(S, kind) for S in saved]
    refs = {}
    for dt in (torch.float64, torch.float32):
        ref = BYOL(rep, 256, 1000, 10, arch=arch)
        ref.load_state_dict(sd)
        ref = ref.to(dt).train()
        blocks = [blk for m in ref.base_network if isinstance(m, torch.nn.Sequential) for blk in m]
        for k in range(2):
            stem, bm, hm, pm = masks[k]
            ref.base_network[2] = _ForcedRelu([stem])
            for blk, ms in zip(blocks, bm):
                blk.relu = _ForcedRelu(ms)
            ref.head[2], ref.predictor[2] = _ForcedRelu([hm]), _ForcedRelu([pm])
            pred = ref.predictor(ref.head(ref.base_network(views[k].to(dt)).flatten(1)))
            (pred * Rs[k].to(dt)).sum().backward()
        refs[dt] = {n: p.grad for n, p in ref.named_parameters()}
    worst, checked = 0.0, 0
    scale = max(float(q.abs().max()) for q in refs[torch.float64].values() if q is not None)
    for n, q in refs[torch.float64].items():
        if q is None:
            assert float(ours[n].abs().max()) == 0.0, n
            continue
        q32 = refs[torch.float32][n]
        if float(q.abs().max()) < 1e-12 * scale:
            # zero by construction (a bias in front of a BatchNorm, or the projector's output bias, whose gradient
            # the predictor's BatchNorm sums to zero): rounding noise below 1e-6 of the largest gradient entry
            assert float(ours[n].abs().max()) <= 1e-6 * scale, n
            continue
        e, e32 = _rel(ours[n], q), _rel(q32, q)
        worst = max(worst, e / max(e32, 3e-4))
        checked += 1
        assert e <= max(2 * e32, 3e-4), (n, e, e32)
    print("%s %dx%d^2: %d tensors, worst error / max(fp32 autograd error, 3e-4) = %.2f" % (arch, b, r, checked, worst))


@pytest.mark.gpu
def test_fp32_backward_follows_reference_loss_curve(cuda):
    """20 steps (graphs on) against the reference's curve: first 5 within 5e-4, all within 2e-2, BYOL loss within
    2e-3 absolute."""
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    z = np.load(os.path.join(GOLDEN, "curve_rn18_b16_r64.npz"))
    arch, rep, b, r, steps, seed, lr, total = z["config"]
    rep, b, r, steps, seed, lr, total = int(rep), int(b), int(r), int(steps), int(seed), float(lr), int(total)
    torch.manual_seed(seed)
    model = BYOL(rep, 256, 1000, total, arch=str(arch), precision="fp32", backward_precision="fp32").cuda().train()
    opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(model, 1e-6), lr=lr, momentum=0.9), eps=0.0)
    data = [(a.cuda(), c.cuda(), l.cuda()) for a, c, l in _batches(seed, 4, b, r)]
    got, byol = [], []
    for s in range(steps):
        st = wiring.train_step(model, opt, *data[s % 4])
        got.append(float(st["loss_mean"]))
        byol.append(float(st["byol_loss_mean"]))
    assert any(v != "warm" for v in model._engine.graphs.values())
    dev = np.abs(np.array(got) / z["loss"] - 1.0)
    db = np.abs(np.array(byol) - z["byol_loss"]).max()
    print("fp32 backward loss curve: max rel dev first 5 %.2e, all %.2e; byol max abs dev %.2e" %
          (dev[:5].max(), dev.max(), db))
    assert dev[:5].max() < 5e-4 and dev.max() < 2e-2 and db < 2e-3


@pytest.mark.gpu
def test_fp32_backward_unusual_gradient_pattern_matches_fp64_autograd(cuda):
    """A loss on online_projection1 and online_representation2 only (no predictions): the captured step's backward
    graph does not cover it, so the eager kernels run over the graph's saved buffers.  Every parameter gradient
    equals a float64 CPU autograd run of the same torchvision modules (loaded from the model's state_dict)."""
    from byol_b200.model import BYOL
    torch.manual_seed(31)
    b, r = 8, 64
    kw = dict(arch="resnet18", precision="fp32", backward_precision="fp32")
    model = BYOL(512, 256, 1000, 10, **kw).cuda().train()
    g = torch.Generator().manual_seed(32)
    a1, a2 = torch.rand(b, 3, r, r, generator=g), torch.rand(b, 3, r, r, generator=g)
    R1, R2 = torch.randn(b, 256, generator=g), torch.randn(b, 512, generator=g)
    for _ in range(2):        # warm-up, then the capture: the third forward replays the graph
        out = model(a1.cuda(), a2.cuda())
        out["online_prediction1"].sum().backward()
    sd = {k: v.cpu() for k, v in model.state_dict().items()}
    model.zero_grad(set_to_none=True)
    out = model(a1.cuda(), a2.cuda())
    assert any(v != "warm" for v in model._engine.graphs.values())
    ((out["online_projection1"] * R1.cuda()).sum() + (out["online_representation2"] * R2.cuda()).sum()).backward()
    torch.cuda.synchronize()
    refs = {}
    for dt in (torch.float64, torch.float32):
        ref = BYOL(512, 256, 1000, 10, **kw)
        ref.load_state_dict(sd)
        ref = ref.to(dt).train()
        rep1 = ref.base_network(a1.to(dt)).flatten(1)
        rep2 = ref.base_network(a2.to(dt)).flatten(1)
        ((ref.head(rep1) * R1.to(dt)).sum() + (rep2 * R2.to(dt)).sum()).backward()
        refs[dt] = dict(ref.named_parameters())
    # BatchNorm over 8 images cancels heavily: plain fp32 autograd itself misses float64 by up to ~7e-2 on some
    # tensors here.  And a ReLU input within rounding of zero may fall on either side in any fp32 forward: after the
    # head's BatchNorm1d (8 samples x 4096 channels) one such input moves one channel's gradient by one sample's share
    # (measured: up to 15 % of a tensor's largest entry; test_fp32_mlp_backward_matches_fp64 checks the head alone on
    # identical inputs).  So: the whole gradient vector within 5e-2 relative L2, every tensor within 0.25.
    # A bias followed by BatchNorm has a gradient of exactly zero; only its size is checked.
    worst, scale = 0.0, max(float(q.grad.abs().max()) for q in refs[torch.float64].values() if q.grad is not None)
    ours, r64, r32 = [], [], []
    for name, p in model.named_parameters():
        q, q32 = refs[torch.float64][name], refs[torch.float32][name]
        if q.grad is None or float(q.grad.abs().max()) < 1e-9 * scale:
            assert p.grad is None or float(p.grad.abs().max()) < 1e-5 * scale, name
            continue
        e, e32 = _rel(p.grad, q.grad), _rel(q32.grad, q.grad)
        worst = max(worst, e)
        assert e < 0.25, (name, e, e32)
        ours.append(p.grad.detach().double().cpu().reshape(-1))
        r64.append(q.grad.detach().reshape(-1))
        r32.append(q32.grad.detach().double().reshape(-1))
    ours, r64, r32 = torch.cat(ours), torch.cat(r64), torch.cat(r32)
    l2, l2_32 = float((ours - r64).norm() / r64.norm()), float((r32 - r64).norm() / r64.norm())
    print("unusual gradient pattern vs float64: worst tensor %.2e, relative L2 %.2e (fp32 autograd %.2e)" %
          (worst, l2, l2_32))
    assert l2 < 5e-2, (l2, l2_32)


@pytest.mark.gpu
@pytest.mark.parametrize("b", [8, 64])
def test_fp32_mlp_backward_matches_fp64(cuda, b):
    """The projector's backward (Linear -> BatchNorm1d -> ReLU -> Linear) on the representation the fp32 forward
    produced, against float64 autograd of the same module on that same input: the input gradient and every parameter
    gradient within 1e-4 (the first bias, followed by BatchNorm, has a gradient of exactly zero)."""
    from byol_b200.model import BYOL
    torch.manual_seed(31)
    model = BYOL(512, 256, 1000, 10, arch="resnet18", precision="fp32", backward_precision="fp32").cuda().train()
    eng = model._engine
    g = torch.Generator().manual_seed(32)
    a = torch.rand(b, 3, 64, 64, generator=g).cuda()
    R = torch.randn(b, 256, generator=g)
    with torch.no_grad():
        model(a, a)                                  # plan and weight layouts
    saved = [{}, {}]
    eng.prep_step(model.target_network.mean, True)
    res, _ = eng.forward_lanes([a, a], [(eng.theta, eng.w_online, s) for s in saved], True)
    eng.grad.zero_()
    rep_g = eng._mlp_bwd_split(eng.mlps[0], [saved[0]["head"]], [R.cuda()])[0]
    torch.cuda.synchronize()
    head = model.head
    ref = torch.nn.Sequential(*[type(m)(*([m.in_features, m.out_features] if hasattr(m, "in_features") else
                                          [m.num_features] if hasattr(m, "num_features") else [])) for m in head])
    ref.load_state_dict({k: v.cpu() for k, v in head.state_dict().items()})
    ref = ref.double().train()
    x = res[0][0].detach().cpu().double().requires_grad_(True)
    (ref(x) * R.double()).sum().backward()
    errs = {"input": _rel(rep_g, x.grad)}
    for (name, p), q in zip(head.named_parameters(), ref.parameters()):
        off = eng.offsets[id(p)]
        gp = eng.grad[off:off + p.numel()].view(p.shape)      # the flat gradient (not attached outside autograd)
        if name == "0.bias":
            assert float(gp.abs().max()) < 1e-5
            continue
        errs[name] = _rel(gp, q.grad)
    print("fp32 MLP backward b=%d: %s" % (b, {k: "%.2e" % v for k, v in errs.items()}))
    assert max(errs.values()) < 1e-4, errs


@pytest.mark.gpu
def test_fp32_backward_graph_replay_is_bit_reproducible(cuda):
    """Bit-equal losses, theta, momentum, EMA target and BN running statistics eager/eager, graph/graph, eager/graph."""
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    arch, b, r = "resnet:bottleneck:1,1,1,1", 8, 64
    g = torch.Generator().manual_seed(3)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 1000, (b,), generator=g).cuda()) for _ in range(4)]
    res = {}
    for mode in ("eager", "eager2", "graph", "graph2"):
        torch.manual_seed(11)
        model = BYOL(2048, 256, 1000, 20, arch=arch, precision="fp32", backward_precision="fp32").cuda().train()
        model._engine.use_graphs = mode.startswith("graph")
        opt = wiring.build_optimizer(model, global_batch_size=256)
        losses = [wiring.train_step(model, opt, *bt)["loss_mean"].detach().clone() for bt in batches]
        torch.cuda.synchronize()
        captured = [v for v in model._engine.graphs.values() if v != "warm"]
        assert (len(captured) == 1) == mode.startswith("graph")
        sd = model.state_dict()
        res[mode] = {"loss": torch.stack(losses), "theta": model._engine.theta.clone(),
                     "momentum": _momentum_flat(model, opt), "target": model.target_network.mean.clone(),
                     "bn": torch.cat([v.reshape(-1).float() for k, v in sd.items() if "running_" in k])}
        model = opt = None
    for a, b_ in (("eager", "eager2"), ("graph", "graph2"), ("eager", "graph")):
        for key in res[a]:
            assert torch.equal(res[a][key], res[b_][key]), "%s differs between %s and %s" % (key, a, b_)


@pytest.mark.parametrize("precision", ["bf16", "bf16x2"])
def test_fp32_backward_needs_fp32_forward(precision):
    from byol_b200.model import BYOL
    with pytest.raises(ValueError, match="backward_precision"):
        BYOL(512, 256, 1000, 10, arch="resnet18", precision=precision, backward_precision="fp32")
    with pytest.raises(ValueError, match="backward_precision"):
        BYOL(512, 256, 1000, 10, arch="resnet18", precision="fp32", backward_precision="fp64")
    assert BYOL(512, 256, 1000, 10, arch="resnet18", precision="fp32").backward_precision == "bf16"


ARCH, REP, B, R, SEED, LR = "resnet:bottleneck:2,1,1,1", 2048, 8, 64, 41, 0.3


def _dist_worker(rank, world, port, ret, peer_xchg):
    import faulthandler
    faulthandler.dump_traceback_later(150, exit=True)
    os.environ["BYOL_B200_PEER_XCHG"] = "1" if peer_xchg else "0"
    import torch.distributed as dist
    import torch.nn as nn
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    torch.manual_seed(SEED)
    model = BYOL(REP, 256, 1000, 10, arch=ARCH, precision="fp32", backward_precision="fp32")
    model = nn.SyncBatchNorm.convert_sync_batchnorm(model).cuda().train()
    net = wiring.DistributedDataParallelPassthrough(model)
    opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(model, 1e-6), lr=LR, momentum=0.9), eps=0.0)
    g = torch.Generator().manual_seed(77)
    a1, a2 = torch.rand(world * B, 3, R, R, generator=g), torch.rand(world * B, 3, R, R, generator=g)
    lab = torch.randint(0, 1000, (world * B,), generator=g)
    sl = slice(rank * B, (rank + 1) * B)
    for _ in range(3):
        wiring.train_step(net, opt, a1[sl].cuda(), a2[sl].cuda(), lab[sl].cuda())
    torch.cuda.synchronize()
    sd = model.state_dict()
    ret[rank] = {"theta": model._engine.theta.cpu(), "ema": model.target_network.mean.cpu(),
                 "rm": sd["base_network.1.running_mean"].cpu()}
    dist.destroy_process_group()


@pytest.mark.gpu
@pytest.mark.parametrize("peer_xchg", [False, True], ids=["nccl-stats-eager", "peer-exchange-graphs"])
def test_fp32_backward_two_rank_syncbn(cuda, peer_xchg):
    """SyncBatchNorm over 2 ranks: the backward sums go through the same exchange as the forward statistics and the
    replicas stay bit-identical."""
    import torch.multiprocessing as mp
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ret = mp.Manager().dict()
    mp.spawn(_dist_worker, args=(2, 29644 + int(peer_xchg), ret, peer_xchg), nprocs=2, join=True)
    for key in ("theta", "ema", "rm"):
        assert torch.equal(ret[0][key], ret[1][key]), "replicas diverged (%s)" % key
