"""GPU: GroupNorm and weight standardisation (BYOL(norm="group_ws"), csrc/groupnorm.cu).

* Weight standardisation at the real fan-ins: (mean, rstd) and w^ within one fp32 ulp of float64 (each is an fp64
  value rounded once), the same bits on every run; its backward against float64 autograd of the WSConv2d formula.
* GroupNorm statistics: the sums equal the float64 sums of the bf16 inputs to the fixed-point resolution (2^-50 per
  block partial), (mean, rstd) within one fp32 ulp of float64.  Apply (plain, residual, GroupNorm-applied residual,
  mask bits) and the fused stem kernel bit for bit against a restatement of their fp32 arithmetic, and within one bf16
  ulp of float64 rounded once.  The backward against float64 autograd of F.group_norm in every mask mode.
* Whole nets: one encoder step (the fine-tune step) of ResNet-18, a bottleneck net and a ResNeXt net against fp32
  torch autograd of the same GroupNorm + WSConv2d encoder; a BYOL step's graph replay bit-equal to eager, two runs
  bit-equal; representations() equal to the eval forward's and independent of the rest of the batch (64 and 224 px).
* The recompute refusal names the batch size; FineTune.step runs on a GroupNorm model.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

F32U = 2.0 ** -23


def _bits(t):
    return t.detach().contiguous().view(torch.int32).cpu() if t.dtype == torch.float32 else \
        t.detach().contiguous().view(torch.int16).cpu()


def _ws_desc(shapes, cuda):
    """(desc, rows, numel) for weights of `shapes` [(cout, fan_in)] laid out back to back in flat and in the scratch."""
    rows, off, row0 = [], 0, 0
    for cout, fan in shapes:
        rows.append([off, off, cout, fan, row0])
        off += cout * fan
        row0 += cout
    return torch.tensor(rows, dtype=torch.int64, device=cuda), row0, off


# stem 3*7*7, 1x1 convs 64 / 256 / 1024 / 2048, 3x3 convs 64*9 / 512*9, grouped 3x3 (4 and 8 channels per group)
FAN_INS = [147, 64, 256, 576, 1024, 2048, 4608, 36, 72]


def test_ws_fwd_against_float64_and_run_to_run(cuda):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(0)
    shapes = [(64 if f != 4608 else 16, f) for f in FAN_INS]
    desc, rows, numel = _ws_desc(shapes, cuda)
    flat = (torch.randn(numel, generator=g) * 0.05 + 0.01).cuda()
    out = torch.empty(numel, dtype=torch.float32, device=cuda)
    stats = torch.empty((rows, 2), dtype=torch.float32, device=cuda)
    ops.ws_fwd(flat, desc, rows, out, stats)
    out2, stats2 = torch.empty_like(out), torch.empty_like(stats)
    ops.ws_fwd(flat, desc, rows, out2, stats2)
    torch.cuda.synchronize()
    assert torch.equal(_bits(out), _bits(out2)) and torch.equal(_bits(stats), _bits(stats2))
    off, r0 = 0, 0
    for cout, fan in shapes:
        w = flat[off:off + cout * fan].double().cpu().view(cout, fan)
        mean = w.mean(1, keepdim=True)
        var = ((w - mean) ** 2).mean(1, keepdim=True)
        rstd = 1.0 / torch.sqrt(var + 1e-5)
        wh = (w - mean) * rstd
        got = out[off:off + cout * fan].double().cpu().view(cout, fan)
        st = stats[r0:r0 + cout].double().cpu()
        # one rounding of an fp64 value: within one fp32 ulp (half an ulp plus the fp64 sums' error)
        assert ((got - wh).abs() <= F32U * wh.abs() + 1e-30).all(), fan
        assert ((st[:, 0] - mean[:, 0]).abs() <= F32U * mean[:, 0].abs()).all(), fan
        assert ((st[:, 1] - rstd[:, 0]).abs() <= F32U * rstd[:, 0]).all(), fan
        off += cout * fan
        r0 += cout


def test_ws_bwd_against_float64_autograd(cuda):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(1)
    shapes = [(32, f) for f in (147, 64, 576, 36, 4608)]
    desc, rows, numel = _ws_desc(shapes, cuda)
    flat = (torch.randn(numel, generator=g) * 0.05).cuda()
    dwh = torch.randn(numel, generator=g).cuda()
    wh = torch.empty_like(flat)
    stats = torch.empty((rows, 2), dtype=torch.float32, device=cuda)
    ops.ws_fwd(flat, desc, rows, wh, stats)
    base = torch.randn(numel, generator=g).cuda()
    grad = base.clone()
    ops.ws_bwd(dwh, wh, stats, desc, rows, grad)
    grad2 = base.clone()
    ops.ws_bwd(dwh, wh, stats, desc, rows, grad2)
    torch.cuda.synchronize()
    assert torch.equal(_bits(grad), _bits(grad2))
    off = 0
    for cout, fan in shapes:
        w = flat[off:off + cout * fan].double().cpu().view(cout, fan).requires_grad_(True)
        mean = w.mean(1, keepdim=True)
        var = w.var(1, unbiased=False, keepdim=True)
        ((w - mean) / torch.sqrt(var + 1e-5) * dwh[off:off + cout * fan].double().cpu().view(cout, fan)).sum().backward()
        ref = w.grad + base[off:off + cout * fan].double().cpu().view(cout, fan)
        got = grad[off:off + cout * fan].double().cpu().view(cout, fan)
        err = float((got - ref).abs().max() / ref.abs().max())
        assert err < 1e-5, (fan, err)
        off += cout * fan


SHAPES = [(3, 8, 8, 64), (2, 7, 7, 2048), (2, 9, 5, 96), (4, 14, 14, 256), (1, 4, 4, 4096)]


def _bf16(shape, g, scale=1.0, shift=0.0):
    return (torch.randn(shape, generator=g) * scale + shift).bfloat16()


def _gn_ref(y64, eps=1e-5):
    n, c = y64.shape[0], y64.shape[-1]
    v = y64.reshape(n, -1, 32, c // 32)
    s = v.sum((1, 3))
    q = (v * v).sum((1, 3))
    m = v.shape[1] * v.shape[3]
    mean = s / m
    var = (q / m - mean * mean).clamp_min(0)
    return s, q, mean, 1.0 / torch.sqrt(var + eps)


@pytest.mark.parametrize("shape", SHAPES)
def test_gn_stats(cuda, shape):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(2)
    y = _bf16(shape, g, 1.5, 0.3)
    sums = torch.empty((shape[0], 32, 2), dtype=torch.float64, device=cuda)
    st = ops.gn_stats(y.cuda(), 1e-5, sums64=sums)
    st2 = ops.gn_stats(y.cuda(), 1e-5)
    torch.cuda.synchronize()
    assert torch.equal(_bits(st), _bits(st2))
    s, q, mean, rstd = _gn_ref(y.double())
    tol = 2.0 ** -50 * (y.numel() // 8 + 1)
    assert (sums[..., 0].cpu() - s).abs().max() <= tol
    assert (sums[..., 1].cpu() - q).abs().max() <= tol
    st = st.double().cpu()
    assert ((st[..., 0] - mean).abs() <= F32U * mean.abs() + 1e-12).all()
    assert ((st[..., 1] - rstd).abs() <= F32U * rstd).all()


def _fma32(a, b, c):
    """fp32 fma: the fp64 product of two fp32 values is exact, the sum rounds at 2^-53, then once to fp32."""
    return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(np.float32)


def _coeffs(gamma, beta, st, c):
    """scale / shift [n, c] as the kernel forms them: sc = fl(gamma*rstd), sh = fma(-mean, sc, beta)."""
    grp = np.arange(c) // (c // 32)
    mean, rstd = st[:, grp, 0], st[:, grp, 1]
    sc = (gamma[None, :] * rstd).astype(np.float32)
    return sc, _fma32(-mean, sc, np.broadcast_to(beta[None, :], sc.shape))


def _to_bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).bfloat16()


@pytest.mark.parametrize("shape", SHAPES[:4])
@pytest.mark.parametrize("mode", ["plain", "resid", "down"])
def test_gn_apply_exact(cuda, shape, mode):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(3)
    n, h, w, c = shape
    x = _bf16(shape, g, 2.0, 0.5)
    r = _bf16(shape, g, 1.0, -0.2)
    gamma, beta = (torch.randn(c, generator=g) * 0.5 + 1).float(), (torch.randn(c, generator=g) * 0.3).float()
    rgamma, rbeta = (torch.randn(c, generator=g) * 0.5 + 1).float(), (torch.randn(c, generator=g) * 0.3).float()
    xc, rc = x.cuda(), r.cuda()
    st, rst = ops.gn_stats(xc, 1e-5), ops.gn_stats(rc, 1e-5)
    rgn = (rgamma.cuda(), rbeta.cuda(), rst) if mode == "down" else None
    mask = torch.empty(x.numel() // 8, dtype=torch.uint8, device=cuda)
    y = ops.gn_apply(xc, gamma.cuda(), beta.cuda(), st, True, resid=None if mode == "plain" else rc, rgn=rgn,
                     mask_out=mask)
    torch.cuda.synchronize()
    sc, sh = _coeffs(gamma.numpy(), beta.numpy(), st.cpu().numpy(), c)
    xv = x.float().numpy().reshape(n, -1, c)
    o = _fma32(xv, sc[:, None, :], sh[:, None, :])
    o64 = xv.astype(np.float64) * sc[:, None, :] + sh[:, None, :]
    if mode != "plain":
        rv = r.float().numpy().reshape(n, -1, c)
        if mode == "down":
            rs, rb = _coeffs(rgamma.numpy(), rbeta.numpy(), rst.cpu().numpy(), c)
            add = _fma32(rv, rs[:, None, :], rb[:, None, :])
            o64 = o64 + rv.astype(np.float64) * rs[:, None, :] + rb[:, None, :]
        else:
            add = rv
            o64 = o64 + rv
        o = (o + add).astype(np.float32)
    o = np.maximum(o, np.float32(0))
    ref = _to_bf16(o).view(shape)
    assert torch.equal(_bits(y), _bits(ref)), "gn_apply differs from its fp32 restatement"
    bits = np.packbits((o.reshape(-1, 8) > 0).astype(np.uint8), axis=1, bitorder="little").reshape(-1)
    assert np.array_equal(mask.cpu().numpy(), bits)
    # against float64 rounded once: at most one bf16 ulp apart
    r64 = _to_bf16(np.maximum(o64, 0)).view(shape).float()
    ulp = 2.0 ** (torch.floor(torch.log2(r64.abs().clamp_min(1e-30))) - 7)
    assert ((y.float().cpu() - r64).abs() <= ulp).all()


@pytest.mark.parametrize("want_idx", [True, False])
def test_gn_relu_maxpool_equals_apply_then_pool(cuda, want_idx):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(4)
    x = _bf16((2, 16, 14, 64), g, 1.0, 0.0).cuda()
    gamma, beta = (torch.randn(64, generator=g) + 1).cuda(), (torch.randn(64, generator=g) * 0.5).cuda()
    st = ops.gn_stats(x, 1e-5)
    y, idx = ops.gn_relu_maxpool_fwd(x, gamma, beta, st, 3, 2, 1, want_idx=want_idx)
    a = ops.gn_apply(x, gamma, beta, st, True)
    y2, i2 = ops.maxpool_fwd(a, 3, 2, 1, want_idx=True)
    torch.cuda.synchronize()
    assert torch.equal(_bits(y), _bits(y2))
    if want_idx:
        assert torch.equal(idx, i2)


@pytest.mark.parametrize("shape", [(3, 8, 8, 64), (2, 7, 7, 2048), (2, 9, 5, 96), (4, 14, 14, 256)])
@pytest.mark.parametrize("mask_mode", [0, 1, 2, 3])
def test_gn_backward_against_float64_autograd(cuda, shape, mask_mode):
    from byol_b200 import ops
    g = torch.Generator().manual_seed(5)
    n, h, w, c = shape
    x = _bf16(shape, g, 1.0, 0.2)
    gr = _bf16(shape, g, 1.0, 0.0)
    gamma, beta = (torch.randn(c, generator=g) * 0.5 + 1).float(), (torch.randn(c, generator=g) * 0.3).float()
    xc, gc = x.cuda(), gr.cuda()
    st = ops.gn_stats(xc, 1e-5)
    act = None
    if mask_mode == 3:
        act = torch.randint(0, 256, (x.numel() // 8,), generator=g, dtype=torch.uint8)
        keep = torch.from_numpy(np.unpackbits(act.numpy(), bitorder="little").astype(bool)).view(shape)
        act = act.cuda()
    elif mask_mode == 2:
        act = _bf16(shape, g).cuda()
        keep = act.float().cpu() > 0
    dgamma = torch.zeros(c, device=cuda)
    dbeta = torch.zeros(c, device=cuda)
    s12 = torch.zeros((n, 32, 2), device=cuda)
    ops.gn_bwd_reduce(gc, xc, gamma.cuda(), beta.cuda(), st, s12, mask_mode, act=act, dgamma=dgamma, dbeta=dbeta)
    dz = torch.empty_like(xc)
    dy = ops.gn_bwd_apply(gc, xc, gamma.cuda(), beta.cuda(), st, s12, mask_mode, act=act, dz_out=dz)
    dy2 = ops.gn_bwd_apply(gc, xc, gamma.cuda(), beta.cuda(), st, s12, mask_mode, act=act)
    torch.cuda.synchronize()
    assert torch.equal(_bits(dy), _bits(dy2))
    x64 = x.double().permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    g64, b64 = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
    z = F.group_norm(x64, 32, g64, b64, 1e-5)
    gg = gr.double().permute(0, 3, 1, 2)
    if mask_mode == 1:
        z = torch.relu(z)
    elif mask_mode in (2, 3):
        gg = gg * keep.permute(0, 3, 1, 2).double()
    (z * gg).sum().backward()
    ref_dy = x64.grad.permute(0, 2, 3, 1)
    rel = lambda a, b: float((a.double().cpu() - b).norm() / b.norm())
    assert rel(dy, ref_dy) < 1e-2, rel(dy, ref_dy)
    assert rel(dgamma, g64.grad) < 1e-4 and rel(dbeta, b64.grad) < 1e-4
    if mask_mode == 0:
        assert torch.equal(_bits(dz), _bits(gc))


# ---- whole nets ----
NETS = [("resnet18", 512, 8), ("resnet:bottleneck:1,1,1,1", 2048, 8), ("resnext:32x4:1,1,1,1", 2048, 8)]


def _model(arch, d, classes=10):
    from byol_b200.model import BYOL
    torch.manual_seed(21)
    return BYOL(d, 64, classes, 10, arch=arch, head_latent_size=128, norm="group_ws").cuda().train()


def _cos(a, b):
    a, b = a.double().flatten().cpu(), b.double().flatten().cpu()
    return float(a @ b / (a.norm() * b.norm()))


@pytest.mark.parametrize("arch,d,b", NETS)
def test_encoder_step_against_fp32_autograd(cuda, arch, d, b):
    """One fine-tune step (the engine's one-lane forward and backward through every GroupNorm / WS kernel) against torch
    fp32 autograd of the GroupNorm + WSConv2d encoder: loss within 1e-2; the gradient cosine of the whole encoder (within
    0.01), of every conv and of all GroupNorm parameters together (within 0.02) as close as torch's own bf16 autocast
    gets, and at least 0.9.  The bf16 forward alone moves the features by a few percent on these random-init nets, so
    the bar is autocast's, as in tests/test_gpu_finetune.py."""
    import copy
    from byol_b200.finetune import FineTune
    model = _model(arch, d)
    C = 5
    ft = FineTune(model, C, 0.1, seed=2)
    W = ft.classifier_weight.clone().requires_grad_(True)
    bias = ft.classifier_bias.clone().requires_grad_(True)
    ref = copy.deepcopy(ft.model.base_network).float()
    for p in ref.parameters():
        p.data = p.data.clone()
    ref_ac = copy.deepcopy(ref)
    g = torch.Generator().manual_seed(6)
    x = torch.rand(b, 3, 64, 64, generator=g).cuda()
    lab = torch.randint(0, C, (b,), generator=g).cuda()
    loss_sum, _ = ft.gradients(x, lab)
    xb = x.bfloat16().float()

    def run(net, autocast):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            f = net(xb).flatten(1).float()
        loss = F.cross_entropy(f @ W.t() + bias, lab)
        loss.backward()
        return loss.item(), [p.grad.clone() for p in net.parameters()]

    ref_loss, ref_g = run(ref, False)
    _, ac_g = run(ref_ac, True)
    torch.cuda.synchronize()
    loss = loss_sum.item() / b
    assert abs(loss - ref_loss) <= 1e-2 * abs(ref_loss), (loss, ref_loss)
    eng = ft.eng
    n_enc = sum(p.numel() for p in ref.parameters())
    whole = _cos(eng.grad[:n_enc], torch.cat([t.reshape(-1) for t in ref_g]))
    whole_ac = _cos(torch.cat([t.reshape(-1) for t in ac_g]), torch.cat([t.reshape(-1) for t in ref_g]))
    print("%s: whole-encoder gradient cosine %.4f (torch autocast %.4f)" % (arch, whole, whole_ac))
    assert whole >= 0.9 and whole >= whole_ac - 0.01
    off, mine_gn, ref_gn, ac_gn = 0, [], [], []
    for (name, p), t, t_ac in zip(ref.named_parameters(), ref_g, ac_g):
        if p.dim() == 4:
            c, c_ac = _cos(eng.grad[off:off + p.numel()], t), _cos(t_ac, t)
            assert c >= 0.9 and c >= c_ac - 0.02, (name, c, c_ac)
        else:
            mine_gn.append(eng.grad[off:off + p.numel()])
            ref_gn.append(t.reshape(-1))
            ac_gn.append(t_ac.reshape(-1))
        off += p.numel()
    c, c_ac = _cos(torch.cat(mine_gn), torch.cat(ref_gn)), _cos(torch.cat(ac_gn), torch.cat(ref_gn))
    print("%s: GroupNorm parameter gradient cosine %.4f (torch autocast %.4f)" % (arch, c, c_ac))
    assert c >= 0.9 and c >= c_ac - 0.02


def _byol_steps(arch, d, b, steps, graphs, seed=0):
    from byol_b200.lars import LARS
    from byol_b200.objective import loss_function
    from byol_b200.wiring import add_weight_decay
    model = _model(arch, d)
    model._engine.use_graphs = graphs
    opt = LARS(torch.optim.SGD(add_weight_decay(model, 1e-6), lr=0.1, momentum=0.9), eps=0.0)
    g = torch.Generator().manual_seed(seed)
    outs = []
    for _ in range(steps):
        a1, a2 = torch.rand(b, 3, 64, 64, generator=g).cuda(), torch.rand(b, 3, 64, 64, generator=g).cuda()
        out = model(a1, a2)
        loss = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                             target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
        opt.zero_grad()
        loss.backward()
        opt.step()
        outs.append(loss.detach().clone())
    torch.cuda.synchronize()
    return model, torch.stack(outs)


def test_byol_step_graph_replay_equals_eager_and_runs_repeat(cuda):
    eager, l_e = _byol_steps("resnet18", 512, 8, 4, graphs=False)
    graphed, l_g = _byol_steps("resnet18", 512, 8, 4, graphs=True)
    again, l_a = _byol_steps("resnet18", 512, 8, 4, graphs=True)
    from byol_b200.engine import _GraphedStep
    assert any(isinstance(v, _GraphedStep) for v in graphed._engine.graphs.values())
    assert torch.isfinite(l_e).all()
    assert torch.equal(_bits(l_e), _bits(l_g)) and torch.equal(_bits(l_g), _bits(l_a))
    for m in (graphed, again):
        assert torch.equal(_bits(m._engine.theta), _bits(eager._engine.theta))
        assert torch.equal(_bits(m.target_network.mean), _bits(eager.target_network.mean))


def test_representations_are_batch_independent(cuda):
    """An image's representation has the same bits alone and inside a batch of 64 (the fprop kernels accumulate each
    output element in an order that does not depend on the image count), and representations() has the bits of the
    eval forward."""
    model = _model("resnet:bottleneck:1,1,1,1", 2048)
    g = torch.Generator().manual_seed(7)
    x = torch.rand(64, 3, 64, 64, generator=g).cuda()
    model.eval()
    with torch.no_grad():
        out = model(x[:8], x[8:16])
    rep = model.representations(x[:8])
    torch.cuda.synchronize()
    assert torch.equal(_bits(rep), _bits(out["online_representation1"]))
    full = model.representations(x)
    for i in (0, 5, 63):
        alone = model.representations(x[i:i + 1])
        assert torch.equal(_bits(alone[0]), _bits(full[i])), i
    tgt = model.representations(x[:8], network="target")
    assert torch.equal(_bits(tgt), _bits(out["target_representation1"]))


def test_batch_independence_at_224(cuda):
    """At 224 px the statistics pass splits each stem output over many blocks; the split depends on the image's shape
    only, so an image's representation has the same bits alone and inside a batch of 16."""
    model = _model("resnet:bottleneck:1,1,1,1", 2048)
    x = torch.rand(16, 3, 224, 224, generator=torch.Generator().manual_seed(8)).cuda()
    full = model.representations(x)
    for i in (0, 15):
        alone = model.representations(x[i:i + 1])
        assert torch.equal(_bits(alone[0]), _bits(full[i])), i


def test_recompute_is_refused_with_the_batch_size(cuda):
    """A GroupNorm net that would have to recompute activations raises instead, naming the batch size."""
    model = _model("resnet18", 512)
    model._engine._mem_budget = 0          # nothing fits: the planner would recompute every block
    g = torch.Generator().manual_seed(9)
    a1, a2 = torch.rand(4, 3, 64, 64, generator=g).cuda(), torch.rand(4, 3, 64, 64, generator=g).cuda()
    with pytest.raises(RuntimeError, match="at 4 images per view"):
        model(a1, a2)
    model._engine._mem_budget = None
    out = model(a1, a2)                    # the refusal left the engine usable
    torch.cuda.synchronize()
    assert torch.isfinite(out["online_prediction1"]).all()


def test_finetune_step_runs(cuda):
    """FineTune.step (gradients + the Nesterov-SGD update) on a GroupNorm model: finite loss, the encoder and the
    classifier move, every GroupNorm layer among them."""
    from byol_b200.finetune import FineTune
    model = _model("resnet18", 512)
    ft = FineTune(model, 5, 0.1, seed=3)
    n_enc = sum(p.numel() for p in ft.model.base_network.parameters())
    before = ft.eng.theta.clone()
    g = torch.Generator().manual_seed(10)
    x = torch.rand(8, 3, 64, 64, generator=g).cuda()
    lab = torch.randint(0, 5, (8,), generator=g).cuda()
    loss = ft.step(x, lab, 1.0)
    torch.cuda.synchronize()
    assert torch.isfinite(loss).all()
    moved = (ft.eng.theta != before)
    assert moved[:n_enc].float().mean() > 0.9
    u = ft.eng.cls
    assert moved[u.w_off:u.w_off + u.w_numel].all()
    # every GroupNorm layer's affine parameters move (single entries may not: an update below half an ulp of 1.0)
    for m in ft.model.base_network.modules():
        if isinstance(m, torch.nn.GroupNorm):
            for p in (m.weight, m.bias):
                off = ft.eng.offsets[id(p)]
                assert moved[off:off + p.numel()].any()
