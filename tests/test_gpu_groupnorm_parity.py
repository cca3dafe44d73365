"""GPU parity of BYOL(norm="group_ws") against torch autograd of the same GroupNorm + WSConv2d model, with the engine's
bf16 storage points restated (straight-through bf16 rounding of every conv output, normalised activation, standardised
weight and head operand, fp32 arithmetic in between: oracle.byol_oracle.bf16_storage), as the BatchNorm parity tests
do with the oracle:

* teacher-forced blocks, each run forward and backward from its own saved input with the same upstream gradient:
  basic blocks (identity and stride-2 downsample), bottleneck blocks (identity with the residual gradient fused into
  the conv1 dgrad, and downsample), ResNeXt blocks; at the tests/test_gpu_blocks.py bars: forward l2 < 5e-3, input
  gradient l2 < 5e-2, every parameter gradient (the conv weights through the weight-standardisation backward, the
  GroupNorm affine parameters) cosine > 0.995 with a norm ratio in (0.97, 1.03);
* the whole four-lane BYOL step (online pair with the two-view concurrent backward, target pair on the EMA weights'
  own standardisation) of two shallow nets, ResNet-18 and ResNet-50 at 8 x 64 x 64: the BYOL loss within the band of
  tests/test_gpu_step.py (5e-2 relative + 2e-4) of the restatement, and the gradient and LARS update as close to fp32
  autograd (the restatement without its bf16 storage points) as the restatement itself is, within 0.02 in cosine.

Why that last bar and not "gradient cosine > 0.99, update cosine > 0.95 against the restatement" as for BatchNorm: the
first step's gradient of these GroupNorm + WS nets is not determined at bf16 precision.  The bf16 restatement, an
implementation independent of the engine, agrees with fp32 autograd only to gradient cosine 0.81 (bottleneck
2,1,1,1), 0.96 (basic 2,1,1,1), 0.88 (ResNet-18) and 0.00 (ResNet-50), measured on an H100; the engine lands within
0.01 of each (0.81, 0.96, 0.87, -0.01), and 0.92 / 0.98 / 0.93 / 0.15 against the restatement.  The same holds with
the target set equal to the online weights, so it is not the EMA initialisation.  The per-block comparison above is
where the engine's arithmetic is held to bf16-level bars.
"""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle.byol_oracle import bf16_storage

_STORAGE = [True]      # False: the same restatement without the bf16 storage points (plain fp32 autograd)


def q(t):
    return bf16_storage(t) if _STORAGE[0] else t

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _no_tf32():
    """The restatement runs in fp32 proper: no TF32 in cuDNN convolutions or matmuls (restored afterwards)."""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def _model(arch, d, seed=31):
    from byol_b200.model import BYOL
    torch.manual_seed(seed)
    return BYOL(d, 256, 1000, 10, arch=arch, norm="group_ws").cuda().train()


def _rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).norm() / (b.norm() + 1e-30))


def _cos(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return float((a @ b) / (a.norm() * b.norm() + 1e-30))


def _nchw(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


# ---- the restatement ----
def _conv_gn(conv, gn, x):
    y = q(F.conv2d(x, q(conv.standardized_weight()), None, conv.stride, conv.padding, 1, conv.groups))
    return F.group_norm(y, 32, gn.weight, gn.bias, gn.eps)


def _block(blk, x):
    a = q(torch.relu(_conv_gn(blk.conv1, blk.bn1, x)))
    z = _conv_gn(blk.conv2, blk.bn2, a)
    if hasattr(blk, "conv3"):
        z = _conv_gn(blk.conv3, blk.bn3, q(torch.relu(z)))
    idt = x if blk.downsample is None else _conv_gn(blk.downsample[0], blk.downsample[1], x)
    return q(torch.relu(z + idt))


def _encoder(base, x):
    ch = list(base.children())
    a = q(torch.relu(_conv_gn(ch[0], ch[1], x)))
    a = F.max_pool2d(a, ch[3].kernel_size, ch[3].stride, ch[3].padding)
    for layer in ch[4:-1]:
        for blk in layer.children():
            a = _block(blk, a)
    return a.mean((2, 3))


def _mlp(seq, x):
    l1, bn, _, l2 = list(seq.children())
    h = q(F.linear(q(x), q(l1.weight), l1.bias))
    a = q(torch.relu(F.batch_norm(h, None, None, bn.weight, bn.bias, True, 0.0, bn.eps)))
    return F.linear(a, q(l2.weight), l2.bias)


def _blocks_of(model):
    return [blk for layer in list(model.base_network.children())[4:-1] for blk in layer.children()]


# ---- teacher-forced blocks ----
@pytest.mark.parametrize("arch,rep", [("resnet:bottleneck:2,1,1,1", 2048), ("resnet:basic:2,1,2,1", 512),
                                      ("resnext:32x4:2,1,1,1", 2048)])
def test_blocks_teacher_forced(cuda, arch, rep):
    from byol_b200 import engine as E, ops
    b, r = 16, 64
    model = _model(arch, rep)
    eng = model._ensure_ready(b)
    eng.prep_weights(eng.theta, eng.w_online, want_dgrad=True)
    a1 = torch.rand(b, 3, r, r, generator=torch.Generator().manual_seed(3)).cuda()
    saved = {}
    with torch.no_grad():
        eng.forward_lanes([a1], [(eng.theta, eng.w_online, saved)], True)
    routes = set()
    for bi, blk in enumerate(_blocks_of(model)):
        S, eb = saved["blocks"][bi], eng.blocks[bi]
        routes.add((eb.kind, eb.down is not None, eb.down is None and eb.c1.k == 1))
        g_out = torch.randn(S["out"].shape, generator=torch.Generator().manual_seed(100 + bi)).to(torch.bfloat16)
        eng.grad.zero_()
        eng.w_online.ws_grad.zero_()
        eng._bpool = E._Pool(2 * eng.bn_channels, eng.device, zero=True)
        g_in = eng._block_bwd(eb, [S], [g_out.cuda()])[0]
        eng._join_side_stream()
        w = eng.w_online
        ops.ws_bwd(w.ws_grad, w.ws_w, w.ws_stats, eng.ws_desc, eng.ws_rows, eng.grad)
        torch.cuda.synchronize()
        ref = copy.deepcopy(blk).float()
        x = _nchw(S["x"]).requires_grad_(True)
        out = _block(ref, x)
        out.backward(_nchw(g_out.cuda()))
        ef, eg = _rel_l2(_nchw(S["out"]), out), _rel_l2(_nchw(g_in), x.grad)
        print("block %d (%s, down %s) fwd l2 %.2e  g_in l2 %.2e" % (bi, eb.kind, eb.down is not None, ef, eg))
        assert ef < 5e-3 and eg < 5e-2, (bi, ef, eg)
        for (name, p), (_, pr) in zip(blk.named_parameters(), ref.named_parameters()):
            off = eng.offsets[id(p)]
            got = eng.grad[off:off + p.numel()]
            c = _cos(got, pr.grad)
            ratio = float(got.double().norm().cpu() / pr.grad.double().norm().cpu())
            assert c > 0.995 and 0.97 < ratio < 1.03, (bi, name, c, ratio)
    # every residual route of the net ran: identity and downsample, and for bottlenecks the fused residual gradient
    if "bottleneck" in arch or "resnext" in arch:
        assert ("bottleneck", False, True) in routes and ("bottleneck", True, False) in routes
    else:
        assert ("basic", False, False) in routes and ("basic", True, False) in routes


# ---- the whole BYOL step ----
@pytest.mark.parametrize("arch,rep", [("resnet:bottleneck:2,1,1,1", 2048), ("resnet:basic:2,1,1,1", 512),
                                      ("resnet18", 512), ("resnet50", 2048)])
def test_byol_step_against_torch_autograd(cuda, arch, rep):
    from byol_b200.lars import LARS
    from byol_b200.objective import loss_function, regression_loss
    from byol_b200.wiring import add_weight_decay
    b, r, lr = 8, 64, 0.3
    model = _model(arch, rep, seed=7)
    online = torch.nn.ModuleList([copy.deepcopy(model.base_network), copy.deepcopy(model.head),
                                  copy.deepcopy(model.predictor)]).float()
    target = copy.deepcopy(online)
    n = sum(p.numel() for p in online.parameters())
    torch.nn.utils.vector_to_parameters(model.target_network.mean[:n].clone().cuda(), target.parameters())
    theta0 = torch.nn.utils.parameters_to_vector(model.parameters()).detach().clone().cuda()
    g = torch.Generator().manual_seed(99)
    a1, a2 = torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda()

    opt = LARS(torch.optim.SGD(add_weight_decay(model, 1e-6), lr=lr, momentum=0.9), eps=0.0)
    out = model(a1, a2)
    loss = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                         target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
    opt.zero_grad()
    loss.backward()
    grad = model._engine.grad[:n].clone()
    opt.step()
    upd = model._engine.theta[:n] - theta0[:n]

    def lane(net, x):
        rep_ = _encoder(net[0], x.bfloat16().float())
        proj = _mlp(net[1], rep_)
        return proj, _mlp(net[2], proj)

    def reference(storage):
        _STORAGE[0] = storage
        try:
            net = copy.deepcopy(online)
            with torch.no_grad():
                tp1, _ = lane(target, a1)
                tp2, _ = lane(target, a2)
            _, p1 = lane(net, a1)
            _, p2 = lane(net, a2)
            ref_loss = (regression_loss(p1, tp2) + regression_loss(p2, tp1)).mean()
            ref_loss.backward()
        finally:
            _STORAGE[0] = True
        ref_grad = torch.cat([p.grad.reshape(-1) for p in net.parameters()])
        # the same LARS step on a twin model fed this gradient
        twin = _model(arch, rep, seed=7)
        eng2 = twin._ensure_ready(b)
        eng2.attach_grads()
        eng2.grad[:n].copy_(ref_grad)
        LARS(torch.optim.SGD(add_weight_decay(twin, 1e-6), lr=lr, momentum=0.9), eps=0.0).step()
        return ref_loss.item(), ref_grad, eng2.theta[:n] - theta0[:n]

    q_loss, q_grad, q_upd = reference(True)
    f_loss, f_grad, f_upd = reference(False)
    torch.cuda.synchronize()
    gc, uc = _cos(grad, q_grad), _cos(upd, q_upd)
    gf, qf = _cos(grad, f_grad), _cos(q_grad, f_grad)
    uf, quf = _cos(upd, f_upd), _cos(q_upd, f_upd)
    print("%s: loss %.6f (restated %.6f, fp32 %.6f); engine against the restatement: gradient cosine %.5f, update "
          "cosine %.5f; against fp32 (engine / restatement): gradient %.5f / %.5f, update %.5f / %.5f"
          % (arch, loss.item(), q_loss, f_loss, gc, uc, gf, qf, uf, quf))
    assert abs(loss.item() - q_loss) < 5e-2 * abs(q_loss) + 2e-4
    assert gf >= qf - 0.02 and uf >= quf - 0.02
