"""GPU: grouped 3x3 convolutions (ResNeXt conv2) on the block-diagonal tile kernels, from single kernels to whole
training steps.

Kernel parity runs on bf16-representable inputs against float64 grouped convolutions, at the tolerances
tests/test_gpu_conv.py holds the dense kernels to.  The block and step tests reuse the criteria of
tests/test_gpu_blocks.py and tests/test_gpu_step.py.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ops_ref as R
from tests import resnext_oracle
from tests.util import assert_close

pytestmark = pytest.mark.gpu

CGS = [4, 8, 16, 32, 64]
# (H, stride, N): stride 1 at 56 / 28 (patch kernel) and 14 / 7 (gather), stride 2 from 56, 28 and 14
MAPS = [(56, 1, 2), (28, 1, 2), (14, 1, 4), (7, 1, 8), (56, 2, 2), (28, 2, 2), (14, 2, 4)]
C = 128


def _mk(n, h, c, cg, stride, dev, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = R.bf16_round(torch.randn(n, c, h, h, generator=g))
    w = R.bf16_round(torch.randn(c, cg, 3, 3, generator=g) / (cg * 9) ** 0.5)
    ho = (h - 1) // stride + 1
    dy = R.bf16_round(torch.randn(n, c, ho, ho, generator=g))
    return x, w, dy


def _nhwc(t, dev):
    return t.permute(0, 2, 3, 1).contiguous().to(dev, torch.bfloat16)


def _refs(x, w, dy, stride):
    """float64 grouped conv and its autograd input / weight gradients (NHWC outputs)."""
    g = x.shape[1] // w.shape[1]
    xd = x.double().requires_grad_(True)
    wd = w.double().requires_grad_(True)
    y = F.conv2d(xd, wd, None, stride, 1, 1, g)
    y.backward(dy.double())
    return (y.detach().permute(0, 2, 3, 1), xd.grad.permute(0, 2, 3, 1), wd.grad)


def _cases():
    out = [(cg, h, s, n, C) for cg in CGS for (h, s, n) in MAPS]
    # C = 192 is not a multiple of the 128-wide wgrad tiles: the second chunk of the last tile lies past C
    out += [(32, 28, 1, 2, 192), (16, 14, 2, 2, 192)]
    return out


CASES = _cases()
IDS = ["cg%d_h%d_s%d_c%d" % (cg, h, s, c) for cg, h, s, n, c in CASES]


@pytest.mark.parametrize("cg,h,stride,n,c", CASES, ids=IDS)
def test_grouped_kernels_match_float64(cuda, cg, h, stride, n, c):
    from byol_b200 import ops
    x, w, dy = _mk(n, h, c, cg, stride, cuda)
    yref, dxref, dwref = _refs(x, w, dy, stride)
    wf, wdg = ops.prep_weight_grouped(w.to(cuda))
    assert wf.shape == (c // 64, 64, 576) and wdg.shape == (c // 64, 64, 576)
    xd, dyd = _nhwc(x, cuda), _nhwc(dy, cuda)
    # fprop with fused BatchNorm statistics
    stats = torch.zeros(2 * c, device=cuda)
    y = ops.conv_fprop(xd, wf, 3, 3, stride, 1, stats=stats)
    torch.cuda.synchronize()
    scale = float(yref.abs().max())
    assert_close("gfprop", y, yref, atol=1e-2 * scale, rtol=0)
    yr = y.float().cpu().reshape(-1, c)
    assert_close("gfprop_sum", stats[:c], yr.sum(0), atol=1e-3 * yr.abs().sum(0).max().item(), rtol=0)
    assert_close("gfprop_sq", stats[c:], (yr * yr).sum(0), atol=0, rtol=1e-3)
    # dgrad
    dx = ops.conv_dgrad(dyd, wdg, h, h, 3, 3, stride, 1)
    torch.cuda.synchronize()
    assert_close("gdgrad", dx, dxref, atol=1e-2 * float(dxref.abs().max()), rtol=0)
    # wgrad into a guarded buffer: += semantics, and nothing outside the [C, Cg, 3, 3] slice is touched
    guard = 4096
    buf = torch.full((guard + c * cg * 9 + guard,), 7.0, device=cuda)
    dw = buf[guard:guard + c * cg * 9].view(c, cg, 3, 3)
    dw.zero_()
    ops.conv_wgrad(xd, dyd, dw, 3, 3, stride, 1)
    torch.cuda.synchronize()
    assert_close("gwgrad", dw, dwref, atol=2e-3 * float(dwref.abs().max()), rtol=0)
    ops.conv_wgrad(xd, dyd, dw, 3, 3, stride, 1)
    torch.cuda.synchronize()
    assert_close("gwgrad_acc", dw, 2 * dwref, atol=4e-3 * float(dwref.abs().max()), rtol=0)
    assert bool((buf[:guard] == 7.0).all()) and bool((buf[guard + c * cg * 9:] == 7.0).all())


def test_grouped_entry_points_reject_bad_arguments(cuda):
    from byol_b200 import ops
    from byol_b200._lib import ByolLibraryError
    x = torch.zeros(1, 8, 8, 128, device=cuda, dtype=torch.bfloat16)
    wf, wd = ops.prep_weight_grouped(torch.zeros(128, 4, 3, 3, device=cuda))
    with pytest.raises(ByolLibraryError, match="unsupported geometry"):
        ops.conv_fprop(x, wf, 3, 3, 3, 1)                      # stride 3
    with pytest.raises(ByolLibraryError, match="unsupported geometry"):
        ops.conv_dgrad(x, wd, 8, 8, 3, 3, 1, 0)                # pad 0
    with pytest.raises(ByolLibraryError, match="must divide 64"):
        ops.conv_wgrad(x, x, torch.zeros(128, 3, 3, 3, device=cuda), 3, 3, 1, 1)
    with pytest.raises(ByolLibraryError, match="unsupported geometry"):
        ops.conv_fprop(x[..., :96].contiguous(), wf, 3, 3, 1, 1)   # C = 96: not a multiple of 64
    # the compact layout never reaches a dense kernel: its ldw (576) is short of 9 * C
    with pytest.raises(ByolLibraryError, match="bad ldw"):
        ops.conv_fprop(x, wf.view(128, 576), 3, 3, 1, 1)


@pytest.mark.parametrize("h,stride", [(28, 1), (14, 1), (28, 2)])
def test_grouped_reductions_bit_reproducible(cuda, h, stride):
    """Statistics and weight gradients are fixed-point sums: two runs and a CUDA-graph replay give the same bits."""
    from byol_b200 import ops
    cg, n = 8, 4
    x, w, dy = _mk(n, h, C, cg, stride, cuda, seed=4)
    wf, _ = ops.prep_weight_grouped(w.to(cuda), want_dgrad=False)
    xd, dyd = _nhwc(x, cuda), _nhwc(dy, cuda)

    def run(stats, dw):
        stats.zero_()
        dw.zero_()
        ops.conv_fprop(xd, wf, 3, 3, stride, 1, stats=stats)
        ops.conv_wgrad(xd, dyd, dw, 3, 3, stride, 1)

    outs = []
    for _ in range(2):
        stats, dw = torch.empty(2 * C, device=cuda), torch.empty(C, cg, 3, 3, device=cuda)
        run(stats, dw)
        torch.cuda.synchronize()
        outs.append((stats.clone(), dw.clone()))
    stats, dw = torch.empty(2 * C, device=cuda), torch.empty(C, cg, 3, 3, device=cuda)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        run(stats, dw)                       # warm-up on the capture stream (its fixed-point scratch)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=s):
        run(stats, dw)
    graph.replay()
    torch.cuda.synchronize()
    outs.append((stats.clone(), dw.clone()))
    for a in outs[1:]:
        assert torch.equal(outs[0][0], a[0]) and torch.equal(outs[0][1], a[1])


@pytest.mark.parametrize("arch", ["resnext:32x4:2,1,1,1", "resnext:32x8:1,1,1,1"])
def test_resnext_blocks_teacher_forced(cuda, monkeypatch, arch):
    """Every block of a shallow ResNeXt against autograd on the oracle's block (tests/test_gpu_blocks.py criteria);
    resnext:32x8 reaches 64 channels per group in its last stage."""
    from tests.test_gpu_blocks import test_blocks_teacher_forced as blocks_teacher_forced
    resnext_oracle.install(monkeypatch)
    blocks_teacher_forced(cuda, arch, 2048)


def test_resnext50_steps_vs_reference_golden(cuda, monkeypatch):
    """Two ResNeXt-50 training steps against the unmodified reference (bf16 criteria of
    test_training_steps_vs_reference_golden)."""
    from tests.test_gpu_step import _run_steps
    from tests.test_oracle_golden import load_case
    resnext_oracle.install(monkeypatch)
    z, arch, rep, b, r, steps, seed, lr, total = load_case("rnx50_b8_r64")
    _run_steps(cuda, arch, rep, b, r, steps, seed, lr, total, out_tol=None, golden=z)


def _train(arch, rep, graphs, steps=3, b=8, r=64, seed=11):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    g = torch.Generator().manual_seed(3)
    batches = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
                torch.randint(0, 1000, (b,), generator=g).cuda()) for _ in range(steps)]
    torch.manual_seed(seed)
    model = BYOL(rep, 256, 1000, 20, arch=arch).cuda().train()
    model._engine.use_graphs = graphs
    opt = wiring.build_optimizer(model, global_batch_size=256)
    losses = torch.stack([wiring.train_step(model, opt, *bt)["loss_mean"].detach().clone() for bt in batches])
    torch.cuda.synchronize()
    sd = model.state_dict()
    return {"loss": losses, "theta": model._engine.theta.clone(), "target": model.target_network.mean.clone(),
            "bn": torch.cat([v.reshape(-1).float() for k, v in sd.items() if "running_" in k])}


def test_resnext_graph_replay_bit_equal_to_eager(cuda):
    arch = "resnext:32x4:1,1,1,1"
    a, b = _train(arch, 2048, graphs=False), _train(arch, 2048, graphs=True)
    for key in a:
        assert torch.equal(a[key], b[key]), key


def test_resnext_eval_forward(cuda, monkeypatch):
    from byol_b200.model import BYOL
    from oracle import byol_oracle as O
    resnext_oracle.install(monkeypatch)
    arch = "resnext:32x4:1,1,1,1"
    torch.manual_seed(4)
    model = BYOL(2048, 256, 1000, 10, arch=arch).cuda().eval()
    params, buffers = O.init_reference_state(arch, 4)
    oracle = O.OracleBYOL(arch, params, buffers, 10)
    g = torch.Generator().manual_seed(6)
    a1, a2 = torch.rand(4, 3, 64, 64, generator=g), torch.rand(4, 3, 64, 64, generator=g)
    with torch.no_grad():
        out = model(a1.cuda(), a2.cuda())
        ref = oracle.forward(a1, a2, training=False)
    for key in ("online_representation1", "online_prediction2", "target_projection1", "linear_preds"):
        e = float((out[key].float().cpu() - ref[key]).abs().max() / ref[key].abs().max())
        print(key, e)
        assert e < 4e-2, key


FAMILY = [("resnet18", 512), ("resnet34", 512), ("resnet50", 2048), ("resnet101", 2048), ("resnet152", 2048),
          ("wide_resnet50_2", 2048), ("wide_resnet101_2", 2048), ("resnext50_32x4d", 2048),
          ("resnext101_32x8d", 2048), ("resnext101_64x4d", 2048)]


@pytest.mark.parametrize("arch,rep", FAMILY, ids=[a for a, _ in FAMILY])
def test_resnet_family_trains(cuda, arch, rep):
    res = _train(arch, rep, graphs=True, steps=2)
    print(arch, res["loss"].tolist())
    assert torch.isfinite(res["loss"]).all() and torch.isfinite(res["theta"]).all()


def test_reference_execute_graph_resnext50(cuda):
    """The reference's own main.execute_graph with --arch=resnext50_32x4d and the byol_b200 classes dropped in (as in
    tests/test_gpu_zz_dropin.py): every loss within 3 % of the golden run."""
    import functools
    import byol_b200.model
    import byol_b200.objective
    import byol_b200.lars
    import byol_b200.wiring
    from tests.test_gpu_zz_dropin import _import_reference_main
    from tests.test_oracle_golden import _batches, load_case
    z, arch, rep, b, r, steps, seed, lr, total = load_case("rnx50_b8_r64")
    main = _import_reference_main(arch, rep, b, r)
    main.BYOL = functools.partial(byol_b200.model.BYOL, arch=main.args.arch, head_latent_size=main.args.head_latent_size)
    main.loss_function = byol_b200.objective.loss_function
    main.LARS = byol_b200.lars.LARS
    main.layers.DistributedDataParallelPassthrough = byol_b200.wiring.DistributedDataParallelPassthrough
    torch.manual_seed(seed)
    model = main.BYOL(base_network_output_size=rep, projection_output_size=256, classifier_output_size=1000,
                      total_training_steps=total, base_decay=0.996).cuda()
    opt = main.LARS(torch.optim.SGD(main.layers.add_weight_decay(model, 1e-6), lr=lr, momentum=0.9), eps=0.0)
    got = [main.execute_graph(1, model, [(a1, a2, lab)], None, optimizer=opt, prefix="train")
           for a1, a2, lab in _batches(seed, steps, b, r)]
    ref = [float(z["s%d_loss" % s]) for s in range(steps)]
    print("execute_graph losses %s   reference %s" % (got, ref))
    np.testing.assert_allclose(got, ref, rtol=3e-2)
