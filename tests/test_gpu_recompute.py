"""GPU: block-level activation recomputation (Engine.recompute_plan).  A block the plan marks keeps only its input, its
BN coefficients and its output mask; its backward re-runs the forward's kernels on them.  Every cross-block sum is
fixed-point (DESIGN.md §4), so a step that recomputes must give the same bits as one that stores: losses, outputs,
gradients, parameters, LARS momentum, EMA target and running statistics are compared with torch.equal."""
import os

import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

STEPS = 3     # step 1 eager, step 2 captured into CUDA graphs and replayed, step 3 replayed


def _order(mm):
    b = mm["blocks"]
    return sorted(range(len(b)), key=lambda i: (-(b[i]["stored"] - b[i]["kept"]) / b[i]["flops"], i))


def _force(eng, plan, b, r):
    """Set the private budget so that the planner picks `plan` ("stored", "all" or "half"); returns that block set."""
    eng.walk_layers()
    mm = eng.memory_model(b, r, r)
    if plan == "stored":
        return frozenset()
    if plan == "all":
        eng._mem_budget = 0
        return frozenset(range(len(eng.blocks)))
    order = _order(mm)
    want = frozenset(order[:len(order) // 2])
    eng._mem_budget = eng.step_need(mm, want)
    return want


def _bn_state(model):
    return torch.cat([v.reshape(-1).float() for k, v in model.state_dict().items() if "running_" in k])


def _train(arch, rep, b, r, plan, proj_loss=False):
    from byol_b200.model import BYOL
    from byol_b200.objective import loss_function
    from byol_b200 import wiring
    g = torch.Generator().manual_seed(5)
    data = [(torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda(),
             torch.randint(0, 1000, (b,), generator=g).cuda()) for _ in range(STEPS)]
    torch.manual_seed(17)
    model = BYOL(rep, 256, 1000, 20, arch=arch).cuda().train()
    eng = model._engine
    want = _force(eng, plan, b, r)
    opt = wiring.build_optimizer(model, global_batch_size=256)
    res = {"loss": [], "out": [], "grad": []}
    for a1, a2, lab in data:
        out = model(a1, a2)
        loss = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                             target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
        loss = loss + wiring.cross_entropy_topk(out["linear_preds"], lab)[0]
        if proj_loss:        # a gradient on the projections: the graphed step takes the eager backward fallback
            loss = loss + 1e-2 * out["online_projection1"].pow(2).mean()
        opt.zero_grad()
        loss.backward()
        res["grad"].append(eng.grad.clone())
        opt.step()
        res["loss"].append(loss.detach().clone())
        res["out"].append(torch.cat([out[k].detach().reshape(-1).float() for k in sorted(out)]))
    torch.cuda.synchronize()
    assert eng.recompute_plan(b, r, r) == want
    captured = [v for v in eng.graphs.values() if v != "warm"]
    assert len(captured) == 1
    for saved in captured[0].saved:
        assert frozenset(i for i, d in enumerate(saved["blocks"]) if d.get("recompute")) == want
    assert int(model.state_dict()["base_network.1.num_batches_tracked"]) == 4 * STEPS      # Q7: 4 updates per step
    res.update(loss=torch.stack(res["loss"]), out=torch.stack(res["out"]), grad=torch.stack(res["grad"]),
               theta=eng.theta.clone(), momentum=torch.cat([s["momentum_buffer"].reshape(-1) for s in
                                                             opt.state_dict()["state"].values()
                                                             if s.get("momentum_buffer") is not None]),
               ema=model.target_network.mean.clone(), bn=_bn_state(model))
    return res


NETS = [("resnet18", 512, 8, 64), ("resnet:bottleneck:1,1,1,1", 2048, 8, 96), ("resnext:32x4:1,1,1,1", 2048, 8, 64)]


@pytest.mark.parametrize("arch,rep,b,r", NETS, ids=[n[0] for n in NETS])
def test_recompute_is_bit_identical(cuda, arch, rep, b, r):
    ref = _train(arch, rep, b, r, "stored")
    for plan in ("all", "half"):
        got = _train(arch, rep, b, r, plan)
        for key in ref:
            assert torch.equal(got[key], ref[key]), "%s: %s differs from the stored plan" % (plan, key)
    print("%s: losses %s" % (arch, ref["loss"].tolist()))


def test_recompute_eager_fallback_is_bit_identical(cuda):
    arch, rep, b, r = "resnet:bottleneck:1,1,1,1", 2048, 8, 96
    ref = _train(arch, rep, b, r, "stored", proj_loss=True)
    got = _train(arch, rep, b, r, "all", proj_loss=True)
    for key in ref:
        assert torch.equal(got[key], ref[key]), "%s differs from the stored plan" % key


def _saved_bytes(blocks):
    """Bytes of the distinct bf16 / uint8 tensors the block dicts hold (the fp32 BN coefficients are views of one
    per-pass pool)."""
    seen = {}
    for d in blocks:
        for v in d.values():
            if isinstance(v, torch.Tensor) and v.dtype != torch.float32:
                s = v.untyped_storage()
                seen[s.data_ptr()] = s.nbytes()
    return sum(seen.values())


def test_recompute_memory(cuda):
    """The saved block tensors have exactly the planner's size, and recomputing every block lowers the step's peak
    by at least 80 % of the planned saving (ResNet-50, 64 images of 128x128)."""
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    arch, b, r = "resnet50", 64, 128
    g = torch.Generator().manual_seed(9)
    a1, a2 = torch.rand(b, 3, r, r, generator=g).cuda(), torch.rand(b, 3, r, r, generator=g).cuda()
    lab = torch.randint(0, 1000, (b,), generator=g).cuda()
    peaks, lane = {}, {}
    for plan in ("stored", "all"):
        torch.manual_seed(3)
        model = BYOL(2048, 256, 1000, 20, arch=arch).cuda().train()
        eng = model._engine
        eng.use_graphs = False
        want = _force(eng, plan, b, r)
        opt = wiring.build_optimizer(model, global_batch_size=256)
        wiring.train_step(model, opt, a1, a2, lab)
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        wiring.train_step(model, opt, a1, a2, lab)
        torch.cuda.synchronize()
        peaks[plan] = torch.cuda.max_memory_allocated() - base
        mean = model.target_network.mean
        saved = [{}, {}]
        lanes = [(eng.theta, eng.w_online, saved[0]), (eng.theta, eng.w_online, saved[1]),
                 (mean, eng.w_target, None), (mean, eng.w_target, None)]
        with torch.no_grad():
            eng.prep_step(mean, True)
            eng.forward_lanes([a1, a2, a1, a2], lanes, True)
        assert eng.recompute_plan(b, r, r) == want
        lane[plan] = eng.lane_bytes(eng.memory_model(b, r, r), want)
        for s in saved:
            assert _saved_bytes(s["blocks"]) == lane[plan]
        model = eng = opt = saved = lanes = mean = None
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    planned = 2 * (lane["stored"] - lane["all"])
    drop = peaks["stored"] - peaks["all"]
    print("per online lane saved: stored %.1f MB, recompute all %.1f MB; step peak above the model: stored %.1f MB, "
          "recompute all %.1f MB; drop %.1f MB = %.2f of the planned %.1f MB" %
          (lane["stored"] / 1e6, lane["all"] / 1e6, peaks["stored"] / 1e6, peaks["all"] / 1e6, drop / 1e6,
           drop / planned, planned / 1e6))
    assert drop >= 0.8 * planned


# every (arch, images per view, resolution) the other GPU tests train
EXISTING_SIZES = [("resnet18", 512, 8, 64), ("resnet18", 512, 16, 64), ("resnet18", 512, 32, 224),
                  ("resnet50", 2048, 8, 64), ("resnet:bottleneck:2,1,1,1", 2048, 16, 64),
                  ("resnet:bottleneck:2,1,1,1", 2048, 8, 64), ("resnet:basic:2,1,1,1", 512, 16, 64),
                  ("resnet:basic:1,1,1,1", 512, 8, 64), ("resnet:bottleneck:1,1,1,1", 2048, 8, 64),
                  ("resnet:bottleneck:1,1,1,1", 2048, 8, 96), ("resnext:32x4:1,1,1,1", 2048, 8, 64),
                  ("resnext50_32x4d", 2048, 8, 64), ("resnext101_32x8d", 2048, 8, 64),
                  ("wide_resnet101_2", 2048, 8, 64)]


def test_default_plan_is_empty_at_test_sizes(cuda):
    from byol_b200.model import BYOL
    for arch, rep, b, r in EXISTING_SIZES:
        model = BYOL(rep, 256, 1000, 10, arch=arch).cuda().train()
        eng = model._ensure_ready(b)
        assert eng.recompute_plan(b, r, r) == frozenset(), (arch, b, r)
        model = eng = None


ARCH, REP, B, R, SEED, LR = "resnet:bottleneck:2,1,1,1", 2048, 8, 64, 41, 0.3


def _worker(rank, world, port, ret):
    import faulthandler
    faulthandler.dump_traceback_later(150, exit=True)      # a cross-rank deadlock must not eat the GPU lease
    os.environ["BYOL_B200_PEER_XCHG"] = "1"
    import torch.distributed as dist
    import torch.nn as nn
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    os.environ["MASTER_ADDR"], os.environ["MASTER_PORT"] = "127.0.0.1", str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    g = torch.Generator().manual_seed(77)
    a1, a2 = torch.rand(world * B, 3, R, R, generator=g), torch.rand(world * B, 3, R, R, generator=g)
    lab = torch.randint(0, 1000, (world * B,), generator=g)
    sl = slice(rank * B, (rank + 1) * B)
    out = {}
    for plan in ("stored", "all"):
        torch.manual_seed(SEED)
        model = BYOL(REP, 256, 1000, 10, arch=ARCH)
        model = nn.SyncBatchNorm.convert_sync_batchnorm(model).cuda().train()
        _force(model._engine, plan, B, R)
        net = wiring.DistributedDataParallelPassthrough(model)
        opt = wiring.LARS(torch.optim.SGD(wiring.add_weight_decay(model, 1e-6), lr=LR, momentum=0.9), eps=0.0)
        losses = [wiring.train_step(net, opt, a1[sl].cuda(), a2[sl].cuda(), lab[sl].cuda())["loss_mean"].item()
                  for _ in range(STEPS)]
        torch.cuda.synchronize()
        out[plan] = {"theta": model._engine.theta.cpu(), "ema": model.target_network.mean.cpu(),
                     "bn": _bn_state(model).cpu(), "loss": torch.tensor(losses)}
    ret[rank] = out
    dist.destroy_process_group()


def test_two_rank_syncbn_recompute(cuda):
    """Under SyncBatchNorm the recompute runs no statistics exchange: the replicas stay bit-identical and equal the
    stored plan."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, 29561, ret), nprocs=world, join=True)
    r0, r1 = ret[0], ret[1]
    for key in r0["stored"]:
        assert torch.equal(r0["all"][key], r1["all"][key]), "replicas diverged (%s)" % key
        assert torch.equal(r0["all"][key], r0["stored"][key]), "recompute differs from the stored plan (%s)" % key
