"""Cost of BYOL(norm="group_ws") against the default BatchNorm encoder on one GPU, with the card's name and power limit
read in the same run:

* the ResNet-50 training step at 224 px (forward of the four lanes, loss, backward, LARS) at each --batches size:
  device ms per step over --steps steps, the two norms alternated for --rounds rounds (each arm builds its model, warms
  up and captures its CUDA graphs anew, then frees everything), and the peak device memory of a step;
* per-kernel device time of the GroupNorm and weight-standardisation launches of one eager GroupNorm step
  (torch.profiler, a run of its own) against the least time HBM allows for the bytes each launch must move
  (3.35 TB/s, the H100 SXM data-sheet figure).

    python tools/bench_groupnorm.py --out profiles/groupnorm_h100_rn50.jsonl

One JSON line per measurement; all are written to --out as well.
"""
import argparse
import gc
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_fp32_backward import card   # noqa: E402

LINES = []
CARD = {}
HBM = 3.35e12


def emit(**kw):
    kw.update(CARD)
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def _setup(norm, batch, graphs=True):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50", norm=norm).cuda().train()
    model._engine.use_graphs = graphs
    opt = wiring.build_optimizer(model, global_batch_size=batch)
    g = torch.Generator(device="cuda").manual_seed(1)
    a1 = torch.rand(batch, 3, 224, 224, device="cuda", generator=g)
    a2 = torch.rand(batch, 3, 224, 224, device="cuda", generator=g)
    return model, opt, a1, a2


def _step(model, opt, a1, a2):
    from byol_b200.objective import loss_function
    out = model(a1, a2)
    loss = loss_function(online_prediction1=out["online_prediction1"], online_prediction2=out["online_prediction2"],
                         target_projection1=out["target_projection1"], target_projection2=out["target_projection2"])
    opt.zero_grad()
    loss.backward()
    opt.step()


def time_arm(norm, batch, steps, warmup):
    model, opt, a1, a2 = _setup(norm, batch)
    for _ in range(warmup):
        _step(model, opt, a1, a2)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        _step(model, opt, a1, a2)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    peak = torch.cuda.max_memory_allocated()
    del model, opt, a1, a2
    gc.collect()
    torch.cuda.empty_cache()
    return ms, peak


# bytes each launch must move, from its arguments (the kernels' own reads and writes; the fixed-point flushes aside)
def _nbytes(name, args, kw):
    if name == "gn_stats":
        return args[0].numel() * 2
    if name == "gn_apply":
        x = args[0]
        n = x.numel() * 4 + (x.numel() * 2 if kw.get("resid") is not None else 0)
        return n + (x.numel() // 8 if kw.get("mask_out") is not None else 0)
    if name == "gn_relu_maxpool_fwd":
        x = args[0]
        n, h, w, c = x.shape
        ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
        return x.numel() * 2 + n * ho * wo * c * (3 if kw.get("want_idx", True) else 2)
    if name in ("gn_bwd_reduce", "gn_bwd_apply"):
        x = args[1]
        mode = args[6]
        n = x.numel() * 4 + (x.numel() // 8 if mode == 3 else x.numel() * 2 if mode == 2 else 0)
        if name == "gn_bwd_apply":
            n += x.numel() * 2 + (x.numel() * 2 if kw.get("dz_out") is not None else 0)
        return n
    if name == "ws_fwd":
        return args[3].numel() * 8
    if name == "ws_bwd":
        return args[0].numel() * 16
    return 0


KERNELS = {"gn_stats": ("gn_stats_kernel", "gn_finalize_kernel"), "gn_apply": ("gn_apply_kernel",),
           "gn_relu_maxpool_fwd": ("gn_relu_maxpool_fwd_kernel",), "gn_bwd_reduce": ("gn_bwd_reduce_kernel",),
           "gn_bwd_apply": ("gn_bwd_apply_kernel",), "ws_fwd": ("ws_fwd_kernel",), "ws_bwd": ("ws_bwd_kernel",)}


def kernel_table(batch):
    from byol_b200 import ops
    model, opt, a1, a2 = _setup("group_ws", batch, graphs=False)
    _step(model, opt, a1, a2)
    torch.cuda.synchronize()
    moved = {k: [0, 0] for k in KERNELS}
    orig = {k: getattr(ops, k) for k in KERNELS}

    def wrap(k):
        def f(*args, **kw):
            moved[k][0] += 1
            moved[k][1] += _nbytes(k, args, kw)
            return orig[k](*args, **kw)
        return f

    for k in KERNELS:
        setattr(ops, k, wrap(k))
    try:
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            _step(model, opt, a1, a2)
            torch.cuda.synchronize()
    finally:
        for k in KERNELS:
            setattr(ops, k, orig[k])
    dev = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            dev[e.name] = dev.get(e.name, 0.0) + e.device_time_total
    step_us = sum(dev.values())
    for k, names in KERNELS.items():
        us = sum(t for n, t in dev.items() if any(n.startswith(m) or ("::" + m) in n for m in names))
        calls, nbytes = moved[k]
        emit(kind="kernel", op=k, batch=batch, calls=calls, device_us=round(us, 1), bytes=nbytes,
             hbm_bound_us=round(nbytes / HBM * 1e6, 1), share_of_hbm_bound=round(nbytes / HBM * 1e6 / us, 3) if us else None)
    emit(kind="kernel_step_total", batch=batch, device_us=round(step_us, 1))
    del model, opt, a1, a2
    gc.collect()
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, nargs="+", default=[256, 512])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--kernel-batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_groupnorm needs a GPU")
    import __graft_entry__ as g
    g.build()
    name, limit = card()
    CARD.update(card=name, power_limit_w=limit)
    for batch in args.batches:
        for rnd in range(args.rounds):
            for norm in ("batch", "group_ws"):
                ms, peak = time_arm(norm, batch, args.steps, args.warmup)
                emit(kind="step", norm=norm, batch=batch, round=rnd, ms_per_step=round(ms, 2),
                     peak_alloc_gib=round(peak / 2 ** 30, 2))
    kernel_table(args.kernel_batch)
    if args.out:
        with open(args.out, "w") as f:
            for line in LINES:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
