"""Cost of the BYOL paper's loss (loss_function(..., variant="byol")) against the default reference loss on one GPU,
with the card's name and power limit read in the same run:

* per-call time of forward + backward at D = 256 and each --rows size, for three implementations: the paper's loss on
  the loss_rows kernels, the reference loss, and torch's composition of the paper's loss in ATen with autograd.
  CUDA events around --calls calls after --warmup, repeated --repeats times (with the host enqueueing one call after
  the other, this is the rate at which calls complete); and, in a run of its own under torch.profiler, the device time
  of the kernels each call launches (the sum of their durations).  Each record holds the HBM bound of the forward's
  reads, 4 B D 4 bytes at 3.35 TB/s (the H100 SXM data-sheet figure); at these sizes a call is expected to be bound by
  launch overhead, not by bandwidth;
* the ResNet-50 training step at 224 px with --batch images: device ms per step over --steps steps, the two loss
  variants alternated for --rounds rounds (each arm builds its model, warms up and captures its CUDA graphs anew).

    python tools/bench_loss.py --out profiles/loss_h100.jsonl

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


def torch_paper_loss(q1, q2, z1, z2):
    def nrm(x):
        return x * torch.rsqrt(torch.clamp((x * x).sum(-1, keepdim=True), min=1e-12))
    return (((nrm(q1) - nrm(z2.detach())) ** 2).sum(-1) + ((nrm(q2) - nrm(z1.detach())) ** 2).sum(-1)).mean()


def time_calls(impl, rows, dim, calls, warmup):
    from byol_b200.objective import loss_function
    g = torch.Generator(device="cuda").manual_seed(rows)
    q1, q2, z1, z2 = (torch.randn(rows, dim, device="cuda", generator=g) for _ in range(4))
    q1.requires_grad_(True)
    q2.requires_grad_(True)

    def call():
        if impl == "torch":
            loss = torch_paper_loss(q1, q2, z1, z2)
        else:
            loss = loss_function(q1, q2, z1, z2, variant=impl)
        q1.grad = q2.grad = None
        loss.backward()

    for _ in range(warmup):
        call()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        call()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / calls


def kernel_time(impl, rows, dim, calls):
    """Device time per call: the summed durations of the CUDA kernels `calls` calls launch, over `calls`."""
    time_calls(impl, rows, dim, 20, 5)
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        time_calls(impl, rows, dim, calls, 0)
    us, n = 0.0, 0
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            us += e.device_time_total
            n += 1
    return us / calls, n / calls


def _setup(batch):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50").cuda().train()
    opt = wiring.build_optimizer(model, global_batch_size=batch)
    g = torch.Generator(device="cuda").manual_seed(1)
    a1 = torch.rand(batch, 3, 224, 224, device="cuda", generator=g)
    a2 = torch.rand(batch, 3, 224, 224, device="cuda", generator=g)
    lab = torch.randint(0, 1000, (batch,), device="cuda", generator=g)
    return model, opt, a1, a2, lab


def time_step(variant, batch, steps, warmup):
    from byol_b200 import wiring
    model, opt, a1, a2, lab = _setup(batch)
    for _ in range(warmup):
        wiring.train_step(model, opt, a1, a2, lab, loss_variant=variant)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        wiring.train_step(model, opt, a1, a2, lab, loss_variant=variant)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    del model, opt, a1, a2, lab
    gc.collect()
    torch.cuda.empty_cache()
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, nargs="+", default=[512, 4096])
    ap.add_argument("--dim", type=int, default=256)
    ap.add_argument("--calls", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--profile-calls", type=int, default=200)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--step-warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_loss needs a GPU")
    import __graft_entry__ as g
    g.build()
    name, limit = card()
    CARD.update(card=name, power_limit_w=limit)
    for rows in args.rows:
        nbytes = 4 * rows * args.dim * 4
        for rep in range(args.repeats):
            for impl in ("byol", "reference", "torch"):
                us = time_calls(impl, rows, args.dim, args.calls, args.warmup)
                emit(kind="loss_call", impl=impl, rows=rows, dim=args.dim, repeat=rep, us_per_fwd_bwd=round(us, 2),
                     fwd_read_bytes=nbytes, fwd_hbm_bound_us=round(nbytes / HBM * 1e6, 2))
        for impl in ("byol", "reference", "torch"):
            us, kernels = kernel_time(impl, rows, args.dim, args.profile_calls)
            emit(kind="loss_kernels", impl=impl, rows=rows, dim=args.dim, device_us_per_fwd_bwd=round(us, 2),
                 kernels_per_call=round(kernels, 2), fwd_read_bytes=nbytes, fwd_hbm_bound_us=round(nbytes / HBM * 1e6, 2))
    for rnd in range(args.rounds):
        for variant in ("reference", "byol"):
            ms = time_step(variant, args.batch, args.steps, args.step_warmup)
            emit(kind="step", variant=variant, arch="resnet50", image=224, batch=args.batch, round=rnd,
                 ms_per_step=round(ms, 2))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in LINES:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
