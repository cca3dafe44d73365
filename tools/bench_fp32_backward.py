"""Cost of the fp32-accurate backward pass: ResNet-50 @224 with precision="fp32", backward_precision "bf16" against
"fp32", alternating in one process (CUDA graphs on, as in training).  For each: device-timed ms per training step,
images/s and peak device memory.  Prints one JSON line per measurement and a summary line, with the card name and
its power limit.

    python tools/bench_fp32_backward.py --batch 256 --steps 5 --warmup 3 --rounds 2

Every measurement runs in a fresh Python process, so no earlier model, CUDA-graph pool or failed attempt holds device
memory while it runs.  A batch that does not fit is halved until it does; the batch that ran is part of every result
line.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        limit = None
    return name, limit


def measure(bwd, batch, steps, warmup, res):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50", precision="fp32", backward_precision=bwd).cuda().train()
    opt = wiring.build_optimizer(model, global_batch_size=batch)
    g = torch.Generator(device="cuda").manual_seed(1)
    a1 = torch.rand(batch, 3, res, res, device="cuda", generator=g)
    a2 = torch.rand(batch, 3, res, res, device="cuda", generator=g)
    lab = torch.randint(0, 1000, (batch,), device="cuda", generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(warmup):
        wiring.train_step(model, opt, a1, a2, lab)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        st = wiring.train_step(model, opt, a1, a2, lab)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / steps
    out = {"backward_precision": bwd, "batch": batch, "resolution": res, "ms_per_step": round(ms, 2),
           "images_per_s": round(batch * 1000.0 / ms, 1), "peak_mem_gb": round(torch.cuda.max_memory_allocated() / 2 ** 30, 2),
           "loss": float(st["loss_mean"])}
    return out


def run_one(bwd, batch, args):
    """One measurement in a child process -> result dict, or None when it ran out of device memory."""
    cmd = [sys.executable, os.path.abspath(__file__), "--one", bwd, "--batch", str(batch), "--res", str(args.res),
           "--steps", str(args.steps), "--warmup", str(args.warmup)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    if p.returncode == 0 and lines:
        return json.loads(lines[-1])
    if "OutOfMemoryError" in p.stderr or "out of memory" in p.stderr:
        return None
    raise RuntimeError("measurement %s / %d failed:\n%s" % (bwd, batch, p.stderr[-4000:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--one", choices=["bf16", "fp32"], help=argparse.SUPPRESS)   # child process: one measurement
    args = ap.parse_args()
    if args.one:
        print(json.dumps(measure(args.one, args.batch, args.steps, args.warmup, args.res)))
        return
    name, limit = card()
    print(json.dumps({"card": name, "power_limit_w": limit}))
    batch = {"bf16": args.batch, "fp32": args.batch}
    results = {"bf16": [], "fp32": []}
    for _ in range(args.rounds):
        for bwd in ("bf16", "fp32"):
            while True:
                r = run_one(bwd, batch[bwd], args)
                if r is not None:
                    break
                if batch[bwd] <= 8:
                    raise RuntimeError("%s backward: 8 images do not fit" % bwd)
                print(json.dumps({"backward_precision": bwd, "out_of_memory_at": batch[bwd]}))
                batch[bwd] //= 2
            r.update({"card": name, "power_limit_w": limit})
            print(json.dumps(r))
            results[bwd].append(r)
    summary = {bwd: {"batch": rs[-1]["batch"], "ms_per_step_min": min(x["ms_per_step"] for x in rs),
                     "images_per_s_max": max(x["images_per_s"] for x in rs),
                     "peak_mem_gb": max(x["peak_mem_gb"] for x in rs)} for bwd, rs in results.items()}
    print(json.dumps({"summary": summary, "card": name, "power_limit_w": limit}))


if __name__ == "__main__":
    main()
