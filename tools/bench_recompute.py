"""Cost of activation recomputation (Engine.recompute_plan): a bf16 BYOL training step that stores every block's
activations against one that recomputes every block in the backward pass, forced through the engine's private budget
override, alternating (CUDA graphs on, as in training).  For each: device-timed ms per training step, images/s, peak
device memory, the planner's figures and the blocks it recomputed.  Prints one JSON line per measurement and a summary
line, with the card name and its power limit.

    python tools/bench_recompute.py --arch resnet50 --batch 256 --steps 10 --warmup 3 --rounds 2
    python tools/bench_recompute.py --arch resnet200 --batch 256 --plans auto --plan-only

"auto" is the plan the engine picks by itself from the device's free memory.  --plan-only builds the model and reports
the plan and the planner's figures without running a step.  Every measurement runs in a fresh Python process, so no
earlier model or CUDA-graph pool holds device memory while it runs.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_fp32_backward import card   # noqa: E402


def measure(plan, args):
    from byol_b200.model import BYOL
    from byol_b200 import wiring
    b, r = args.batch, args.res
    torch.manual_seed(0)
    model = BYOL(args.rep, 256, 1000, 1000, arch=args.arch).cuda().train()
    eng = model._ensure_ready(b)
    if plan == "stored":
        eng._mem_budget = 1 << 62
    elif plan == "all":
        eng._mem_budget = 0
    chosen = sorted(eng.recompute_plan(b, r, r))
    mm = eng.memory_model(b, r, r)
    out = {"arch": args.arch, "plan": plan, "batch": b, "resolution": r, "blocks": len(eng.blocks),
           "recomputed_blocks": chosen,
           "planner_lane_gb": round(eng.lane_bytes(mm, frozenset(chosen)) / 1e9, 3),
           "planner_need_gb": round(eng.step_need(mm, frozenset(chosen)) / 1e9, 2),
           "planner_need_stored_gb": round(eng.step_need(mm, frozenset()) / 1e9, 2)}
    if args.plan_only:
        free, total = torch.cuda.mem_get_info()
        out.update(free_gb=round(free / 1e9, 2), total_gb=round(total / 1e9, 2))
        return out
    opt = wiring.build_optimizer(model, global_batch_size=b)
    g = torch.Generator(device="cuda").manual_seed(1)
    a1 = torch.rand(b, 3, r, r, device="cuda", generator=g)
    a2 = torch.rand(b, 3, r, r, device="cuda", generator=g)
    lab = torch.randint(0, 1000, (b,), device="cuda", generator=g)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    for _ in range(args.warmup):
        wiring.train_step(model, opt, a1, a2, lab)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(args.steps):
        st = wiring.train_step(model, opt, a1, a2, lab)
    end.record()
    torch.cuda.synchronize()
    ms = start.elapsed_time(end) / args.steps
    out.update(ms_per_step=round(ms, 2), images_per_s=round(b * 1000.0 / ms, 1),
               peak_mem_gb=round(torch.cuda.max_memory_allocated() / 1e9, 2),
               reserved_gb=round(torch.cuda.max_memory_reserved() / 1e9, 2), loss=float(st["loss_mean"]))
    return out


def run_one(plan, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--one", plan, "--arch", args.arch, "--batch", str(args.batch),
           "--rep", str(args.rep), "--res", str(args.res), "--steps", str(args.steps), "--warmup", str(args.warmup)]
    if args.plan_only:
        cmd.append("--plan-only")
    p = subprocess.run(cmd, capture_output=True, text=True)
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("{")]
    if p.returncode == 0 and lines:
        return json.loads(lines[-1])
    raise RuntimeError("measurement %s failed:\n%s" % (plan, p.stderr[-4000:]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--arch", default="resnet50")
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--rep", type=int, default=2048, help="representation size (512 for ResNet-18 / 34)")
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--plans", default="stored,all")
    ap.add_argument("--plan-only", action="store_true")
    ap.add_argument("--one", choices=["stored", "all", "auto"], help=argparse.SUPPRESS)   # child: one measurement
    args = ap.parse_args()
    if args.one:
        print(json.dumps(measure(args.one, args)))
        return
    name, limit = card()
    plans = args.plans.split(",")
    results = {p: [] for p in plans}
    for _ in range(1 if args.plan_only else args.rounds):
        for plan in plans:
            r = run_one(plan, args)
            r.update({"card": name, "power_limit_w": limit})
            print(json.dumps(r), flush=True)
            results[plan].append(r)
    if args.plan_only:
        return
    summary = {p: {"ms_per_step_min": min(x["ms_per_step"] for x in rs),
                   "ms_per_step_all": [x["ms_per_step"] for x in rs],
                   "peak_mem_gb": max(x["peak_mem_gb"] for x in rs)} for p, rs in results.items()}
    if "stored" in summary and "all" in summary:
        summary["all_over_stored"] = round(summary["all"]["ms_per_step_min"] / summary["stored"]["ms_per_step_min"], 4)
    print(json.dumps({"summary": summary, "arch": args.arch, "batch": args.batch, "resolution": args.res,
                      "card": name, "power_limit_w": limit}))


if __name__ == "__main__":
    main()
