"""Time the weight-gradient convolutions of ResNet-50: every distinct wgrad shape of the encoder (the 7x7 stem on its
own kernel, the 1x1 convolutions on the TMA-operand wgrad GEMM, the stride-1 3x3 ones on the shared-memory patch
kernel, the stride-2 and 7x7 3x3 ones on the gather route) and the projector, predictor and classifier linears, each
through ops.conv_wgrad / ops.stem_conv_wgrad as the engine calls them.

Per shape: the route, the launches of one training step (2 online backward passes; the classifier runs once over both
views), the FLOPs and the bytes the launch must move (read X and dY, read and write the fp32 dW), both from the shapes,
the bound that applies at the H100 SXM data-sheet rates (989 TFLOP/s dense bf16, 3.35 TB/s HBM3), the median of --reps
launches timed with CUDA events with L2 flushed before each, and its fraction of the bound.  Totals are weighted by
the launches of one step, per route and overall.

--profile-steps K instead profiles K BYOL training steps (ResNet-50 @224, --batch images, after 3 warm-up steps) with
torch.profiler and sums the device time per kernel name: the wgrad kernels and the rest of the step.

    python tools/bench_wgrad.py                        # batch 512, 224 px
    python tools/bench_wgrad.py --shapes-only          # the shape table and its bounds, no GPU needed
    python tools/bench_wgrad.py --out table.json
    python tools/bench_wgrad.py --profile-steps 3 --out profile.json
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_gemm1x1 import BF16_FLOPS, HBM_BPS, STAGES, card  # noqa: E402

WGRAD_PASSES = 2
# (name, Cin, Cout): the linears of BYOL's heads (projector 2048 -> 4096 -> 256, predictor 256 -> 4096 -> 256)
LINEARS = [("proj1", 2048, 4096), ("proj2", 4096, 256), ("pred1", 256, 4096), ("pred2", 4096, 256)]
WGRAD_KERNELS = ("conv_wgrad_kernel", "conv3x3_wgrad_patch_kernel", "stem_wgrad_kernel", "wgrad_reduce_kernel")


def resnet50_shapes(image_size):
    """{(kind, Cin, Cout, k, stride, hw_in): layers per pass}; kind 'stem', 'conv' (hw_in: the input the wgrad kernel
    reads; the stride-2 1x1 downsample reads the compacted input, so it is a 1x1 / stride 1 at the output size)."""
    h = (image_size + 1) // 2
    shapes = {("stem", 3, 64, 7, 2, image_size): 1}
    h = (h + 1) // 2
    cin = 64

    def add(key):
        shapes[key] = shapes.get(key, 0) + 1
    for planes, blocks, stride in STAGES:
        for i in range(blocks):
            s = stride if i == 0 else 1
            hout = (h - 1) // s + 1
            add(("conv", cin, planes, 1, 1, h))
            add(("conv", planes, planes, 3, s, h))
            add(("conv", planes, 4 * planes, 1, 1, hout))
            if i == 0:
                add(("conv", cin, 4 * planes, 1, 1, hout))
            cin, h = 4 * planes, hout
    return shapes


def route(kind, cin, k, s, hw):
    if kind == "stem":
        return "stem"
    if k == 1:
        return "gemm1x1"
    return "patch3x3" if s == 1 and hw >= 12 and cin % 64 == 0 else "gather3x3"


def shape_rows(batch, image_size):
    rows = []
    for (kind, cin, cout, k, s, hw), count in sorted(resnet50_shapes(image_size).items(), key=lambda kv: -kv[0][5]):
        pad = (k - 1) // 2
        ho = (hw + 2 * pad - k) // s + 1
        rows.append(dict(name="%s_%dx%d_%d_%d_s%d_%d" % (kind, k, k, cin, cout, s, hw), kind=kind, Cin=cin, Cout=cout,
                         k=k, stride=s, hw=hw, M=batch * ho * ho, launches_per_step=WGRAD_PASSES * count))
    for name, cin, cout in LINEARS:
        rows.append(dict(name=name, kind="linear", Cin=cin, Cout=cout, k=1, stride=1, hw=1, M=batch,
                         launches_per_step=WGRAD_PASSES))
    rows.append(dict(name="classifier", kind="linear", Cin=2048, Cout=1000, k=1, stride=1, hw=1, M=2 * batch,
                     launches_per_step=1))
    for r in rows:
        ho2 = r["M"] // batch if r["kind"] != "linear" else 1
        x_elems = (r["M"] // ho2) * r["hw"] * r["hw"] * r["Cin"] if r["kind"] != "linear" else r["M"] * r["Cin"]
        ndw = r["Cout"] * r["Cin"] * r["k"] * r["k"]
        r["route"] = route(r["kind"], r["Cin"], r["k"], r["stride"], r["hw"])
        r["bytes"] = 2 * (x_elems + r["M"] * r["Cout"]) + 8 * ndw
        r["gflop"] = 2.0 * r["M"] * ndw / 1e9
        t_c, t_b = r["gflop"] * 1e9 / BF16_FLOPS, r["bytes"] / HBM_BPS
        r["bound"] = "compute" if t_c >= t_b else "HBM"
        r["bound_ms"] = 1e3 * max(t_c, t_b)
    return rows


def time_rows(rows, batch, reps):
    import torch
    from byol_b200 import _lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_wgrad: no CUDA device (use --shapes-only for the shape table)")
    dev = torch.device("cuda", 0)
    BF = torch.bfloat16
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)

    def timed(fn):
        for _ in range(2):
            fn()
        ts = []
        for _ in range(reps):
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2], ts[-1] - ts[0]

    for r in rows:
        cin, cout, k, s, hw = r["Cin"], r["Cout"], r["k"], r["stride"], r["hw"]
        dw = torch.zeros(cout, cin, k, k, device=dev)
        if r["kind"] == "stem":
            ho = (hw + 1) // 2
            xs4 = ops.nchw_to_stem4(torch.rand(batch, 3, hw, hw, device=dev, generator=g))
            dy = torch.randn(batch, ho, ho, cout, device=dev, generator=g).to(BF)
            ms, spread = timed(lambda: ops.stem_conv_wgrad(xs4, dy, dw, hw, hw))
            del xs4
        else:
            pad = (k - 1) // 2
            ho = (hw + 2 * pad - k) // s + 1
            n = r["M"] // (ho * ho)
            x = torch.randn(n, hw, hw, cin, device=dev, generator=g).to(BF)
            dy = torch.randn(n, ho, ho, cout, device=dev, generator=g).to(BF)
            ms, spread = timed(lambda: ops.conv_wgrad(x, dy, dw, k, k, s, pad))
            del x
        r["ms"], r["spread_ms"] = ms, spread
        r["frac_of_bound"] = r["bound_ms"] / ms
        del dy, dw
    return _lib.LIB_PATH


def totals(rows):
    tot = {}
    for key in ("stem", "gemm1x1", "patch3x3", "gather3x3", "all"):
        sel = [r for r in rows if key in ("all", r["route"])]
        t = {"launches_per_step": sum(r["launches_per_step"] for r in sel),
             "TFLOP_per_step": sum(r["launches_per_step"] * r["gflop"] for r in sel) / 1e3,
             "GB_per_step": sum(r["launches_per_step"] * r["bytes"] for r in sel) / 1e9,
             "bound_ms_per_step": sum(r["launches_per_step"] * r["bound_ms"] for r in sel)}
        if sel and "ms" in sel[0]:
            t["ms_per_step"] = sum(r["launches_per_step"] * r["ms"] for r in sel)
            t["frac_of_bound"] = t["bound_ms_per_step"] / t["ms_per_step"]
        tot[key] = t
    return tot


def profile_steps(batch, image_size, steps):
    """Device time per kernel name over `steps` training steps (the engine replays its CUDA graphs)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    from byol_b200 import wiring
    from byol_b200.model import BYOL
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, total_training_steps=1000, arch="resnet50").cuda().train()
    opt = wiring.build_optimizer(model, base_lr=0.2, global_batch_size=batch)
    g = torch.Generator(device=dev).manual_seed(1234)
    a1 = torch.rand(batch, 3, image_size, image_size, generator=g, device=dev)
    a2 = torch.rand(batch, 3, image_size, image_size, generator=g, device=dev)
    lab = torch.randint(0, 1000, (batch,), generator=g, device=dev)
    for _ in range(3):
        wiring.train_step(model, opt, a1, a2, lab)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            wiring.train_step(model, opt, a1, a2, lab)
        torch.cuda.synchronize()
    per = {}
    for e in prof.events():
        if e.device_type.name == "CUDA":
            d = per.setdefault(e.name, [0, 0.0])
            d[0] += 1
            d[1] += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
    kernels = sorted(({"name": k, "calls_per_step": v[0] / steps, "ms_per_step": v[1] / 1e3 / steps}
                      for k, v in per.items()), key=lambda d: -d["ms_per_step"])
    groups = {w: sum(d["ms_per_step"] for d in kernels if w in d["name"]) for w in WGRAD_KERNELS}
    groups["fix_flush_kernel"] = sum(d["ms_per_step"] for d in kernels if "fix_flush_kernel" in d["name"])
    groups["device_total"] = sum(d["ms_per_step"] for d in kernels)
    return {"steps": steps, "groups_ms_per_step": groups, "kernels": kernels[:40]}


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--shapes-only", action="store_true", help="print the shapes and their bounds without timing")
    ap.add_argument("--profile-steps", type=int, default=0, help="profile this many training steps instead")
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    args = ap.parse_args()
    assert args.reps >= 7, "at least 7 timed launches per shape"
    if args.profile_steps:
        result = {"workload": "ResNet-50 BYOL @%d, batch %d" % (args.image_size, args.batch), "card": card()}
        result.update(profile_steps(args.batch, args.image_size, args.profile_steps))
        print("# %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"]))
        for k, v in result["groups_ms_per_step"].items():
            print("%-28s %8.3f ms/step" % (k, v))
        for d in result["kernels"][:25]:
            print("%8.3f ms %6.1f calls  %s" % (d["ms_per_step"], d["calls_per_step"], d["name"][:110]))
    else:
        rows = shape_rows(args.batch, args.image_size)
        result = {"workload": "ResNet-50 wgrad, batch %d, %d px" % (args.batch, args.image_size)}
        if not args.shapes_only:
            result["card"] = card()
            result["library"] = time_rows(rows, args.batch, args.reps)
            print("# %s | %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"],
                                      result["library"]))
        print("%-26s %-9s %6s %8s %8s %7s %8s %9s %8s %7s" % ("shape", "route", "n/step", "GFLOP", "MB", "bound",
                                                             "bound_ms", "ms", "spread", "of_bnd"))
        for r in rows:
            print("%-26s %-9s %6d %8.1f %8.1f %7s %8.3f %9s %8s %7s" % (
                r["name"], r["route"], r["launches_per_step"], r["gflop"], r["bytes"] / 1e6, r["bound"], r["bound_ms"],
                "%.3f" % r["ms"] if "ms" in r else "-", "%.3f" % r["spread_ms"] if "ms" in r else "-",
                "%.1f%%" % (100 * r["frac_of_bound"]) if "ms" in r else "-"))
        result["rows"], result["totals"] = rows, totals(rows)
        for key, t in result["totals"].items():
            line = "%s: %d launches/step, %.2f TFLOP, %.1f GB, bound %.2f ms" % (
                key, t["launches_per_step"], t["TFLOP_per_step"], t["GB_per_step"], t["bound_ms_per_step"])
            if "ms_per_step" in t:
                line += ", measured %.2f ms (%.1f%% of the bound's speed)" % (t["ms_per_step"], 100 * t["frac_of_bound"])
            print("# total " + line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
