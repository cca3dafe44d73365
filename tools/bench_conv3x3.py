"""Time the 3x3 convolutions of ResNet-50: every distinct stride-1 3x3 shape that takes the shared-memory patch route
(conv3x3_patch_kernel: 56x56 with 64 channels, 28x28 with 128, 14x14 with 256), as a fprop with fused BatchNorm
statistics (as the engine calls it) and as a dgrad (the patch kernel with flipped taps).  --gather times the 3x3
shapes that take the implicit-GEMM gather route instead (stride 2, and 7x7 where W < 12).

Per shape: median of --reps launches timed with CUDA events, L2 flushed before each launch (as bench.py's layer
table does), the FLOPs and the bytes the launch must move (read the input and the weight, write the output), both
from the shapes, the achieved TFLOP/s and its fraction of the H100 SXM data-sheet dense bf16 rate (989 TFLOP/s), the
fraction of the larger of the compute and HBM bounds, and totals weighted by the launches of one training step
(fprop: 4 encoder passes, dgrad: the 2 online backward passes).

    python tools/bench_conv3x3.py                      # batch 512, 224 px, patch-route shapes
    python tools/bench_conv3x3.py --gather             # the gather-route 3x3 shapes
    python tools/bench_conv3x3.py --shapes-only        # the shape table and its bounds, no GPU needed
    python tools/bench_conv3x3.py --out table.json
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_gemm1x1 import BF16_FLOPS, DGRAD_PASSES, FPROP_PASSES, HBM_BPS, STAGES, card  # noqa: E402


def resnet50_shapes(image_size, gather):
    """{(kind, C, hw_in, stride): layers per pass} of the bottleneck conv2 (3x3, pad 1, C -> C channels).
    gather=False: the stride-1 layers with W >= 12 (patch route); True: the stride-2 and the W < 12 ones."""
    h = (image_size + 1) // 2          # stem 7x7 / 2
    h = (h + 1) // 2                   # max pool 3x3 / 2
    shapes = {}
    for planes, blocks, stride in STAGES:
        for i in range(blocks):
            s = stride if i == 0 else 1
            patch = s == 1 and h >= 12
            if patch != gather:
                for kind in ("fprop", "dgrad"):
                    key = (kind, planes, h, s)
                    shapes[key] = shapes.get(key, 0) + 1
            h = (h - 1) // s + 1
    return shapes


def shape_rows(batch, image_size, gather):
    rows = []
    for (kind, c, hw, s), count in sorted(resnet50_shapes(image_size, gather).items()):
        ho = (hw - 1) // s + 1
        m = batch * ho * ho
        launches = count * (FPROP_PASSES if kind == "fprop" else DGRAD_PASSES)
        nbytes = 2 * (batch * hw * hw * c + m * c + 9 * c * c)
        flop = 2.0 * m * c * 9 * c
        rows.append({"kind": kind, "C": c, "Ndim": c, "hw": hw, "stride": s, "M": m, "launches_per_step": launches,
                     "bytes": nbytes, "gflop": flop / 1e9,
                     "bound": "compute" if flop / BF16_FLOPS >= nbytes / HBM_BPS else "HBM",
                     "bound_ms": 1e3 * max(nbytes / HBM_BPS, flop / BF16_FLOPS)})
    return rows


def time_rows(rows, batch, reps):
    import torch
    from byol_b200 import _lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_conv3x3: no CUDA device (use --shapes-only for the shape table)")
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
        return ts[len(ts) // 2]

    for r in rows:
        c, hw, s = r["C"], r["hw"], r["stride"]
        ho = (hw - 1) // s + 1
        # [Ndim][9 * C] with k = tap * C + c (fprop) and [Cin][9 * Cout] (dgrad): both [C][9 * C] here
        w = (torch.randn(c, 9 * c, device=dev, generator=g) / (3 * c ** 0.5)).to(BF)
        if r["kind"] == "fprop":
            x = torch.randn(batch, hw, hw, c, device=dev, generator=g).to(BF)
            out = torch.empty(batch, ho, ho, c, device=dev, dtype=BF)
            stats = torch.zeros(2 * c, device=dev)
            ms = timed(lambda: ops.conv_fprop(x, w, 3, 3, s, 1, stats=stats, out=out))
        else:
            x = torch.randn(batch, ho, ho, c, device=dev, generator=g).to(BF)
            out = torch.empty(batch, hw, hw, c, device=dev, dtype=BF)
            ms = timed(lambda: ops.conv_dgrad(x, w, hw, hw, 3, 3, s, 1, out=out))
        r["ms"] = ms
        r["TFLOPs"] = r["gflop"] / ms     # GFLOP per ms
        r["frac_peak"] = r["gflop"] * 1e9 / (ms * 1e-3) / BF16_FLOPS
        r["frac_bound"] = r["bound_ms"] / ms
        del x, w, out
    return _lib.LIB_PATH


def totals(rows):
    tot = {}
    for kind in ("fprop", "dgrad"):
        sel = [r for r in rows if r["kind"] == kind]
        t = {"launches_per_step": sum(r["launches_per_step"] for r in sel),
             "TFLOP_per_step": sum(r["launches_per_step"] * r["gflop"] for r in sel) / 1e3,
             "bound_ms_per_step": sum(r["launches_per_step"] * r["bound_ms"] for r in sel)}
        if sel and "ms" in sel[0]:
            t["ms_per_step"] = sum(r["launches_per_step"] * r["ms"] for r in sel)
            t["TFLOPs"] = t["TFLOP_per_step"] / t["ms_per_step"] * 1e3
        tot[kind] = t
    return tot


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--gather", action="store_true", help="the gather-route 3x3 shapes instead of the patch route")
    ap.add_argument("--shapes-only", action="store_true", help="print the shapes and their bounds without timing")
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    args = ap.parse_args()
    assert args.reps >= 5, "at least 5 timed launches per shape"
    rows = shape_rows(args.batch, args.image_size, args.gather)
    route = "gather" if args.gather else "patch"
    result = {"workload": "ResNet-50 3x3 convolutions (%s route), batch %d, %d px" % (route, args.batch,
                                                                                      args.image_size)}
    if not args.shapes_only:
        result["card"] = card()
        result["library"] = time_rows(rows, args.batch, args.reps)
        print("# %s | %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"],
                                  result["library"]))
    print("%-5s %5s %4s %2s %8s %6s %8s %7s %9s %8s %7s %7s %8s" % (
        "kind", "C", "hw", "s", "M", "n/step", "GFLOP", "bound", "bound_ms", "ms", "TFLOP/s", "of_peak", "of_bound"))
    for r in rows:
        timed = "ms" in r
        print("%-5s %5d %4d %2d %8d %6d %8.1f %7s %9.3f %8s %7s %7s %8s" % (
            r["kind"], r["C"], r["hw"], r["stride"], r["M"], r["launches_per_step"], r["gflop"], r["bound"],
            r["bound_ms"], "%.3f" % r["ms"] if timed else "-", "%.0f" % r["TFLOPs"] if timed else "-",
            "%.1f%%" % (100 * r["frac_peak"]) if timed else "-", "%.1f%%" % (100 * r["frac_bound"]) if timed else "-"))
    result["rows"], result["totals"] = rows, totals(rows)
    for kind, t in result["totals"].items():
        line = "%s: %d launches/step, %.2f TFLOP, bound %.2f ms" % (
            kind, t["launches_per_step"], t["TFLOP_per_step"], t["bound_ms_per_step"])
        if "ms_per_step" in t:
            line += ", measured %.2f ms (%.0f TFLOP/s)" % (t["ms_per_step"], t["TFLOPs"])
        print("# total " + line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
