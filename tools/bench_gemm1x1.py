"""Time the 1x1 convolutions of ResNet-50 that run as plain TMA-fed GEMMs (conv_igemm_kernel with a TMA A operand):
every distinct 1x1 fprop with fused BatchNorm statistics (c1, c3 and the downsample of each bottleneck; the stride-2
downsample reads its compacted input) and every plain 1x1 dgrad without a residual (c3 and the downsample).

Per shape: median of --reps launches timed with CUDA events, L2 flushed before each launch (as bench.py's layer
table does), the bytes the launch must move (read the input and the weight, write the output) and its FLOPs, both
from the shapes, the achieved bandwidth and its fraction of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s), and
totals weighted by the launches of one training step (fprop: 4 encoder passes, dgrad: the 2 online backward passes).

    python tools/bench_gemm1x1.py                      # batch 512, 224 px
    python tools/bench_gemm1x1.py --shapes-only        # the shape table and its bounds, no GPU needed
    python tools/bench_gemm1x1.py --out table.json
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BPS = 3.35e12        # H100 SXM data sheet, HBM3
BF16_FLOPS = 989.4e12    # H100 SXM data sheet, dense bf16 (700 W)
FPROP_PASSES, DGRAD_PASSES = 4, 2
# ResNet-50 bottleneck stages: (planes, blocks, stride of the first block); the stride sits in conv2 (v1.5)
STAGES = [(64, 3, 1), (128, 4, 2), (256, 6, 2), (512, 3, 2)]


def resnet50_shapes(image_size):
    """{(kind, C, Ndim, hw): launches per pass}: kind 'fprop' (C -> Ndim at hw x hw, with statistics) or 'dgrad'
    (dY with C channels -> dX with Ndim channels at hw x hw)."""
    h = (image_size + 1) // 2          # stem 7x7 / 2
    h = (h + 1) // 2                   # max pool 3x3 / 2
    cin = 64
    shapes = {}

    def add(key):
        shapes[key] = shapes.get(key, 0) + 1
    for planes, blocks, stride in STAGES:
        for i in range(blocks):
            s = stride if i == 0 else 1
            hout = (h - 1) // s + 1
            add(("fprop", cin, planes, h))                 # c1 at the block's input resolution
            add(("fprop", planes, 4 * planes, hout))       # c3
            add(("dgrad", 4 * planes, planes, hout))       # c3 dgrad (c1's dgrad carries the residual gradient)
            if i == 0:
                add(("fprop", cin, 4 * planes, hout))      # downsample (stride 2: on the compacted input)
                add(("dgrad", 4 * planes, cin, hout))
            cin, h = 4 * planes, hout
    return shapes


def shape_rows(batch, image_size):
    rows = []
    for (kind, c, n, hw), count in sorted(resnet50_shapes(image_size).items()):
        m = batch * hw * hw
        launches = count * (FPROP_PASSES if kind == "fprop" else DGRAD_PASSES)
        nbytes = 2 * (m * c + m * n + n * c)
        flop = 2.0 * m * c * n
        rows.append({"kind": kind, "C": c, "Ndim": n, "hw": hw, "M": m, "launches_per_step": launches,
                     "bytes": nbytes, "gflop": flop / 1e9,
                     "bound_ms": 1e3 * max(nbytes / HBM_BPS, flop / BF16_FLOPS)})
    return rows


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # the card name still identifies the number
        q = "nvidia-smi unavailable (%s)" % e
    return {"name": name, "power_limit_and_max_sm_clock": q}


def time_rows(rows, reps):
    import torch
    from byol_b200 import _lib, ops
    if not torch.cuda.is_available():
        raise SystemExit("bench_gemm1x1: no CUDA device (use --shapes-only for the shape table)")
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
        c, n, hw = r["C"], r["Ndim"], r["hw"]
        src = torch.randn(r["M"] // (hw * hw), hw, hw, c, device=dev, generator=g).to(BF)
        w = (torch.randn(n, c, device=dev, generator=g) / c ** 0.5).to(BF)     # [Ndim][K], K = C for a 1x1
        out = torch.empty(src.shape[0], hw, hw, n, device=dev, dtype=BF)
        if r["kind"] == "fprop":
            stats = torch.zeros(2 * n, device=dev)
            ms = timed(lambda: ops.conv_fprop(src, w, 1, 1, 1, 0, stats=stats, out=out))
        else:
            ms = timed(lambda: ops.conv_dgrad(src, w, hw, hw, 1, 1, 1, 0, out=out))
        r["ms"] = ms
        r["GBps"] = r["bytes"] / ms / 1e6
        r["frac_hbm"] = r["bytes"] / (ms * 1e-3) / HBM_BPS
        del src, w, out
    return _lib.LIB_PATH


def totals(rows):
    tot = {}
    for kind in ("fprop", "dgrad"):
        sel = [r for r in rows if r["kind"] == kind]
        t = {"launches_per_step": sum(r["launches_per_step"] for r in sel),
             "GB_per_step": sum(r["launches_per_step"] * r["bytes"] for r in sel) / 1e9,
             "TFLOP_per_step": sum(r["launches_per_step"] * r["gflop"] for r in sel) / 1e3,
             "bound_ms_per_step": sum(r["launches_per_step"] * r["bound_ms"] for r in sel)}
        if sel and "ms" in sel[0]:
            t["ms_per_step"] = sum(r["launches_per_step"] * r["ms"] for r in sel)
            t["frac_of_bound"] = t["bound_ms_per_step"] / t["ms_per_step"]
        tot[kind] = t
    return tot


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--shapes-only", action="store_true", help="print the shapes and their bounds without timing")
    ap.add_argument("--out", default=None, help="also write the table as JSON")
    args = ap.parse_args()
    assert args.reps >= 5, "at least 5 timed launches per shape"
    rows = shape_rows(args.batch, args.image_size)
    result = {"workload": "ResNet-50 1x1 GEMMs, batch %d, %d px" % (args.batch, args.image_size)}
    if not args.shapes_only:
        result["card"] = card()
        result["library"] = time_rows(rows, args.reps)
        print("# %s | %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"],
                                  result["library"]))
    print("%-5s %5s %5s %4s %8s %6s %9s %9s %8s %8s %7s" % ("kind", "C", "Ndim", "hw", "M", "n/step", "MB", "bound_ms",
                                                         "ms", "GB/s", "of_HBM"))
    for r in rows:
        print("%-5s %5d %5d %4d %8d %6d %9.1f %9.3f %8s %8s %7s" % (
            r["kind"], r["C"], r["Ndim"], r["hw"], r["M"], r["launches_per_step"], r["bytes"] / 1e6, r["bound_ms"],
            "%.3f" % r["ms"] if "ms" in r else "-", "%.0f" % r["GBps"] if "ms" in r else "-",
            "%.1f%%" % (100 * r["frac_hbm"]) if "ms" in r else "-"))
    result["rows"], result["totals"] = rows, totals(rows)
    for kind, t in result["totals"].items():
        line = "%s: %d launches/step, %.1f GB, %.2f TFLOP, bound %.2f ms" % (
            kind, t["launches_per_step"], t["GB_per_step"], t["TFLOP_per_step"], t["bound_ms_per_step"])
        if "ms_per_step" in t:
            line += ", measured %.2f ms (%.1f%% of the bound's speed)" % (t["ms_per_step"], 100 * t["frac_of_bound"])
        print("# total " + line)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
