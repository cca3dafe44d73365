"""Grouped 3x3 convolutions of ResNeXt-50 (32x4d) at 224x224: every distinct conv2 shape, timed per kernel (fprop with
BatchNorm statistics, dgrad, wgrad) and through torch's cuDNN grouped convolution (bf16, channels_last) in the same
process.  CUDA events, L2 flushed before every timed launch, warmed up, median of --reps.

    python tools/bench_grouped.py --batch 256 --out out/bench_grouped.jsonl

Per shape: time, algorithmic FLOPs (2*M*C*Cg*9, what the convolution needs), executed FLOPs (2*M*C*64*9: the
block-diagonal 64-channel tiles multiply 64 / Cg times the algorithmic work), the bytes each pass must move (inputs,
outputs, weights; bf16 activations, fp32 weight gradient) and which bound applies: the larger of executed FLOPs over
the data-sheet dense BF16 rate and bytes over the HBM3 bandwidth of an H100 SXM (989 TFLOP/s, 3.35 TB/s).  The card
name and power limit are printed with the results.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

PEAK_FLOPS = 989e12
PEAK_BW = 3.35e12
# ResNeXt-50 32x4d at 224: conv2 (C channels, Cg per group) per stage; input map, stride
SHAPES = [(128, 4, 56, 1), (256, 8, 56, 2), (256, 8, 28, 1), (512, 16, 28, 2), (512, 16, 14, 1), (1024, 32, 14, 2),
          (1024, 32, 7, 1)]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                               capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        limit = None
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grouped.py needs a GPU")
    from byol_b200 import ops
    dev = torch.device("cuda:0")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    def timed(fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(args.reps):
            flush.fill_(1)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        return ts[len(ts) // 2]

    name, limit = card()
    rows = []
    n = args.batch
    for c, cg, h, s in SHAPES:
        ho = (h - 1) // s + 1
        m = n * ho * ho
        g = torch.Generator(device=dev).manual_seed(c + h)
        x = torch.randn(n, h, h, c, device=dev, generator=g).to(torch.bfloat16)
        dy = torch.randn(n, ho, ho, c, device=dev, generator=g).to(torch.bfloat16)
        w = torch.randn(c, cg, 3, 3, device=dev, generator=g) / (cg * 9) ** 0.5
        wf, wd = ops.prep_weight_grouped(w)
        dw = torch.zeros(c, cg, 3, 3, device=dev)
        stats = torch.zeros(2 * c, device=dev)
        t = {"fprop": timed(lambda: ops.conv_fprop(x, wf, 3, 3, s, 1, stats=stats)),
             "dgrad": timed(lambda: ops.conv_dgrad(dy, wd, h, h, 3, 3, s, 1)),
             "wgrad": timed(lambda: ops.conv_wgrad(x, dy, dw, 3, 3, s, 1))}
        # cuDNN on the same shapes (bf16, channels_last)
        xc = x.permute(0, 3, 1, 2)          # NHWC memory = channels_last NCHW view
        wc = w.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dyc = dy.permute(0, 3, 1, 2)
        t_cudnn = {"fprop": timed(lambda: F.conv2d(xc, wc, None, s, 1, 1, c // cg)),
                   "dgrad": timed(lambda: torch.nn.grad.conv2d_input(xc.shape, wc, dyc, s, 1, 1, c // cg)),
                   "wgrad": timed(lambda: torch.nn.grad.conv2d_weight(xc, wc.shape, dyc, s, 1, 1, c // cg))}
        alg = 2.0 * m * c * cg * 9
        exe = 2.0 * m * c * 64 * 9
        act_in, act_out = n * h * h * c * 2, m * c * 2
        byts = {"fprop": act_in + act_out + c * 576 * 2, "dgrad": act_out + act_in + c * 576 * 2,
                "wgrad": act_in + act_out + c * cg * 9 * 4 * 2}
        for op in ("fprop", "dgrad", "wgrad"):
            t_flop, t_mem = exe / PEAK_FLOPS, byts[op] / PEAK_BW
            row = {"op": op, "C": c, "Cg": cg, "hin": h, "stride": s, "batch": n, "ms": round(t[op], 4),
                   "cudnn_ms": round(t_cudnn[op], 4), "alg_gflop": round(alg / 1e9, 3),
                   "exec_gflop": round(exe / 1e9, 3), "gbytes": round(byts[op] / 1e9, 4),
                   "bound": "compute" if t_flop > t_mem else "memory",
                   "share_of_bound": round(max(t_flop, t_mem) * 1e3 / t[op], 3),
                   "alg_tflops": round(alg / t[op] / 1e9, 1), "exec_tflops": round(exe / t[op] / 1e9, 1),
                   "gpu": name, "power_limit_w": limit}
            rows.append(row)
            print(json.dumps(row))
        del x, dy, xc, dyc, wc, w, wf, wd, dw
    tot = {op: sum(r["ms"] for r in rows if r["op"] == op) for op in ("fprop", "dgrad", "wgrad")}
    tot_c = {op: sum(r["cudnn_ms"] for r in rows if r["op"] == op) for op in ("fprop", "dgrad", "wgrad")}
    summary = {"summary": "sum over the distinct shapes (one launch each)", "ms": tot, "cudnn_ms": tot_c, "gpu": name,
               "power_limit_w": limit, "batch": n}
    print(json.dumps(summary))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in rows + [summary]:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
