"""Time the fixed-route BatchNorm kernels of ResNet-50: every distinct bn_apply / bn_bwd_reduce / bn_bwd_apply launch of
one BYOL training step that takes the channel-pinned ("fixed") kernels, each through ops.bn_* as the engine calls it.

Shapes (M rows x C channels, NHWC bf16), per step:
  apply_ff  inner bn1 / bn2 + ReLU, no residual (4 forward lanes)
  apply_tf  block output bn3 + identity residual + ReLU, mask bits written (4 lanes)
  apply_tt  block output bn3 + downsample-BN residual + ReLU, mask bits written (4 lanes)
  reduce1 / bwd_apply1  inner bn1 / bn2, the stem BN and the heads' BatchNorm1d (4096 x batch), ReLU mask recomputed
            from x (2 online backward passes)
  reduce3 / bwd_apply3  bn3 and the downsample BN, mask bits from the forward (2 passes)
The stem's forward BN runs fused with its max pool and the heads' forward BN inside the fused MLP kernel, so neither
appears here.

Per shape: launches per step, the bytes the launch must move (from the shapes: bf16 operands, 1 bit per element of
mask), the HBM bound at the H100 SXM data-sheet rate (3.35 TB/s), the median of --reps launches timed with CUDA events
with L2 flushed before each, and its fraction of the bound.  A reduction's time includes its fix_flush_kernel, which
adds the fixed-point sums to the fp32 output.  Totals are weighted by the launches of one step, per
family and overall.

--profile-steps K instead profiles K BYOL training steps (ResNet-50 @224, --batch images) with torch.profiler and sums
the device time per kernel name (tools/bench_wgrad.py's profile), with the BatchNorm families split out.

    python tools/bench_bn.py                           # batch 512, 224 px
    python tools/bench_bn.py --shapes-only             # the shape table and its bounds, no GPU needed
    python tools/bench_bn.py --out table.json --tag bn # adds {"bn": result} to table.json (kept if it exists)
    python tools/bench_bn.py --profile-steps 3 --out table.json --tag profile_bn
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_gemm1x1 import HBM_BPS, STAGES, card  # noqa: E402

FWD_LANES, BWD_PASSES = 4, 2
HEAD_BN = [("proj", 4096), ("pred", 4096)]       # BatchNorm1d of the projector and the predictor
# bytes per element: bf16 operands, mask bits at 1/8 byte
BYTES = {"apply_ff": 4.0, "apply_tf": 6.125, "apply_tt": 6.125, "reduce1": 4.0, "reduce3": 4.125,
         "bwd_apply1": 6.0, "bwd_apply3": 6.125}
FAMILIES = {"apply_ff": "bn_apply_fixed_kernel<false,false>", "apply_tf": "bn_apply_fixed_kernel<true,false>",
            "apply_tt": "bn_apply_fixed_kernel<true,true>", "reduce1": "bn_bwd_reduce_fixed_kernel<1>",
            "reduce3": "bn_bwd_reduce_fixed_kernel<3>", "bwd_apply1": "bn_bwd_apply_fixed_kernel<1>",
            "bwd_apply3": "bn_bwd_apply_fixed_kernel<3>"}


def resnet50_bn_shapes(batch, image_size):
    """{(kind, M, C): launches per step}."""
    shapes = {}

    def add(kind, m, c, n):
        shapes[(kind, m, c)] = shapes.get((kind, m, c), 0) + n
    h = (image_size + 1) // 2
    add("reduce1", batch * h * h, 64, BWD_PASSES)                 # stem
    add("bwd_apply1", batch * h * h, 64, BWD_PASSES)
    h = (h + 1) // 2
    for planes, blocks, stride in STAGES:
        for i in range(blocks):
            s = stride if i == 0 else 1
            hout = (h - 1) // s + 1
            for m in (batch * h * h, batch * hout * hout):       # bn1 at the input resolution, bn2 after the stride
                add("apply_ff", m, planes, FWD_LANES)
                add("reduce1", m, planes, BWD_PASSES)
                add("bwd_apply1", m, planes, BWD_PASSES)
            mo = batch * hout * hout
            add("apply_tt" if i == 0 else "apply_tf", mo, 4 * planes, FWD_LANES)
            n3 = 2 if i == 0 else 1                               # bn3, and the downsample BN in the first block
            add("reduce3", mo, 4 * planes, n3 * BWD_PASSES)
            add("bwd_apply3", mo, 4 * planes, n3 * BWD_PASSES)
            h = hout
    for _, c in HEAD_BN:
        add("reduce1", batch, c, BWD_PASSES)
        add("bwd_apply1", batch, c, BWD_PASSES)
    return shapes


def shape_rows(batch, image_size):
    rows = []
    for (kind, m, c), n in sorted(resnet50_bn_shapes(batch, image_size).items(),
                                  key=lambda kv: (list(FAMILIES).index(kv[0][0]), -kv[0][1] * kv[0][2])):
        nbytes = BYTES[kind] * m * c
        rows.append({"name": "%s_%dx%d" % (kind, m, c), "kind": kind, "kernel": FAMILIES[kind], "M": m, "C": c,
                     "launches_per_step": n, "bytes": nbytes, "bound_ms": 1e3 * nbytes / HBM_BPS})
    return rows


def operands(kind, m, c, dev, g):
    """Seeded operands at the magnitudes of real data: activations ~N(0, 1), gradients ~1e-3, random mask bits,
    coefficients that are not powers of two, drawn on the generator's device and moved to `dev`.  Returns a function
    running the launch and its outputs.  (torch's CUDA sampling kernels size their grids from the SM count, so only a
    CPU generator gives the same operands on every GPU.)"""
    import torch
    from byol_b200 import ops
    BF = torch.bfloat16
    gd = g.device

    def coef(lo, hi):
        return (torch.rand(c, device=gd, generator=g) * (hi - lo) + lo).to(dev)
    x = torch.randn(m, c, device=gd, generator=g).to(dev, BF)
    scale, shift = coef(0.5, 1.5), coef(-0.3, 0.3)
    mean, invstd = coef(-0.2, 0.2), coef(0.7, 1.9)
    coeffs = torch.stack([scale, shift, mean, invstd])
    if kind.startswith("apply"):
        out = torch.empty_like(x)
        if kind == "apply_ff":
            return (lambda: ops.bn_apply(x, scale, shift, True, out=out)), {"y": out}
        resid = torch.randn(m, c, device=gd, generator=g).to(dev, BF)
        mask = torch.empty(m * c // 8, dtype=torch.uint8, device=dev)
        rsc, rsh = (coef(0.5, 1.5), coef(-0.3, 0.3)) if kind == "apply_tt" else (None, None)
        return (lambda: ops.bn_apply(x, scale, shift, True, resid=resid, rscale=rsc, rshift=rsh, out=out,
                                     mask_out=mask)), {"y": out, "mask": mask}
    gr = (torch.randn(m, c, device=gd, generator=g) * 1e-3).to(dev, BF)
    mode = 1 if kind.endswith("1") else 3
    act = (torch.randint(0, 256, (m * c // 8,), dtype=torch.uint8, device=gd, generator=g).to(dev) if mode == 3
           else None)
    if kind.startswith("reduce"):
        s12 = torch.zeros(2 * c, device=dev)     # the first launch's sums (timed launches keep adding to them)
        return (lambda: ops.bn_bwd_reduce(gr, x, coeffs, s12, mode, act=act)), {"s12": s12}
    s12 = (torch.cat([torch.randn(c, device=gd, generator=g), torch.randn(c, device=gd, generator=g)]) * 0.3).to(dev)
    gamma = coef(0.5, 1.5)
    dy = torch.empty_like(x)
    return (lambda: ops.bn_bwd_apply(gr, x, coeffs, gamma, s12, m, mode, act=act, dy=dy)), {"dy": dy}


def time_rows(rows, reps):
    import torch
    from byol_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("bench_bn: no CUDA device (use --shapes-only for the shape table)")
    dev = torch.device("cuda", 0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    for r in rows:
        fn, _ = operands(r["kind"], r["M"], r["C"], dev, g)
        for _ in range(2):
            fn()
        ts = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(reps):
            flush.fill_(1)
            # ~100 us of device work queued before the window opens, so that the window holds the launch's device
            # time and not the host's time to enqueue it (the small shapes run for tens of microseconds)
            torch.cuda._sleep(200_000)
            e0.record(); fn(); e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        ts.sort()
        r["ms"], r["spread_ms"] = ts[len(ts) // 2], ts[-1] - ts[0]
        r["frac_of_bound"] = r["bound_ms"] / r["ms"]
        del fn
        torch.cuda.empty_cache()
    return os.path.basename(_lib.LIB_PATH)   # the file name only: a record must not carry this machine's paths


def totals(rows):
    tot = {}
    for key in list(FAMILIES) + ["all"]:
        sel = [r for r in rows if key in ("all", r["kind"])]
        t = {"launches_per_step": sum(r["launches_per_step"] for r in sel),
             "GB_per_step": sum(r["launches_per_step"] * r["bytes"] for r in sel) / 1e9,
             "bound_ms_per_step": sum(r["launches_per_step"] * r["bound_ms"] for r in sel)}
        if sel and "ms" in sel[0]:
            t["ms_per_step"] = sum(r["launches_per_step"] * r["ms"] for r in sel)
            t["frac_of_bound"] = t["bound_ms_per_step"] / t["ms_per_step"]
        tot[key] = t
    return tot


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--shapes-only", action="store_true", help="print the shapes and their bounds without timing")
    ap.add_argument("--profile-steps", type=int, default=0, help="profile this many training steps instead")
    ap.add_argument("--out", default=None, help="also write the result as JSON")
    ap.add_argument("--tag", default=None, help="with --out: store the result under this key of the file's object")
    args = ap.parse_args()
    assert args.reps >= 9, "at least 9 timed launches per shape"
    if args.profile_steps:
        from bench_wgrad import profile_steps
        result = {"workload": "ResNet-50 BYOL @%d, batch %d" % (args.image_size, args.batch), "card": card()}
        prof = profile_steps(args.batch, args.image_size, args.profile_steps)
        groups = {f: sum(d["ms_per_step"] for d in prof["kernels"] if fam.replace(",", ", ") in d["name"])
                  for f, fam in FAMILIES.items()}
        groups["bn_fixed_total"] = sum(groups.values())
        groups["device_total"] = prof["groups_ms_per_step"]["device_total"]
        result.update({"steps": prof["steps"], "groups_ms_per_step": groups, "kernels": prof["kernels"]})
        print("# %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"]))
        for k, v in groups.items():
            print("%-28s %8.3f ms/step" % (k, v))
    else:
        rows = shape_rows(args.batch, args.image_size)
        result = {"workload": "ResNet-50 BatchNorm (fixed route), batch %d, %d px" % (args.batch, args.image_size)}
        if not args.shapes_only:
            result["card"] = card()
            result["library"] = time_rows(rows, args.reps)
            print("# %s | %s | %s" % (result["card"]["name"], result["card"]["power_limit_and_max_sm_clock"],
                                      result["library"]))
        print("%-24s %6s %6s %9s %8s %8s %8s %7s" % ("shape", "n/step", "C", "MB", "bound_ms", "ms", "spread",
                                                     "of_bnd"))
        for r in rows:
            print("%-24s %6d %6d %9.1f %8.3f %8s %8s %7s" % (
                r["name"], r["launches_per_step"], r["C"], r["bytes"] / 1e6, r["bound_ms"],
                "%.3f" % r["ms"] if "ms" in r else "-", "%.3f" % r["spread_ms"] if "ms" in r else "-",
                "%.1f%%" % (100 * r["frac_of_bound"]) if "ms" in r else "-"))
        result["rows"], result["totals"] = rows, totals(rows)
        for key, t in result["totals"].items():
            line = "%s: %d launches/step, %.1f GB, bound %.2f ms" % (key, t["launches_per_step"], t["GB_per_step"],
                                                                    t["bound_ms_per_step"])
            if "ms_per_step" in t:
                line += ", measured %.2f ms (%.1f%% of the bound's speed)" % (t["ms_per_step"],
                                                                           100 * t["frac_of_bound"])
            print("# total " + line)
    if args.out:
        if args.tag:
            doc = {}
            if os.path.exists(args.out):
                with open(args.out) as f:
                    doc = json.load(f)
            doc[args.tag] = result
            result = doc
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
