#!/usr/bin/env python
"""bench.py — images/sec of the BYOL training step (ResNet-50 @224, synthetic data) on N H100s of one node.

    python bench.py --gpus 1 --steps 10 --warmup 3
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port P \
        bench.py --gpus 8 --steps 10 --warmup 3
    python bench.py --impl reference --steps 2 --warmup 1     # the reference algorithm on the host CPU cores
    python bench.py --steps 10 --warmup 3 --dump-outputs out/  # + what the last timed step computed, as .npy

One "step" = one pass of the hot path (/root/reference/main.py:579-624) over one synthetic batch: 4 encoder
passes (online x2 with grad, EMA target x2), loss, backward, gradient all-reduce, LARS+SGD, EMA update.  One
"image" = one dataset sample = one (aug1, aug2) pair (main.py:609).  Rank 0 prints ONE JSON line.

Workload (same per-GPU work at every N => weak scaling): ResNet-50 BYOL, 224x224, per-GPU batch 512, bf16
tensor-core compute with fp32 master weights / statistics / loss / optimizer, SyncBatchNorm + flat gradient
all-reduce when N > 1.  At N = 8 this is exactly BASELINE.json configs[2] (global batch 4096).
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ALG_GFLOP_PER_IMAGE = {("resnet50", 224): 65.1067, ("resnet18", 224): 28.6288, ("resnet50", 384): 190.9761,
                       ("resnet200", 224): 239.7994}   # BASELINE.md section 4
REP_DIM = {"resnet18": 512, "resnet34": 512}


_T0 = time.perf_counter()


def note(msg):
    """Progress on stderr (the JSON line on stdout stays alone)."""
    sys.stderr.write("[bench %7.1fs] %s\n" % (time.perf_counter() - _T0, msg))
    sys.stderr.flush()


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--arch", default="resnet50")
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--batch-per-gpu", type=int, default=512)
    ap.add_argument("--ref-batch", type=int, default=8, help="bounded sample batch for the CPU reference arm")
    ap.add_argument("--precision", default="bf16", choices=["bf16", "bf16x2", "fp32"],
                    help="forward arithmetic: bf16 operands (default) or the fp32-accurate split path (configs[1])")
    ap.add_argument("--no-sync-bn", action="store_true")
    ap.add_argument("--no-layers", action="store_true", help="skip the per-layer kernel roofline pass")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--layers-out", default=None, help="write the per-layer kernel table (JSON) to this path")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR",
                    help="after the timed steps write what the last timed step computed to DIR/<name>.npy (float32)")
    return ap.parse_args()


DUMP_SAMPLE = 1 << 20   # parameter vectors are dumped as a fixed, seeded sample of this many entries (4 MB each)


def dump_outputs(path, stats, model):
    """The step's results as a caller receives them: the returned losses / accuracies and the parameters the step
    updated (online weights after LARS, EMA target), the latter as the same seeded sample in every run."""
    import numpy as np
    import torch
    os.makedirs(path, exist_ok=True)
    arrays = dict(stats)
    theta, mean = model._engine.theta.detach(), model.target_network.mean.detach()
    idx = torch.randperm(theta.numel(), generator=torch.Generator().manual_seed(0))[:DUMP_SAMPLE].to(theta.device)
    arrays["params_sample"] = theta[idx]
    arrays["ema_params_sample"] = mean[idx]
    for name, t in arrays.items():
        np.save(os.path.join(path, name + ".npy"), t.detach().float().cpu().numpy())


# ------------------------------------------------------------------------------------------------
# clocks
# ------------------------------------------------------------------------------------------------
class ClockSampler(object):
    Q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
         "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
         "clocks_event_reasons.sw_power_cap")

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + self.Q,
                                          "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            threading.Thread(target=self._read, daemon=True).start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        sm, mx, reasons = [], None, set()
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx = float(r[1])
            except Exception:
                continue
            for name, v in zip(("hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"), r[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        busy = [x for x in sm if mx and x > 0.3 * mx] or sm
        return {"sm_mhz": busy[len(busy) // 2] if busy else None, "sm_max_mhz": mx, "reasons": sorted(reasons),
                "samples": len(sm)}


# ------------------------------------------------------------------------------------------------
# CPU reference arm / cpu_baseline (the ONLY place bench.py touches oracle/)
# ------------------------------------------------------------------------------------------------
def _host_threads():
    """Threads for the CPU arm.  torchrun exports OMP_NUM_THREADS=1 for its workers, which would silently turn the CPU
    arm into a single-thread run; all 128 hyper-threads of the GPU box, on the other hand, make the eager reference
    ~20x SLOWER than 64 (measured: oversubscribed OpenMP spin-waits around its many tiny ops).  So: one thread per
    physical core (half the visible CPUs), at most 64 — the count torch itself picks on that box."""
    import torch
    n = os.cpu_count() or 1
    try:
        n = len(os.sched_getaffinity(0))
    except Exception:
        pass
    torch.set_num_threads(max(1, min(64, n // 2 if n > 8 else n)))
    return torch.get_num_threads()


def _run_reference_main(arch, image_size, batch, steps, warmup):
    """The UNMODIFIED reference (oracle/_ref, byte-compiled by build()) on the host cores: its
    BYOL / loss_function / LARS(SGD) driven by its own main.execute_graph, --no-cuda, synthetic batches."""
    import torch
    ref = os.path.join(ROOT, "oracle", "_ref")
    if not os.path.exists(os.path.join(ref, "main.pyc")):
        return None
    rep = REP_DIM.get(arch, 2048)
    argv, path = sys.argv, list(sys.path)
    sys.argv = ["main.py", "--arch=%s" % arch, "--representation-size=%d" % rep, "--num-replicas=1", "--no-cuda",
                "--batch-size=%d" % batch, "--image-size-override=%d" % image_size]
    sys.path[:0] = [ref, os.path.join(ROOT, "oracle", "ref_shims")]
    try:
        import main
    finally:
        sys.argv, sys.path[:] = argv, path
    main.args.cuda, main.args.distributed_rank = False, 0
    from helpers import layers
    from optimizers.lars import LARS
    torch.manual_seed(0)
    model = main.BYOL(base_network_output_size=rep, projection_output_size=256, classifier_output_size=1000,
                      total_training_steps=1000, base_decay=0.996)
    opt = LARS(torch.optim.SGD(layers.add_weight_decay(model, 1e-6), lr=0.2 * batch / 256, momentum=0.9), eps=0.0)
    g = torch.Generator().manual_seed(1234)
    bt = (torch.rand(batch, 3, image_size, image_size, generator=g),
          torch.rand(batch, 3, image_size, image_size, generator=g), torch.randint(0, 1000, (batch,), generator=g))
    if warmup:
        main.execute_graph(0, model, [bt] * warmup, None, optimizer=opt, prefix="train")
    t0 = time.perf_counter()
    main.execute_graph(1, model, [bt] * steps, None, optimizer=opt, prefix="train")
    return time.perf_counter() - t0


def run_cpu_reference(arch, image_size, batch, steps, warmup):
    """The reference's own CPU implementation of the step on all host cores, on a bounded sample of the workload
    (`batch` images per step at the same geometry): the unmodified reference when it was shipped to this box
    (kind "reference"), else the oracle port of main.py's step, which is pinned against it (kind "port")."""
    import contextlib
    import io
    import torch
    cores = _host_threads()
    kind, what = "reference", "unmodified reference main.execute_graph (oracle/_ref)"
    with contextlib.redirect_stdout(io.StringIO()):        # the reference prints a log line per call
        dt = _run_reference_main(arch, image_size, batch, steps, warmup)
    if dt is None:
        from oracle import byol_oracle as O
        kind, what = "port", "oracle/byol_oracle.py"
        torch.manual_seed(0)
        params, buffers = O.init_reference_state(arch, 0)
        model = O.OracleBYOL(arch, params, buffers, 1000)
        g = torch.Generator().manual_seed(1234)
        a1 = torch.rand(batch, 3, image_size, image_size, generator=g)
        a2 = torch.rand(batch, 3, image_size, image_size, generator=g)
        lab = torch.randint(0, 1000, (batch,), generator=g)
        for _ in range(warmup):
            model.train_step(a1, a2, lab, 0.2 * batch / 256)
        t0 = time.perf_counter()
        for _ in range(steps):
            model.train_step(a1, a2, lab, 0.2 * batch / 256)
        dt = time.perf_counter() - t0
    return {"value": steps * batch / dt, "unit": "images/sec", "cores": cores, "kind": kind,
            "sample": "%d step(s) of %s BYOL at batch %d, %dx%d, fp32, torch CPU, %d threads (%s)"
                      % (steps, arch, batch, image_size, image_size, cores, what), "ms_per_step": 1000 * dt / steps}


def main_reference(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cb = run_cpu_reference(args.arch, args.image_size, args.ref_batch, args.steps, args.warmup)
    line = {"impl": "reference", "metric": "images/sec", "value": cb["value"], "unit": "images/sec",
            "n_gpus": args.gpus, "steps": args.steps, "warmup": args.warmup, "ms_per_step": cb["ms_per_step"],
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "fp32", "data": "synthetic",
            "config": {"workload": "%s BYOL training step %dx%d, CPU, bounded sample batch %d"
                                   % (args.arch, args.image_size, args.image_size, args.ref_batch)},
            "cpu_baseline": {k: cb[k] for k in ("value", "unit", "cores", "kind", "sample")},
            "e2e": {"value": cb["value"], "unit": "images/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
            "gpu_launches": 0}
    print(json.dumps(line))


# ------------------------------------------------------------------------------------------------
# per-layer kernel roofline (dominant kernel = wgmma implicit-GEMM conv, fprop + dgrad + wgrad)
# ------------------------------------------------------------------------------------------------
def layer_table(model, batch, image_size, reps=5):
    """Time every distinct conv shape of the encoder in isolation (CUDA events on the launching stream, L2
    flushed between launches by overwriting a 256 MiB buffer) and aggregate over the layer mix of one step."""
    import torch
    from byol_b200 import ops
    eng = model._engine
    dev = eng.device
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    shapes = {}
    h = image_size

    def add(u, hin):
        key = (u.cin, u.cout, u.k, u.stride, u.pad, hin)
        shapes.setdefault(key, [0, u])[0] += 1
        return ops.conv_out_size(hin, u.k, u.stride, u.pad)

    hcur = add(eng.stem, h)
    hcur = ops.conv_out_size(hcur, eng.pool_k, eng.pool_s, eng.pool_p)
    for b in eng.blocks:
        hin = hcur
        h1 = add(b.c1, hin)
        h2 = add(b.c2, h1)
        hout = add(b.c3, h2) if b.c3 is not None else h2
        if b.down is not None:
            add(b.down, hin)
        hcur = hout

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

    rows = []
    tot = {"fprop": [0.0, 0.0], "dgrad": [0.0, 0.0], "wgrad": [0.0, 0.0]}
    for (cin, cout, k, s, p, hin), (count, u) in sorted(shapes.items(), key=lambda kv: -kv[0][5]):
        ho = ops.conv_out_size(hin, k, s, p)
        x = torch.randn(batch, hin, hin, u.cpad, device=dev).to(torch.bfloat16)
        dy = torch.randn(batch, ho, ho, cout, device=dev).to(torch.bfloat16)
        wf, wd = eng.w_online.wf[u.idx], eng.w_online.wd[u.idx]
        dw = torch.zeros(cout, cin, k, k, device=dev)
        stats = torch.zeros(2 * cout, device=dev)
        flops = 2.0 * batch * ho * ho * cout * cin * k * k
        if u is eng.stem and eng.w_online.stem4_ok and ops.stem4_supported(cin, cout, hin, hin, k, s, p):
            # the engine's stem path: padded NHWC4 image + the dedicated kernels
            xs4 = ops.nchw_to_stem4(torch.randn(batch, cin, hin, hin, device=dev))
            t_f = timed(lambda: ops.stem_conv_fprop(xs4, eng.w_online.w_stem4, hin, hin, stats=stats))
            t_w = timed(lambda: ops.stem_conv_wgrad(xs4, dy, dw, hin, hin))
            del xs4
        elif k == 1 and s == 2 and p == 0 and hin % 2 == 0:
            # the engine's downsample path: compact the strided pixels once, then a plain TMA-fed GEMM (the
            # compaction is charged to fprop)
            xsub = ops.subsample2(x)
            t_f = timed(lambda: ops.conv_fprop(ops.subsample2(x), wf, 1, 1, 1, 0, stats=stats))
            t_w = timed(lambda: ops.conv_wgrad(xsub, dy, dw, 1, 1, 1, 0))
            del xsub
        else:
            t_f = timed(lambda: ops.conv_fprop(x, wf, k, k, s, p, stats=stats))
            t_w = timed(lambda: ops.conv_wgrad(x, dy, dw, k, k, s, p))
        t_d = timed(lambda: ops.conv_dgrad(dy, wd, hin, hin, k, k, s, p)) if wd is not None else None
        row = {"cin": cin, "cout": cout, "k": k, "stride": s, "hin": hin, "count": count, "gflop": flops / 1e9,
               "fprop_ms": t_f, "fprop_tflops": flops / t_f / 1e9, "wgrad_ms": t_w, "wgrad_tflops": flops / t_w / 1e9,
               "dgrad_ms": t_d, "dgrad_tflops": (flops / t_d / 1e9) if t_d else None}
        rows.append(row)
        # per step: fprop runs in 4 passes, dgrad / wgrad in the 2 online backward passes
        tot["fprop"][0] += 4 * count * flops; tot["fprop"][1] += 4 * count * t_f
        tot["wgrad"][0] += 2 * count * flops; tot["wgrad"][1] += 2 * count * t_w
        if t_d:
            tot["dgrad"][0] += 2 * count * flops; tot["dgrad"][1] += 2 * count * t_d
        del x, dy, dw
    agg = {k: {"tflops": v[0] / v[1] / 1e9 if v[1] else None, "ms_per_step": v[1], "launch_gflop": v[0] / 1e9}
           for k, v in tot.items()}
    return rows, agg


# ------------------------------------------------------------------------------------------------
# main arm
# ------------------------------------------------------------------------------------------------
def main_b200(args):
    import torch
    import torch.distributed as dist
    import torch.nn as nn
    from byol_b200 import _lib
    from byol_b200.model import BYOL
    from byol_b200 import wiring

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    if world != args.gpus:
        if world == 1 and args.gpus > 1:
            raise SystemExit("launch with torch.distributed.run --nproc-per-node %d for --gpus %d" % (args.gpus, args.gpus))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)

    b = args.batch_per_gpu
    gb = b * world
    R = args.image_size
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    # without a measured peak: NVIDIA's H100 SXM data sheet, dense bf16 at 700 W (a rate, not one reached here)
    peak_sustained = peaks.get("bf16_tflops_sustained", 989.4)
    peak_burst = peaks.get("bf16_tflops", 989.4)
    peak_src = "measured (MEASURED_PEAKS.json)" if peaks else "H100 SXM data sheet, dense bf16"

    torch.manual_seed(0)
    rep = REP_DIM.get(args.arch, 2048)
    model = BYOL(rep, 256, 1000, total_training_steps=1000, arch=args.arch, precision=args.precision)
    sync_bn = world > 1 and not args.no_sync_bn
    if sync_bn:
        model = nn.SyncBatchNorm.convert_sync_batchnorm(model)
    model = model.cuda().train()
    net = wiring.DistributedDataParallelPassthrough(model) if world > 1 else model
    opt = wiring.build_optimizer(model, base_lr=0.2, global_batch_size=gb)

    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    aug1 = torch.rand(b, 3, R, R, generator=g, device=dev)
    aug2 = torch.rand(b, 3, R, R, generator=g, device=dev)
    labels = torch.randint(0, 1000, (b,), generator=g, device=dev)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(ms):
        if world > 1:
            t = torch.tensor([ms], device=dev, dtype=torch.float64)
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            return float(t.item())
        return ms

    # ---- device-resident timing ---------------------------------------------------------------
    note("model built; warm-up")
    for _ in range(args.warmup):
        wiring.train_step(net, opt, aug1, aug2, labels)
    barrier()
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()
    l0 = _lib.launch_count[0]
    ms0 = torch.cuda.memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    t_host0 = time.perf_counter()
    for _ in range(args.steps):
        stats = wiring.train_step(net, opt, aug1, aug2, labels)
    host_ms = 1000.0 * (time.perf_counter() - t_host0) / args.steps   # Python time to ENQUEUE one step
    e1.record()
    barrier()
    if args.dump_outputs and rank == 0:
        dump_outputs(args.dump_outputs, stats, model)
    ms = max_over_ranks(e0.elapsed_time(e1))
    launches = (_lib.launch_count[0] - l0) // args.steps
    ms1 = torch.cuda.memory_stats()
    alloc_info = {"cudaMalloc_calls_in_timed_region": ms1.get("num_device_alloc", 0) - ms0.get("num_device_alloc", 0),
                  "cudaFree_calls_in_timed_region": ms1.get("num_device_free", 0) - ms0.get("num_device_free", 0),
                  "alloc_retries": ms1.get("num_alloc_retries", 0), "reserved_gb": torch.cuda.memory_reserved() / 1e9}
    clocks = sampler.stop() if rank == 0 else None
    loss_val = float(stats["loss_mean"].item())
    value = args.steps * gb / (ms / 1000.0)

    note("device-resident timing done: %.2f ms/step" % (ms / args.steps))
    # ---- end to end: pinned host inputs -> H2D -> step -> D2H loss, every step ------------------
    h1, h2 = aug1.cpu().pin_memory(), aug2.cpu().pin_memory()
    hl = labels.cpu().pin_memory()
    h2d = h1.numel() * 4 + h2.numel() * 4 + hl.numel() * 8
    d2h = 4

    # Every step copies ITS inputs host->device (pinned memory, on a side stream so the copy of step i+1 overlaps the
    # compute of step i, as a prefetching loader would) and reads ITS loss device->host (asynchronously into pinned
    # memory; all values are checked after the timed region).
    copy_stream = torch.cuda.Stream()
    loss_host = torch.zeros(args.steps + 1, dtype=torch.float32).pin_memory()

    def prefetch():
        with torch.cuda.stream(copy_stream):
            t = (h1.to(dev, non_blocking=True), h2.to(dev, non_blocking=True), hl.to(dev, non_blocking=True))
            ev = torch.cuda.Event()
            ev.record(copy_stream)
        return t, ev

    def e2e_step(i, cur):
        (a1, a2, lb), ev = cur
        torch.cuda.current_stream().wait_event(ev)
        nxt = prefetch()
        out = wiring.train_step(net, opt, a1, a2, lb)
        for t in (a1, a2, lb):
            t.record_stream(torch.cuda.current_stream())
        loss_host[i].copy_(out["loss_mean"], non_blocking=True)     # D2H read of the step's loss
        return nxt

    cur = prefetch()
    cur = e2e_step(args.steps, cur)
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        cur = e2e_step(i, cur)
    e1.record()
    barrier()
    assert bool(torch.isfinite(loss_host).all()), "non-finite loss in the end-to-end loop"
    ms_e2e = max_over_ranks(e0.elapsed_time(e1))
    e2e_value = args.steps * gb / (ms_e2e / 1000.0)

    note("end-to-end timing done: %.2f ms/step" % (ms_e2e / args.steps))
    # ---- roofline --------------------------------------------------------------------------------
    alg = ALG_GFLOP_PER_IMAGE.get((args.arch, R))
    step_tflops = (value / world) * alg / 1000.0 if alg else None
    roofline = {"bound": "tensor", "achieved": step_tflops, "peak": peak_sustained, "unit": "TFLOP/s",
                "frac": (step_tflops / peak_sustained) if step_tflops else None, "traffic": None,
                "what": "whole step: images/s/GPU x %.4f algorithmic GFLOP/image vs sustained bf16 peak, %s"
                        % (alg or 0.0, peak_src)}
    if rank == 0 and world == 1 and not args.no_layers:
        rows, agg = layer_table(model, b, R)
        conv_flops = sum(v["launch_gflop"] for v in agg.values())
        conv_ms = sum(v["ms_per_step"] for v in agg.values())
        roofline["dominant_kernel"] = {
            "name": "conv_igemm_kernel / conv_wgrad_kernel (wgmma implicit GEMM)",
            "achieved": conv_flops / conv_ms, "peak": peak_burst, "unit": "TFLOP/s",
            "frac": conv_flops / conv_ms / peak_burst, "isolated_ms_per_step": conv_ms,
            "share_of_step": conv_ms / (ms / args.steps), "by_kind": agg,
            "traffic": None,
            "how": "every distinct conv shape timed alone with CUDA events, L2 flushed between launches, weighted "
                   "by its count in one step (4 fprop passes, 2 dgrad/wgrad passes); peak = burst bf16, %s" % peak_src}
        if args.layers_out:
            with open(args.layers_out, "w") as f:
                json.dump({"batch": b, "image_size": R, "rows": rows, "agg": agg}, f, indent=1)

    cpu_baseline = None
    note("per-layer table done")
    if rank == 0 and world == 1 and not args.no_cpu_baseline:
        # in a child process with a hard limit: a pathological host (thread oversubscription) must not stall the bench
        try:
            out = subprocess.run([sys.executable, os.path.abspath(__file__), "--impl", "reference", "--steps", "1",
                                  "--warmup", "1", "--arch", args.arch, "--image-size", str(R), "--ref-batch",
                                  str(args.ref_batch)], capture_output=True, text=True, timeout=240,
                                 env={k: v for k, v in os.environ.items() if k != "OMP_NUM_THREADS"})
            cpu_baseline = json.loads(out.stdout.strip().splitlines()[-1])["cpu_baseline"]
            note("cpu baseline done: %s" % cpu_baseline["sample"])
        except Exception as e:
            cpu_baseline = {"value": None, "unit": "images/sec", "cores": None, "kind": "unavailable",
                            "sample": "CPU arm did not finish within 240 s (%s)" % type(e).__name__}
            note("cpu baseline failed: %r" % (e,))

    if rank == 0:
        line = {
            "metric": "images/sec", "value": value, "unit": "images/sec", "n_gpus": world, "steps": args.steps,
            "warmup": args.warmup, "ms_per_step": ms / args.steps, "higher_is_better": True, "scaling": "weak",
            "vs_baseline": None, "data": "synthetic",
            "dtype": "bf16" if args.precision == "bf16" else
                     "fp32 forward via %d-term bf16 split products (fp32 accumulate, fp64 BN statistics); bf16-operand "
                     "backward" % (6 if args.precision == "fp32" else 3),
            "config": {"workload": "%s BYOL training step, %dx%d, global batch %d (%d/GPU), %s, LARS+SGD momentum, "
                                   "EMA target; inputs (%.0f MB/step/GPU) larger than L2"
                                   % (args.arch, R, R, gb, b, "SyncBN + flat grad all-reduce" if sync_bn else
                                      "local BN", (aug1.numel() + aug2.numel()) * 4 / 1e6),
                       "global_batch": gb, "image_size": R, "parallelism": "dp%d" % world,
                       "compute": "bf16 tensor-core inputs, fp32 accumulate / master weights / BN / loss / optimizer"
                                  if args.precision == "bf16" else
                                  "fp32-accurate forward (precision=%s, csrc/split.cu), bf16-operand backward, fp32 "
                                  "master weights / loss / optimizer" % args.precision,
                       "cuda_graphs": bool(model._engine.use_graphs)},
            "e2e": {"value": e2e_value, "unit": "images/sec", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                    "ms_per_step": ms_e2e / args.steps},
            "gpu_launches": launches, "clocks": clocks, "roofline": roofline, "cpu_baseline": cpu_baseline,
            "loss": loss_val, "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
            "host_enqueue_ms_per_step": host_ms, "allocator": alloc_info,
        }
        print(json.dumps(line))
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    a = parse()
    if a.impl == "reference":
        main_reference(a)
    else:
        main_b200(a)
