#!/usr/bin/env python
"""The UNMODIFIED reference's stock PyTorch path timed on the same GPUs (the ">= 1.5x the reference PyTorch/DDP
images/sec" target of BASELINE.json's north_star; BASELINE.md section 5.2).

    python tools/ref_gpu_baseline.py --mode fp32 --batch-per-gpu 256                       # configs[1], 1 GPU
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29511 \
        tools/ref_gpu_baseline.py --mode bf16 --batch-per-gpu 512 --sync-bn               # configs[2], 8 GPUs

What runs: the reference's `main.py`, byte-compiled into oracle/_ref by build() (oracle/build_ref.py)
— its `BYOL`, its `loss_function`, its `LARS` around torch.optim.SGD(momentum 0.9), SyncBatchNorm conversion and
DistributedDataParallel(find_unused_parameters=True) exactly as main.build_loader_model_grapher wires them
(main.py:428-443) — driven by its own `main.execute_graph` over a synthetic on-device loader.  None of byol_b200's
code is on this path.  Harness deviations (stated in the JSON line): the three missing submodules come from
oracle/ref_shims; `--mode bf16` wraps the model call in torch.autocast(bfloat16) because the reference's own
`--half` needs apex, which is not installed (BASELINE.md 5.2); the learning rate is fixed instead of the lr = 0 first
epoch (Q11).  Timing: CUDA events around one execute_graph call over K batches, max over ranks.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.path.join(ROOT, "oracle", "_ref")


def parse():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="bf16", choices=["fp32", "tf32", "bf16"])
    ap.add_argument("--arch", default="resnet50")
    ap.add_argument("--image-size", type=int, default=224)
    ap.add_argument("--batch-per-gpu", type=int, default=512)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--sync-bn", action="store_true")
    ap.add_argument("--out", default=None)
    return ap.parse_args()


def main_():
    a = parse()
    import torch
    import torch.distributed as dist
    import torch.nn as nn
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    rep = 512 if a.arch in ("resnet18", "resnet34") else 2048
    argv = sys.argv
    sys.argv = ["main.py", "--arch=%s" % a.arch, "--representation-size=%d" % rep, "--num-replicas=%d" % world,
                "--batch-size=%d" % a.batch_per_gpu, "--image-size-override=%d" % a.image_size]
    sys.path[:0] = [REF, os.path.join(ROOT, "oracle", "ref_shims")]
    import main
    sys.argv = argv
    assert os.path.realpath(main.__file__).startswith(os.path.realpath(REF)), "not the shipped reference"
    main.args.cuda, main.args.distributed_rank = True, rank
    if a.mode == "fp32":          # strict fp32 (the CPU semantics of the reference); "tf32" = torch's GPU defaults
        torch.backends.cudnn.allow_tf32 = False
        torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    model = main.BYOL(base_network_output_size=rep, projection_output_size=256, classifier_output_size=1000,
                      total_training_steps=1000, base_decay=0.996)
    if a.sync_bn and world > 1:
        model = nn.SyncBatchNorm.convert_sync_batchnorm(model)          # main.py:433
    model = model.cuda()                                                # main.py:434
    from helpers import layers
    from optimizers.lars import LARS
    net = model
    if world > 1:                                                       # main.py:440-443
        net = layers.DistributedDataParallelPassthrough(model, device_ids=[local], output_device=local,
                                                        find_unused_parameters=True)
    if a.mode == "bf16":
        inner = net

        class _Autocast(nn.Module):     # harness deviation: autocast instead of apex AMP O2 (--half)
            def __init__(self):
                super().__init__()
                self.inner = inner

            def forward(self, x1, x2):
                with torch.autocast("cuda", dtype=torch.bfloat16):
                    out = self.inner(x1, x2)
                return {k: v.float() for k, v in out.items()}
        net = _Autocast()
    gb = a.batch_per_gpu * world
    groups = layers.add_weight_decay(model, 1e-6)                       # main.py:321
    opt = LARS(torch.optim.SGD(groups, lr=0.2 * gb / 256, momentum=0.9), eps=0.0)   # main.py:334-340
    g = torch.Generator(device=dev).manual_seed(1234 + rank)
    b, R = a.batch_per_gpu, a.image_size
    batch = (torch.rand(b, 3, R, R, generator=g, device=dev), torch.rand(b, 3, R, R, generator=g, device=dev),
             torch.randint(0, 1000, (b,), generator=g, device=dev))

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    main.execute_graph(0, net, [batch] * a.warmup, None, optimizer=opt, prefix="train")
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    loss = main.execute_graph(1, net, [batch] * a.steps, None, optimizer=opt, prefix="train")
    e1.record()
    barrier()
    ms = e0.elapsed_time(e1)
    if world > 1:
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        ms = float(t.item())
    if rank == 0:
        line = {"impl": "reference-gpu", "what": "unmodified /root/reference main.py (BYOL, loss_function, LARS+SGD, "
                "execute_graph) on torch %s eager" % torch.__version__, "mode": a.mode, "arch": a.arch,
                "image_size": R, "n_gpus": world, "batch_per_gpu": b, "global_batch": gb, "sync_bn": bool(a.sync_bn),
                "steps": a.steps, "warmup": a.warmup, "ms_per_step": ms / a.steps,
                "value": a.steps * gb / (ms / 1000.0), "unit": "images/sec", "loss": loss,
                "peak_mem_gb": torch.cuda.max_memory_allocated() / 1e9,
                "deviations": ["import shims for helpers/datasets/tree (oracle/ref_shims)", "fixed lr",
                               "synthetic on-device batch"] +
                              (["torch.autocast(bfloat16) instead of apex --half"] if a.mode == "bf16" else [])}
        s = json.dumps(line)
        print(s)
        if a.out:
            with open(a.out, "a") as f:
                f.write(s + "\n")
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main_()
