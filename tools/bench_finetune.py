"""Cost of semi-supervised fine-tuning (byol_b200.finetune) on one GPU, with the card's name and power limit read in
the same run:

* the fine-tune step of a ResNet-50 copy at 224 px and --batches images (1000 classes): device ms per step over
  --rounds windows of --steps steps alternated with the torch arm below (min / median / max), the host time to enqueue
  one step (the step is eager: this is what a CUDA graph could save), the peak device memory of a step with the
  recompute plan the planner chose, and the device memory one copy holds;
* the same step in torch: torchvision ResNet-50 in channels_last under bf16 autocast, nn.Linear + F.cross_entropy,
  torch.optim.SGD(nesterov=True, foreach=True);
* one epoch over a generated JPEG folder (tools/bench_image_folder.py's generator) with 5 runs sharing every decoded
  batch, against the same epoch with 1 run: how far sharing the decode helps.

    python tools/bench_finetune.py --out profiles/finetune_h100_rn50.jsonl

One JSON line per measurement; all are written to --out as well.
"""
import argparse
import gc
import json
import os
import shutil
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_fp32_backward import card   # noqa: E402

LINES = []
CARD = {}


def emit(**kw):
    kw.update(CARD)
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def spread(values):
    v = sorted(values)
    return {"min": round(v[0], 3), "median": round(float(np.median(v)), 3), "max": round(v[-1], 3)}


def window_ms(step, steps):
    """Device ms per step over `steps` steps (CUDA events around the window)."""
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(steps):
        step()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / steps


def torch_step_fn(x, lab):
    import torchvision
    net = torchvision.models.resnet50(num_classes=1000).cuda().to(memory_format=torch.channels_last).train()
    opt = torch.optim.SGD(net.parameters(), lr=0.01, momentum=0.9, nesterov=True, weight_decay=1e-4, foreach=True)
    xc = x.contiguous(memory_format=torch.channels_last)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = torch.nn.functional.cross_entropy(net(xc), lab)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        opt.step()
    return step, net, opt


def bench_step(b, steps, warmup, rounds):
    from byol_b200.finetune import FineTune
    from byol_b200.model import BYOL
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50").cuda()
    g = torch.Generator().manual_seed(1)
    x = torch.rand(b, 3, 224, 224, generator=g).cuda()
    lab = torch.randint(0, 1000, (b,), generator=g).cuda()
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    ft = FineTune(model, 1000, 0.01, 1e-4)
    torch.cuda.synchronize()
    copy_bytes = torch.cuda.memory_allocated() - m0
    ours = lambda: ft.step(x, lab, 0.5)
    for _ in range(warmup):
        ours()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    ours()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    plan = sorted(ft.eng.recompute_plan(b, 224, 224, 1, False, False))
    enqueue = []
    for _ in range(10):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ours()
        enqueue.append(1e3 * (time.perf_counter() - t0))
    torch.cuda.synchronize()
    theirs, net, opt = torch_step_fn(x, lab)
    for _ in range(warmup):
        theirs()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base_t = torch.cuda.memory_allocated()
    theirs()
    torch.cuda.synchronize()
    peak_t = torch.cuda.max_memory_allocated() - base_t
    t_ours, t_torch = [], []
    for _ in range(rounds):
        t_ours.append(window_ms(ours, steps))
        t_torch.append(window_ms(theirs, steps))
    emit(stage="finetune_step", arch="resnet50", res=224, batch=b, classes=1000, steps=steps, rounds=rounds,
         ms_per_step=spread(t_ours), torch_ms_per_step=spread(t_torch),
         images_per_s=round(b / float(np.median(t_ours)) * 1e3, 1),
         host_enqueue_ms=spread(enqueue), peak_step_gb=round(peak / 1e9, 2), torch_peak_step_gb=round(peak_t / 1e9, 2),
         recompute_blocks=plan, copy_gb=round(copy_bytes / 1e9, 3))
    del ft, model, net, opt, theirs, ours
    gc.collect()
    torch.cuda.empty_cache()


def bench_sweep_epoch(images, batch, workers, rounds, data_dir):
    from tools.bench_image_folder import make_folder
    root = data_dir or tempfile.mkdtemp(prefix="byol_finetune_")
    try:
        if not os.path.isdir(os.path.join(root, "train")):
            make_folder(root, images, 100, seed=0)
        _sweep_epoch(os.path.join(root, "train"), batch, workers, rounds)
    finally:
        if data_dir is None:
            shutil.rmtree(root, ignore_errors=True)      # the generated folder goes with the run


def _sweep_epoch(train_dir, batch, workers, rounds):
    """One epoch as finetune_accuracy runs it (decode + crop / flip once per batch, then every run's step)."""
    from byol_b200.augment import TwoViewAugment
    from byol_b200.data import ImageFolderLoader, _scan
    from byol_b200.finetune import FineTune
    from byol_b200.linear_eval import cosine_factor
    from byol_b200.model import BYOL
    _, samples = _scan(train_dir)
    torch.manual_seed(0)
    model = BYOL(2048, 256, 100, 1000, arch="resnet50").cuda()
    runs = [FineTune(model, 100, lr, 0.0) for lr in (0.1, 0.05, 0.02, 0.01, 0.005)]
    crop = TwoViewAugment(image_size=224, seed=0, p_jitter=0.0, p_gray=0.0, p_blur=0.0, blur=False)
    loader = ImageFolderLoader(samples, batch, crop, train=True, seed=0, workers=workers)

    def epoch(k, e):
        loader.set_epoch(e)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        n = 0
        for v1, _, lab in loader:
            for r in runs[:k]:
                r.step(v1, lab, cosine_factor(n, len(loader)))
            n += 1
        torch.cuda.synchronize()
        return time.perf_counter() - t0, n

    epoch(5, 0)                                           # warm-up: module loads, decoder, GEMM shapes
    res = {1: [], 5: []}
    for rnd in range(rounds):
        for k in (1, 5):
            s, n = epoch(k, rnd + 1)
            res[k].append(s)
    emit(stage="sweep_epoch", arch="resnet50", res=224, batch=batch, images=n * batch, rounds=rounds, workers=workers,
         epoch_s_1_run=spread(res[1]), epoch_s_5_runs=spread(res[5]),
         images_per_s_1_run=round(n * batch / float(np.median(res[1])), 1),
         images_per_s_5_runs=round(n * batch / float(np.median(res[5])), 1),
         ratio_5_to_1=round(float(np.median(res[5])) / float(np.median(res[1])), 3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="256,1024")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--sweep-batch", type=int, default=256)
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--data-dir", default=None, help="where the JPEG folder is generated (default: a temporary dir)")
    ap.add_argument("--skip-sweep", action="store_true")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__  # noqa: F401  (repository root on sys.path)
    name, limit = card()
    CARD.update(card=name, power_limit_w=limit)
    for b in [int(v) for v in args.batches.split(",") if v]:
        bench_step(b, args.steps, args.warmup, args.rounds)
    if not args.skip_sweep:
        bench_sweep_epoch(args.images, args.sweep_batch, args.workers, args.rounds, args.data_dir)
    if args.out:
        with open(args.out, "w") as f:
            for line in LINES:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
