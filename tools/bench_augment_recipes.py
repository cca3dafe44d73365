"""The two augmentation recipes of byol_b200.augment ("reference" and the BYOL paper's "byol") on the image-folder
path, alternated in one run.

    python tools/bench_augment_recipes.py --out profiles/augment_recipes_h100_r224_b512.jsonl

The seeded synthetic JPEG folder of tools/bench_image_folder.py (sizes around 500 x 375, quality 90) is generated in a
temporary directory and --batch images of it are decoded once on the GPU.  Then, for --rounds rounds, each recipe in
turn:
- augment: the ragged uint8 two-view augmentation of those images at --res, in the loader's sub-batches (sampler +
  apply, --reps passes timed with CUDA events), in images/s;
- loader: the whole train loader with that recipe (read, GPU decode, augment), one epoch after its first batch, host
  clock ending in a synchronise, in images/s, with the least and greatest value of the views it produced (main.py
  rejects a batch outside [0, 1]).
The card's name and power limit are read in the same run.  One JSON line per measurement, then a summary line with
the median of each; all of them are written to --out as well.
"""
import argparse
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
from tools.bench_image_folder import make_folder   # noqa: E402

RECIPES = ("reference", "byol")
LINES = []


def emit(**kw):
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def augment_rate(aug, decoded, reps, device):
    from byol_b200.data import DECODE_BATCH
    chunks = [decoded[s:s + DECODE_BATCH] for s in range(0, len(decoded), DECODE_BATCH)]
    sizes = [[tuple(t.shape[1:]) for t in ch] for ch in chunks]

    def augment_all(step):
        for s, ch in enumerate(chunks):
            p = aug.sample_params_ragged(sizes[s], device, n0=s * DECODE_BATCH, total=len(decoded), step=step)
            aug.apply_ragged(ch, p)

    augment_all(0)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for r in range(reps):
        augment_all(r + 1)
    e1.record()
    torch.cuda.synchronize()
    return reps * len(decoded) / (e0.elapsed_time(e1) / 1e3)


def loader_rate(loader, batch):
    tl = loader.train_loader
    it = iter(tl)
    next(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    k, lo, hi = 0, [], []
    for a1, a2, _ in it:
        k += 1
        for v in (a1, a2):
            mn, mx = torch.aminmax(v)
            lo.append(mn)
            hi.append(mx)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return k, k * batch / dt, float(torch.stack(lo).min()), float(torch.stack(hi).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=100)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="timed augmentation passes over the decoded batch per round")
    ap.add_argument("--workers", type=int, default=4, help="host threads reading file bytes (workers_per_replica)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_augment_recipes needs a GPU"
    name, limit = card()
    emit(card=name, power_limit_w=limit)
    tmp = tempfile.mkdtemp(prefix="byol_augment_recipes_")
    try:
        t0 = time.perf_counter()
        mean_bytes = make_folder(tmp, args.images, args.classes, seed=0)
        emit(stage="generate", images=args.images, mean_file_kb=round(mean_bytes / 1024, 1),
             seconds=round(time.perf_counter() - t0, 1))
        from byol_b200.data import DECODE_BATCH, _read, decode_batch, get_loader
        device = torch.device("cuda", 0)
        loaders = {r: get_loader(task="multi_augment_image_folder", data_dir=tmp, batch_size=args.batch,
                                 image_size_override=args.res, color_jitter_strength=1.0, seed=0, num_replicas=1,
                                 distributed_rank=0, workers_per_replica=args.workers, augmentation=r)
                   for r in RECIPES}
        paths = [p for p, _ in loaders[RECIPES[0]].train_loader.samples[:args.batch]]
        datas = [_read(p) for p in paths]
        decoded = []
        for s in range(0, len(datas), DECODE_BATCH):
            decoded += decode_batch(datas[s:s + DECODE_BATCH], device)
        torch.cuda.synchronize()
        emit(stage="decoded", images=len(decoded), mean_hw=[round(float(np.mean([t.shape[1] for t in decoded])), 1),
                                                            round(float(np.mean([t.shape[2] for t in decoded])), 1)])
        rates = {r: {"augment": [], "loader": []} for r in RECIPES}
        for rnd in range(args.rounds):
            for r in RECIPES:
                a = augment_rate(loaders[r].train_loader.augment, decoded, args.reps, device)
                rates[r]["augment"].append(a)
                emit(stage="augment", recipe=r, round=rnd, images=len(decoded), image_size=args.res,
                     sub_batch=DECODE_BATCH, reps=args.reps, images_per_s=round(a, 1))
            for r in RECIPES:
                k, l, vmin, vmax = loader_rate(loaders[r], args.batch)
                rates[r]["loader"].append(l)
                emit(stage="loader", recipe=r, round=rnd, batches=k, batch=args.batch, images_per_s=round(l, 1),
                     view_min=vmin, view_max=vmax)
        emit(summary=True, card=name, power_limit_w=limit, batch=args.batch, res=args.res, rounds=args.rounds,
             **{"%s_%s_images_per_s" % (r, s): round(float(np.median(v[s])), 1)
                for r, v in rates.items() for s in ("augment", "loader")},
             byol_over_reference_augment=round(float(np.median(rates["byol"]["augment"]) /
                                                     np.median(rates["reference"]["augment"])), 4))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for l in LINES:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
