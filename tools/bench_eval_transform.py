"""The two evaluation transforms of byol_b200.augment ("resize", the whole image to R x R, and the BYOL paper's "byol",
the shorter side to (8R + 3) // 7 by bicubic and the centre R x R crop) on the image-folder path, alternated in one run.

    python tools/bench_eval_transform.py --out profiles/eval_transform_h100_r224.jsonl

The seeded synthetic JPEG folder of tools/bench_image_folder.py (sizes around 500 x 375, quality 90) is generated in a
temporary directory and --batch images of it are decoded once on the GPU.  Then, for --rounds rounds, each transform
in turn:
- apply: ``apply_ragged`` of those images at --res with the transform's records, built once, in the loader's
  sub-batches (--reps passes timed with CUDA events), in images/s;
- loader: the test-split loader (read, GPU decode, records, apply) over the generated training images, which are many
  more than its test split holds, one pass after its first batch, host clock ending in a synchronise, in images/s,
  with the least and greatest value of the views it produced.
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

TRANSFORMS = ("resize", "byol")
LINES = []


def emit(**kw):
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def apply_rate(aug, decoded, reps, device):
    from byol_b200.data import DECODE_BATCH
    chunks = [decoded[s:s + DECODE_BATCH] for s in range(0, len(decoded), DECODE_BATCH)]
    records = [aug.eval_params([tuple(t.shape[1:]) for t in ch], device) for ch in chunks]

    def apply_all():
        for ch, p in zip(chunks, records):
            aug.apply_ragged(ch, p)

    apply_all()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        apply_all()
    e1.record()
    torch.cuda.synchronize()
    return reps * len(decoded) / (e0.elapsed_time(e1) / 1e3)


def loader_rate(ld):
    it = iter(ld)
    n0 = next(it)[0].shape[0]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    n, lo, hi = 0, [], []
    for a1, a2, _ in it:
        n += a1.shape[0]
        for v in (a1, a2):
            mn, mx = torch.aminmax(v)
            lo.append(mn)
            hi.append(mx)
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    return n0 + n, n / dt, float(torch.stack(lo).min()), float(torch.stack(hi).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=100)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="timed apply passes over the decoded batch per round")
    ap.add_argument("--workers", type=int, default=4, help="host threads reading file bytes (workers_per_replica)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_eval_transform needs a GPU"
    name, limit = card()
    emit(card=name, power_limit_w=limit)
    tmp = tempfile.mkdtemp(prefix="byol_eval_transform_")
    try:
        t0 = time.perf_counter()
        mean_bytes = make_folder(tmp, args.images, args.classes, seed=0)
        emit(stage="generate", images=args.images, mean_file_kb=round(mean_bytes / 1024, 1),
             seconds=round(time.perf_counter() - t0, 1))
        from byol_b200.data import DECODE_BATCH, ImageFolderLoader, _read, decode_batch, get_loader
        device = torch.device("cuda", 0)
        loaders = {t: get_loader(task="multi_augment_image_folder", data_dir=tmp, batch_size=args.batch,
                                 image_size_override=args.res, color_jitter_strength=1.0, seed=0, num_replicas=1,
                                 distributed_rank=0, workers_per_replica=args.workers, eval_transform=t)
                   for t in TRANSFORMS}
        samples = loaders[TRANSFORMS[0]].train_loader.samples
        evals = {t: ImageFolderLoader(samples, args.batch, ld.test_loader.augment, train=False, workers=args.workers)
                 for t, ld in loaders.items()}
        datas = [_read(p) for p, _ in samples[:args.batch]]
        decoded = []
        for s in range(0, len(datas), DECODE_BATCH):
            decoded += decode_batch(datas[s:s + DECODE_BATCH], device)
        torch.cuda.synchronize()
        emit(stage="decoded", images=len(decoded), mean_hw=[round(float(np.mean([t.shape[1] for t in decoded])), 1),
                                                            round(float(np.mean([t.shape[2] for t in decoded])), 1)])
        rates = {t: {"apply": [], "loader": []} for t in TRANSFORMS}
        for rnd in range(args.rounds):
            for t in TRANSFORMS:
                a = apply_rate(loaders[t].test_loader.augment, decoded, args.reps, device)
                rates[t]["apply"].append(a)
                emit(stage="apply", eval_transform=t, round=rnd, images=len(decoded), image_size=args.res,
                     sub_batch=DECODE_BATCH, reps=args.reps, images_per_s=round(a, 1))
            for t in TRANSFORMS:
                n, r, vmin, vmax = loader_rate(evals[t])
                rates[t]["loader"].append(r)
                emit(stage="loader", eval_transform=t, round=rnd, images=n, batch=args.batch, images_per_s=round(r, 1),
                     view_min=vmin, view_max=vmax)
        emit(summary=True, card=name, power_limit_w=limit, batch=args.batch, res=args.res, rounds=args.rounds,
             **{"%s_%s_images_per_s" % (t, s): round(float(np.median(v[s])), 1)
                for t, v in rates.items() for s in ("apply", "loader")},
             byol_over_resize_apply=round(float(np.median(rates["byol"]["apply"]) /
                                                np.median(rates["resize"]["apply"])), 4),
             byol_over_resize_loader=round(float(np.median(rates["byol"]["loader"]) /
                                                 np.median(rates["resize"]["loader"])), 4))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for l in LINES:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
