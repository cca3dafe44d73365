"""Image-folder input (byol_b200.data) on one GPU: what each stage of the loader sustains, and the ResNet-50 BYOL step
fed by it against the same step on synthetic inputs.

    python tools/bench_image_folder.py --out profiles/image_folder_h100_rn50_b512.json

A seeded synthetic JPEG folder is generated first (ImageNet-like sizes around 500 x 375, quality 90, nothing
downloaded) in --data-dir, a temporary directory by default.  Reported, in images/s:
- read: the file bytes, read by the loader's host thread pool (the files are in the page cache after generation);
- decode: byol_b200.data.decode_batch (nvJPEG through torchvision) in the loader's sub-batches;
- augment: the ragged two-view augmentation of those decoded images at 224;
- loader: the whole train loader, iterated without a training step;
- step_synthetic / step_loader: ms per BYOL training step (ResNet-50 @224, --batch images) on fixed random views and
  on the loader's batches, alternated for --rounds rounds, host clock around --steps steps ending in a synchronise.
The card's name and power limit are read in the same run.  One JSON line per measurement, then a summary line; all of
them are written to --out as well.
"""
import argparse
import json
import os
import shutil
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_fp32_backward import card   # noqa: E402

LINES = []


def emit(**kw):
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def make_folder(root, n, classes, seed):
    """n JPEGs of sizes around 500 x 375 (either orientation) over `classes` classes, and a small test split."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    jobs = []
    for split, count in (("train", n), ("test", max(classes, n // 64))):
        for i in range(count):
            w, h = int(rng.integers(400, 601)), int(rng.integers(300, 451))
            if rng.random() < 0.25:
                w, h = h, w
            jobs.append((os.path.join(root, split, "c%03d" % (i % classes), "%06d.JPEG" % i), h, w,
                         int(rng.integers(0, 2 ** 31))))

    def write(job):
        path, h, w, s = job
        r = np.random.default_rng(s)
        # smooth content plus fine noise: about the entropy of a photograph at quality 90
        small = r.integers(0, 256, size=(h // 16 + 1, w // 16 + 1, 3), dtype=np.uint8)
        img = np.asarray(Image.fromarray(small).resize((w, h), Image.BICUBIC)).astype(np.int16)
        img = np.clip(img + r.integers(-12, 13, size=img.shape), 0, 255).astype(np.uint8)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        Image.fromarray(img).save(path, format="JPEG", quality=90)
        return os.path.getsize(path)

    with ThreadPoolExecutor(max_workers=min(32, os.cpu_count() or 4)) as ex:
        sizes = list(ex.map(write, jobs))
    return float(np.mean(sizes))


def stage_rates(loader, batch, device):
    from byol_b200.data import DECODE_BATCH, _read, decode_batch
    tl = loader.train_loader
    paths = [p for p, _ in tl.samples]
    with ThreadPoolExecutor(max_workers=tl.workers) as ex:
        list(ex.map(_read, paths[:batch]))
        t0 = time.perf_counter()
        datas = list(ex.map(_read, paths))
        t_read = time.perf_counter() - t0
    emit(stage="read", images=len(datas), threads=tl.workers, images_per_s=round(len(datas) / t_read, 1),
         mb_per_s=round(sum(len(d) for d in datas) / t_read / 1e6, 1))
    subs = [datas[s:s + DECODE_BATCH] for s in range(0, len(datas), DECODE_BATCH)]
    for sb in subs[:2]:
        decode_batch(sb, device)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    decoded = []
    for sb in subs:
        imgs = decode_batch(sb, device)
        if len(decoded) < batch:
            decoded += imgs
    torch.cuda.synchronize()
    t_dec = time.perf_counter() - t0
    emit(stage="decode", images=len(datas), sub_batch=DECODE_BATCH, images_per_s=round(len(datas) / t_dec, 1))
    aug = tl.augment
    chunks = [decoded[s:s + DECODE_BATCH] for s in range(0, len(decoded), DECODE_BATCH)]

    def augment_all():
        for s, ch in enumerate(chunks):
            p = aug.sample_params_ragged([tuple(t.shape[1:]) for t in ch], device, n0=s * DECODE_BATCH,
                                         total=len(decoded), step=0)
            aug.apply_ragged(ch, p)

    augment_all()
    torch.cuda.synchronize()
    reps = 5
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        augment_all()
    e1.record()
    torch.cuda.synchronize()
    emit(stage="augment", images=len(decoded), image_size=aug.R, sub_batch=DECODE_BATCH,
         images_per_s=round(reps * len(decoded) / (e0.elapsed_time(e1) / 1e3), 1))
    del decoded, chunks
    it = iter(tl)
    next(it)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    k = 0
    for _ in it:
        k += 1
    torch.cuda.synchronize()
    emit(stage="loader", batches=k, batch=batch, images_per_s=round(k * batch / (time.perf_counter() - t0), 1))


def batches_forever(tl):
    epoch = 0
    while True:
        tl.set_epoch(epoch)
        for b in tl:
            yield b
        epoch += 1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=4096)
    ap.add_argument("--classes", type=int, default=100)
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--workers", type=int, default=4, help="host threads reading file bytes (workers_per_replica)")
    ap.add_argument("--data-dir", default=None, help="where the JPEG folder is generated (default: a temporary dir)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_image_folder needs a GPU"
    name, limit = card()
    emit(card=name, power_limit_w=limit)
    tmp = args.data_dir or tempfile.mkdtemp(prefix="byol_image_folder_")
    try:
        t0 = time.perf_counter()
        mean_bytes = make_folder(tmp, args.images, args.classes, seed=0)
        emit(stage="generate", images=args.images, mean_file_kb=round(mean_bytes / 1024, 1),
             seconds=round(time.perf_counter() - t0, 1))
        from byol_b200 import wiring
        from byol_b200.data import get_loader
        from byol_b200.model import BYOL
        device = torch.device("cuda", 0)
        loader = get_loader(task="multi_augment_image_folder", data_dir=tmp, batch_size=args.batch,
                            image_size_override=args.res, color_jitter_strength=1.0, seed=0, num_replicas=1,
                            distributed_rank=0, workers_per_replica=args.workers)
        stage_rates(loader, args.batch, device)

        torch.manual_seed(0)
        model = BYOL(2048, 256, loader.output_size, 1000, arch="resnet50").cuda().train()
        opt = wiring.build_optimizer(model, global_batch_size=args.batch)
        g = torch.Generator(device="cuda").manual_seed(1)
        syn = (torch.rand(args.batch, 3, args.res, args.res, device="cuda", generator=g),
               torch.rand(args.batch, 3, args.res, args.res, device="cuda", generator=g),
               torch.randint(0, loader.output_size, (args.batch,), device="cuda", generator=g))
        feed = batches_forever(loader.train_loader)
        sources = {"synthetic": lambda: syn, "loader": lambda: next(feed)}
        for src in sources.values():
            for _ in range(args.warmup):
                wiring.train_step(model, opt, *src())
        torch.cuda.synchronize()
        times = {k: [] for k in sources}
        for rnd in range(args.rounds):
            for k, src in sources.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                for _ in range(args.steps):
                    out = wiring.train_step(model, opt, *src())
                torch.cuda.synchronize()
                ms = (time.perf_counter() - t0) * 1e3 / args.steps
                assert np.isfinite(float(out["loss_mean"]))
                times[k].append(ms)
                emit(step=k, round=rnd, arch="resnet50", batch=args.batch, res=args.res, steps=args.steps,
                     ms_per_step=round(ms, 2), images_per_s=round(args.batch / ms * 1e3, 1))
        syn_ms, ld_ms = np.median(times["synthetic"]), np.median(times["loader"])
        emit(summary=True, card=name, power_limit_w=limit, arch="resnet50", batch=args.batch, res=args.res,
             step_synthetic_ms=[round(v, 2) for v in times["synthetic"]],
             step_loader_ms=[round(v, 2) for v in times["loader"]],
             loader_over_synthetic=round(float(ld_ms / syn_ms), 4),
             stages={l["stage"]: l["images_per_s"] for l in LINES if "stage" in l and "images_per_s" in l})
    finally:
        if args.data_dir is None:
            shutil.rmtree(tmp, ignore_errors=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for l in LINES:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
