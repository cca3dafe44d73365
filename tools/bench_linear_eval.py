"""Cost of the linear evaluation on one GPU, with the card's name and power limit read in the same run:

* head training on random cached features at ImageNet size (N = 1 281 167, D = 2048, C = 1000, H = 5, B = 1024):
  ms per step (--rounds windows of --steps steps, alternated with the torch arm below; min / median / max), a
  torch.profiler split of one step's device time by kernel, the CUDA-event time of each of the step's five launches
  and its share of the least time the data sheet allows (989 dense BF16 TFLOP/s for the GEMMs, 3.35 TB/s for the
  rest), and --rounds whole epochs as ``train_linear_heads`` runs them (permutation and row gathers included);
* the same step in torch for comparison: one bf16 nn.Linear(2048, 5000) under autocast, per-head F.cross_entropy and
  torch.optim.SGD(nesterov=True, foreach=True) (one learning rate: torch's SGD has no per-row lr);
* augment=True feature throughput: images/s of JPEG decode + random resized crop / flip + ResNet-50 representations
  on a synthetic JPEG folder (tools/bench_image_folder.py's generator), which prices an epoch of that mode.

    python tools/bench_linear_eval.py --out profiles/linear_eval_h100_rn50.jsonl

One JSON line per measurement; all are written to --out as well.
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

PEAK_BF16_TFLOPS = 989.0
PEAK_HBM_TBPS = 3.35
LINES = []
CARD = {}


def emit(**kw):
    kw.update(CARD)
    LINES.append(kw)
    print(json.dumps(kw), flush=True)


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def spread(values):
    v = sorted(values)
    return dict(ms_min=round(v[0], 4), ms_median=round(float(np.median(v)), 4), ms_max=round(v[-1], 4),
                rounds=len(v))


def torch_step_fn(feats, labels, c, h, b):
    """One step of the torch arm: bf16 nn.Linear(D, H * C) under autocast, per-head cross-entropy, foreach Nesterov
    SGD (one learning rate)."""
    import torch.nn.functional as F
    lin = torch.nn.Linear(feats.shape[1], h * c).cuda()
    opt = torch.optim.SGD(lin.parameters(), lr=0.1, momentum=0.9, nesterov=True, foreach=True)
    x, y = feats[:b].contiguous(), labels[:b].contiguous()

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            z = lin(x)
        z = z.float().view(b, h, c)
        loss = sum(F.cross_entropy(z[:, k], y) for k in range(h))
        opt.zero_grad(set_to_none=False)
        loss.backward()
        opt.step()

    return step


def profile_step(step, reps):
    """Device time per step of every kernel one step launches (torch.profiler, a run of its own)."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            step()
        torch.cuda.synchronize()
    rows = []
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0 and ev.count >= reps:
            rows.append((t / reps / 1e3, ev.key, ev.count // reps))
    return sorted(rows, reverse=True)


def bench_heads(n, d, c, h, b, steps, warmup, rounds):
    from byol_b200 import ops
    from byol_b200.linear_eval import LinearHeads, _fit, multihead_ce
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cuda").manual_seed(0)
    feats = torch.empty((n, d), dtype=torch.bfloat16, device=dev)
    for r0 in range(0, n, 65536):
        feats[r0:r0 + 65536] = torch.randn((min(n, r0 + 65536) - r0, d), device=dev, generator=g)
    labels = torch.randint(0, c, (n,), device=dev, generator=g)
    lrs = (0.4, 0.3, 0.2, 0.1, 0.05)[:h]
    heads = LinearHeads(d, c, lrs, (0.0,), seed=0, device=dev)
    hp = heads.H * heads.Cp
    x, y = feats[:b].contiguous(), labels[:b].contiguous()
    for _ in range(warmup):
        heads.step(x, y, 0.5)
    torch.cuda.synchronize()
    step = lambda: heads.step(x, y, 0.5)        # noqa: E731
    torch_step = torch_step_fn(feats, labels, c, heads.H, b)
    for _ in range(warmup):
        torch_step()
    torch.cuda.synchronize()
    ours, theirs = [], []
    for _ in range(rounds):                      # alternated windows of `steps` steps each
        ours.append(timed(step, steps))
        theirs.append(timed(torch_step, steps))
    ms_step = float(np.median(ours))
    emit(stage="torch_step", d=d, classes=c, heads=heads.H, batch=b, steps_per_round=steps,
         ms_per_step=round(float(np.median(theirs)), 4), **spread(theirs))
    torch_step = None
    # which kernels the step's time goes to (the wgrad launch is its GEMM kernel plus the fixed-point flush)
    try:
        for ms, name, per_step in profile_step(step, 20):
            emit(stage="profile", kernel=name[:120], launches_per_step=per_step, ms_per_step=round(ms, 4))
    except Exception as e:                       # the profiler is optional: the timings below do not depend on it
        emit(stage="profile", error=repr(e)[:200])
    # the five launches, each between its own events
    logits = torch.empty((b, hp), dtype=torch.float32, device=dev)
    dl = torch.empty((b, hp), dtype=torch.bfloat16, device=dev)
    loss = torch.zeros(heads.H, dtype=torch.float32, device=dev)
    nw = hp * d
    stages = [
        ("fprop_gemm", lambda: heads.logits(x, out=logits), 2.0 * b * hp * d, None),
        ("cross_entropy", lambda: multihead_ce(logits, y, heads.H, c, dlogits=dl, loss_sum=loss), None,
         4.0 * b * hp + 2.0 * b * hp),
        ("wgrad_gemm", lambda: ops.linear_wgrad(x, dl, heads.grads[:nw].view(hp, d)), 2.0 * b * hp * d, None),
        ("bias_col_sum", lambda: ops.col_sum(dl, heads.grads[nw:]), None, 2.0 * b * hp),
        ("sgd_update", lambda: heads.apply_gradients(0.5), None, 26.0 * c * heads.H * d),
    ]
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(len(stages) + 1)] for _ in range(steps)]
    for fn in (s[1] for s in stages):
        fn()
    torch.cuda.synchronize()
    for e in ev:
        e[0].record()
        for i, s in enumerate(stages):
            s[1]()
            e[i + 1].record()
    torch.cuda.synchronize()
    total_bound = 0.0
    for i, (name, _, flops, nbytes) in enumerate(stages):
        ms = float(np.median([e[i].elapsed_time(e[i + 1]) for e in ev]))
        if flops is not None:
            bound_ms = flops / (PEAK_BF16_TFLOPS * 1e12) * 1e3
            emit(stage="launch", name=name, ms=round(ms, 4), tflops=round(flops / ms / 1e9, 1),
                 bound="bf16 tensor core", bound_ms=round(bound_ms, 4), share_of_bound=round(bound_ms / ms, 3))
        else:
            bound_ms = nbytes / (PEAK_HBM_TBPS * 1e12) * 1e3
            emit(stage="launch", name=name, ms=round(ms, 4), tb_per_s=round(nbytes / ms / 1e9, 3),
                 bound="HBM", bound_ms=round(bound_ms, 4), share_of_bound=round(bound_ms / ms, 3))
        total_bound += bound_ms
    steps_per_epoch = n // b
    emit(stage="head_step", n=n, d=d, classes=c, heads=heads.H, batch=b, steps_per_round=steps,
         ms_per_step=round(ms_step, 4), **spread(ours),
         bound_ms=round(total_bound, 4), share_of_bound=round(total_bound / ms_step, 3),
         steps_per_epoch=steps_per_epoch, s_per_epoch_from_step=round(ms_step * steps_per_epoch / 1e3, 3),
         s_per_80_epochs_from_step=round(80 * ms_step * steps_per_epoch / 1e3, 1))

    def batches(epoch):
        perm = torch.from_numpy(np.random.default_rng([0, epoch]).permutation(n)).to(dev)
        for i in range(steps_per_epoch):
            idx = perm[i * b:(i + 1) * b]
            yield feats.index_select(0, idx), labels.index_select(0, idx)

    for rnd in range(rounds):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _fit(heads, 1, steps_per_epoch, batches)
        torch.cuda.synchronize()
        s_epoch = time.perf_counter() - t0
        emit(stage="cached_epoch", n=n, batch=b, round=rnd, s_per_epoch=round(s_epoch, 3),
             ms_per_step=round(s_epoch * 1e3 / steps_per_epoch, 4), s_per_80_epochs=round(80 * s_epoch, 1))
    del heads, logits, dl
    return feats, labels


def bench_augment_features(images, batch, res, steps, workers, data_dir):
    """images/s of decode + crop / flip + representations over a JPEG folder at `data_dir`, or over a generated one
    in a temporary directory that is removed afterwards."""
    from tools.bench_image_folder import make_folder
    root = data_dir or tempfile.mkdtemp(prefix="byol_linear_eval_")
    try:
        if not os.path.isdir(os.path.join(root, "train")):
            make_folder(root, images, 100, seed=0)
        _measure_augment_features(os.path.join(root, "train"), batch, res, steps, workers)
    finally:
        if data_dir is None:
            shutil.rmtree(root, ignore_errors=True)      # the generated folder goes with the run


def _measure_augment_features(train_dir, batch, res, steps, workers):
    from byol_b200.augment import TwoViewAugment
    from byol_b200.data import ImageFolderLoader, _scan
    from byol_b200 import ops
    from byol_b200.model import BYOL
    _, samples = _scan(train_dir)
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50").cuda()
    crop = TwoViewAugment(image_size=res, seed=0, p_jitter=0.0, p_gray=0.0, p_blur=0.0, blur=False)
    loader = ImageFolderLoader(samples, batch, crop, train=True, seed=0, workers=workers)
    for v1, _, _ in loader:          # warm-up epoch (module loads, decoder and GEMM shapes)
        ops.cast_bf16(model.representations(v1))
    torch.cuda.synchronize()
    for rnd in range(steps):
        loader.set_epoch(rnd + 1)
        t0 = time.perf_counter()
        k = 0
        for v1, _, _ in loader:
            ops.cast_bf16(model.representations(v1))
            k += 1
        torch.cuda.synchronize()
        ips = k * batch / (time.perf_counter() - t0)
        emit(stage="augment_features", arch="resnet50", res=res, batch=batch, images=k * batch, round=rnd,
             workers=workers, images_per_s=round(ips, 1), imagenet_epoch_s=round(1281167 / ips, 1),
             imagenet_80_epochs_h=round(80 * 1281167 / ips / 3600, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1281167)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--classes", type=int, default=1000)
    ap.add_argument("--heads", type=int, default=5)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=1000, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--images", type=int, default=4096, help="JPEGs in the synthetic folder (augment=True arm)")
    ap.add_argument("--image-batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--rounds", type=int, default=3, help="alternated windows / epochs / folder passes")
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--data-dir", default=None)
    ap.add_argument("--out", default="profiles/linear_eval_h100_rn50.jsonl")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_linear_eval needs a GPU"
    name, limit = card()
    CARD.update(card=name, power_limit_w=limit)
    feats, labels = bench_heads(args.n, args.dim, args.classes, args.heads, args.batch, args.steps, args.warmup,
                                args.rounds)
    del feats, labels
    torch.cuda.empty_cache()
    if args.images:
        bench_augment_features(args.images, args.image_batch, args.res, args.rounds, args.workers, args.data_dir)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in LINES:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
