"""Cost of the k-NN evaluation on one GPU, with the card's name and power limit read in the same run:

* BYOL.representations of ResNet-50 @224 on synthetic batches (images/s, device-timed after warm-up), next to the
  eval-mode BYOL forward it replaces (four encoder lanes, MLPs, classifier);
* the search over a random ImageNet-sized bank (N = 1 281 167, Q = 50 000, D = 2048) for each k: device time of the
  similarity GEMM chunks, of the top-k selection and of the vote, the GEMM's TFLOP/s against the H100 SXM data
  sheet's 989 dense BF16 TFLOP/s and the selection's read rate of the fp32 similarities against 3.35 TB/s.

    python tools/bench_knn.py --out profiles/knn_h100_rn50.jsonl

One JSON line per measurement; all are written to --out as well.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tools.bench_fp32_backward import card   # noqa: E402

PEAK_BF16_TFLOPS = 989.0
PEAK_HBM_TBPS = 3.35
LINES = []


def emit(**kw):
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


def bench_representations(batch, res, steps, warmup):
    from byol_b200.model import BYOL
    torch.manual_seed(0)
    model = BYOL(2048, 256, 1000, 1000, arch="resnet50").cuda().eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.rand(batch, 3, res, res, device="cuda", generator=g)
    for _ in range(warmup):
        model.representations(x)
        with torch.no_grad():
            model(x, x)
    torch.cuda.synchronize()
    for rnd in range(2):     # alternate the two, twice
        ms_rep = timed(lambda: model.representations(x), steps)
        with torch.no_grad():
            ms_fwd = timed(lambda: model(x, x), steps)
        emit(stage="representations", arch="resnet50", batch=batch, res=res, round=rnd, ms=round(ms_rep, 3),
             images_per_s=round(batch / ms_rep * 1e3, 1), eval_forward_ms=round(ms_fwd, 3),
             eval_forward_over_representations=round(ms_fwd / ms_rep, 3))
    del model, x
    torch.cuda.empty_cache()


def bench_search(n, q, d, ks, classes, seed):
    from byol_b200 import knn, ops
    dev = torch.device("cuda", 0)
    g = torch.Generator(device="cuda").manual_seed(seed)
    bank = torch.empty((n, d), dtype=torch.bfloat16, device=dev)
    for r0 in range(0, n, 65536):
        r1 = min(n, r0 + 65536)
        knn.l2_normalize_rows(torch.randn((r1 - r0, d), device=dev, generator=g), out=bank[r0:r1])
    queries = knn.l2_normalize_rows(torch.randn((q, d), device=dev, generator=g))
    labels = torch.randint(0, classes, (n,), device=dev, generator=g)
    qc = min(q, knn.QUERY_CHUNK)
    nc = min(n, max(128, knn.SIM_BUDGET // (4 * qc) // 128 * 128))
    sim = torch.empty(qc * nc, dtype=torch.float32, device=dev)
    for k in ks:
        vals = torch.empty((q, k), dtype=torch.float32, device=dev)
        idx = torch.empty((q, k), dtype=torch.int32, device=dev)
        # warm-up: one chunk of each shape class
        s = sim[:qc * nc].view(qc, nc)
        ops.linear_fprop(queries[:qc], bank[:nc], out_fp32=True, out=s)
        knn.topk_update(s, 0, vals[:qc], idx[:qc], merge=False)
        torch.cuda.synchronize()
        ev = []
        for q0 in range(0, q, qc):
            qn = min(qc, q - q0)
            for n0 in range(0, n, nc):
                bn = min(nc, n - n0)
                s = sim[:qn * bn].view(qn, bn)
                e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
                e[0].record()
                ops.linear_fprop(queries[q0:q0 + qn], bank[n0:n0 + bn], out_fp32=True, out=s)
                e[1].record()
                knn.topk_update(s, n0, vals[q0:q0 + qn], idx[q0:q0 + qn], merge=n0 > 0)
                e[2].record()
                ev.append(e)
        v0, v1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        v0.record()
        knn.vote(vals, idx, labels, classes, 0.07)
        v1.record()
        torch.cuda.synchronize()
        gemm_s = sum(e[0].elapsed_time(e[1]) for e in ev) / 1e3
        sel_s = sum(e[1].elapsed_time(e[2]) for e in ev) / 1e3
        vote_s = v0.elapsed_time(v1) / 1e3
        flops = 2.0 * q * n * d
        sim_bytes = 4.0 * q * n          # the selection reads every fp32 similarity at least once
        emit(stage="search", n=n, q=q, d=d, k=k, query_chunk=qc, bank_chunk=nc, chunks=len(ev),
             gemm_s=round(gemm_s, 4), gemm_tflops=round(flops / gemm_s / 1e12, 1),
             gemm_share_of_989=round(flops / gemm_s / 1e12 / PEAK_BF16_TFLOPS, 3),
             select_s=round(sel_s, 4), select_tb_per_s=round(sim_bytes / sel_s / 1e12, 3),
             select_share_of_3p35=round(sim_bytes / sel_s / 1e12 / PEAK_HBM_TBPS, 3),
             vote_s=round(vote_s, 5), total_s=round(gemm_s + sel_s + vote_s, 4))
        del vals, idx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=512)
    ap.add_argument("--res", type=int, default=224)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--bank", type=int, default=1281167)
    ap.add_argument("--queries", type=int, default=50000)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--k", type=int, nargs="+", default=[20, 200])
    ap.add_argument("--out", default="profiles/knn_h100_rn50.jsonl")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_knn needs a GPU"
    name, limit = card()
    emit(card=name, power_limit_w=limit)
    bench_representations(args.batch, args.res, args.steps, args.warmup)
    bench_search(args.bank, args.queries, args.dim, args.k, 1000, seed=0)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in LINES:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
