"""Transfer linear evaluation: the batched L-BFGS fit of byol_b200.logreg against torch.optim.LBFGS run one head at a
time, on synthetic features (N train rows, D = 2048, C classes, the 45 values of L2_GRID).

    python tools/bench_logreg.py --out profiles/logreg_h100_c10_c100.jsonl

Per C and round, one JSON line per method: fit time (host clock around work that ends in a device synchronise), the
batched fit's function evaluations and device-timed ms per evaluation (CUDA events around one evaluation of every head,
averaged over repeats), peak memory, and each head's float64 objective at the returned (W, b) (computed by the same
float64 code for both methods, so their solutions are compared at equal accuracy).  Rounds alternate the two methods.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:                                    # noqa: BLE001
        q = "unknown (%s)" % e
    return q


def _features(n, d, c, seed, device):
    g = torch.Generator(device=device).manual_seed(seed)
    teacher = torch.randn(c, d, generator=g, device=device) / d ** 0.5
    x = torch.randn(n, d, generator=g, device=device)
    y = (x @ teacher.T + 2.0 * torch.randn(n, c, generator=g, device=device)).argmax(1)
    y[:c] = torch.arange(c, device=device)
    return x, y


def _objective64(x, y, w, b, l2):
    """float64 f(W, b) on the device, in row chunks."""
    total = 0.0
    for r0 in range(0, x.shape[0], 8192):
        z = x[r0:r0 + 8192].double() @ w.T + b
        total += float(torch.nn.functional.cross_entropy(z, y[r0:r0 + 8192], reduction="sum"))
    return total / x.shape[0] + 0.5 * l2 * float((w * w).sum())


def _torch_fit(x, y, c, l2, max_iter, tol):
    d = x.shape[1]
    w = torch.zeros(c, d, device=x.device, requires_grad=True)
    b = torch.zeros(c, device=x.device, requires_grad=True)
    opt = torch.optim.LBFGS([w, b], lr=1.0, max_iter=max_iter, history_size=10, tolerance_grad=tol,
                            tolerance_change=0.0, line_search_fn="strong_wolfe")

    def closure():
        opt.zero_grad()
        f = torch.nn.functional.cross_entropy(x @ w.T + b, y) + 0.5 * l2 * (w * w).sum()
        f.backward()
        return f

    opt.step(closure)
    return w.detach(), b.detach(), opt.state[opt._params[0]]["func_evals"]


def _eval_ms(x, y, c, l2s, reps=5):
    """Device time of one function evaluation of every head (the solver's evaluate), CUDA events."""
    from byol_b200 import logreg, ops
    planes, _ = ops.split_planes(x, logreg.T_PLANES)
    s = logreg._Solver(planes, y, x.shape[0], x.shape[1], c, l2s, x.device)
    s.set_modes(np.full(s.H, logreg._SEARCH), np.ones(s.H))
    s.evaluate(logreg._bit(logreg._SEARCH))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        s.evaluate(logreg._bit(logreg._SEARCH))
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=50000)
    ap.add_argument("--n-test", type=int, default=10000)
    ap.add_argument("--dim", type=int, default=2048)
    ap.add_argument("--classes", default="10,100")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--max-iter", type=int, default=1000)
    ap.add_argument("--tol", type=float, default=1e-5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    from byol_b200.logreg import L2_GRID, fit_logistic_regression
    dev = torch.device("cuda")
    card = _card()
    l2s = tuple(float(v) for v in L2_GRID)
    lines = []
    for c in (int(v) for v in args.classes.split(",")):
        x, y = _features(args.n + args.n_test, args.dim, c, 7 + c, dev)
        xt, yt, x, y = x[args.n:], y[args.n:], x[:args.n].contiguous(), y[:args.n].contiguous()
        eval_ms = _eval_ms(x, y, c, l2s)
        for rnd in range(args.rounds):
            for method in (("batched", "torch") if rnd % 2 == 0 else ("torch", "batched")):
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                t0 = time.perf_counter()
                if method == "batched":
                    fit = fit_logistic_regression(x, y, c, l2s, args.max_iter, args.tol)
                    torch.cuda.synchronize()
                    secs = time.perf_counter() - t0
                    ws, bs = fit.weight, fit.bias
                    extra = {"evaluations": fit.evaluations, "device_ms_per_evaluation": eval_ms,
                             "converged": sum(e["converged"] for e in fit.heads),
                             "iterations": [e["iterations"] for e in fit.heads],
                             "test_top1": [float(v) for v in fit.evaluate(xt, yt, "top1")]}
                else:
                    ws, bs, evals = [], [], []
                    for l2 in l2s:
                        w, b, n_eval = _torch_fit(x, y, c, l2, args.max_iter, args.tol)
                        ws.append(w); bs.append(b); evals.append(n_eval)
                    torch.cuda.synchronize()
                    secs = time.perf_counter() - t0
                    extra = {"evaluations": evals}
                peak = torch.cuda.max_memory_allocated() - base
                obj = [_objective64(x, y, ws[h].double(), bs[h].double(), l2s[h]) for h in range(len(l2s))]
                rec = dict(card=card, method=method, round=rnd, C=c, N=args.n, D=args.dim, heads=len(l2s),
                           fit_seconds=secs, peak_mem_gb=peak / 1e9, objective64=obj, **extra)
                lines.append(rec)
                print(json.dumps({k: v for k, v in rec.items() if k not in ("objective64", "iterations",
                                                                             "test_top1")}), flush=True)
                fit = ws = bs = None
        # summary: medians and spread of the fit times, and the per-head objective difference batched - torch
        for m in ("batched", "torch"):
            t = [r["fit_seconds"] for r in lines if r["C"] == c and r["method"] == m]
            print(json.dumps({"C": c, "method": m, "median_fit_seconds": float(np.median(t)),
                              "min": min(t), "max": max(t)}), flush=True)
        ob = np.array([r["objective64"] for r in lines if r["C"] == c and r["method"] == "batched"][0])
        ot = np.array([r["objective64"] for r in lines if r["C"] == c and r["method"] == "torch"][0])
        print(json.dumps({"C": c, "objective64_batched_minus_torch": {"min": float((ob - ot).min()),
                                                                      "max": float((ob - ot).max())}}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
