"""The harness of the exact kernel tests (test_gpu_*_exact.py, test_gpu_paper_loss.py, test_gpu_conv_patch_h16.py).

A test file keeps its operands, references, kernel tables, matching rules and replay dispatch; this module holds what
does not depend on a kernel family:
* comparisons with the float64 reference or a restatement;
* Case and the row rule: each row's generator is seeded from its name;
* launch checks under torch.profiler, run in a fresh Python process;
* the replay of the calls one eager training step makes.
"""
import contextlib
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.util import gen, report_mismatch

BF = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------------
# comparison
# ------------------------------------------------------------------------------------------------------------------
def rounded_like(got, ref64):
    """The float64 reference rounded once to the kernel's output dtype."""
    if got.dtype in (torch.bool, torch.uint8):
        return ref64.to(got.dtype)
    return ref64.float() if got.dtype == torch.float32 else ref64.float().to(BF)


def same(a, b):
    """torch.equal with NaN == NaN."""
    if a.shape != b.shape or a.dtype != b.dtype:
        return False
    if not a.is_floating_point():
        return torch.equal(a, b)
    na, nb = torch.isnan(a), torch.isnan(b)
    return torch.equal(na, nb) and torch.equal(torch.where(na, 0, a), torch.where(nb, 0, b))


def expect_same(name, got, ref, equal=same, note=None):
    """equal(got, ref); note(got, ref) adds to the mismatch message."""
    if equal(got, ref):
        return
    _, msg = report_mismatch(name, got.float(), ref.float(), 0.0, 0.0)
    raise AssertionError(msg + (note(got, ref) if note else ""))


def expect(name, got, ref64, equal=same, note=None):
    """got == ref64 rounded once to got's dtype.  equal=torch.equal: a NaN matches nothing."""
    expect_same(name, got, rounded_like(got, ref64.reshape(got.shape)), equal, note)


def bits_same(got, ref):
    """got (torch) == ref (numpy fp32 or torch) bit for bit (every NaN matches every NaN)."""
    g = got.detach().float().cpu().numpy().reshape(-1)
    w = ref.detach().float().cpu().numpy() if torch.is_tensor(ref) else np.asarray(ref, dtype=np.float32)
    w = w.reshape(-1)
    if g.shape != w.shape:
        return False
    gn, wn = np.isnan(g), np.isnan(w)
    return bool(np.array_equal(gn, wn) and np.array_equal(np.where(gn, 0, g).view(np.uint32),
                                                          np.where(wn, 0, w).view(np.uint32)))


def expect_bits(name, got, ref):
    if bits_same(got, ref):
        return
    g = got.detach().float().cpu().reshape(1, -1)
    w = ref.detach().float().cpu().reshape(1, -1) if torch.is_tensor(ref) else \
        torch.from_numpy(np.asarray(ref, dtype=np.float32).reshape(1, -1).copy())
    _, msg = report_mismatch(name, g, w, 0.0, 0.0)
    raise AssertionError(msg + " (bits)")


def expect_within(name, got, ref64, tol):
    """|got - ref64| <= tol where ref64 is finite; non-finite entries must match in kind (NaN, +inf, -inf)."""
    g = np.asarray(got.detach().cpu().double().numpy() if torch.is_tensor(got) else got, dtype=np.float64).reshape(-1)
    r, tol = np.asarray(ref64, dtype=np.float64).reshape(-1), np.broadcast_to(np.asarray(tol, np.float64), g.shape)
    fin, inf = np.isfinite(r), np.isinf(r)
    same_kind = np.array_equal(np.isnan(g), np.isnan(r)) and np.array_equal(g[inf], r[inf]) and \
        bool(np.isfinite(g[fin]).all())
    err = np.where(fin, np.abs(g - np.where(fin, r, 0)), 0)
    bad = fin & ~(err <= tol)
    print("%s: max |err| / bound %.3g over %d finite values" % (name, float((err / np.maximum(tol, 1e-300))[fin].max())
                                                                if fin.any() else 0.0, int(fin.sum())))
    assert same_kind, "%s: non-finite entries differ from float64" % name
    assert not bad.any(), "%s: %d of %d beyond the float64 bound (first %s: got %r, ref %r)" % (
        name, int(bad.sum()), bad.size, np.nonzero(bad)[0][:8].tolist(), g[bad][:4].tolist(), r[bad][:4].tolist())


# ------------------------------------------------------------------------------------------------------------------
# float64 convolution references (cuDNN off: im2col + GEMM, exact on integers); activations NHWC, weights OIHW
# ------------------------------------------------------------------------------------------------------------------
def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1)


def conv64(x, w, s, p, groups=1):
    with torch.backends.cudnn.flags(enabled=False):
        return nhwc(F.conv2d(nchw(x), w, None, s, p, 1, groups))


def dgrad64(dy, w, h, wd, s, p, groups=1):
    n, cin = dy.shape[0], w.shape[1] * groups
    with torch.backends.cudnn.flags(enabled=False):
        return nhwc(torch.nn.grad.conv2d_input((n, cin, h, wd), w, nchw(dy), s, p, 1, groups))


def wgrad64(x, dy, wshape, s, p, groups=1):
    with torch.backends.cudnn.flags(enabled=False):
        return torch.nn.grad.conv2d_weight(nchw(x), wshape, nchw(dy), s, p, 1, groups)


# ------------------------------------------------------------------------------------------------------------------
# rows
# ------------------------------------------------------------------------------------------------------------------
class Case:
    """run() launches the kernel(s) under test on fresh outputs and returns them; check(outs) compares them with the
    reference.  What the row is meant for, as the file's launch check reads it: route (the kernel the restated host
    predicate picks), parity (parity-mode dgrad), launches (the byol:: kernels run() launches, in order), branch (the
    restated in-kernel predicates)."""

    def __init__(self, run, check, route=None, parity=False, launches=None, branch=None):
        self.run, self.check = run, check
        self.route, self.parity, self.launches, self.branch = route, parity, launches, branch


def row_case(dev, name, builder, kw):
    """The case of row `name`: builder(dev, generator, **kw) with a generator seeded from the name."""
    return builder(dev, gen(dev, sum(map(ord, name))), **kw)


def run_and_check(case):
    outs = case.run()
    torch.cuda.synchronize()
    case.check(outs)


# ------------------------------------------------------------------------------------------------------------------
# launch checks
# ------------------------------------------------------------------------------------------------------------------
NO_EVENTS = "SKIP: torch.profiler recorded no CUDA kernel events on this system"


def kernel_names(run):
    """The CUDA kernels one run() launches, names without spaces."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        run()
        torch.cuda.synchronize()
    return [e.name.replace(" ", "") for e in prof.events() if "kernel" in e.name]


def check_row_launches(runs, complaints, names_of=kernel_names):
    """Every run() once outside the profiler (first launches: shared-memory opt-in, scratch), then each in a profiler
    session of its own; complaints(name, launched) lists what is wrong with a row's launched = names_of(run).  Even a
    fresh process now and then loses some of a session's kernel events, so a row fails only when three sessions in a
    row show it wrong: the kernels a row launches do not vary from run to run."""
    for run in runs.values():
        run()
    torch.cuda.synchronize()
    wrong, seen_any = [], False
    for name, run in runs.items():
        for _ in range(3):
            launched = names_of(run)
            seen_any = seen_any or bool(launched)
            row_wrong = complaints(name, launched)
            if not row_wrong:
                break
        wrong += row_wrong
    if not seen_any:
        print(NO_EVENTS)
        return
    assert not wrong, "\n".join(wrong)
    print("%d rows launched their kernels" % len(runs))


def byol_kernel_sequence(runs):
    """The byol:: kernels of one profiler session over runs (each followed by a device synchronisation), in
    device-time order, names without their template arguments and signature."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for run in runs:
            run()
            torch.cuda.synchronize()
    events = sorted((e for e in prof.events() if "byol::" in e.name), key=lambda e: e.time_range.start)
    return [re.sub(r"^byol::([A-Za-z0-9_]+).*$", r"\1", e.name) for e in events]


def check_in_fresh_process(module, func="_check_launches"):
    """module.func() in a fresh Python process: one that has already held many profiler sessions (the rest of the GPU
    suite) can drop CUDA kernel events.  Output starting with SKIP skips the test."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([root] + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "from %s import %s; %s()" % (module, func, func)]
    r = subprocess.run(cmd, cwd=root, env=env, capture_output=True, text=True, timeout=900)
    print(r.stdout[-2000:])
    assert r.returncode == 0, r.stderr[-4000:]
    if r.stdout.startswith("SKIP"):
        pytest.skip(r.stdout.strip())


# ------------------------------------------------------------------------------------------------------------------
# replay of the engine's own calls
# ------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def recording(recorders):
    """Within the block, a call of byol_b200.ops.<name> (or of ops.lib.<symbol> for a name "lib.<symbol>") first
    calls recorders[name] with the same arguments, which notes the call's signature, then goes through."""
    from byol_b200 import ops
    saved = []
    try:
        for name, rec in recorders.items():
            owner, attr = (ops.lib, name[4:]) if name.startswith("lib.") else (ops, name)
            orig = getattr(owner, attr)

            def wrapped(*a, _orig=orig, _rec=rec, **k):
                _rec(*a, **k)
                return _orig(*a, **k)
            saved.append((owner, attr, orig))
            setattr(owner, attr, wrapped)
        yield
    finally:
        for owner, attr, orig in reversed(saved):
            setattr(owner, attr, orig)


def byol_model(dev, arch, rep, b, r, classes=1000, projection=256, **model_kw):
    """(model, view 1, view 2, labels): an eager BYOL(rep, projection, classes, 10 steps) built under seed 5, and
    b random r x r views and labels from seed 6."""
    from byol_b200.model import BYOL
    torch.manual_seed(5)
    model = BYOL(rep, projection, classes, 10, arch=arch, **model_kw).to(dev).train()
    model._engine.use_graphs = False
    g = torch.Generator().manual_seed(6)
    a1, a2 = torch.rand(b, 3, r, r, generator=g).to(dev), torch.rand(b, 3, r, r, generator=g).to(dev)
    lab = torch.randint(0, classes, (b,), generator=g).to(dev)
    return model, a1, a2, lab


def byol_train_step(dev, arch, rep, b, r, classes=1000, **model_kw):
    """One eager wiring.train_step of byol_model(...)."""
    from byol_b200 import wiring
    model, a1, a2, lab = byol_model(dev, arch, rep, b, r, classes, **model_kw)
    opt = wiring.build_optimizer(model, global_batch_size=256)
    wiring.train_step(model, opt, a1, a2, lab)
    torch.cuda.synchronize()


def replay(dev, calls, case_of, seed0, detail=""):
    """Every recorded call, in repr order, as case_of(dev, generator seeded seed0 + i, signature): run, synchronise,
    check.  Fails listing every call whose check failed."""
    failures = []
    for i, sig in enumerate(sorted(calls, key=repr)):
        case = case_of(dev, gen(dev, seed0 + i), sig)
        outs = case.run()
        torch.cuda.synchronize()
        try:
            case.check(outs)
        except AssertionError as e:
            failures.append("%s: %s" % (str(sig)[:200], e))
        del outs, case
    print("replayed %d distinct calls%s" % (len(calls), detail))
    assert not failures, "%d of %d replayed calls differ:\n%s" % (len(failures), len(calls), "\n".join(failures))
