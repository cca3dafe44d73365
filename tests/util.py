"""Shared helpers for the parity tests."""
from fractions import Fraction

import numpy as np
import torch


# exact operands for the bit-for-bit kernel tests (the test_gpu_*_exact files and test_gpu_paper_loss; tests/exact.py
# seeds their rows and replays with gen)
def gen(dev, seed):
    return torch.Generator(device=dev).manual_seed(seed)


def ints(shape, dev, g, amp, density=1.0):
    """fp64 integers in [-amp, amp], a fraction `density` of them non-zero (exactly representable in bf16)."""
    v = torch.randint(-amp, amp + 1, shape, generator=g, device=dev).to(torch.float64)
    if density < 1.0:
        v = v * (torch.rand(shape, generator=g, device=dev) < density)
    return v


def pow2(n, dev, g, signed=False):
    """fp64 [n] powers of two in {1/2, 1, 2} (signed: either sign)."""
    v = torch.pow(2.0, torch.randint(-1, 2, (n,), generator=g, device=dev).to(torch.float64))
    if signed:
        v = v * (torch.randint(0, 2, (n,), generator=g, device=dev) * 2 - 1)
    return v


# fp32 and fp64 roundings for the numpy restatements of compiled kernel arithmetic (test_gpu_elementwise_exact,
# test_gpu_groupnorm_exact, test_gpu_optim_exact, test_gpu_paper_loss)
def _rn32(fr):
    """Fraction -> the nearest fp32 (ties to even), without double rounding."""
    f = np.float32(float(fr))
    if Fraction(float(f)) == fr or not np.isfinite(f):
        return f
    up = Fraction(float(f)) < fr
    other = np.nextafter(f, np.float32(np.inf if up else -np.inf), dtype=np.float32)
    mid = (Fraction(float(f)) + Fraction(float(other))) / 2
    if fr == mid:
        return f if (f.view(np.uint32) & 1) == 0 else other
    return other if (fr > mid) == up else f


def _fma32(a, b, c):
    """fp32 fused multiply-add a*b + c, rounded once (elementwise over equal-length sequences)."""
    return np.array([_rn32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z)))
                     for x, y, z in zip(a, b, c)], dtype=np.float32)


def fma32(a, b, c):
    """Vectorised _fma32 over fp32 arrays.  The fp64 product of two fp32 values is exact; the fp64 sum is turned into
    its round-to-odd value with the exact TwoSum error, and rounding a round-to-odd fp64 value to fp32 is a correct
    single rounding (53 >= 24 + 2 bits)."""
    a, b, c = (np.asarray(v, dtype=np.float32).astype(np.float64) for v in np.broadcast_arrays(a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = p + c
        bb = s - p
        e = (p - (s - bb)) + (c - bb)
        odd = (s.view(np.int64) & 1) == 1
        fix = np.isfinite(s) & (e != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def fma64(a, b, c):
    """fp64 fused multiply-add a*b + c, rounded once (elementwise over equal-length sequences)."""
    return np.array([float(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)])


def gn_finalize_restated(sums, count, eps):
    """csrc/groupnorm.cu gn_finalize_kernel as compiled, from fp64 (sum, sum of squares) [..., 2]: mean = s / count and
    q / count correctly rounded fp64 divisions, var = q/count - mean*mean contracted to one DFMA (rounded once), clamped
    at 0, rstd = 1.0 / sqrt(var + eps) (fp64 IEEE sqrt and division, eps the fp32 value widened); both rounded once to
    fp32.  Returns fp32 [..., 2] (mean, rstd)."""
    sums = np.asarray(sums, dtype=np.float64)
    s, q = sums[..., 0].reshape(-1), sums[..., 1].reshape(-1)
    eps = float(np.float32(eps))
    out = np.empty((s.size, 2), dtype=np.float32)
    for i in range(s.size):
        mean = s[i] / count
        qc = q[i] / count
        if np.isfinite(mean) and np.isfinite(qc):
            var = float(Fraction(qc) - Fraction(mean) * Fraction(mean))
        else:
            with np.errstate(invalid="ignore"):
                var = qc - mean * mean
        var = 0.0 if var < 0.0 else var
        out[i, 0] = np.float32(mean)
        with np.errstate(divide="ignore", invalid="ignore"):
            out[i, 1] = np.float32(1.0 / np.sqrt(np.float64(var) + eps))
    return out.reshape(sums.shape[:-1] + (2,))


def pack_bits(keep):
    """bool [..., C] -> uint8 bits, element i of the flat index space in bit i % 8 of byte i // 8 (bn_apply's mask)."""
    k = keep.reshape(-1, 8).to(torch.int32) * (2 ** torch.arange(8, dtype=torch.int32, device=keep.device))
    return k.sum(1).to(torch.uint8)


def unpack_bits(bits, shape):
    b = bits.to(torch.int32).unsqueeze(1) >> torch.arange(8, device=bits.device, dtype=torch.int32)
    return (b & 1).bool().reshape(shape)


def report_mismatch(name, got, ref, atol, rtol):
    """Return (ok, message) with enough structure to diagnose layout / swizzle / descriptor bugs remotely."""
    got = got.detach().float().cpu()
    ref = ref.detach().float().cpu()
    if got.shape != ref.shape:
        return False, "%s: shape %s vs %s" % (name, tuple(got.shape), tuple(ref.shape))
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    nbad = int(bad.sum())
    finite = bool(torch.isfinite(got).all())
    msg = "%s: max_err=%.4g max_ref=%.4g bad=%d/%d finite=%s" % (name, float(err.max()), float(ref.abs().max()), nbad,
                                                                 err.numel(), finite)
    if nbad:
        flat = bad.reshape(-1, bad.shape[-1]) if bad.dim() > 1 else bad.reshape(1, -1)
        rows = flat.any(1).nonzero().flatten()
        cols = flat.any(0).nonzero().flatten()
        msg += " | bad rows %d/%d (first %s) bad cols %d/%d (first %s)" % (
            rows.numel(), flat.shape[0], rows[:12].tolist(), cols.numel(), flat.shape[1], cols[:12].tolist())
        i = int(err.reshape(-1).argmax())
        msg += " | worst got=%.5g ref=%.5g" % (float(got.reshape(-1)[i]), float(ref.reshape(-1)[i]))
    return nbad == 0 and finite, msg


def assert_close(name, got, ref, atol, rtol):
    ok, msg = report_mismatch(name, got, ref, atol, rtol)
    print(msg)
    assert ok, msg
