"""Shared helpers for the parity tests."""
import torch


# exact operands for the bit-for-bit kernel tests (test_gpu_conv_exact, test_gpu_elementwise_exact)
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
