"""Thin Python wrappers over the C-ABI kernels (``include/byol_b200.h``).

PyTorch is used only as the owner of device memory and of the CUDA stream: every function borrows
``tensor.data_ptr()`` for the duration of one asynchronous launch on ``torch.cuda.current_stream()``.
There is no CPU / ATen fallback; calling any of these without the CUDA extension raises at import time.

Layout conventions: activations NHWC bf16 with channels padded to a multiple of 8; weights for the
tensor-core kernels bf16 ``[Cout, KH*KW*Cpad]`` (fprop) / ``[Cin, KH*KW*Cout]`` (dgrad) made by
:func:`prep_weight` from the fp32 master in the reference's ``[Cout, Cin, KH, KW]`` layout.
"""
import torch

from ._lib import lib, check

BF16 = torch.bfloat16
F32 = torch.float32


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _chk(t, dtype, name):
    if t is None:
        return
    if not t.is_cuda:
        raise ValueError("%s must be a CUDA tensor (byol_b200 has no CPU path)" % name)
    if t.dtype != dtype:
        raise ValueError("%s must be %s, got %s" % (name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("%s must be contiguous" % name)


def conv_out_size(h, k, s, p):
    return (h + 2 * p - k) // s + 1


# ------------------------------------------------------------------------------------------------
# layout / weights
# ------------------------------------------------------------------------------------------------
def nchw_to_nhwc8(x, out=None):
    """fp32 NCHW [N, C<=8, H, W] -> bf16 NHWC [N, H, W, 8] (zero padded channels)."""
    _chk(x, F32, "x")
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty((n, h, w, 8), dtype=BF16, device=x.device)
    check(lib.byol_nchw_to_nhwc8(_ptr(x), _ptr(out), n, c, h, w, _stream()), "byol_nchw_to_nhwc8")
    return out


def stem4_supported(cin, cout, h, w, k, stride, pad):
    """True if the dedicated stem kernels (7x7/s2/p3, <= 4 -> 64 channels, W <= 256) handle this geometry."""
    return bool(lib.byol_stem4_supported(cin, cout, h, w, k, stride, pad))


def nchw_to_stem4(x, out=None):
    """fp32 NCHW [N, C<=4, H, W] -> zero-padded bf16 NHWC4 [N, H+6, Wp, 4] (input format of the stem kernels)."""
    _chk(x, F32, "x")
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty((n, h + 6, lib.byol_stem4_row_pixels(), 4), dtype=BF16, device=x.device)
    check(lib.byol_nchw_to_stem4(_ptr(x), _ptr(out), n, c, h, w, _stream()), "byol_nchw_to_stem4")
    return out


def prep_weight_stem4(w, out=None):
    """fp32 [64, Cin, 7, 7] -> bf16 [7, 4, 64, 8] (stem kernel layout)."""
    _chk(w, F32, "w")
    if out is None:
        out = torch.empty(7 * 4 * 64 * 8, dtype=BF16, device=w.device)
    check(lib.byol_prep_weight_stem4(_ptr(w), _ptr(out), w.shape[1], _stream()), "byol_prep_weight_stem4")
    return out


def stem_conv_fprop(xs4, w_stem4, h, w, stats=None):
    """y[N, H/2, W/2, 64] = conv7x7/s2/p3 over the padded NHWC4 image; stats (fp32 [128], zeroed): += sum | sum sq."""
    _chk(xs4, BF16, "xs4"); _chk(w_stem4, BF16, "w_stem4")
    n = xs4.shape[0]
    y = torch.empty((n, h // 2, w // 2, 64), dtype=BF16, device=xs4.device)
    cs = _ptr(stats) if stats is not None else 0
    cq = _ptr(stats[64:]) if stats is not None else 0
    check(lib.byol_stem_conv_fprop(_ptr(xs4), _ptr(w_stem4), _ptr(y), cs, cq, n, h, w, _stream()),
          "byol_stem_conv_fprop")
    return y


def stem_conv_wgrad(xs4, dy, dw, h, w):
    """dw[64, Cin, 7, 7] (fp32) += dy^T * im2col(image) for the 7x7/s2/p3 stem; xs4 from nchw_to_stem4."""
    _chk(xs4, BF16, "xs4"); _chk(dy, BF16, "dy"); _chk(dw, F32, "dw")
    check(lib.byol_stem_conv_wgrad(_ptr(xs4), _ptr(dy), _ptr(dw), xs4.shape[0], dw.shape[1], h, w, _stream()),
          "byol_stem_conv_wgrad")
    return dw


def subsample2(x):
    """x[N,H,W,C] -> x[:, ::2, ::2, :] compacted (H, W even): the input of a 1x1 / stride-2 convolution."""
    _chk(x, BF16, "x")
    n, h, w, c = x.shape
    y = torch.empty((n, h // 2, w // 2, c), dtype=BF16, device=x.device)
    check(lib.byol_subsample2(_ptr(x), _ptr(y), n, h, w, c, _stream()), "byol_subsample2")
    return y


def prep_weight(w, cpad=None, want_dgrad=True, out_f=None, out_d=None):
    """fp32 [Cout, Cin, KH, KW] (or [out, in] for Linear) -> (w_fprop bf16 [Cout, taps*Cpad], w_dgrad bf16 [Cin, taps*Cout])."""
    _chk(w, F32, "w")
    if w.dim() == 2:
        cout, cin = w.shape
        kh = kw = 1
    else:
        cout, cin, kh, kw = w.shape
    if cpad is None:
        cpad = (cin + 7) // 8 * 8
    if out_f is None:
        out_f = torch.empty((cout, kh * kw * cpad), dtype=BF16, device=w.device)
    if want_dgrad and out_d is None:
        out_d = torch.empty((cin, kh * kw * cout), dtype=BF16, device=w.device)
    check(lib.byol_prep_weight(_ptr(w), _ptr(out_f), _ptr(out_d) if want_dgrad else 0, cout, cin, cpad, kh, kw,
                               _stream()), "byol_prep_weight")
    return out_f, (out_d if want_dgrad else None)


def prep_weight_fold(w, out_f=None):
    """Stem layout: fp32 [Cout, Cin<=8, KH, KW<=8] -> bf16 [Cout, KH*64] (column = kh*64 + kw*8 + c)."""
    _chk(w, F32, "w")
    cout, cin, kh, kw = w.shape
    if out_f is None:
        out_f = torch.empty((cout, kh * 64), dtype=BF16, device=w.device)
    check(lib.byol_prep_weight_fold(_ptr(w), _ptr(out_f), cout, cin, kh, kw, _stream()), "byol_prep_weight_fold")
    return out_f


def prep_weights_multi(flat, pool_f, pool_d, desc, num_blocks=None):
    """All weights of one parameter set (flat fp32 vector) -> bf16 tensor-core layouts, one launch.
    num_blocks: sum of prep_unit_blocks over the rows of `desc` (computed from the device table when not given)."""
    if num_blocks is None:
        num_blocks = prep_blocks(desc.cpu().tolist())
    check(lib.byol_prep_weights_multi(_ptr(flat), _ptr(pool_f), _ptr(pool_d), _ptr(desc), desc.shape[0], num_blocks,
                                      _stream()), "byol_prep_weights_multi")


def prep_weights_grouped(flat, pool_f, pool_d, desc, max_c):
    """All grouped 3x3 weights of one parameter set -> block-diagonal tile layouts, one launch.
    desc: device int64 [units, 5] = [src offset, fprop offset, dgrad offset or -1, C, Cg]; max_c: the largest C."""
    check(lib.byol_prep_weights_grouped(_ptr(flat), _ptr(pool_f), _ptr(pool_d), _ptr(desc), desc.shape[0], max_c,
                                        _stream()), "byol_prep_weights_grouped")


def prep_weight_grouped(w, want_dgrad=True):
    """fp32 [C, Cg, 3, 3] -> (w_fprop, w_dgrad) bf16 [C/64, 64, 9*64] block-diagonal tiles (w_dgrad None unless
    want_dgrad)."""
    _chk(w, F32, "w")
    c, cg = w.shape[0], w.shape[1]
    if tuple(w.shape[2:]) != (3, 3) or c % 64 != 0 or 64 % cg != 0:
        raise ValueError("prep_weight_grouped: need a [C, Cg, 3, 3] weight, C a multiple of 64 and Cg dividing 64, got %s"
                         % (tuple(w.shape),))
    wf = torch.empty((c // 64, 64, 9 * 64), dtype=BF16, device=w.device)
    wd = torch.empty_like(wf) if want_dgrad else None
    desc = torch.tensor([[0, 0, 0 if want_dgrad else -1, c, cg]], dtype=torch.int64, device=w.device)
    prep_weights_grouped(w.reshape(-1), wf, wd, desc, c)
    return wf, wd


def prep_blocks(rows):
    """Grid size for prep_weights_multi: rows = [[src, dstf, dstd, Cout, Cin, Cpad, taps, fold], ...]."""
    return sum(lib.byol_prep_unit_blocks(int(r[3]), int(r[4]), int(r[5]), int(r[6]), int(r[7])) for r in rows)


def cast_bf16_pitched(x2d, ldy):
    """fp32 [rows, cols] (any row stride) -> bf16 [rows, ldy] with zero padding columns (ldy >= cols)."""
    if x2d.dtype != F32 or not x2d.is_cuda or x2d.stride(1) != 1:
        raise ValueError("cast_bf16_pitched: need a CUDA fp32 matrix with unit column stride")
    rows, cols = x2d.shape
    out = torch.empty((rows, ldy), dtype=BF16, device=x2d.device)
    check(lib.byol_cast_f32_bf16_2d(_ptr(x2d), _ptr(out), rows, cols, x2d.stride(0), ldy, _stream()),
          "byol_cast_f32_bf16_2d")
    return out


def cast_bf16(x, out=None):
    _chk(x, F32, "x")
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    check(lib.byol_cast_f32_bf16(_ptr(x), _ptr(out), x.numel(), _stream()), "byol_cast_f32_bf16")
    return out


# ------------------------------------------------------------------------------------------------
# tensor-core convolution / linear
# ------------------------------------------------------------------------------------------------
def _grouped_unsupported(**options):
    bad = sorted(k for k, v in options.items() if v is not None and v is not False)
    if bad:
        raise ValueError("grouped convolutions do not support %s" % ", ".join(bad))


def conv_fprop(x, w_f, kh, kw, stride, pad, bias=None, resid=None, stats=None, relu=False, out_fp32=False,
               out=None, force_gather=False):
    """y[N,Ho,Wo,Cout] = conv(x[N,H,W,C], w).  stats: optional zeroed fp32 [2*Cout] receiving column sum / sqsum.
    A 3-D w_f is the grouped tile layout [C/64, 64, 9*64] of :func:`prep_weights_grouped` (grouped 3x3 conv)."""
    _chk(x, BF16, "x"); _chk(w_f, BF16, "w_f"); _chk(bias, F32, "bias"); _chk(resid, BF16, "resid")
    _chk(stats, F32, "stats")
    n, h, w, c = x.shape
    if w_f.dim() == 3:
        _grouped_unsupported(bias=bias, resid=resid, relu=relu, out_fp32=out_fp32, force_gather=force_gather)
        ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
        if out is None:
            out = torch.empty((n, ho, wo, c), dtype=BF16, device=x.device)
        cq = (stats.data_ptr() + 4 * c) if stats is not None else 0
        check(lib.byol_conv_fprop_grouped(_ptr(x), _ptr(w_f), _ptr(out), _ptr(stats), cq, n, h, w, c, ho, wo, kh, kw,
                                          stride, pad, _stream()), "byol_conv_fprop_grouped")
        return out
    cout, ldw = w_f.shape
    ho, wo = conv_out_size(h, kh, stride, pad), conv_out_size(w, kw, stride, pad)
    if out is None:
        out = torch.empty((n, ho, wo, cout), dtype=F32 if out_fp32 else BF16, device=x.device)
    cs = _ptr(stats)
    cq = (stats.data_ptr() + 4 * cout) if stats is not None else 0
    check(lib.byol_conv_igemm(_ptr(x), _ptr(w_f), _ptr(out), _ptr(resid), 0, 0, _ptr(bias), cs, cq, n, h, w, c, ho, wo,
                              cout, kh, kw, stride, pad, 0, ldw, cout, int(out_fp32), int(relu), int(force_gather),
                              _stream()), "byol_conv_igemm(fprop)")
    return out


def conv_dgrad(dy, w_d, h, w, kh, kw, stride, pad, resid=None, out=None, force_gather=False, resid_mask=None,
               resid_up=False):
    """dx[N,H,W,Cin] = conv_transpose(dy[N,Ho,Wo,Cout], w) (+ resid, optionally only where the bits of resid_mask,
    the uint8 ReLU mask written by bn_apply, are set; resid_up: resid is the compact [N, h/2, w/2, Cin] gradient of a
    stride-2 branch, added to the even pixels);  w_d is the dgrad layout [Cin, taps*Cout], or the grouped tile
    layout [C/64, 64, 9*64] (3-D) of :func:`prep_weights_grouped`."""
    _chk(dy, BF16, "dy"); _chk(w_d, BF16, "w_d"); _chk(resid, BF16, "resid"); _chk(resid_mask, torch.uint8, "mask")
    n, ho, wo, cout = dy.shape
    if w_d.dim() == 3:
        _grouped_unsupported(resid=resid, resid_mask=resid_mask, resid_up=resid_up, force_gather=force_gather)
        if out is None:
            out = torch.empty((n, h, w, cout), dtype=BF16, device=dy.device)
        check(lib.byol_conv_dgrad_grouped(_ptr(dy), _ptr(w_d), _ptr(out), n, ho, wo, cout, h, w, kh, kw, stride, pad,
                                          _stream()), "byol_conv_dgrad_grouped")
        return out
    cin, ldw = w_d.shape
    if out is None:
        out = torch.empty((n, h, w, cin), dtype=BF16, device=dy.device)
    check(lib.byol_conv_igemm(_ptr(dy), _ptr(w_d), _ptr(out), _ptr(resid), _ptr(resid_mask), int(resid_up), 0, 0, 0, n, ho, wo, cout, h, w, cin,
                              kh, kw, stride, pad, 1, ldw, cin, 0, 0, int(force_gather), _stream()),
          "byol_conv_igemm(dgrad)")
    return out


def conv_wgrad(x, dy, dw, kh, kw, stride, pad, force_gather=False):
    """dw[Cout,Cin,KH,KW] (fp32, reference layout) += dy^T * im2col(x).  x: [N,H,W,Cpad], dy: [N,Ho,Wo,ldy] whose
    first Cout = dw.shape[0] columns are the gradient (ldy > Cout: pitched rows, e.g. a 10-class classifier).
    dw.shape[1] < C (C a multiple of 64, so not channel padding): a grouped 3x3 convolution with dw.shape[1] input
    channels per group; only the in-group entries of dw are accumulated."""
    _chk(x, BF16, "x"); _chk(dy, BF16, "dy"); _chk(dw, F32, "dw")
    n, h, w, c = x.shape
    _, ho, wo, ldy = dy.shape
    cout, cin_real = dw.shape[0], dw.shape[1]
    if cin_real < c and c % 64 == 0:
        _grouped_unsupported(force_gather=force_gather)
        if cout != c or ldy != c:
            raise ValueError("grouped conv_wgrad: dw [%d, %d] and dy with %d channels do not match x with %d channels"
                             % (cout, cin_real, ldy, c))
        check(lib.byol_conv_wgrad_grouped(_ptr(x), _ptr(dy), _ptr(dw), n, h, w, c, cin_real, ho, wo, kh, kw, stride,
                                          pad, _stream()), "byol_conv_wgrad_grouped")
        return dw
    check(lib.byol_conv_wgrad(_ptr(x), _ptr(dy), _ptr(dw), n, h, w, c, cin_real, ho, wo, cout, ldy, kh, kw, stride,
                              pad, int(force_gather), _stream()), "byol_conv_wgrad")
    return dw


def mlp_fused_supported(b, k1, h, o):
    return bool(lib.byol_mlp_fused_supported(b, k1, h, o))


def mlp_fused_fwd(x2d, w1, b1, gamma, beta, w2, b2, stats, running_mean, running_var, momentum, eps, count, coeffs,
                  grid_bar, train, save, peer=None):
    """Linear -> BatchNorm1d -> ReLU -> Linear of one lane in ONE cooperative kernel (csrc/mlp_fused.cu).
    stats: zeroed fp32 [2H] (train); coeffs: fp32 [4, H] out; grid_bar: persistent zeroed int32 [2] (one per stream);
    peer: comm.PeerExchange of this stream's channel under SyncBatchNorm (world > 1), else None.
    Returns (out fp32 [B, O], h bf16 [B, H] | None, a bf16 [B, H] | None)."""
    _chk(x2d, BF16, "x"); _chk(w1, BF16, "w1"); _chk(w2, BF16, "w2"); _chk(stats, F32, "stats")
    b, k1 = x2d.shape
    h, ldw1 = w1.shape
    o, ldw2 = w2.shape
    dev = x2d.device
    out = torch.zeros((b, o), dtype=F32, device=dev)
    hs = torch.empty((b, h), dtype=BF16, device=dev) if save else None
    as_ = torch.empty((b, h), dtype=BF16, device=dev) if save else None
    pp, world, rank, cap, ctr = 0, 1, 0, 0, 0
    if peer is not None:
        pp, world, rank, cap, ctr = peer.ptrs, peer.world, peer.rank, peer.cap_bytes, peer.counter.data_ptr()
    check(lib.byol_mlp_fused_fwd(_ptr(x2d), _ptr(w1), _ptr(b1), _ptr(gamma), _ptr(beta), _ptr(w2), _ptr(b2), _ptr(stats),
                                 _ptr(running_mean), _ptr(running_var), float(momentum), float(eps), float(count),
                                 _ptr(coeffs), _ptr(out), _ptr(hs), _ptr(as_), _ptr(grid_bar), b, k1, h, o, ldw1, ldw2,
                                 int(train), pp, world, rank, cap, ctr, _stream()), "byol_mlp_fused_fwd")
    return out, hs, as_


def linear_fprop(x2d, w_f, bias=None, stats=None, relu=False, out_fp32=False, out=None):
    """y[M, out] = x[M, in] @ W^T (+bias): a 1x1 'convolution' over M pixels."""
    m, k = x2d.shape
    y = conv_fprop(x2d.view(m, 1, 1, k), w_f, 1, 1, 1, 0, bias=bias, stats=stats, relu=relu, out_fp32=out_fp32,
                   out=None if out is None else out.view(m, 1, 1, -1))
    return y.view(m, -1)


def linear_dgrad(dy2d, w_d, out=None):
    m, n = dy2d.shape
    dx = conv_dgrad(dy2d.view(m, 1, 1, n), w_d, 1, 1, 1, 1, 1, 0, out=None if out is None else out.view(m, 1, 1, -1))
    return dx.view(m, -1)


def linear_wgrad(x2d, dy2d, dw):
    m, k = x2d.shape
    n = dy2d.shape[1]
    conv_wgrad(x2d.view(m, 1, 1, k), dy2d.view(m, 1, 1, n), dw.view(n, dw.shape[1], 1, 1), 1, 1, 1, 0)
    return dw


# ------------------------------------------------------------------------------------------------
# batch norm
# ------------------------------------------------------------------------------------------------
def bn_stats(x2d, stats):
    """stats (zeroed fp32 [2C]) += [column sums, column sums of squares] of x2d [M, C] bf16."""
    _chk(x2d, BF16, "x"); _chk(stats, F32, "stats")
    m, c = x2d.shape
    check(lib.byol_bn_stats(_ptr(x2d), _ptr(stats), m, c, _stream()), "byol_bn_stats")
    return stats


def bn_finalize(stats, count, gamma, beta, running_mean, running_var, momentum, eps, coeffs):
    """Single-lane form of :func:`bn_finalize_lanes`; coeffs: fp32 [4, C] receiving scale, shift, mean, invstd."""
    bn_finalize_lanes(stats, count, [gamma], [beta], running_mean, running_var, momentum, eps, coeffs)
    return coeffs


def bn_finalize_lanes(stats, count, gammas, betas, running_mean, running_var, momentum, eps, coeffs):
    """One launch for all lock-step lanes: stats [L*2C], coeffs [L,4,C]; gammas/betas: per-lane fp32 [C] tensors."""
    L = len(gammas)
    c = gammas[0].numel()
    g = [_ptr(t) for t in gammas] + [0] * (4 - L)
    b = [_ptr(t) for t in betas] + [0] * (4 - L)
    check(lib.byol_bn_finalize_lanes(_ptr(stats), float(count), L, g[0], b[0], g[1], b[1], g[2], b[2], g[3], b[3],
                                     _ptr(running_mean), _ptr(running_var), float(momentum), float(eps),
                                     _ptr(coeffs), c, _stream()), "byol_bn_finalize_lanes")
    return coeffs


def bn_eval_coeffs(gamma, beta, running_mean, running_var, eps, coeffs):
    c = gamma.numel()
    check(lib.byol_bn_eval_coeffs(_ptr(gamma), _ptr(beta), _ptr(running_mean), _ptr(running_var), float(eps),
                                  _ptr(coeffs[0]), _ptr(coeffs[1]), c, _stream()), "byol_bn_eval_coeffs")
    return coeffs


def bn_apply(x2d, scale, shift, relu, resid=None, rscale=None, rshift=None, out=None, out_f32=None, mask_out=None):
    """y = act(x*scale + shift (+ resid | resid*rscale + rshift)); mask_out (uint8 [M*C/8]) receives the bits y > 0."""
    _chk(x2d, BF16, "x"); _chk(resid, BF16, "resid"); _chk(mask_out, torch.uint8, "mask_out")
    m, c = x2d.shape
    if out is None and out_f32 is None:
        out = torch.empty_like(x2d)
    check(lib.byol_bn_apply(_ptr(x2d), _ptr(scale), _ptr(shift), _ptr(resid), _ptr(rscale), _ptr(rshift), _ptr(out),
                            _ptr(out_f32), _ptr(mask_out), m, c, int(relu), _stream()), "byol_bn_apply")
    return out if out is not None else out_f32


def bn_bwd_reduce(g, x, coeffs, s12, mask_mode, act=None):
    """s12 (zeroed fp32 [2C]) += [sum dz, sum dz*xhat];  mask_mode 0 none / 1 relu(x*scale+shift) / 2 act>0 /
    3 mask bits (act = the uint8 mask written by bn_apply)."""
    _chk(g, BF16, "g"); _chk(x, BF16, "x"); _chk(act, torch.uint8 if mask_mode == 3 else BF16, "act")
    m, c = x.shape
    check(lib.byol_bn_bwd_reduce(_ptr(g), _ptr(x), _ptr(act), _ptr(coeffs[0]), _ptr(coeffs[1]), _ptr(coeffs[2]),
                                 _ptr(coeffs[3]), _ptr(s12), m, c, mask_mode, _stream()), "byol_bn_bwd_reduce")
    return s12


def bn_bwd_apply(g, x, coeffs, gamma, s12, count, mask_mode, act=None, dy=None, dz_out=None, s12_local=None,
                 dgamma=None, dbeta=None):
    """dy = gamma*invstd*(dz - s1/n - xhat*s2/n) with the (global) sums s12 over `count` rows; when dgamma/dbeta
    are given they are incremented by the rank-local sums (s12_local, default s12)."""
    _chk(g, BF16, "g"); _chk(x, BF16, "x"); _chk(act, torch.uint8 if mask_mode == 3 else BF16, "act")
    m, c = x.shape
    if dy is None:
        dy = torch.empty_like(x)
    check(lib.byol_bn_bwd_apply(_ptr(g), _ptr(x), _ptr(act), _ptr(coeffs[0]), _ptr(coeffs[1]), _ptr(coeffs[2]),
                                _ptr(coeffs[3]), _ptr(gamma), _ptr(s12), float(count), _ptr(dy), _ptr(dz_out), m, c,
                                mask_mode, _ptr(s12_local), _ptr(dgamma), _ptr(dbeta), _stream()),
          "byol_bn_bwd_apply")
    return dy


def col_sum(x2d, out):
    """out[c] (fp32) += sum_r x2d[r, c]."""
    m, c = x2d.shape
    check(lib.byol_col_sum(_ptr(x2d), _ptr(out), m, c, x2d.stride(0), int(x2d.dtype == F32), _stream()),
          "byol_col_sum")
    return out


# ------------------------------------------------------------------------------------------------
# GroupNorm (32 groups) and weight standardisation (BYOL(norm="group_ws"); csrc/groupnorm.cu)
# ------------------------------------------------------------------------------------------------
GN_GROUPS = 32


def _chk_shape(t, dtype, shape, name):
    """_chk, and t has exactly `shape` (nothing to check when t is None)."""
    if t is None:
        return
    _chk(t, dtype, name)
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s must have shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))


def _chk_bits(t, x, name):
    """t (optional): contiguous CUDA uint8 mask bits of x, one bit per element of x."""
    if t is None:
        return
    _chk(t, torch.uint8, name)
    if t.numel() * 8 != x.numel():
        raise ValueError("%s must hold %d mask bytes (one bit per element of x), got %d" % (name, x.numel() // 8,
                                                                                           t.numel()))


def _chk_gn(x, gamma, beta, stats, gamma_name="gamma", beta_name="beta", stats_name="stats"):
    """x bf16 [N, ..., C]; gamma / beta fp32 [C]; stats fp32 [N, 32, 2].  Checked on the host only: these wrappers run
    inside CUDA-graph capture, where a device sync is not allowed."""
    _chk(x, BF16, "x")
    if x.dim() < 2:
        raise ValueError("x must be [N, ..., C], got shape %s" % (tuple(x.shape),))
    n, c = x.shape[0], x.shape[-1]
    for t, name in ((gamma, gamma_name), (beta, beta_name)):
        if t is None:
            raise ValueError("%s is required" % name)
        _chk_shape(t, F32, (c,), name)
    if stats is None:
        raise ValueError("%s is required" % stats_name)
    _chk_shape(stats, F32, (n, GN_GROUPS, 2), stats_name)
    return n, c


def _chk_act(act, x, mask_mode):
    if mask_mode not in (0, 1, 2, 3):
        raise ValueError("mask_mode must be 0, 1, 2 or 3, got %r" % (mask_mode,))
    if mask_mode >= 2 and act is None:
        raise ValueError("mask_mode %d needs act" % mask_mode)
    if mask_mode == 3:
        _chk_bits(act, x, "act")
    elif mask_mode == 2:
        _chk_shape(act, BF16, x.shape, "act")


def _chk_ws(desc, num_rows, stats):
    """desc: contiguous CUDA int64 [units, 5]; stats fp32 [num_rows, 2]."""
    _chk(desc, torch.int64, "desc")
    if desc.dim() != 2 or desc.shape[1] != 5 or desc.shape[0] < 1:
        raise ValueError("desc must be [units, 5] with at least one unit, got shape %s" % (tuple(desc.shape),))
    if int(num_rows) <= 0:
        raise ValueError("num_rows must be positive, got %d" % int(num_rows))
    _chk_shape(stats, F32, (int(num_rows), 2), "stats")


def ws_fwd(flat, desc, num_rows, w_out, stats):
    """Standardise every weight row listed in `desc` (device int64 [units, 5] = src offset in flat, offset in w_out,
    Cout, fan-in, first row): w_out[row] = (w - mean) / sqrt(var + 1e-5) (biased variance); stats fp32 [rows, 2] =
    (mean, rstd)."""
    _chk(flat, F32, "flat"); _chk(w_out, F32, "w_out"); _chk_ws(desc, num_rows, stats)
    check(lib.byol_ws_fwd(_ptr(flat), _ptr(desc), desc.shape[0], int(num_rows), _ptr(w_out), _ptr(stats), _stream()),
          "byol_ws_fwd")


def ws_bwd(dwhat, what, stats, desc, num_rows, grad):
    """grad[row] (flat fp32, at the row's src offset) += rstd * (dw^ - mean(dw^) - w^ * mean(dw^ * w^))."""
    _chk(dwhat, F32, "dwhat"); _chk(what, F32, "what"); _chk(grad, F32, "grad"); _chk_ws(desc, num_rows, stats)
    check(lib.byol_ws_bwd(_ptr(dwhat), _ptr(what), _ptr(stats), _ptr(desc), desc.shape[0], int(num_rows), _ptr(grad),
                          _stream()), "byol_ws_bwd")


def gn_stats(y, eps, out=None, sums64=None):
    """y bf16 [N, H, W, C] -> fp32 [N, 32, 2] (mean, rstd) per (image, group); sums64 (fp64 [N, 32, 2], optional)
    receives the sums and sums of squares."""
    _chk(y, BF16, "y")
    n, c = y.shape[0], y.shape[-1]
    _chk_shape(out, F32, (n, GN_GROUPS, 2), "out"); _chk_shape(sums64, F64, (n, GN_GROUPS, 2), "sums64")
    if out is None:
        out = torch.empty((n, GN_GROUPS, 2), dtype=F32, device=y.device)
    check(lib.byol_gn_stats(_ptr(y), _ptr(out), _ptr(sums64), n, y.numel() // (n * c), c, float(eps), _stream()),
          "byol_gn_stats", kernels=2)
    return out


def gn_apply(x, gamma, beta, stats, relu, resid=None, rgn=None, out=None, mask_out=None):
    """act(x*scale + shift (+ resid | + GroupNorm(resid))) of bf16 [N, H, W, C] with scale = gamma*rstd, shift =
    beta - mean*scale per (image, channel); rgn = (gamma, beta, stats) of a GroupNorm-applied residual."""
    n, c = _chk_gn(x, gamma, beta, stats)
    _chk_shape(resid, BF16, x.shape, "resid"); _chk_shape(out, BF16, x.shape, "out"); _chk_bits(mask_out, x, "mask_out")
    rg, rb, rs = rgn if rgn is not None else (None, None, None)
    if rgn is not None:
        if resid is None:
            raise ValueError("rgn needs resid")
        _chk_gn(resid, rg, rb, rs, "rgamma", "rbeta", "rstats")
    if out is None:
        out = torch.empty_like(x)
    check(lib.byol_gn_apply(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(resid), _ptr(rg), _ptr(rb), _ptr(rs),
                            _ptr(out), _ptr(mask_out), n, x.numel() // (n * c), c, int(relu), _stream()),
          "byol_gn_apply")
    return out


def gn_relu_maxpool_fwd(x, gamma, beta, stats, k=3, s=2, p=1, want_idx=True):
    """maxpool(relu(GroupNorm(x))) in one pass (stem); bit-identical to gn_apply(relu) + maxpool_fwd."""
    _chk_gn(x, gamma, beta, stats)
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, k, s, p), conv_out_size(w, k, s, p)
    y = torch.empty((n, ho, wo, c), dtype=BF16, device=x.device)
    idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=x.device) if want_idx else None
    check(lib.byol_gn_relu_maxpool_fwd(_ptr(x), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(y), _ptr(idx), n, h, w, c,
                                       k, s, p, _stream()), "byol_gn_relu_maxpool_fwd")
    return y, idx


def gn_bwd_reduce(g, x, gamma, beta, stats, s12, mask_mode, dgamma, dbeta, act=None):
    """s12 (zeroed fp32 [N, 32, 2]) += per (image, group) [sum gamma*dz, sum gamma*dz*xhat]; dgamma / dbeta (fp32 [C],
    required) += the per-channel sums dz*xhat / dz.  mask_mode as bn_bwd_reduce."""
    n, c = _chk_gn(x, gamma, beta, stats)
    _chk_shape(g, BF16, x.shape, "g"); _chk_act(act, x, mask_mode)
    for t, name in ((s12, "s12"), (dgamma, "dgamma"), (dbeta, "dbeta")):
        if t is None:
            raise ValueError("%s is required" % name)
    _chk_shape(s12, F32, (n, GN_GROUPS, 2), "s12")
    _chk_shape(dgamma, F32, (c,), "dgamma"); _chk_shape(dbeta, F32, (c,), "dbeta")
    check(lib.byol_gn_bwd_reduce(_ptr(g), _ptr(x), _ptr(act), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(s12),
                                 _ptr(dgamma), _ptr(dbeta), n, x.numel() // (n * c), c, mask_mode, _stream()),
          "byol_gn_bwd_reduce", kernels=4)
    return s12


def gn_bwd_apply(g, x, gamma, beta, stats, s12, mask_mode, act=None, dy=None, dz_out=None):
    """dy = rstd*(gamma*dz - s1/m - xhat*s2/m) per (image, group), m = H*W*C/32; dz_out (optional) receives dz."""
    n, c = _chk_gn(x, gamma, beta, stats)
    _chk_shape(g, BF16, x.shape, "g"); _chk_act(act, x, mask_mode)
    if s12 is None:
        raise ValueError("s12 is required")
    _chk_shape(s12, F32, (n, GN_GROUPS, 2), "s12")
    _chk_shape(dy, BF16, x.shape, "dy"); _chk_shape(dz_out, BF16, x.shape, "dz_out")
    if dy is None:
        dy = torch.empty_like(x)
    check(lib.byol_gn_bwd_apply(_ptr(g), _ptr(x), _ptr(act), _ptr(gamma), _ptr(beta), _ptr(stats), _ptr(s12), _ptr(dy),
                                _ptr(dz_out), n, x.numel() // (n * c), c, mask_mode, _stream()), "byol_gn_bwd_apply")
    return dy


# ------------------------------------------------------------------------------------------------
# pooling
# ------------------------------------------------------------------------------------------------
def maxpool_fwd(x, k=3, s=2, p=1, want_idx=True):
    _chk(x, BF16, "x")
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, k, s, p), conv_out_size(w, k, s, p)
    y = torch.empty((n, ho, wo, c), dtype=BF16, device=x.device)
    idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=x.device) if want_idx else None
    check(lib.byol_maxpool_fwd(_ptr(x), _ptr(y), _ptr(idx), n, h, w, c, k, s, p, _stream()), "byol_maxpool_fwd")
    return y, idx


def bn_relu_maxpool_fwd(x, scale, shift, k=3, s=2, p=1, want_idx=True):
    """maxpool(relu(x*scale + shift)) in one pass (stem); bit-identical to bn_apply(relu) + maxpool_fwd."""
    _chk(x, BF16, "x")
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, k, s, p), conv_out_size(w, k, s, p)
    y = torch.empty((n, ho, wo, c), dtype=BF16, device=x.device)
    idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=x.device) if want_idx else None
    check(lib.byol_bn_relu_maxpool_fwd(_ptr(x), _ptr(scale), _ptr(shift), _ptr(y), _ptr(idx), n, h, w, c, k, s, p,
                                       _stream()), "byol_bn_relu_maxpool_fwd")
    return y, idx


def maxpool_bwd(dy, idx, h, w, k=3, s=2, p=1):
    _chk(dy, BF16, "dy")
    n, ho, wo, c = dy.shape
    dx = torch.empty((n, h, w, c), dtype=BF16, device=dy.device)
    check(lib.byol_maxpool_bwd(_ptr(dy), _ptr(idx), _ptr(dx), n, h, w, c, k, s, p, _stream()), "byol_maxpool_bwd")
    return dx


def avgpool_fwd(x, want_f32=True, want_bf16=True):
    _chk(x, BF16, "x")
    n, h, w, c = x.shape
    yf = torch.empty((n, c), dtype=F32, device=x.device) if want_f32 else None
    yb = torch.empty((n, c), dtype=BF16, device=x.device) if want_bf16 else None
    check(lib.byol_avgpool_fwd(_ptr(x), _ptr(yf), _ptr(yb), n, h * w, c, _stream()), "byol_avgpool_fwd")
    return yf, yb


def avgpool_bwd(g_bf16, g_f32, n, h, w, c):
    _chk(g_bf16, BF16, "g_bf16"); _chk(g_f32, F32, "g_f32")
    dev = (g_bf16 if g_bf16 is not None else g_f32).device
    dx = torch.empty((n, h, w, c), dtype=BF16, device=dev)
    check(lib.byol_avgpool_bwd(_ptr(g_bf16), _ptr(g_f32), _ptr(dx), n, h * w, c, _stream()), "byol_avgpool_bwd")
    return dx


# ------------------------------------------------------------------------------------------------
# objective / EMA / LARS
# ------------------------------------------------------------------------------------------------
def loss_fwd(q1, q2, z1, z2, workspace, loss, saved):
    for t, nm in ((q1, "q1"), (q2, "q2"), (z1, "z1"), (z2, "z2")):
        _chk(t, F32, nm)
    rows, dim = q1.shape
    check(lib.byol_loss_fwd(_ptr(q1), _ptr(q2), _ptr(z1), _ptr(z2), rows, dim, _ptr(workspace), _ptr(loss),
                            _ptr(saved), _stream()), "byol_loss_fwd", kernels=2)
    return loss


def loss_bwd(q1, q2, z1, z2, saved, grad_out, dq1, dq2):
    rows, dim = q1.shape
    check(lib.byol_loss_bwd(_ptr(q1), _ptr(q2), _ptr(z1), _ptr(z2), _ptr(saved), _ptr(grad_out), _ptr(dq1),
                            _ptr(dq2), rows, dim, _stream()), "byol_loss_bwd")
    return dq1, dq2


def _loss_rows_shape(q1, q2, z1, z2):
    for t, nm in ((q1, "q1"), (q2, "q2"), (z1, "z1"), (z2, "z2")):
        _chk(t, F32, nm)
    if q1.dim() != 2 or any(t.shape != q1.shape for t in (q2, z1, z2)):
        raise ValueError("the paper's loss needs four [rows, dim] tensors of one shape")
    return q1.shape


def loss_rows_fwd(q1, q2, z1, z2, loss, saved):
    """The BYOL paper's loss of fp32 [rows, dim] predictions q and targets z (dim a multiple of 4): loss (fp32 [1]) =
    mean over rows of |q1^ - z2^|^2 + |q2^ - z1^|^2, per-row L2-normalised; saved: fp32 [rows, 8] for the backward."""
    rows, dim = _loss_rows_shape(q1, q2, z1, z2)
    _chk(loss, F32, "loss"); _chk(saved, F32, "saved")
    if saved.numel() != 8 * rows:
        raise ValueError("saved must hold 8 floats per row")
    check(lib.byol_loss_rows_fwd(_ptr(q1), _ptr(q2), _ptr(z1), _ptr(z2), rows, dim, _ptr(loss), _ptr(saved),
                                 _stream()), "byol_loss_rows_fwd", kernels=2)
    return loss


def loss_rows_bwd(q1, q2, z1, z2, saved, grad_out, dq1, dq2):
    """dq1, dq2 of loss_rows_fwd's loss, scaled by grad_out (fp32 [1], or None: 1)."""
    rows, dim = _loss_rows_shape(q1, q2, z1, z2)
    _chk(saved, F32, "saved"); _chk(grad_out, F32, "grad_out"); _chk(dq1, F32, "dq1"); _chk(dq2, F32, "dq2")
    check(lib.byol_loss_rows_bwd(_ptr(q1), _ptr(q2), _ptr(z1), _ptr(z2), _ptr(saved), _ptr(grad_out), _ptr(dq1),
                                 _ptr(dq2), rows, dim, _stream()), "byol_loss_rows_bwd")
    return dq1, dq2


def ema_update(x, mean, one_minus_decay, decay):
    """mean <- fl(fl(a*x) + fl(d*mean)) in place; a, d already rounded to fp32 by the caller."""
    _chk(x, F32, "x"); _chk(mean, F32, "mean")
    if x.numel() != mean.numel():
        raise ValueError("ema_update: size mismatch")
    check(lib.byol_ema_update(_ptr(x), _ptr(mean), float(one_minus_decay), float(decay), x.numel(), _stream()),
          "byol_ema_update")
    return mean


def lars_sgd_step(table, trust_coef, eps, momentum, first_step):
    """table: dict of device tensors p_ptrs/g_ptrs/m_ptrs (int64 pointer tables, m_ptrs may be None),
    chunk_start (int64), chunk_len / chunk_tensor / tensor_first_chunk (int32), wd / lr (fp32), ignore (int32),
    partial (fp64 [2 * chunks])."""
    check(lib.byol_lars_sgd_step(_ptr(table["p_ptrs"]), _ptr(table["g_ptrs"]), _ptr(table.get("m_ptrs")),
                                 _ptr(table["chunk_start"]), _ptr(table["chunk_len"]), _ptr(table["chunk_tensor"]),
                                 table["chunk_start"].numel(), _ptr(table["tensor_first_chunk"]), _ptr(table["wd"]),
                                 _ptr(table["lr"]), _ptr(table["ignore"]), table["wd"].numel(),
                                 _ptr(table["partial"]), float(trust_coef), float(eps), float(momentum),
                                 int(first_step), _stream()),
          "byol_lars_sgd_step", kernels=2)


def sgd_nesterov_step(table, lr_scale, momentum):
    """One Nesterov-SGD step over the tensors of `table` (lars.chunk_table plus int64 pointer tables p_ptrs / g_ptrs /
    m_ptrs and fp32 [tensors] wd / lr); tensor t's learning rate is fp32(lr[t] * lr_scale).  Zeroes the gradients."""
    check(lib.byol_sgd_nesterov_step(_ptr(table["p_ptrs"]), _ptr(table["g_ptrs"]), _ptr(table["m_ptrs"]),
                                     _ptr(table["chunk_start"]), _ptr(table["chunk_len"]), _ptr(table["chunk_tensor"]),
                                     table["chunk_start"].numel(), _ptr(table["wd"]), _ptr(table["lr"]),
                                     float(lr_scale), float(momentum), _stream()), "byol_sgd_nesterov_step")


def _ce_args(logits, labels):
    """The checks both cross-entropy entry points share: fp32 CUDA logits [R, C] with unit column stride (rows may be
    pitched, e.g. a column slice), contiguous CUDA int64 labels whose count divides R."""
    if logits.dtype != F32 or not logits.is_cuda or logits.dim() != 2 or logits.stride(1) != 1:
        raise ValueError("logits must be a CUDA fp32 matrix with unit column stride")
    if labels.dtype != torch.int64 or not labels.is_cuda or not labels.is_contiguous():
        raise ValueError("labels must be a contiguous CUDA int64 tensor")
    r, c = logits.shape
    if labels.numel() == 0 or r % labels.numel() != 0:
        raise ValueError("labels: %d entries do not tile %d rows" % (labels.numel(), r))
    return r, c


def ce_topk_fwd(logits, labels, scratch=None):
    """Softmax cross-entropy (mean) + top-1 / top-5 accuracy (%) of fp32 logits [R, C] in one launch; `labels` has R
    entries or a divisor of R (row r uses labels[r % len]: both views of a sample share its label).
    Rows may be pitched (a column slice: unit column stride, row stride >= C).
    Returns (out fp32 [3] = loss, top1, top5; row_lse fp32 [R] for the backward pass)."""
    r, c = _ce_args(logits, labels)
    dev = logits.device
    fl = torch.empty(2 * r + 3, dtype=F32, device=dev)            # row_lse | row_loss | out
    it = torch.zeros(r + 1, dtype=torch.int32, device=dev)        # row_rank | ticket (must start at 0)
    check(lib.byol_ce_topk_fwd(_ptr(logits), _ptr(labels), labels.numel(), r, c, logits.stride(0), _ptr(fl), _ptr(fl[r:]), _ptr(it),
                               _ptr(it[r:]), _ptr(fl[2 * r:]), _stream()), "byol_ce_topk_fwd")
    return fl[2 * r:], fl[:r]


def ce_bwd(logits, labels, row_lse, grad_out):
    """dlogits fp32 [R, C] (contiguous) = grad_out / R * (softmax - onehot) from ce_topk_fwd's row_lse; the same
    logits / labels checks as ce_topk_fwd."""
    r, c = _ce_args(logits, labels)
    _chk(row_lse, F32, "row_lse"); _chk(grad_out, F32, "grad_out")
    if row_lse.numel() != r:
        raise ValueError("row_lse: %d entries for %d rows" % (row_lse.numel(), r))
    d = torch.empty((r, c), dtype=F32, device=logits.device)
    check(lib.byol_ce_bwd(_ptr(logits), _ptr(labels), labels.numel(), _ptr(row_lse), _ptr(grad_out), r, c, logits.stride(0), _ptr(d), c,
                          _stream()), "byol_ce_bwd")
    return d


# ------------------------------------------------------------------------------------------------
# fp32-accurate forward path ("split-bf16"; csrc/split.cu)
# ------------------------------------------------------------------------------------------------
F64 = torch.float64


def split_planes(x2d, T, cpad=None, want_copy=False, copy_out=None):
    """fp32 [M, C] (unit column stride) -> bf16 planes [M, T*cpad] (+ the plane x0 [M, C]: the bf16 rounding, saturated
    at the largest finite bf16)."""
    if x2d.dtype != F32 or not x2d.is_cuda or x2d.stride(-1) != 1:
        raise ValueError("split_planes: need a CUDA fp32 matrix with unit column stride")
    m, c = x2d.shape
    cpad = cpad or c
    planes = torch.empty((m, T * cpad), dtype=BF16, device=x2d.device)
    copy = copy_out if copy_out is not None else \
        (torch.empty((m, c), dtype=BF16, device=x2d.device) if want_copy else None)
    _chk(copy, BF16, "copy_out")
    check(lib.byol_split_planes(_ptr(x2d), _ptr(planes), _ptr(copy), m, c, cpad, x2d.stride(0), T, _stream()),
          "byol_split_planes")
    return planes, copy


def nchw_to_planes(x, T, cpad=8, out=None):
    """fp32 NCHW [N, C<=cpad, H, W] -> bf16 NHWC planes [N, H, W, T*cpad]."""
    _chk(x, F32, "x")
    n, c, h, w = x.shape
    if out is None:
        out = torch.empty((n, h, w, T * cpad), dtype=BF16, device=x.device)
    check(lib.byol_nchw_to_planes(_ptr(x), _ptr(out), n, c, h, w, cpad, T, _stream()), "byol_nchw_to_planes")
    return out


def prep_weight_planes(w, T, cpad, out):
    """fp32 [Cout, Cin, KH, KW] / [out, in] -> bf16 [Cout, taps*T*cpad] with the weight-side plane pattern."""
    _chk(w, F32, "w")
    cout, cin = w.shape[0], w.shape[1]
    taps = w.numel() // (cout * cin)
    check(lib.byol_prep_weight_planes(_ptr(w), _ptr(out), cout, cin, cpad, taps, T, _stream()),
          "byol_prep_weight_planes")
    return out


def stats_f32(y2d, stats64):
    """stats64 (zeroed fp64 [2C]) += [column sums, column sums of squares] of the fp32 matrix y2d."""
    _chk(y2d, F32, "y"); _chk(stats64, F64, "stats")
    m, c = y2d.shape
    check(lib.byol_stats_f32(_ptr(y2d), _ptr(stats64), m, c, _stream()), "byol_stats_f32")
    return stats64


def bn_finalize_lanes_f64(stats64, count, gammas, betas, running_mean, running_var, momentum, eps, coeffs):
    L = len(gammas)
    c = gammas[0].numel()
    g = [_ptr(t) for t in gammas] + [0] * (4 - L)
    b = [_ptr(t) for t in betas] + [0] * (4 - L)
    check(lib.byol_bn_finalize_lanes_f64(_ptr(stats64), float(count), L, g[0], b[0], g[1], b[1], g[2], b[2], g[3],
                                         b[3], _ptr(running_mean), _ptr(running_var), float(momentum), float(eps),
                                         _ptr(coeffs), c, _stream()), "byol_bn_finalize_lanes_f64")
    return coeffs


def bn_apply_f32(y2d, scale, shift, relu, T, resid=None, rscale=None, rshift=None, want_out32=False, want_planes=True,
                 want_copy=False, want_mask=False):
    """act(y*scale + shift (+ residual)) on fp32 [M, C] -> (out32, planes [M, T*C], bf16 copy, mask bits)."""
    _chk(y2d, F32, "y"); _chk(resid, F32, "resid")
    m, c = y2d.shape
    dev = y2d.device
    out32 = torch.empty((m, c), dtype=F32, device=dev) if want_out32 else None
    planes = torch.empty((m, T * c), dtype=BF16, device=dev) if want_planes else None
    copy = torch.empty((m, c), dtype=BF16, device=dev) if want_copy else None
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device=dev) if want_mask else None
    check(lib.byol_bn_apply_f32(_ptr(y2d), _ptr(scale), _ptr(shift), _ptr(resid), _ptr(rscale), _ptr(rshift),
                                _ptr(out32), _ptr(planes), _ptr(copy), _ptr(mask), m, c, int(relu), T, _stream()),
          "byol_bn_apply_f32")
    return out32, planes, copy, mask


def maxpool_f32(x, k=3, s=2, p=1, want_idx=True):
    _chk(x, F32, "x")
    n, h, w, c = x.shape
    ho, wo = conv_out_size(h, k, s, p), conv_out_size(w, k, s, p)
    y = torch.empty((n, ho, wo, c), dtype=F32, device=x.device)
    idx = torch.empty((n, ho, wo, c), dtype=torch.uint8, device=x.device) if want_idx else None
    check(lib.byol_maxpool_f32(_ptr(x), _ptr(y), _ptr(idx), n, h, w, c, k, s, p, _stream()), "byol_maxpool_f32")
    return y, idx


def avgpool_f32(x):
    _chk(x, F32, "x")
    n, h, w, c = x.shape
    y = torch.empty((n, c), dtype=F32, device=x.device)
    check(lib.byol_avgpool_f32(_ptr(x), _ptr(y), n, h * w, c, _stream()), "byol_avgpool_f32")
    return y


# ------------------------------------------------------------------------------------------------
# fp32-accurate backward path (BYOL(backward_precision="fp32"); csrc/split.cu, csrc/conv_igemm.cu)
# ------------------------------------------------------------------------------------------------
def prep_weight_dgrad_planes(w, T, out):
    """fp32 [Cout, Cin, KH, KW] / [out, in] -> bf16 [Cin, taps*T*Cout] (dgrad layout, weight-side plane pattern)."""
    _chk(w, F32, "w"); _chk(out, BF16, "out")
    cout, cin = w.shape[0], w.shape[1]
    taps = w.numel() // (cout * cin)
    check(lib.byol_prep_weight_dgrad_planes(_ptr(w), _ptr(out), cout, cin, taps, T, _stream()),
          "byol_prep_weight_dgrad_planes")
    return out


def conv_dgrad_planes(dyp, wdp, h, w, kh, kw, stride, pad, T, resid=None):
    """dx[N, h, w, Cin] fp32 = conv_transpose(dY, W) (+ resid, fp32 [N, h, w, Cin]).
    dyp: bf16 planes [N, Ho, Wo, T*Cout]; wdp: [Cin, taps*T*Cout] from prep_weight_dgrad_planes."""
    _chk(dyp, BF16, "dy"); _chk(wdp, BF16, "wd"); _chk(resid, F32, "resid")
    n, ho, wo, tc = dyp.shape
    cin = wdp.shape[0]
    dx = torch.empty((n, h, w, cin), dtype=F32, device=dyp.device)
    check(lib.byol_conv_dgrad_planes(_ptr(dyp), _ptr(wdp), _ptr(dx), _ptr(resid), n, ho, wo, tc // T, h, w, cin, kh, kw,
                                     stride, pad, T, _stream()), "byol_conv_dgrad_planes")
    return dx


def linear_dgrad_planes(dyp, wdp, T):
    m, tn = dyp.shape
    return conv_dgrad_planes(dyp.view(m, 1, 1, tn), wdp, 1, 1, 1, 1, 1, 0, T).view(m, -1)


def conv_wgrad_planes(xp, dyp, dw, kh, kw, stride, pad, T):
    """dw[Cout, Cin, KH, KW] (fp32) += dY^T * im2col(X) over the T product terms.  xp: bf16 planes [N, H, W, T*C]
    (C >= Cin, a multiple of 8); dyp: bf16 planes [N, Ho, Wo, T*ldy] (ldy >= Cout, a multiple of 8)."""
    _chk(xp, BF16, "x"); _chk(dyp, BF16, "dy"); _chk(dw, F32, "dw")
    n, h, w, tc = xp.shape
    _, ho, wo, tl = dyp.shape
    check(lib.byol_conv_wgrad_planes(_ptr(xp), _ptr(dyp), _ptr(dw), n, h, w, tc // T, dw.shape[1], ho, wo, dw.shape[0],
                                     tl // T, kh, kw, stride, pad, T, _stream()), "byol_conv_wgrad_planes")
    return dw


def bn_bwd_reduce_f32(g, y, coeffs, s12, mask_mode, mask=None):
    """s12 (zeroed fp64 [2C]) += [sum dz, sum dz*xhat] of fp32 g, y [M, C]; mask_mode 1: dz = g where
    y*scale + shift > 0, 3: where the bits of `mask` (bn_apply_f32) are set."""
    _chk(g, F32, "g"); _chk(y, F32, "y"); _chk(s12, F64, "s12"); _chk(mask, torch.uint8, "mask")
    m, c = y.shape
    check(lib.byol_bn_bwd_reduce_f32(_ptr(g), _ptr(y), _ptr(mask), _ptr(coeffs[0]), _ptr(coeffs[1]), _ptr(coeffs[2]),
                                     _ptr(coeffs[3]), _ptr(s12), m, c, mask_mode, _stream()), "byol_bn_bwd_reduce_f32")
    return s12


def bn_bwd_apply_f32(g, y, coeffs, gamma, s12, count, mask_mode, T, mask=None, want_planes=True, want_f32=False,
                     want_dz=False, s12_local=None, dgamma=None, dbeta=None):
    """dy = gamma*invstd*(dz - s1/n - xhat*s2/n) of fp32 [M, C] -> (planes bf16 [M, T*C] | None, fp32 dy | None,
    fp32 dz | None); dgamma / dbeta += the rank-local sums (s12_local, default s12)."""
    _chk(g, F32, "g"); _chk(y, F32, "y"); _chk(s12, F64, "s12"); _chk(mask, torch.uint8, "mask")
    m, c = y.shape
    dev = y.device
    planes = torch.empty((m, T * c), dtype=BF16, device=dev) if want_planes else None
    dy32 = torch.empty((m, c), dtype=F32, device=dev) if want_f32 else None
    dz = torch.empty((m, c), dtype=F32, device=dev) if want_dz else None
    check(lib.byol_bn_bwd_apply_f32(_ptr(g), _ptr(y), _ptr(mask), _ptr(coeffs[0]), _ptr(coeffs[1]), _ptr(coeffs[2]),
                                    _ptr(coeffs[3]), _ptr(gamma), _ptr(s12), _ptr(s12_local), float(count),
                                    _ptr(planes), _ptr(dy32), _ptr(dz), _ptr(dgamma), _ptr(dbeta), m, c, mask_mode, T,
                                    _stream()), "byol_bn_bwd_apply_f32")
    return planes, dy32, dz


def maxpool_bwd_f32(dy, idx, h, w, k=3, s=2, p=1):
    _chk(dy, F32, "dy"); _chk(idx, torch.uint8, "idx")
    n, _, _, c = dy.shape
    dx = torch.empty((n, h, w, c), dtype=F32, device=dy.device)
    check(lib.byol_maxpool_bwd_f32(_ptr(dy), _ptr(idx), _ptr(dx), n, h, w, c, k, s, p, _stream()),
          "byol_maxpool_bwd_f32")
    return dx


def avgpool_bwd_f32(ga, gb, n, h, w, c):
    """dx[n, h, w, c] fp32 = (ga + gb)[n, c] / (h*w); ga / gb fp32 [n, c], either may be None."""
    _chk(ga, F32, "ga"); _chk(gb, F32, "gb")
    dev = (ga if ga is not None else gb).device
    dx = torch.empty((n, h, w, c), dtype=F32, device=dev)
    check(lib.byol_avgpool_bwd_f32(_ptr(ga), _ptr(gb), _ptr(dx), n, h * w, c, _stream()), "byol_avgpool_bwd_f32")
    return dx
