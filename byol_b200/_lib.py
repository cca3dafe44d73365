"""ctypes loader for the C-ABI shared library ``libbyol_b200.so`` (declared in ``include/byol_b200.h``).

There is deliberately NO fallback: if the library is missing or a symbol cannot be resolved the import of
any product module fails loudly.  Build it with ``python -c "import __graft_entry__ as g; g.build()"`` (or
``make -C byol_b200/csrc``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# BYOL_B200_LIB: A/B timing of an older build of the same C ABI (tools/time_cases.py); the product path never sets it
LIB_PATH = os.environ.get("BYOL_B200_LIB") or os.path.join(_HERE, "libbyol_b200.so")

c_void_p = ctypes.c_void_p
c_int = ctypes.c_int
c_int64 = ctypes.c_int64
c_float = ctypes.c_float
c_double = ctypes.c_double

# name -> argtypes (all functions return int status unless listed in _SPECIAL)
_SIGNATURES = {
    "byol_conv_igemm": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,               # src wt dst resid resid_mask resid_up
                        c_void_p, c_void_p, c_void_p,                                          # bias col_sum col_sqsum
                        c_int, c_int, c_int, c_int, c_int, c_int, c_int,                      # Nimg Hs Ws C Ho Wo Ndim
                        c_int, c_int, c_int, c_int, c_int, c_int, c_int,                      # KH KW stride pad mode ldw ldc
                        c_int, c_int, c_int, c_void_p],                                        # out_fp32 relu force_gather stream
    "byol_stem4_supported": [c_int, c_int, c_int, c_int, c_int, c_int, c_int],
    "byol_stem4_row_pixels": [],
    "byol_nchw_to_stem4": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_prep_weight_stem4": [c_void_p, c_void_p, c_int, c_void_p],
    "byol_stem_conv_fprop": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "byol_stem_conv_wgrad": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_conv_wgrad": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                        c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_bn_stats": [c_void_p, c_void_p, c_int, c_int, c_void_p],
    "byol_bn_finalize_lanes": [c_void_p, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                               c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_void_p, c_int, c_void_p],
    "byol_bn_eval_coeffs": [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_int, c_void_p],
    "byol_bn_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                      c_int, c_int, c_int, c_void_p],
    "byol_bn_bwd_reduce": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_int, c_int, c_void_p],
    "byol_bn_bwd_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_double, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "byol_col_sum": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_nchw_to_nhwc8": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_prep_weight": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_prep_weight_fold": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_prep_unit_blocks": [c_int, c_int, c_int, c_int, c_int],
    "byol_prep_weights_multi": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p],
    # grouped 3x3 convolutions (ResNeXt)
    "byol_prep_weights_grouped": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p],
    "byol_conv_fprop_grouped": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_conv_dgrad_grouped": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_void_p],
    "byol_conv_wgrad_grouped": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                                c_int, c_int, c_int, c_void_p],
    "byol_subsample2": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_cast_f32_bf16": [c_void_p, c_void_p, c_int64, c_void_p],
    "byol_cast_f32_bf16_2d": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_maxpool_fwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_bn_relu_maxpool_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                 c_int, c_int, c_void_p],
    "byol_maxpool_bwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_avgpool_fwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "byol_avgpool_bwd": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "byol_loss_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p],
    "byol_loss_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                      c_void_p],
    "byol_loss_rows_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "byol_loss_rows_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_int, c_void_p],
    "byol_ema_update": [c_void_p, c_void_p, c_float, c_float, c_int64, c_void_p],
    "byol_lars_sgd_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                           c_void_p, c_void_p, c_int, c_void_p, c_float, c_float, c_float, c_int, c_void_p],
    "byol_sgd_nesterov_step": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                               c_float, c_float, c_void_p],
    "byol_ce_topk_fwd": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                         c_void_p],
    "byol_ce_bwd": [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p],
    # fp32-accurate ("split-bf16") forward path, csrc/split.cu
    "byol_split_planes": [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p],
    "byol_nchw_to_planes": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_prep_weight_planes": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_stats_f32": [c_void_p, c_void_p, c_int64, c_int, c_void_p],
    "byol_bn_finalize_lanes_f64": [c_void_p, c_double, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                   c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_void_p, c_int,
                                   c_void_p],
    "byol_bn_apply_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_void_p, c_int64, c_int, c_int, c_int, c_void_p],
    "byol_maxpool_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_avgpool_f32": [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    # fp32-accurate backward path
    "byol_prep_weight_dgrad_planes": [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_conv_dgrad_planes": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_conv_wgrad_planes": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int,
                               c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_bn_bwd_reduce_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                               c_int, c_int, c_void_p],
    "byol_bn_bwd_apply_f32": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                              c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int,
                              c_int, c_void_p],
    "byol_maxpool_bwd_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_avgpool_bwd_f32": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "byol_mlp_fused_supported": [c_int, c_int, c_int, c_int],
    "byol_mlp_fused_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_void_p, c_float, c_float, c_double, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int64, c_void_p,
                           c_void_p],
    "byol_augment_record_floats": [],
    "byol_augment_params": [c_void_p, c_int, c_int, c_int, ctypes.c_uint64, ctypes.c_uint64, c_float, c_float, c_float,
                            c_float, c_float, c_void_p],
    "byol_augment_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_augment_params_ragged": [c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_uint64, ctypes.c_uint64, c_float,
                                   c_float, c_float, c_float, c_float, c_void_p],
    "byol_augment_apply_ragged": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p],
    "byol_augment_params_recipe": [c_void_p, c_int, c_int, c_int, ctypes.c_uint64, ctypes.c_uint64, c_float,
                                   c_void_p, c_void_p],
    "byol_augment_params_ragged_recipe": [c_void_p, c_void_p, c_int, c_int, c_int, ctypes.c_uint64, ctypes.c_uint64,
                                          c_float, c_void_p, c_void_p],
    "byol_xchg_layout": [c_void_p, c_void_p, c_void_p],
    "byol_xchg_sum": [c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p],
    # k-NN evaluation, csrc/knn.cu
    "byol_l2_normalize_rows": [c_void_p, c_void_p, c_int64, c_int, c_int64, c_void_p],
    "byol_knn_topk": [c_void_p, c_int, c_int, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p],
    "byol_knn_vote": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p],
    # linear evaluation, csrc/linear_eval.cu
    "byol_linprobe_ce": [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p,
                         c_void_p],
    "byol_linprobe_sgd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_float, c_int, c_int,
                          c_int, c_int, c_void_p],
    # transfer linear evaluation, csrc/logreg.cu
    "byol_logreg_vec_blocks": [c_int, c_int],
    "byol_logreg_ce": [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_double, c_void_p, c_void_p, c_void_p,
                       c_void_p, c_void_p, c_void_p],
    "byol_logreg_grad": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                         c_void_p, c_void_p, c_int, c_void_p],
    "byol_logreg_dots": [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p,
                         c_int, c_void_p],
    "byol_logreg_accept": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p],
    "byol_logreg_twoloop": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                            c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p],
    "byol_logreg_trial": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p],
    # GroupNorm and weight standardisation, csrc/groupnorm.cu
    "byol_ws_fwd": [c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p, c_void_p],
    "byol_ws_bwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int64, c_void_p, c_void_p],
    "byol_gn_stats": [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p],
    "byol_gn_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                      c_void_p, c_int, c_int, c_int, c_int, c_void_p],
    "byol_gn_relu_maxpool_fwd": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int,
                                 c_int, c_int, c_int, c_int, c_void_p],
    "byol_gn_bwd_reduce": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                           c_int, c_int, c_int, c_int, c_void_p],
    "byol_gn_bwd_apply": [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                          c_int, c_int, c_int, c_int, c_void_p],
    "byol_abi_version": [],
    "byol_device_sm_count": [],
}



class AugmentRecipe(ctypes.Structure):
    """``byol_augment_recipe_t``"""
    _fields_ = [("jitter", c_float * 4), ("p_flip", c_float), ("p_jitter", c_float), ("p_gray", c_float),
                ("p_blur", c_float * 2), ("p_solarize", c_float * 2), ("bicubic", c_int)]


EXPORTED_SYMBOLS = sorted(list(_SIGNATURES.keys()) + ["byol_last_error"])


class ByolLibraryError(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "byol_b200: %s not found. The CUDA extension is mandatory (no CPU / PyTorch fallback exists). "
            "Build it with `python -c 'import __graft_entry__ as g; g.build()'` from the repository root." % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, argtypes in _SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is missing: loud by design
        fn.argtypes = argtypes
        fn.restype = c_int
    lib.byol_last_error.argtypes = []
    lib.byol_last_error.restype = ctypes.c_char_p
    return lib


lib = _load()


def last_error():
    return lib.byol_last_error().decode("utf-8", "replace")


# number of byol_b200 CUDA kernels launched through the C-ABI since import (bench.py reports the per-step count)
launch_count = [0]


def check(status, what, kernels=1):
    if status != 0:
        raise ByolLibraryError("%s failed (status %d): %s" % (what, status, last_error()))
    launch_count[0] += kernels
