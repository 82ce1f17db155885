"""ctypes binding of libvjepa_b200.so (the C ABI declared in include/vjepa_b200.h).

There is no CPU fallback: if the library is missing or a call fails the caller gets an exception.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_longlong, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libvjepa_b200.so")

P, I, L, F, Z = c_void_p, c_int, c_longlong, c_float, c_size_t

# name -> (restype, argtypes); must list every symbol include/vjepa_b200.h declares
SIGNATURES = {
    "vj_last_error_string": (c_char_p, []),
    "vj_version": (I, []),
    "vj_launch_count": (L, []),
    "vj_tmap_cache_stats": (L, [I]),
    "vj_set_sm_limit": (I, [I]),
    "vj_clip_preprocess": (I, [P, P, P, I, I, I, I, P, P, P]),
    "vj_clip_views": (I, [P, P, P, P, I, I, I, I, P, P, P]),
    "vj_clip_augment": (I, [P, P, P, P, P, P, I, P, I, I, I, I, P, P, P]),
    "vj_image_views": (I, [P, P, P, P, P, I, I, I, P, P, P]),
    "vj_image_augment": (I, [P, P, P, P, P, P, P, P, P, P, I, P, P, I, I, I, P, P, P, P]),
    "vj_gemm": (I, [P, L, I, P, L, I, P, L, I, I, I, I, P, F, I, P, L, I, P, I, P, L, I, I, P]),
    "vj_gemm_f16": (I, [P, L, I, P, L, I, P, L, I, I, I, I, P, F, I, P, L, I, P, I, P, L, I, I, P]),
    "vj_attn_fwd": (I, [P, P, P, P, I, I, I, I, I, F, P]),
    "vj_attn_fwd_f16": (I, [P, P, P, P, I, I, I, I, I, F, P]),
    "vj_attn_bwd": (I, [P, P, P, P, P, P, P, P, I, I, I, I, I, F, P]),
    "vj_layernorm_fwd": (I, [P, I, P, I, P, P, P, P, I, I, F, P]),
    "vj_layernorm_bwd_workspace": (Z, [I, I]),
    "vj_layernorm_bwd": (I, [P, P, I, P, P, P, P, P, P, P, P, Z, I, I, P]),
    "vj_layernorm_bwd_f16": (I, [P, P, P, P, P, P, P, P, P, P, Z, I, I, P]),
    "vj_colsum": (I, [P, I, P, L, I, L, I, I, I, P]),
    "vj_colsum_f16": (I, [P, P, L, I, L, I, I, I, P]),
    "vj_im2col_tubelets": (I, [P, P, P, I, I, I, I, I, I, I, I, P]),
    "vj_im2col_tubelets_f16": (I, [P, P, P, I, I, I, I, I, I, I, I, P]),
    "vj_pos_interp": (I, [P, P, I, I, I, I, I, I, I, c_double, c_double, c_double, I, P]),
    "vj_gather_rows": (I, [P, P, P, I, I, I, I, P]),
    "vj_scatter_rows_add": (I, [P, P, P, I, I, I, I, I, P]),
    "vj_target_ln_gather": (I, [P, P, P, P, P, I, I, I, I, F, F, P]),
    "vj_pred_assemble_fwd": (I, [P, P, P, P, P, P, I, I, I, I, I, P]),
    "vj_pred_assemble_bwd": (I, [P, I, P, P, I, I, I, I, P]),
    "vj_seq_slice": (I, [P, P, I, I, I, I, I, I, I, P]),
    "vj_l1_loss_fwd": (I, [P, P, P, L, F, P]),
    "vj_l1_loss_bwd": (I, [P, P, P, F, P, L, P]),
    "vj_token_std_accum": (I, [P, P, I, I, I, F, F, P]),
    "vj_lp_loss_fwd": (I, [P, P, P, L, F, F, P]),
    "vj_lp_loss_bwd": (I, [P, P, P, F, P, L, F, P]),
    "vj_cross_attn_fwd": (I, [P, P, P, I, I, I, I, I, F, P]),
    "vj_cross_attn_fwd_lse": (I, [P, P, P, P, I, I, I, I, I, F, P]),
    "vj_cross_attn_bwd_workspace": (Z, [I, I, I, I, I]),
    "vj_cross_attn_bwd": (I, [P, P, P, P, P, P, P, P, Z, I, I, I, I, I, F, P]),
    "vj_cross_attn_fwd_f16": (I, [P, P, P, I, I, I, I, I, F, P]),
    "vj_cross_attn_fwd_lse_f16": (I, [P, P, P, P, I, I, I, I, I, F, P]),
    "vj_cross_attn_bwd_f16": (I, [P, P, P, P, P, P, P, P, Z, I, I, I, I, I, F, P]),
    "vj_token_std_bwd": (I, [P, P, P, F, P, I, I, I, F, F, P]),
    "vj_cast_f32_bf16": (I, [P, P, L, P]),
    "vj_cast_f32_f16": (I, [P, P, L, P]),
    "vj_head_pad": (I, [P, I, P, I, L, I, I, I, L, I, P]),
    "vj_ema_update": (I, [P, P, L, F, F, P]),
    "vj_adamw_step": (I, [P, P, P, P, L, F, F, F, F, F, I, P, P, P]),
    "vj_adamw_flat": (I, [P, P, P, P, P, L, P, P, F, F, F, I, P, P, P, P, P]),
    "vj_ema_update_shadow": (I, [P, P, L, F, F, P, P]),
    "vj_grad_unscale_stats": (I, [P, P, L, P, P, P, I, P]),
    "vj_seg_abs_sum": (I, [P, P, L, P, P]),
    "vj_clip_coef": (I, [P, I, F, P, P, P]),
    "vj_scale_flat": (I, [P, L, P, P]),
    "vj_sumsq": (I, [P, L, P, P]),
}

_lib = None


class VJError(RuntimeError):
    pass


def load():
    """Load the shared library (once) and attach prototypes.  Raises if it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise VJError(
                f"{LIB_PATH} is not built; run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the hot path)")
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def call(name, *args):
    """Invoke an int-returning entry point; translate non-zero codes into exceptions."""
    lib = load()
    rc = getattr(lib, name)(*args)
    if rc != 0:
        msg = lib.vj_last_error_string()
        raise VJError(f"{name} failed (rc={rc}): {msg.decode() if msg else '?'}")
    return rc
