"""ctypes binding of libgligen_b200.so (include/gligen_b200.h).  No torch types cross this boundary:
only raw device pointers, sizes and a stream handle.

The product path fails loudly when the library is missing: there is NO CPU or PyTorch fallback.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libgligen_b200.so")

c_void_p, c_int, c_int64, c_float = C.c_void_p, C.c_int32, C.c_int64, C.c_float


class GlgGemmArgs(C.Structure):
    _fields_ = [
        ("A", c_void_p), ("lda", c_int64), ("W", c_void_p), ("out", c_void_p), ("ldc", c_int64),
        ("M", c_int), ("N", c_int), ("K", c_int), ("out_fp32", c_int),
        ("bias", c_void_p), ("rowbias", c_void_p), ("ld_rowbias", c_int64), ("rows_per_batch", c_int),
        ("act", c_int), ("gate", c_void_p), ("residual", c_void_p), ("ldr", c_int64),
        ("geglu", c_int), ("conv_mode", c_int), ("H", c_int), ("Wd", c_int), ("Bn", c_int),
        ("ln_stats", c_void_p), ("ln_colsum", c_void_p), ("ln_slots", c_int), ("ln_eps", c_float),
        ("stats_out", c_void_p), ("stats_slots", c_int), ("out_rows_per_batch", c_int), ("out_batch_stride", c_int64),
        ("splitk_ws", c_void_p), ("splitk_ws_bytes", c_int64),
        ("ln_slot_stride", c_int64), ("stats_slot_stride", c_int64),
    ]


class GlgAttnArgs(C.Structure):
    _fields_ = [
        ("q", c_void_p), ("k", c_void_p), ("v", c_void_p), ("out", c_void_p),
        ("q_row", c_int64), ("k_row", c_int64), ("v_row", c_int64), ("o_row", c_int64),
        ("q_batch", c_int64), ("k_batch", c_int64), ("v_batch", c_int64), ("o_batch", c_int64),
        ("B", c_int), ("heads", c_int), ("d_head", c_int), ("Lq", c_int), ("Lk", c_int),
        ("scale", c_float), ("causal", c_int),
    ]


# name -> (restype, argtypes); every symbol include/gligen_b200.h declares
SIGNATURES = {
    "glg_abi_version": (c_int, []),
    "glg_last_error": (C.c_char_p, []),
    "glg_launch_count": (c_int64, []),
    "glg_reset_launch_count": (None, []),
    "glg_gemm": (c_int, [C.POINTER(GlgGemmArgs), c_void_p]),
    "glg_attention": (c_int, [C.POINTER(GlgAttnArgs), c_void_p]),
    "glg_groupnorm": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p,
                              c_int, c_int, c_int, c_int, c_float, c_int, c_void_p]),
    "glg_layernorm": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_int, c_int, c_float, c_void_p]),
    "glg_conv_in": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_conv_out": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_upsample2x": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_im2col_s2": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_im2col_s2_pad": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_copy_rows": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int, c_void_p]),
    "glg_timestep_embedding": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "glg_timestep_embedding_f32": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "glg_position_features": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                      c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_cast_f32_bf16": (c_int, [c_void_p, c_void_p, c_int64, c_void_p]),
    "glg_softmax_rows": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int, c_float, c_void_p]),
    "glg_patchify_nchw": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_patchify_nhwc": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_layernorm_rows": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_float, c_void_p]),
    "glg_layernorm_rows_f32": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_float, c_void_p]),
    "glg_embed_tokens": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "glg_clip_vision_embed": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_float, c_void_p]),
    "glg_clip_image_head": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                                    c_int, c_int, c_int, c_float, c_void_p]),
    "glg_dwconv7_ln": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p]),
    "glg_spatial_tokens": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_void_p]),
    "glg_resize_plane": (c_int, [c_void_p, c_int64, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_conv2d_small": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_grid_resample_gate": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p, c_int64, c_int, c_int, c_int, c_int, c_void_p]),
    "glg_engine_load": (c_int, [C.c_char_p, C.POINTER(c_void_p)]),
    "glg_engine_buffer": (c_int, [c_void_p, C.c_char_p, C.POINTER(c_void_p), C.POINTER(c_int64)]),
    "glg_engine_write": (c_int, [c_void_p, C.c_char_p, c_void_p, c_int64, c_void_p]),
    "glg_engine_read": (c_int, [c_void_p, C.c_char_p, c_void_p, c_int64, c_void_p]),
    "glg_engine_run": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "glg_engine_num_ops": (c_int64, [c_void_p]),
    "glg_engine_destroy": (c_int, [c_void_p]),
    "glg_sampler_update": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p,
                                   c_float, c_float, c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_int64, c_void_p]),
    "glg_dpm_update": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p,
                               c_float, c_float, c_float, c_float, c_float, c_float, c_void_p, c_void_p, c_int64, c_void_p]),
    "glg_unipc_update": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_float, c_float]
                         + [c_float] * 9 + [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "glg_sde_update": (c_int, [c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p]
                       + [c_float] * 7 + [c_void_p, c_void_p, c_int64, c_void_p]),
}
# not part of the public header: test hook
_DEBUG_SIGNATURES = {"glg_debug_force_bn": (None, [c_int]), "glg_debug_pick_tile": (None, [c_int, c_int, c_int, c_int, c_int, c_int, c_int64, C.POINTER(c_int)]), "glg_debug_attn_mode": (None, [c_int]), "glg_debug_attn_poly_share": (None, [c_int]), "glg_debug_gemm_cta2": (None, [c_int]), "glg_debug_splitk": (None, [c_int]), "glg_debug_gemm_bres": (None, [c_int]), "glg_debug_gemm_pp": (None, [c_int]), "glg_debug_pick_pingpong": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int64]), "glg_debug_epilogue_kind": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int64, c_int])}

_lib: Optional[C.CDLL] = None


class GligenLibraryError(RuntimeError):
    pass


def load() -> C.CDLL:
    """Load the native library (building it first when nvcc is present and sources changed)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH) or os.environ.get("GLIGEN_B200_REBUILD"):
        from . import build as _build
        _build.build()
    if not os.path.exists(LIB_PATH):
        raise GligenLibraryError(f"{LIB_PATH} is missing: run `python -m gligen_b200.build` (there is no fallback path)")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in {**SIGNATURES, **_DEBUG_SIGNATURES}.items():
        fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.glg_abi_version() != 4:
        raise GligenLibraryError(f"ABI mismatch: library reports {lib.glg_abi_version()}")
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().glg_last_error()
        raise GligenLibraryError(f"{what}: {msg.decode() if msg else 'unknown error'} (rc={rc})")
