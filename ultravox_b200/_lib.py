"""ctypes binding of ``libuvx.so`` (the C ABI in ``include/uvx.h``).

The library is built in-tree by ``__graft_entry__.build()`` (``make -C ultravox_b200/csrc``).  There is no
fallback: if the shared object is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
import os
import pathlib

_HERE = pathlib.Path(__file__).resolve().parent
LIB_PATH = _HERE / "libuvx.so"

c_i64, c_i32, c_f32, c_vp, c_sz = C.c_int64, C.c_int32, C.c_float, C.c_void_p, C.c_size_t


class GemmArgs(C.Structure):
    """``struct uvx_gemm_args`` (include/uvx.h)."""
    _fields_ = [("A", c_vp), ("a_batch", c_i64), ("a_rows", c_i64), ("K", c_i64), ("a_row_stride", c_i64),
                ("a_batch_stride", c_i64), ("W", c_vp), ("N", c_i64), ("w_row_stride", c_i64), ("C", c_vp),
                ("c_row_stride", c_i64), ("c_batch_rows", c_i64), ("c_row_offset", c_i64), ("c_row_map", c_vp),
                ("bias", c_vp), ("R", c_vp), ("r_row_stride", c_i64), ("r_batch_stride", c_i64), ("alpha", c_f32),
                ("act", c_i32), ("out_dtype", c_i32), ("workspace", c_vp), ("workspace_bytes", c_i64),
                ("norm_w", c_vp), ("norm_out", c_vp), ("norm_eps", c_f32), ("w_tiled", c_i32), ("rope_cols", c_i32),
                ("rope_cos", c_vp), ("rope_sin", c_vp), ("rope_positions", c_vp), ("rope_rows_per_seq", c_i64),
                ("rope_pos_offset", c_i64), ("flags", c_i32), ("w_perm", c_i32)]


class AttnArgs(C.Structure):
    """``struct uvx_attn_args`` (include/uvx.h)."""
    _fields_ = [("q", c_vp), ("k", c_vp), ("v", c_vp), ("o", c_vp), ("B", c_i64), ("Hq", c_i64), ("Hkv", c_i64),
                ("Sq", c_i64), ("Skv", c_i64), ("D", c_i64), ("q_rs", c_i64), ("q_bs", c_i64), ("k_rs", c_i64),
                ("k_bs", c_i64), ("v_rs", c_i64), ("v_bs", c_i64), ("o_rs", c_i64), ("o_bs", c_i64), ("kv_len", c_vp),
                ("causal", c_i32), ("block", c_i32), ("scale", c_f32), ("lse", c_vp), ("kv_start", c_vp)]


TL_MAX = 8                 # UVX_TL_MAX
NORM_WS_BYTES = 8 * 1024 + 8   # UVX_NORM_WS_BYTES


class TensorList(C.Structure):
    """``struct uvx_tensor_list`` (include/uvx.h)."""
    _fields_ = [("count", c_i64), ("numel", c_i64 * TL_MAX), ("g", c_vp * TL_MAX), ("acc", c_vp * TL_MAX), ("p", c_vp * TL_MAX),
                ("m", c_vp * TL_MAX), ("v", c_vp * TL_MAX)]


# name -> (restype, argtypes); must list every symbol include/uvx.h declares (tests check this)
SIGNATURES = {
    "uvx_abi_version": (C.c_int, []),
    "uvx_last_error": (C.c_char_p, []),
    "uvx_launch_count": (c_i64, []),
    "uvx_logmel_workspace": (c_sz, [c_i64, c_i64, C.c_int]),
    "uvx_logmel": (C.c_int, [c_vp, c_i64, c_i64, C.c_int, c_vp, c_vp, c_vp, c_sz, c_vp]),
    "uvx_debug_mel_filters": (C.c_int, [C.c_int, c_vp]),
    "uvx_mel_to_timemajor": (C.c_int, [c_vp, c_i64, C.c_int, c_i64, c_vp, c_vp]),
    "uvx_gemm_bf16": (C.c_int, [C.POINTER(GemmArgs), c_vp]),
    "uvx_debug_gemm_override": (C.c_int, [C.c_int, C.c_int]),
    "uvx_debug_gemm_cluster": (C.c_int, [C.c_int, C.c_int]),
    "uvx_debug_gemm_mode": (C.c_int, [C.c_int]),
    "uvx_debug_gemm_pf": (C.c_int, [C.c_int]),
    "uvx_debug_gemm_stages": (C.c_int, [C.c_int]),
    "uvx_debug_gemm_times": (C.c_int, [c_vp]),
    "uvx_debug_gemm_tma_store": (C.c_int, [C.c_int]),
    "uvx_debug_gemm_split_ring": (C.c_int, [C.c_int]),
    "uvx_debug_gemm_ws": (C.c_int, [C.c_int, C.c_int, C.c_int]),
    "uvx_debug_gemm_ws_times": (C.c_int, [C.c_void_p]),
    "uvx_tile_weight": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i32, c_i32, c_vp, c_vp]),
    "uvx_layernorm": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_f32, c_vp]),
    "uvx_rmsnorm": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f32, c_vp]),
    "uvx_attention": (C.c_int, [C.POINTER(AttnArgs), c_vp]),
    "uvx_debug_attn_tc": (C.c_int, [C.c_int]),
    "uvx_attention_enc_tc": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_vp, c_i64, c_vp, c_i32, c_f32, c_vp]),
    "uvx_attention_indexed": (C.c_int, [C.POINTER(AttnArgs), c_i64, c_vp, c_vp, c_vp]),
    "uvx_attention_paged": (C.c_int, [C.POINTER(AttnArgs), c_vp, c_i64, c_vp]),
    "uvx_attention_indexed_paged": (C.c_int, [C.POINTER(AttnArgs), c_i64, c_vp, c_i64, c_vp, c_vp, c_vp]),
    "uvx_kv_page_map": (C.c_int, [c_vp, c_i64, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "uvx_kv_pages_copy": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_i64, c_i32, c_vp]),
    "uvx_rope": (C.c_int, [c_vp, c_i64, c_i64, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "uvx_swiglu": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, C.c_int, c_vp]),
    "uvx_splice_plan": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp]),
    "uvx_embed_splice": (C.c_int, [c_vp, c_vp, c_i64, c_vp, c_vp, c_i64, c_i64, c_vp, c_vp]),
    "uvx_lm_head": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_vp, c_vp]),
    "uvx_gemv_bf16": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, C.c_int, c_vp]),
    "uvx_kv_append": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_vp, c_i64, c_vp]),
    "uvx_gemv_fused_bf16": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_vp, c_i64, C.c_int, c_vp, C.c_float,
                                      C.c_int, c_vp]),
    "uvx_rope_kv_append": (C.c_int, [c_vp, c_i64, c_i64, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "uvx_rope_kv_append_map": (C.c_int, [c_vp, c_i64, c_i64, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp,
                                         c_vp]),
    "uvx_add_i32": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_vp]),
    "uvx_kv_write": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_i64, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_vp]),
    "uvx_repetition_penalty": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_f32, c_vp, c_vp]),
    "uvx_sample": (C.c_int, [c_vp, c_i64, c_i64, c_f32, c_i32, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "uvx_sample_top_p": (C.c_int, [c_vp, c_i64, c_i64, c_f32, c_i32, c_f32, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "uvx_token_finish": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "uvx_sample_slots": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp]),
    "uvx_repetition_penalty_slots": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "uvx_slot_finish": (C.c_int, [c_vp, c_vp, c_vp, c_i32, c_vp, c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp]),
    "uvx_log_softmax": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_vp]),
    "uvx_beam_select": (C.c_int, [c_vp, c_i64, c_i32, c_i64, c_vp, c_i32, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "uvx_beam_update": (C.c_int, [c_vp, c_vp, c_i64, c_i32, c_i32, c_i64, c_vp, c_i32, c_i32, c_vp, c_i32, c_i32, c_vp, c_vp, c_vp,
                                  c_i64, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp,
                                  c_vp]),
    "uvx_kv_reorder": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_i32, c_i64, c_i64, c_vp, c_vp, c_vp]),
    "uvx_argmax": (C.c_int, [c_vp, c_i64, c_i64, c_vp, c_vp]),
    "uvx_rope_bwd": (C.c_int, [c_vp, c_i64, c_i64, C.c_int, C.c_int, C.c_int, c_vp, c_vp, c_vp, c_i64, c_i64, c_vp]),
    "uvx_attention_bwd": (C.c_int, [C.POINTER(AttnArgs), c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64,
                                    c_vp, c_vp]),
    "uvx_transpose_bf16": (C.c_int, [c_vp, c_i64, c_i64, c_i64, c_vp, c_i64, c_vp]),
    "uvx_rmsnorm_bwd": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, c_i64, c_i64, c_i64, c_f32, c_vp]),
    "uvx_swiglu_bwd": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_i64, c_i64, C.c_int, c_vp]),
    "uvx_layernorm_bwd": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_vp, c_i64, c_i64, C.c_float, c_vp]),
    "uvx_gelu": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "uvx_gelu_bwd": (C.c_int, [c_vp, c_vp, c_vp, c_i64, c_vp]),
    "uvx_ce_bwd": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_i64, C.c_int, c_vp, c_vp, c_f32, c_vp, c_vp]),
    "uvx_gather_rows": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_vp, c_vp]),
    "uvx_splice_inverse": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_vp]),
    "uvx_adamw": (C.c_int, [c_vp, c_vp, c_vp, c_vp, c_i64, c_f32, c_f32, c_f32, c_f32, c_f32, c_i64, c_f32, c_vp]),
    "uvx_cast_f32_bf16": (C.c_int, [c_vp, c_vp, c_i64, c_vp]),
    "uvx_grad_norm_clip": (C.c_int, [C.POINTER(TensorList), c_vp, c_f32, c_vp, c_vp, c_vp, c_vp, c_i64, c_vp, c_vp]),
    "uvx_adamw_multi": (C.c_int, [C.POINTER(TensorList), c_vp, c_vp, c_vp, c_vp, C.c_double, C.c_double, C.c_double, C.c_double,
                                  c_vp]),
    "uvx_grad_accumulate": (C.c_int, [C.POINTER(TensorList), c_i32, c_vp]),
    "uvx_kl_loss": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_f32, c_vp, c_vp, c_vp, c_vp, c_vp, c_vp]),
    "uvx_kl_bwd": (C.c_int, [c_vp, c_vp, c_i64, c_i64, c_i64, c_f32, c_vp, c_vp, c_vp, c_f32, c_vp, c_vp]),
    "uvx_ce_loss": (C.c_int, [c_vp, c_i64, c_vp, c_i64, c_i64, c_i64, c_i64, C.c_int, c_vp, c_vp, c_vp, c_vp]),
}

_lib = None


class UvxError(RuntimeError):
    pass


def lib() -> C.CDLL:
    """Load (once) and return the library; raises if it has not been built."""
    global _lib
    if _lib is None:
        path = os.environ.get("UVX_LIB", str(LIB_PATH))
        if not os.path.exists(path):
            raise UvxError(f"{path} not found - run `python -c 'import __graft_entry__ as g; g.build()'` "
                           "(nvcc, sm_90a).  ultravox_b200 has no CPU / PyTorch fallback.")
        handle = C.CDLL(path)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(handle, name)
            fn.restype, fn.argtypes = res, args
        if handle.uvx_abi_version() != 1:
            raise UvxError("libuvx ABI version mismatch")
        _lib = handle
    return _lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = lib().uvx_last_error().decode("utf-8", "replace")
        raise UvxError(f"{what or 'libuvx'} failed (code {rc}): {msg}")


def launch_count() -> int:
    return int(lib().uvx_launch_count())
