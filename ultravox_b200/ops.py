"""Tensor-level wrappers over the C ABI (``libuvx``).  PyTorch is only the owner of device memory and of
the current stream here; every op below is a hand-written sm_90a kernel.  CUDA tensors only - there is no
CPU path (an exception is raised instead).
"""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from . import _lib
from ._lib import AttnArgs, GemmArgs, check, lib

ACT_NONE, ACT_GELU = 0, 1
BF16 = torch.bfloat16


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _cuda(t: torch.Tensor, dtype=None, name="tensor") -> torch.Tensor:
    if not t.is_cuda:
        raise _lib.UvxError(f"{name} must be a CUDA tensor (ultravox_b200 has no CPU path)")
    if dtype is not None and t.dtype != dtype:
        raise TypeError(f"{name} must be {dtype}, got {t.dtype}")
    return t


def _p(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


# ------------------------------------------------------------------------------------------ log-mel
def logmel(wave: torch.Tensor, n_mels: int, want_f32: bool = True, want_tm: bool = False,
           out_f32: Optional[torch.Tensor] = None, out_tm: Optional[torch.Tensor] = None,
           workspace: Optional[torch.Tensor] = None):
    """wave [B, L] fp32 (L % 160 == 0) -> ``audio_values`` [B, n_mels, L/160] fp32 and/or the bf16 time-major
    guard-padded layout [B, L/160 + 2, n_mels] (see include/uvx.h)."""
    _cuda(wave, torch.float32, "wave")
    wave = wave.contiguous()
    B, L = wave.shape
    T = L // 160
    if want_f32 and out_f32 is None:
        out_f32 = torch.empty(B, n_mels, T, dtype=torch.float32, device=wave.device)
    if want_tm and out_tm is None:
        out_tm = torch.empty(B, T + 2, n_mels, dtype=BF16, device=wave.device)
    need = lib().uvx_logmel_workspace(B, L, n_mels)
    if workspace is None or workspace.numel() < need:
        workspace = torch.empty(need, dtype=torch.uint8, device=wave.device)
    check(lib().uvx_logmel(wave.data_ptr(), B, L, n_mels, _p(out_f32), _p(out_tm), workspace.data_ptr(),
                           workspace.numel(), _stream()), "uvx_logmel")
    if want_f32 and want_tm:
        return out_f32, out_tm
    return out_f32 if want_f32 else out_tm


def mel_to_timemajor(audio_values: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(audio_values, torch.float32, "audio_values")
    audio_values = audio_values.contiguous()
    N, n_mels, T = audio_values.shape
    if out is None:
        out = torch.empty(N, T + 2, n_mels, dtype=BF16, device=audio_values.device)
    check(lib().uvx_mel_to_timemajor(audio_values.data_ptr(), N, n_mels, T, out.data_ptr(), _stream()),
          "uvx_mel_to_timemajor")
    return out


# ------------------------------------------------------------------------------------------ GEMM
_GEMM_WS: dict = {}
GEMM_WS_BYTES = 160 << 20


def gemm_workspace(device) -> torch.Tensor:
    """Split-K workspace of the CURRENT stream on ``device`` (fp32 partial sums; contents on entry do not matter).  One buffer per
    (device, stream): GEMMs issued on different streams - e.g. ``infer_stream``'s generation thread next to the main thread,
    ref infer.py:227-241 - never share partial sums.  Kernels recorded into CUDA graphs use one more buffer per device (graph
    replays are serialised by the engines); it is created together with the first eager workspace so that it never comes out of
    a graph's private memory pool."""
    idx = torch.device(device).index if torch.device(device).index is not None else torch.cuda.current_device()
    capturing = torch.cuda.is_current_stream_capturing()
    key = (idx, "graph") if capturing else (idx, torch.cuda.current_stream(idx).cuda_stream)
    ws = _GEMM_WS.get(key)
    if ws is None:
        with torch.cuda.device(idx):
            ws = torch.zeros(GEMM_WS_BYTES, dtype=torch.uint8, device=torch.device("cuda", idx))
            _GEMM_WS[key] = ws
            if not capturing and (idx, "graph") not in _GEMM_WS:
                _GEMM_WS[(idx, "graph")] = torch.zeros(GEMM_WS_BYTES, dtype=torch.uint8, device=torch.device("cuda", idx))
    return ws


def gemm_raw(A_ptr: int, a_batch: int, a_rows: int, K: int, a_row_stride: int, a_batch_stride: int,
             W: torch.Tensor, C_t: torch.Tensor, c_row_stride: int, c_batch_rows: int, c_row_offset: int = 0,
             c_row_map: Optional[torch.Tensor] = None, bias: Optional[torch.Tensor] = None,
             R: Optional[torch.Tensor] = None, r_row_stride: int = 0, r_batch_stride: int = 0,
             alpha: float = 1.0, act: int = ACT_NONE, norm: Optional[tuple] = None, rope: Optional[tuple] = None,
             flags: int = 0) -> None:
    a = GemmArgs()
    a.flags = flags
    a.A, a.a_batch, a.a_rows, a.K = A_ptr, a_batch, a_rows, K
    a.a_row_stride, a.a_batch_stride = a_row_stride, a_batch_stride
    a.W, a.N, a.w_row_stride = W.data_ptr(), W.shape[0], W.stride(0)
    a.C, a.c_row_stride, a.c_batch_rows, a.c_row_offset = C_t.data_ptr(), c_row_stride, c_batch_rows, c_row_offset
    a.c_row_map = _p(c_row_map)
    a.bias, a.R = _p(bias), _p(R)
    a.r_row_stride, a.r_batch_stride = r_row_stride, r_batch_stride
    a.alpha, a.act = alpha, act
    a.out_dtype = 1 if C_t.dtype == torch.float32 else 0
    ws = gemm_workspace(C_t.device)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if norm is not None:                       # (weight, eps, out): fused RMSNorm of the finished rows
        a.norm_w, a.norm_eps, a.norm_out = norm[0].data_ptr(), float(norm[1]), norm[2].data_ptr()
    if rope is not None:                       # (cos, sin, positions|None, rows_per_seq, pos_offset, rope_cols): fused RoPE, head_dim 128
        cos, sin, positions, rows_per_seq, pos_offset, rope_cols = rope
        a.rope_cos, a.rope_sin, a.rope_positions = cos.data_ptr(), sin.data_ptr(), _p(positions)
        a.rope_rows_per_seq, a.rope_pos_offset, a.rope_cols = int(rows_per_seq), int(pos_offset), int(rope_cols)
    check(lib().uvx_gemm_bf16(C.byref(a), _stream()), "uvx_gemm_bf16")


class TiledWeight:
    """Pre-tiled image of an ``nn.Linear`` weight [N, K] for the weight-streaming GEMM (include/uvx.h: ``uvx_tile_weight`` /
    ``uvx_gemm_args.w_tiled``): [ceil(N/R)][K/64][R][64] bf16, every (tile, k-block) box one contiguous R*128-byte run.
    ``swiglu``: gate and up rows of the same features share a tile (fused gate|up projection, N = 2*ffn), which is what
    ``linear_tiled(..., act=ACT_SWIGLU)`` needs to finish act(gate)*up inside the GEMM epilogue: R = 128 -> 16 gate | 16 up
    rows per 32-row quarter, other R -> 8 gate / 8 up rows alternating (gemm_tc.cu)."""

    def __init__(self, w: torch.Tensor, R: int, swiglu: bool = False, rope_pairs: bool = False):
        _cuda(w, BF16, "w")
        self.N, self.K, self.R, self.swiglu = int(w.shape[0]), int(w.shape[1]), int(R), bool(swiglu)
        self.rope_pairs = bool(rope_pairs)
        if rope_pairs and (swiglu or R != 128 or self.N % 128 != 0):
            raise ValueError("rope_pairs: a 128-row image of whole 128-wide heads")
        n_tiles = -(-self.N // R)
        self.image = torch.empty(n_tiles * (self.K // 64) * R * 64, dtype=BF16, device=w.device)
        inter = ((16 if R == 128 else 8) if swiglu else (1 if rope_pairs else 0))
        check(lib().uvx_tile_weight(w.data_ptr(), self.N, self.K, w.stride(0), R, inter, self.image.data_ptr(), _stream()), "uvx_tile_weight")

    @property
    def n_out(self) -> int:
        return self.N // 2 if self.swiglu else self.N


ACT_SWIGLU = 2
GEMM_W_STATIC = 4   # uvx_gemm_args.flags bit 2 (UVX_GEMM_W_STATIC)


def linear_tiled(x: torch.Tensor, wt: TiledWeight, out: Optional[torch.Tensor] = None, residual: Optional[torch.Tensor] = None,
                 act: int = ACT_NONE, norm: Optional[tuple] = None, rope: Optional[tuple] = None, flags: int = 0) -> torch.Tensor:
    """y = x @ W.T (+ residual) over the pre-tiled weight image; ``act=ACT_SWIGLU`` -> y = silu(gate) * up [M, N/2] (needs a
    ``swiglu`` image); ``rope=(cos, sin, positions|None, rows_per_seq, pos_offset, rope_cols)`` rotates the q / k heads in the
    epilogue (head_dim 128); ``norm`` as in ``linear``.  ``flags=GEMM_W_STATIC`` promises that no kernel still running in the
    stream writes the image (a frozen image finished before the call), so the weight stream may start before the previous
    kernel ends."""
    _cuda(x, BF16, "x")
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    M = x2.shape[0]
    n_out = wt.n_out if act == ACT_SWIGLU else wt.N
    if (act == ACT_SWIGLU) != wt.swiglu:
        raise ValueError("ACT_SWIGLU needs (and only works with) the gate|up-interleaved weight image")
    if out is None:
        out = torch.empty(*x.shape[:-1], n_out, dtype=BF16, device=x.device)
    o2 = out.view(-1, n_out)
    a = GemmArgs()
    a.A, a.a_batch, a.a_rows, a.K = x2.data_ptr(), 1, M, K
    a.a_row_stride, a.a_batch_stride = x2.stride(0), 0
    a.W, a.N, a.w_row_stride = wt.image.data_ptr(), wt.N, K
    a.C, a.c_row_stride, a.c_batch_rows, a.c_row_offset = o2.data_ptr(), o2.stride(0), M, 0
    if residual is not None:
        r2 = residual.reshape(-1, n_out)
        a.R, a.r_row_stride = r2.data_ptr(), r2.stride(0)
    a.alpha, a.act, a.out_dtype = 1.0, act, 0
    ws = gemm_workspace(out.device)
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    if norm is not None:
        a.norm_w, a.norm_eps, a.norm_out = norm[0].data_ptr(), float(norm[1]), norm[2].data_ptr()
    a.w_tiled = wt.R
    a.w_perm = 1 if wt.rope_pairs else 0
    a.flags = flags
    if rope is not None:
        cos, sin, positions, rows_per_seq, pos_offset, rope_cols = rope
        a.rope_cos, a.rope_sin, a.rope_positions = cos.data_ptr(), sin.data_ptr(), _p(positions)
        a.rope_rows_per_seq, a.rope_pos_offset, a.rope_cols = int(rows_per_seq), int(pos_offset), int(rope_cols)
    check(lib().uvx_gemm_bf16(C.byref(a), _stream()), "uvx_gemm_bf16(tiled)")
    return out


def linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor] = None, act: int = ACT_NONE,
           residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
           out_dtype=BF16, row_map: Optional[torch.Tensor] = None, alpha: float = 1.0,
           norm: Optional[tuple] = None, rope: Optional[tuple] = None, flags: int = 0) -> torch.Tensor:
    """y = act(alpha * x @ w.T + bias) + residual for x [..., K] (last dim contiguous, uniform row stride).
    ``norm=(weight, eps, out)`` additionally writes out = RMSNorm(y) (fused into the split-K reduction when possible)."""
    _cuda(x, BF16, "x"), _cuda(w, BF16, "w")
    K = x.shape[-1]
    x2 = x.reshape(-1, K)
    if x2.stride(-1) != 1:
        x2 = x2.contiguous()
    M, N = x2.shape[0], w.shape[0]
    if out is None:
        out = torch.empty(*x.shape[:-1], N, dtype=out_dtype, device=x.device)
    o2 = out.view(-1, out.shape[-1]) if row_map is None else out
    r2 = None
    if residual is not None:
        r2 = residual.reshape(-1, N)
    gemm_raw(x2.data_ptr(), 1, M, K, x2.stride(0), 0, w, o2, o2.stride(-2) if o2.dim() >= 2 else N, M, 0,
             row_map, bias, r2, r2.stride(0) if r2 is not None else 0, 0, alpha, act, norm, rope, flags)
    return out


def conv1d_k3(x_tm: torch.Tensor, w_r: torch.Tensor, bias: torch.Tensor, stride: int, out: torch.Tensor,
              out_guard: bool, pos: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Conv1d(k=3, pad=1, stride) + GELU (+ pos) as an implicit GEMM over the guard-padded time-major input.

    x_tm [N, T + 2, C_in] bf16 (rows 0 and T+1 zero), w_r [C_out, 3 * C_in] (= conv.weight.permute(0, 2, 1)
    flattened).  Output rows t' = 0 .. ceil(T/stride)-1 are written to ``out`` [N, T' (+2), C_out]; with
    ``out_guard`` they land at row t'+1 (guard rows must already be zero)."""
    N, Tp, Cin = x_tm.shape
    T = Tp - 2
    Tout = (T + stride - 1) // stride if stride > 1 else T
    Cout = w_r.shape[0]
    rows_out = out.shape[1]
    gemm_raw(x_tm.data_ptr(), N, Tout, 3 * Cin, stride * Cin, Tp * Cin, w_r, out, Cout, rows_out,
             1 if out_guard else 0, None, bias, pos, Cout if pos is not None else 0, 0, 1.0, ACT_GELU)
    return out


# ------------------------------------------------------------------------------------------ norms
def layernorm(x: torch.Tensor, w: torch.Tensor, b: torch.Tensor, eps: float = 1e-5,
              out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, BF16, "x")
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    check(lib().uvx_layernorm(x2.data_ptr(), w.data_ptr(), b.data_ptr(), out.data_ptr(), x2.shape[0], cols,
                              x2.stride(0), eps, _stream()), "uvx_layernorm")
    return out


def rmsnorm(x: torch.Tensor, w: torch.Tensor, eps: float, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, BF16, "x")
    cols = x.shape[-1]
    x2 = x.reshape(-1, cols)
    if out is None:
        out = torch.empty(x.shape, dtype=BF16, device=x.device)
    check(lib().uvx_rmsnorm(x2.data_ptr(), w.data_ptr(), out.data_ptr(), x2.shape[0], cols, x2.stride(0), 0, 0, 0, eps,
                            _stream()), "uvx_rmsnorm")
    return out


def stack_rmsnorm(enc: torch.Tensor, w: torch.Tensor, stack: int, eps: float = 1e-6,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """StackAudioFrames + ln_pre without materialising the padded/stacked tensor.
    enc [N, T, C] contiguous -> [N, ceil(T/stack), stack*C]."""
    _cuda(enc, BF16, "enc")
    enc = enc.contiguous()
    N, T, Cc = enc.shape
    rows = (T + stack - 1) // stack
    cols = Cc * stack
    if out is None:
        out = torch.empty(N, rows, cols, dtype=BF16, device=enc.device)
    check(lib().uvx_rmsnorm(enc.data_ptr(), w.data_ptr(), out.data_ptr(), N * rows, cols, cols, rows, T * Cc, T * Cc, eps,
                            _stream()), "uvx_rmsnorm(stack)")
    return out


# ------------------------------------------------------------------------------------------ attention
def attention(q_ptr: int, k_ptr: int, v_ptr: int, out: torch.Tensor, B: int, Hq: int, Hkv: int, Sq: int,
              Skv: int, D: int, strides: tuple, scale: float, causal: bool = False,
              kv_len: Optional[torch.Tensor] = None, block: int = 0, kv_start: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Raw strided interface: strides = (q_rs, q_bs, k_rs, k_bs, v_rs, v_bs, o_rs, o_bs) in elements; the three
    pointers address element [b=0, i=0, h=0, 0] of q / k / v.  ``kv_len`` / ``kv_start`` [B] int32 bound the visible keys
    of each sequence to [kv_start, kv_len) (right / left padding)."""
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q_ptr, k_ptr, v_ptr, out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, Sq, Skv, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = strides
    a.kv_len = _p(kv_len)
    a.kv_start = _p(kv_start)
    a.causal, a.block, a.scale = int(causal), int(block), float(scale)
    check(lib().uvx_attention(C.byref(a), _stream()), "uvx_attention")
    return out


def attention_indexed(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, out: torch.Tensor, Hq: int, scale: float,
                      kv_row: torch.Tensor, past: torch.Tensor, kv_len: torch.Tensor) -> torch.Tensor:
    """Causal attention of one prompt chunk per query batch against a slot cache, with the cache row and the offset read on
    the device (``uvx_attention_indexed``): q [B, Sq, Hq * D] (rows of any stride), k_cache / v_cache one layer [slots, S_max,
    Hkv, D], kv_row / past / kv_len [B] int32 -> out [B, Sq, Hq * D].  Query i of batch b sees keys j <= i + past[b] and
    j < kv_len[b] of cache row kv_row[b]."""
    _cuda(q, BF16, "q"), _cuda(k_cache, BF16, "k_cache"), _cuda(v_cache, BF16, "v_cache"), _cuda(out, BF16, "out")
    B, Sq = q.shape[0], q.shape[1]
    slots, smax, Hkv, D = k_cache.shape
    if q.shape[2] != Hq * D or q.stride(2) != 1 or out.shape != (B, Sq, Hq * D) or out.stride(2) != 1:
        raise ValueError(f"q / out must be [B, Sq, {Hq * D}] with unit column stride")
    if v_cache.shape != k_cache.shape or v_cache.stride() != k_cache.stride() or not k_cache.is_contiguous():
        raise ValueError("k_cache / v_cache must be contiguous [slots, S_max, Hkv, D] of the same shape")
    for t, name in ((kv_row, "kv_row"), (past, "past"), (kv_len, "kv_len")):
        _rows(t, torch.int32, B, name)
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, Sq, smax, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (q.stride(1), q.stride(0), Hkv * D, smax * Hkv * D, Hkv * D,
                                                                        smax * Hkv * D, out.stride(1), out.stride(0))
    a.kv_len = kv_len.data_ptr()
    a.kv_start = None
    a.causal, a.block, a.scale = 1, 0, float(scale)
    check(lib().uvx_attention_indexed(C.byref(a), slots, kv_row.data_ptr(), past.data_ptr(), _stream()), "uvx_attention_indexed")
    return out


PAGE = 64      # positions per KV page: one key tile of both attention kernels
FP8 = torch.float8_e4m3fn     # the FP8 paged pool's element type (include/uvx.h: quantize / dequantize contract)


def _is_fp8_kv(k: torch.Tensor, v: torch.Tensor, name: str = "k_pool / v_pool") -> bool:
    """Whether a KV pair is an e4m3 pool (True) or bf16 (False); any other dtype, or a mixed pair, raises UvxError."""
    _cuda(k, None, name), _cuda(v, None, name)
    if k.dtype not in (BF16, FP8) or v.dtype != k.dtype:
        raise _lib.UvxError(f"{name} must both be bfloat16 or both float8_e4m3fn, got {k.dtype} / {v.dtype}")
    return k.dtype == FP8


def _kv_scale(scale: Optional[torch.Tensor], fp8: bool, shape: tuple, name: str) -> Optional[int]:
    """Device pointer of the fp32 scales an fp8 pool needs (contiguous, ``shape``); a bf16 pool takes none."""
    if not fp8:
        if scale is not None:
            raise ValueError(f"{name} is for a float8_e4m3fn pool; this pool is bfloat16")
        return None
    if scale is None:
        raise ValueError(f"a float8_e4m3fn pool needs {name} {list(shape)} fp32")
    _cuda(scale, torch.float32, name)
    if tuple(scale.shape) != tuple(shape) or not scale.is_contiguous():
        raise ValueError(f"{name} must be a contiguous {list(shape)} fp32 tensor, got {tuple(scale.shape)}")
    return scale.data_ptr()


def _pool(k_pool: torch.Tensor, v_pool: torch.Tensor, table: torch.Tensor):
    """Checks of a paged pool layer [n_pages, 64, Hkv, D] pair (bf16 or e4m3) and its table [rows, W] int32; returns
    (n_pages, Hkv, D, W, fp8)."""
    fp8 = _is_fp8_kv(k_pool, v_pool)
    _cuda(table, torch.int32, "table")
    if k_pool.dim() != 4 or k_pool.shape[1] != PAGE or not k_pool.is_contiguous():
        raise ValueError(f"k_pool must be a contiguous pool layer [n_pages, {PAGE}, Hkv, D], got {tuple(k_pool.shape)}")
    if v_pool.shape != k_pool.shape or not v_pool.is_contiguous():
        raise ValueError("k_pool / v_pool must be contiguous pool layers of the same shape")
    if table.dim() != 2 or table.stride(1) != 1:
        raise ValueError(f"table must be [rows, W] int32 with unit column stride, got {tuple(table.shape)}")
    n_pages, _, Hkv, D = k_pool.shape
    return n_pages, Hkv, D, table.shape[1], fp8


def attention_rows(q: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, out: torch.Tensor, Hq: int, scale: float,
                   kv_len: torch.Tensor, kv_row: torch.Tensor) -> torch.Tensor:
    """Row-mapped decode attention (``uvx_attention_rows``): q [R, Hq * D] (rows of any stride), one cache layer k_cache /
    v_cache [rows, S_max, Hkv, D] (contiguous), kv_len / kv_row [R] int32 -> out [R, Hq * D].  Row r sees keys [0, kv_len[r]) of
    cache row kv_row[r]; bit-identical to ``attention`` of that row against that cache row."""
    _cuda(q, BF16, "q"), _cuda(k_cache, BF16, "k_cache"), _cuda(v_cache, BF16, "v_cache"), _cuda(out, BF16, "out")
    R = q.shape[0]
    rows, smax, Hkv, D = k_cache.shape
    if q.dim() != 2 or q.shape[1] != Hq * D or q.stride(1) != 1 or out.shape != (R, Hq * D) or out.stride(1) != 1:
        raise ValueError(f"q / out must be [R, {Hq * D}] with unit column stride")
    if v_cache.shape != k_cache.shape or not k_cache.is_contiguous() or not v_cache.is_contiguous():
        raise ValueError("k_cache / v_cache must be contiguous [rows, S_max, Hkv, D] of the same shape")
    _rows(kv_len, torch.int32, R, "kv_len"), _rows(kv_row, torch.int32, R, "kv_row")
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr(), out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = R, Hq, Hkv, 1, smax, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (q.stride(0), q.stride(0), Hkv * D, smax * Hkv * D, Hkv * D,
                                                                        smax * Hkv * D, out.stride(0), out.stride(0))
    a.kv_len = kv_len.data_ptr()
    a.kv_start = None
    a.causal, a.block, a.scale = 0, 0, float(scale)
    check(lib().uvx_attention_rows(C.byref(a), kv_row.data_ptr(), _stream()), "uvx_attention_rows")
    return out


def attention_paged(q: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, out: torch.Tensor, Hq: int, scale: float,
                    table: torch.Tensor, kv_len: torch.Tensor, kv_scale: Optional[torch.Tensor] = None,
                    kv_row: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Decode attention through a page table (``uvx_attention_paged``): q [B, Hq * D] (rows of any stride), one pool layer
    k_pool / v_pool [n_pages, 64, Hkv, D], table [>= B, W] int32 (row b: the pages of batch row b's key tiles), kv_len [B] int32
    -> out [B, Hq * D].  Row b sees keys [0, kv_len[b]); bit-identical to ``attention`` on a contiguous cache holding them.
    A float8_e4m3fn pool takes ``kv_scale`` [2] fp32 (the layer's K and V scales) and runs ``uvx_attention_paged_fp8``:
    bit-identical to the bf16 form on the dequantized pool.  ``kv_row`` [B] int32 (``uvx_attention_paged_rows`` /
    ``_fp8_rows``): row b reads table row kv_row[b] instead of b."""
    _cuda(q, BF16, "q"), _cuda(out, BF16, "out")
    n_pages, Hkv, D, W, fp8 = _pool(k_pool, v_pool, table)
    sc = _kv_scale(kv_scale, fp8, (2,), "kv_scale")
    B = q.shape[0]
    if q.dim() != 2 or q.shape[1] != Hq * D or q.stride(1) != 1 or out.shape != (B, Hq * D) or out.stride(1) != 1:
        raise ValueError(f"q / out must be [B, {Hq * D}] with unit column stride")
    if kv_row is None and table.shape[0] < B:
        raise ValueError(f"table has {table.shape[0]} rows for {B} batch rows")
    _rows(kv_len, torch.int32, B, "kv_len")
    if kv_row is not None:
        _rows(kv_row, torch.int32, B, "kv_row")
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, 1, W * PAGE, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (q.stride(0), q.stride(0), Hkv * D, PAGE * Hkv * D, Hkv * D,
                                                                        PAGE * Hkv * D, out.stride(0), out.stride(0))
    a.kv_len = kv_len.data_ptr()
    a.kv_start = None
    a.causal, a.block, a.scale = 0, 0, float(scale)
    if kv_row is not None and fp8:
        check(lib().uvx_attention_paged_fp8_rows(C.byref(a), table.data_ptr(), table.stride(0), sc, kv_row.data_ptr(), _stream()),
              "uvx_attention_paged_fp8_rows")
    elif kv_row is not None:
        check(lib().uvx_attention_paged_rows(C.byref(a), table.data_ptr(), table.stride(0), kv_row.data_ptr(), _stream()),
              "uvx_attention_paged_rows")
    elif fp8:
        check(lib().uvx_attention_paged_fp8(C.byref(a), table.data_ptr(), table.stride(0), sc, _stream()), "uvx_attention_paged_fp8")
    else:
        check(lib().uvx_attention_paged(C.byref(a), table.data_ptr(), table.stride(0), _stream()), "uvx_attention_paged")
    return out


def attention_indexed_paged(q: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, out: torch.Tensor, Hq: int, scale: float,
                            table: torch.Tensor, kv_row: torch.Tensor, past: torch.Tensor, kv_len: torch.Tensor,
                            kv_scale: Optional[torch.Tensor] = None) -> torch.Tensor:
    """``attention_indexed`` through a page table (``uvx_attention_indexed_paged``): q [B, Sq, Hq * D], one pool layer
    k_pool / v_pool [n_pages, 64, Hkv, D], table [rows, W] int32; kv_row [B] (a table row) / past / kv_len [B] int32 on the
    device -> out [B, Sq, Hq * D].  Bit-identical to ``attention_indexed`` on a contiguous cache holding the same keys.
    A float8_e4m3fn pool takes ``kv_scale`` [2] fp32 and runs ``uvx_attention_indexed_paged_fp8`` (bit-identical to the bf16
    form on the dequantized pool)."""
    _cuda(q, BF16, "q"), _cuda(out, BF16, "out")
    n_pages, Hkv, D, W, fp8 = _pool(k_pool, v_pool, table)
    sc = _kv_scale(kv_scale, fp8, (2,), "kv_scale")
    B, Sq = q.shape[0], q.shape[1]
    if q.shape[2] != Hq * D or q.stride(2) != 1 or out.shape != (B, Sq, Hq * D) or out.stride(2) != 1:
        raise ValueError(f"q / out must be [B, Sq, {Hq * D}] with unit column stride")
    for t, name in ((kv_row, "kv_row"), (past, "past"), (kv_len, "kv_len")):
        _rows(t, torch.int32, B, name)
    a = AttnArgs()
    a.q, a.k, a.v, a.o = q.data_ptr(), k_pool.data_ptr(), v_pool.data_ptr(), out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, Sq, W * PAGE, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (q.stride(1), q.stride(0), Hkv * D, PAGE * Hkv * D, Hkv * D,
                                                                        PAGE * Hkv * D, out.stride(1), out.stride(0))
    a.kv_len = kv_len.data_ptr()
    a.kv_start = None
    a.causal, a.block, a.scale = 1, 0, float(scale)
    if fp8:
        check(lib().uvx_attention_indexed_paged_fp8(C.byref(a), n_pages, table.data_ptr(), table.stride(0), kv_row.data_ptr(),
                                                    past.data_ptr(), sc, _stream()), "uvx_attention_indexed_paged_fp8")
    else:
        check(lib().uvx_attention_indexed_paged(C.byref(a), n_pages, table.data_ptr(), table.stride(0), kv_row.data_ptr(),
                                                past.data_ptr(), _stream()), "uvx_attention_indexed_paged")
    return out


def kv_page_map(table: torch.Tensor, cache_row: torch.Tensor, pos: torch.Tensor, page_out: torch.Tensor, off_out: torch.Tensor,
                frozen: Optional[torch.Tensor] = None) -> None:
    """(table row cache_row[r], position pos[r]) -> (page_out[r], off_out[r]) through ``table`` [rows, W] int32; cache_row < 0,
    or frozen[r] != 0 for the first frozen.numel() rows, gives (-1, 0).  All int32 on the device (``uvx_kv_page_map``)."""
    _cuda(table, torch.int32, "table")
    if table.dim() != 2 or table.stride(1) != 1:
        raise ValueError("table must be [rows, W] int32 with unit column stride")
    R = cache_row.shape[0]
    for t, name in ((cache_row, "cache_row"), (pos, "pos"), (page_out, "page_out"), (off_out, "off_out")):
        _rows(t, torch.int32, R, name)
    nf = 0
    if frozen is not None:
        nf = frozen.numel()
        _rows(frozen, torch.int32, nf, "frozen")
        if nf > R:
            raise ValueError(f"{nf} frozen flags for {R} rows")
    check(lib().uvx_kv_page_map(table.data_ptr(), table.stride(0), cache_row.data_ptr(), pos.data_ptr(), _p(frozen), nf, R,
                                page_out.data_ptr(), off_out.data_ptr(), _stream()), "uvx_kv_page_map")


def kv_pages_copy(k_row: torch.Tensor, v_row: torch.Tensor, k_pool: torch.Tensor, v_pool: torch.Tensor, pages: torch.Tensor,
                  p0: int, p1: int, to_pages: bool, kv_scales: Optional[torch.Tensor] = None) -> None:
    """Positions [p0, p1) of every layer, K and V, between a contiguous one-row cache [L, 1, S_max, Hkv, D] and the pool
    [L, n_pages, 64, Hkv, D] (``uvx_kv_pages_copy``): position p lives in page pages[p // 64] (int32 on the device), row p % 64.
    ``to_pages``: row -> pages (scatter), else pages -> row (gather).  Bit-exact.  A float8_e4m3fn pool takes ``kv_scales``
    [L, 2] fp32 (``uvx_kv_pages_copy_fp8``): the scatter quantizes, the gather dequantizes into the bf16 row."""
    fp8 = _is_fp8_kv(k_pool, v_pool)
    sc = _kv_scale(kv_scales, fp8, (k_pool.shape[0], 2), "kv_scales")
    for t, name in ((k_row, "k_row"), (v_row, "v_row"), (k_pool, "k_pool"), (v_pool, "v_pool")):
        _cuda(t, None if name.endswith("pool") else BF16, name)
        if not t.is_contiguous() or t.dim() != 5:
            raise ValueError(f"{name} must be a contiguous 5-D cache")
    _cuda(pages, torch.int32, "pages")
    L, one, smax, Hkv, D = k_row.shape
    if one != 1 or v_row.shape != k_row.shape:
        raise ValueError(f"k_row / v_row must be one-row caches [L, 1, S_max, Hkv, D], got {tuple(k_row.shape)}")
    if k_pool.shape[0] != L or k_pool.shape[2:] != (PAGE, Hkv, D) or v_pool.shape != k_pool.shape:
        raise ValueError(f"k_pool / v_pool must be [{L}, n_pages, {PAGE}, {Hkv}, {D}], got {tuple(k_pool.shape)}")
    if not 0 <= p0 <= p1 <= smax or pages.numel() * PAGE < p1:
        raise ValueError(f"positions [{p0}, {p1}) outside the row ({smax}) or the page list ({pages.numel()} pages)")
    args = (k_row.data_ptr(), v_row.data_ptr(), smax * Hkv * D, k_pool.data_ptr(), v_pool.data_ptr(), k_pool.shape[1] * PAGE * Hkv * D, L,
            Hkv * D, pages.data_ptr(), int(p0), int(p1), int(bool(to_pages)))
    if fp8:
        check(lib().uvx_kv_pages_copy_fp8(*args, sc, _stream()), "uvx_kv_pages_copy_fp8")
    else:
        check(lib().uvx_kv_pages_copy(*args, _stream()), "uvx_kv_pages_copy")


def kv_pages_move(src_k: torch.Tensor, src_v: torch.Tensor, dst_k: torch.Tensor, dst_v: torch.Tensor, src_pages: torch.Tensor,
                  dst_pages: torch.Tensor) -> None:
    """Whole pages, every layer, K and V, byte for byte, from the pool ``src_k`` / ``src_v`` [L, n_src, 64, Hkv, D] to ``dst_k`` /
    ``dst_v`` [L, n_dst, 64, Hkv, D] of the same dtype (bf16 or float8_e4m3fn; an e4m3 pool's scales do not change): page
    src_pages[j] -> page dst_pages[j] (``uvx_kv_pages_move``).  Either pool may be a pinned CPU tensor, which the kernel reads or
    writes over PCIe; a pageable one raises UvxError and nothing is launched.  The page lists are int32 on the device and are
    not range-checked here (that would need a sync): the caller keeps them inside the pools, destinations distinct."""
    if src_v.dtype != src_k.dtype or dst_k.dtype != src_k.dtype or dst_v.dtype != src_k.dtype or src_k.dtype not in (BF16, FP8):
        raise _lib.UvxError(f"the four pools must share one dtype, bfloat16 or float8_e4m3fn; got {src_k.dtype} / {src_v.dtype} -> "
                            f"{dst_k.dtype} / {dst_v.dtype}")
    for t, name in ((src_k, "src_k"), (src_v, "src_v"), (dst_k, "dst_k"), (dst_v, "dst_v")):
        if not t.is_contiguous() or t.dim() != 5 or t.shape[2] != PAGE:
            raise ValueError(f"{name} must be a contiguous pool [L, n_pages, {PAGE}, Hkv, D], got {tuple(t.shape)}")
    if src_v.shape != src_k.shape or dst_v.shape != dst_k.shape or src_k.shape[0] != dst_k.shape[0] or \
            src_k.shape[2:] != dst_k.shape[2:]:
        raise ValueError(f"pools of different layers or page shapes: {tuple(src_k.shape)} -> {tuple(dst_k.shape)}")
    n = src_pages.numel()
    _rows(src_pages, torch.int32, n, "src_pages")
    _rows(dst_pages, torch.int32, n, "dst_pages")
    page_bytes = src_k[0, 0].numel() * src_k.element_size()
    check(lib().uvx_kv_pages_move(src_k.data_ptr(), src_v.data_ptr(), src_k.shape[1] * page_bytes, dst_k.data_ptr(),
                                  dst_v.data_ptr(), dst_k.shape[1] * page_bytes, src_k.shape[0], page_bytes, src_pages.data_ptr(),
                                  dst_pages.data_ptr(), n, _stream()), "uvx_kv_pages_move")


def attention_fused_qkv(qkv: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int, scale: float, causal: bool,
                        kv_len: Optional[torch.Tensor] = None, block: int = 0,
                        out: Optional[torch.Tensor] = None, kv_start: Optional[torch.Tensor] = None) -> torch.Tensor:
    """qkv [B*S, (Hq + 2*Hkv) * D] (q | k | v sections) -> out [B*S, Hq*D]."""
    _cuda(qkv, BF16, "qkv")
    assert qkv.shape[-1] == (Hq + 2 * Hkv) * D and qkv.stride(-1) == 1
    rs = qkv.stride(-2)
    if out is None:
        out = torch.empty(B * S, Hq * D, dtype=BF16, device=qkv.device)
    base = qkv.data_ptr()
    return attention(base, base + 2 * Hq * D, base + 2 * (Hq + Hkv) * D, out, B, Hq, Hkv, S, S, D,
                     (rs, S * rs, rs, S * rs, rs, S * rs, Hq * D, S * Hq * D), scale, causal, kv_len, block, kv_start)


def attention_encoder_tc(qkv: torch.Tensor, B: int, S: int, H: int, scale: float, kv_len: Optional[torch.Tensor] = None,
                         block: int = 0, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Encoder attention over a fused [B*S, 3*H*64] q|k|v projection (head_dim 64), no q / k / v copies: the TMA + wgmma flash
    kernel from 16 queries on, the mma.sync kernel below that (``uvx_attention``'s dispatch)."""
    _cuda(qkv, BF16, "qkv")
    d = H * 64
    assert qkv.shape[-1] == 3 * d and qkv.stride(-1) == 1
    if out is None:
        out = torch.empty(B * S, d, dtype=BF16, device=qkv.device)
    check(lib().uvx_attention_enc_tc(qkv.data_ptr(), qkv.stride(-2), B, S, H, 0, d, 2 * d, out.data_ptr(), out.stride(-2),
                                     _p(kv_len), int(block), float(scale), _stream()), "uvx_attention_enc_tc")
    return out


# ------------------------------------------------------------------------------------------ rope / swiglu
def rope_tables(inv_freq: torch.Tensor, max_pos: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """cos/sin [max_pos, D/2] fp32 exactly as LlamaRotaryEmbedding computes them (fp32 outer product)."""
    pos = torch.arange(max_pos, dtype=torch.float32)
    freqs = pos[:, None] * inv_freq.to(torch.float32)[None, :]
    return freqs.cos().to(device).contiguous(), freqs.sin().to(device).contiguous()


def rope_(qkv: torch.Tensor, Hq: int, Hkv: int, D: int, cos: torch.Tensor, sin: torch.Tensor, rows_per_seq: int,
          pos_offset: int = 0, positions: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(qkv, BF16, "qkv")
    rows = qkv.numel() // qkv.shape[-1]
    check(lib().uvx_rope(qkv.data_ptr(), rows, qkv.stride(-2), Hq, Hkv, D, cos.data_ptr(), sin.data_ptr(), _p(positions),
                         rows_per_seq, pos_offset, _stream()), "uvx_rope")
    return qkv


def swiglu(x: torch.Tensor, gate_first: bool, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, BF16, "x")
    H = x.shape[-1] // 2
    x2 = x.reshape(-1, 2 * H)
    if out is None:
        out = torch.empty(*x.shape[:-1], H, dtype=BF16, device=x.device)
    check(lib().uvx_swiglu(x2.data_ptr(), out.data_ptr(), x2.shape[0], H, x2.stride(0), int(gate_first), _stream()),
          "uvx_swiglu")
    return out


# ------------------------------------------------------------------------------------------ embed + splice
def splice_plan(start_idx: torch.Tensor, tok_len: torch.Tensor, audio_batch_size: torch.Tensor, B: int, S: int,
                tok_stride: int, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    dev = start_idx.device
    _cuda(start_idx, torch.int64, "audio_token_start_idx"), _cuda(tok_len, torch.int32, "audio_token_len")
    _cuda(audio_batch_size, torch.int64, "audio_batch_size")
    if out is None:
        out = torch.empty(B * S, dtype=torch.int32, device=dev)
    check(lib().uvx_splice_plan(start_idx.data_ptr(), tok_len.data_ptr(), audio_batch_size.data_ptr(), start_idx.numel(),
                                B, S, tok_stride, out.data_ptr(), _stream()), "uvx_splice_plan")
    return out


def embed_splice(input_ids: torch.Tensor, embed_tokens: torch.Tensor, audio_embeds: Optional[torch.Tensor],
                 src: Optional[torch.Tensor], out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(input_ids, torch.int64, "input_ids"), _cuda(embed_tokens, BF16, "embed_tokens")
    ids = input_ids.contiguous()
    d = embed_tokens.shape[1]
    if out is None:
        out = torch.empty(*ids.shape, d, dtype=BF16, device=ids.device)
    check(lib().uvx_embed_splice(ids.data_ptr(), embed_tokens.data_ptr(), embed_tokens.shape[0], _p(audio_embeds), _p(src),
                                 ids.numel(), d, out.data_ptr(), _stream()), "uvx_embed_splice")
    return out


# ------------------------------------------------------------------------------------------ lm head
def lm_head(h: torch.Tensor, w: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """h [B, d] bf16 (row stride arbitrary) x w [V, d] -> fp32 logits [B, V]."""
    _cuda(h, BF16, "h"), _cuda(w, BF16, "w")
    B, d = h.shape
    V = w.shape[0]
    if out is None:
        out = torch.empty(B, V, dtype=torch.float32, device=h.device)
    check(lib().uvx_lm_head(h.data_ptr(), B, h.stride(0), w.data_ptr(), V, d, out.data_ptr(), _stream()), "uvx_lm_head")
    return out


def argmax(logits: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(logits, torch.float32, "logits")
    B, V = logits.shape
    if out is None:
        out = torch.empty(B, dtype=torch.int64, device=logits.device)
    check(lib().uvx_argmax(logits.data_ptr(), B, V, out.data_ptr(), _stream()), "uvx_argmax")
    return out


def llama3_inv_freq(head_dim: int, theta: float, scaling: Optional[dict]) -> torch.Tensor:
    """inv_freq with the llama3 smoothing (hf:modeling_rope_utils.py:550-626); fp32 like the reference."""
    inv = 1.0 / (theta ** (torch.arange(0, head_dim, 2, dtype=torch.int64).to(torch.float32) / head_dim))
    if not scaling or scaling.get("rope_type", scaling.get("type")) != "llama3":
        return inv
    factor, lo, hi = scaling["factor"], scaling["low_freq_factor"], scaling["high_freq_factor"]
    old = scaling["original_max_position_embeddings"]
    wl = 2 * math.pi / inv
    inv_l = torch.where(wl > old / lo, inv / factor, inv)
    smooth = (old / wl - lo) / (hi - lo)
    sm = (1 - smooth) * inv_l / factor + smooth * inv_l
    mid = ~(wl < old / hi) * ~(wl > old / lo)
    return torch.where(mid, sm, inv_l)


# ------------------------------------------------------------------------------------------ backward pieces (a14)
def transpose(x: torch.Tensor, out: Optional[torch.Tensor] = None, pad_cols_to: int = 8) -> torch.Tensor:
    """[R, C] bf16 -> [C, R'] with R' = R rounded up to ``pad_cols_to`` (zero tail) so it can be a GEMM operand."""
    _cuda(x, BF16, "x")
    R, Cc = x.shape
    Rp = -(-R // pad_cols_to) * pad_cols_to
    if out is None:
        out = torch.zeros(Cc, Rp, dtype=BF16, device=x.device) if Rp != R else torch.empty(Cc, Rp, dtype=BF16, device=x.device)
    check(lib().uvx_transpose_bf16(x.data_ptr(), R, Cc, x.stride(0), out.data_ptr(), out.stride(0), _stream()),
          "uvx_transpose_bf16")
    return out


def rmsnorm_bwd(dy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, eps: float, dres: Optional[torch.Tensor] = None,
                want_dx: bool = True, dw: Optional[torch.Tensor] = None, stack: Optional[tuple] = None,
                out: Optional[torch.Tensor] = None) -> Optional[torch.Tensor]:
    """dx (bf16, + dres) and/or dw (fp32, accumulated) of uvx_rmsnorm.  ``stack=(group_rows, T*C)`` for ln_pre: x is the
    encoder output [N, T, C] and dx comes back in the stacked layout [N * group_rows, stack * C]."""
    _cuda(dy, BF16, "dy"), _cuda(x, BF16, "x")
    cols = dy.shape[-1]
    dy = dy.contiguous()                          # the kernel reads dy / dres / dx as dense [rows, cols]
    rows = dy.numel() // cols
    if dres is not None:
        assert dres.shape == dy.shape, "dres must have dy's shape"
        dres = dres.contiguous()
    if want_dx and out is None:
        out = torch.empty(dy.shape, dtype=BF16, device=dy.device)
    assert not want_dx or (out.is_contiguous() and out.numel() == dy.numel()), "out must be a dense [rows, cols] buffer"
    assert dw is None or (dw.dtype == torch.float32 and dw.is_contiguous() and dw.numel() == cols)
    g_rows, g_stride, valid = (stack[0], stack[1], stack[1]) if stack else (0, 0, 0)
    if stack:
        x = x.contiguous()
        xs = cols
    else:
        x = x.reshape(-1, cols)
        if x.stride(-1) != 1 or x.stride(0) % 8 != 0:
            x = x.contiguous()
        xs = x.stride(0)
    check(lib().uvx_rmsnorm_bwd(dy.data_ptr(), x.data_ptr(), w.data_ptr(), _p(dres), _p(out) if want_dx else None, _p(dw), rows,
                                cols, xs, g_rows, g_stride, valid, eps, _stream()), "uvx_rmsnorm_bwd")
    return out if want_dx else None


def layernorm_bwd(dy: torch.Tensor, x: torch.Tensor, w: torch.Tensor, eps: float = 1e-5, dres: Optional[torch.Tensor] = None,
                  out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Data gradient of ``layernorm`` (+ ``dres``, the gradient arriving on the residual branch): rows x cols bf16."""
    _cuda(dy, BF16, "dy"), _cuda(x, BF16, "x")
    cols = x.shape[-1]
    x2, dy2 = x.reshape(-1, cols), dy.reshape(-1, cols)
    assert x2.is_contiguous() and dy2.is_contiguous() and (dres is None or dres.is_contiguous())
    if out is None:
        out = torch.empty_like(x2)
    check(lib().uvx_layernorm_bwd(dy2.data_ptr(), x2.data_ptr(), w.data_ptr(), _p(dres), out.data_ptr(), x2.shape[0], cols, float(eps),
                                  _stream()), "uvx_layernorm_bwd")
    return out.view(x.shape)


def gelu(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, BF16, "x")
    assert x.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    check(lib().uvx_gelu(x.data_ptr(), out.data_ptr(), x.numel(), _stream()), "uvx_gelu")
    return out


def gelu_bwd(x: torch.Tensor, dy: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dx = dy * gelu'(x) for the pre-activation ``x`` (erf form)."""
    _cuda(x, BF16, "x"), _cuda(dy, BF16, "dy")
    assert x.is_contiguous() and dy.is_contiguous()
    if out is None:
        out = torch.empty_like(x)
    check(lib().uvx_gelu_bwd(x.data_ptr(), dy.data_ptr(), out.data_ptr(), x.numel(), _stream()), "uvx_gelu_bwd")
    return out


def swiglu_bwd(x: torch.Tensor, dout: torch.Tensor, gate_first: bool, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _cuda(x, BF16, "x"), _cuda(dout, BF16, "dout")
    H = x.shape[-1] // 2
    x2 = x.reshape(-1, 2 * H)
    if x2.stride(-1) != 1 or x2.stride(0) % 8 != 0:
        x2 = x2.contiguous()
    assert dout.numel() == x2.shape[0] * H, "dout must be [rows, H]"
    dout = dout.contiguous()                      # the kernel reads dout as dense [rows, H]
    if out is None:
        out = torch.empty(x2.shape, dtype=BF16, device=x.device)
    assert out.is_contiguous() and out.numel() == x2.numel(), "out must be a dense [rows, 2H] buffer"
    check(lib().uvx_swiglu_bwd(x2.data_ptr(), dout.data_ptr(), out.data_ptr(), x2.shape[0], H, x2.stride(0), int(gate_first),
                               _stream()), "uvx_swiglu_bwd")
    return out


def rope_bwd_(dqkv: torch.Tensor, Hq: int, Hkv: int, D: int, cos: torch.Tensor, sin: torch.Tensor, rows_per_seq: int,
              pos_offset: int = 0) -> torch.Tensor:
    rows = dqkv.numel() // dqkv.shape[-1]
    check(lib().uvx_rope_bwd(dqkv.data_ptr(), rows, dqkv.stride(-2), Hq, Hkv, D, cos.data_ptr(), sin.data_ptr(), None,
                             rows_per_seq, pos_offset, _stream()), "uvx_rope_bwd")
    return dqkv


def attention_fused_qkv_train(qkv: torch.Tensor, B: int, S: int, Hq: int, Hkv: int, D: int, scale: float, causal: bool,
                              out: torch.Tensor, lse: torch.Tensor, kv_len: Optional[torch.Tensor] = None) -> torch.Tensor:
    """Forward that also records the log-sum-exp ([B, Hq, S] fp32) needed by the backward."""
    rs = qkv.stride(-2)
    base = qkv.data_ptr()
    a = AttnArgs()
    a.q, a.k, a.v, a.o = base, base + 2 * Hq * D, base + 2 * (Hq + Hkv) * D, out.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, S, S, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (rs, S * rs, rs, S * rs, rs, S * rs, Hq * D, S * Hq * D)
    a.kv_len, a.causal, a.block, a.scale, a.lse = _p(kv_len), int(causal), 0, float(scale), lse.data_ptr()
    check(lib().uvx_attention(C.byref(a), _stream()), "uvx_attention")
    return out


def attention_fused_qkv_bwd(qkv: torch.Tensor, o: torch.Tensor, dout: torch.Tensor, lse: torch.Tensor, B: int, S: int, Hq: int,
                            Hkv: int, D: int, scale: float, causal: bool, dqkv: Optional[torch.Tensor] = None,
                            kv_len: Optional[torch.Tensor] = None) -> torch.Tensor:
    """dqkv [B*S, (Hq+2Hkv)*D] (same fused layout as qkv) from dout [B*S, Hq*D]."""
    _cuda(qkv, BF16, "qkv"), _cuda(o, BF16, "o"), _cuda(dout, BF16, "dout"), _cuda(lse, torch.float32, "lse")
    assert qkv.shape[-1] == (Hq + 2 * Hkv) * D and qkv.stride(-1) == 1
    assert o.numel() == dout.numel() == B * S * Hq * D and lse.numel() == B * Hq * S and lse.is_contiguous()
    o, dout = o.contiguous(), dout.contiguous()  # o and dout are read as dense [B*S, Hq*D]
    rs = qkv.stride(-2)
    base = qkv.data_ptr()
    if dqkv is None:
        dqkv = torch.empty_like(qkv)
    assert dqkv.shape == qkv.shape and dqkv.stride(-1) == 1
    a = AttnArgs()
    a.q, a.k, a.v, a.o = base, base + 2 * Hq * D, base + 2 * (Hq + Hkv) * D, o.data_ptr()
    a.B, a.Hq, a.Hkv, a.Sq, a.Skv, a.D = B, Hq, Hkv, S, S, D
    (a.q_rs, a.q_bs, a.k_rs, a.k_bs, a.v_rs, a.v_bs, a.o_rs, a.o_bs) = (rs, S * rs, rs, S * rs, rs, S * rs, Hq * D, S * Hq * D)
    a.kv_len, a.causal, a.block, a.scale, a.lse = _p(kv_len), int(causal), 0, float(scale), lse.data_ptr()
    delta = torch.empty(B * Hq * S, dtype=torch.float32, device=qkv.device)
    drs = dqkv.stride(-2)
    dbase = dqkv.data_ptr()
    check(lib().uvx_attention_bwd(C.byref(a), o.data_ptr(), dout.data_ptr(), dbase, dbase + 2 * Hq * D, dbase + 2 * (Hq + Hkv) * D,
                                  drs, S * drs, drs, S * drs, drs, S * drs, delta.data_ptr(), _stream()), "uvx_attention_bwd")
    return dqkv


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    d = src.shape[-1]
    if out is None:
        out = torch.empty(idx.numel(), d, dtype=BF16, device=src.device)
    check(lib().uvx_gather_rows(src.data_ptr(), idx.data_ptr(), idx.numel(), d, out.data_ptr(), _stream()), "uvx_gather_rows")
    return out


def splice_inverse(src: torch.Tensor, n_audio_rows: int) -> torch.Tensor:
    inv = torch.empty(n_audio_rows, dtype=torch.int32, device=src.device)
    check(lib().uvx_splice_inverse(src.data_ptr(), src.numel(), inv.data_ptr(), n_audio_rows, _stream()), "uvx_splice_inverse")
    return inv


def adamw_(p: torch.Tensor, g: torch.Tensor, m: torch.Tensor, v: torch.Tensor, step: int, lr: float, betas=(0.9, 0.999),
           eps: float = 1e-8, weight_decay: float = 0.0, grad_scale: float = 1.0) -> None:
    _cuda(p, BF16, "p"), _cuda(g, torch.float32, "g")
    check(lib().uvx_adamw(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), p.numel(), lr, betas[0], betas[1], eps,
                          weight_decay, step, grad_scale, _stream()), "uvx_adamw")


def _tensor_list(g, acc=None, p=None, m=None, v=None) -> _lib.TensorList:
    """``uvx_tensor_list`` over parallel lists of contiguous CUDA tensors (g / acc / m / v fp32, p bf16)."""
    if not 1 <= len(g) <= _lib.TL_MAX:
        raise ValueError(f"1 .. {_lib.TL_MAX} tensors per launch, got {len(g)}")
    tl = _lib.TensorList()
    tl.count = len(g)
    for field, ts, dtype in (("g", g, torch.float32), ("acc", acc, torch.float32), ("p", p, BF16), ("m", m, torch.float32),
                             ("v", v, torch.float32)):
        if ts is None:
            continue
        if len(ts) != len(g):
            raise ValueError(f"{field}: {len(ts)} tensors for {len(g)} gradients")
        for i, t in enumerate(ts):
            _cuda(t, dtype, f"{field}[{i}]")
            if not t.is_contiguous() or t.numel() != g[i].numel():
                raise ValueError(f"{field}[{i}] must be contiguous with {g[i].numel()} elements")
            getattr(tl, field)[i] = t.data_ptr()
            tl.numel[i] = t.numel()
    return tl


def norm_workspace(device) -> torch.Tensor:
    """Zeroed workspace of ``grad_norm_clip`` (block partials + the self-resetting ticket); one per stream of calls."""
    return torch.zeros(_lib.NORM_WS_BYTES, dtype=torch.uint8, device=device)


def grad_norm_clip(grads, scale: torch.Tensor, max_norm: Optional[float], workspace: torch.Tensor,
                   out: Optional[torch.Tensor] = None, step: Optional[torch.Tensor] = None, lr_table: Optional[torch.Tensor] = None,
                   lr: Optional[torch.Tensor] = None) -> torch.Tensor:
    """out = [norm, coef] (fp32 device): norm = ||scale[0] * g||_2 over all ``grads`` (deterministic fp64 sum) and
    coef = min(max_norm / (norm + 1e-6), 1) as ``torch.nn.utils.clip_grad_norm_`` forms it; ``max_norm`` None / <= 0 gives
    coef = 1.  With ``step`` (int64 [1]) the same launch does step += 1 and lr[0] = lr_table[min(step, len) - 1]."""
    _cuda(scale, torch.float32, "scale"), _cuda(workspace, torch.uint8, "workspace")
    if workspace.numel() < _lib.NORM_WS_BYTES:
        raise ValueError(f"workspace needs {_lib.NORM_WS_BYTES} bytes")
    if out is None:
        out = torch.empty(2, dtype=torch.float32, device=scale.device)
    if step is not None:
        _cuda(step, torch.int64, "step"), _cuda(lr_table, torch.float32, "lr_table"), _cuda(lr, torch.float32, "lr")
    tl = _tensor_list(list(grads))
    check(lib().uvx_grad_norm_clip(C.byref(tl), scale.data_ptr(), float(max_norm or 0.0), workspace.data_ptr(), out.data_ptr(),
                                   _p(step), _p(lr_table), 0 if lr_table is None else lr_table.numel(), _p(lr), _stream()),
          "uvx_grad_norm_clip")
    return out


def adamw_multi_(params, grads, ms, vs, lr: torch.Tensor, step: torch.Tensor, scale: torch.Tensor,
                 coef: Optional[torch.Tensor] = None, betas=(0.9, 0.999), eps: float = 1e-8, weight_decay: float = 0.0) -> None:
    """torch.optim.AdamW over every tensor of the lists in one launch; lr / step / coef / scale are device scalars (``coef`` may be
    a view of ``grad_norm_clip``'s output)."""
    _cuda(lr, torch.float32, "lr"), _cuda(step, torch.int64, "step"), _cuda(scale, torch.float32, "scale")
    if coef is not None:
        _cuda(coef, torch.float32, "coef")
    tl = _tensor_list(list(grads), p=list(params), m=list(ms), v=list(vs))
    check(lib().uvx_adamw_multi(C.byref(tl), lr.data_ptr(), step.data_ptr(), _p(coef), scale.data_ptr(), betas[0], betas[1], eps,
                                weight_decay, _stream()), "uvx_adamw_multi")


def grad_accumulate_(accs, grads, assign: bool = False) -> None:
    """acc[i] (+)= g[i] in fp32 for every pair, one launch; ``assign`` starts a new accumulation (acc = g)."""
    tl = _tensor_list(list(grads), acc=list(accs))
    check(lib().uvx_grad_accumulate(C.byref(tl), int(bool(assign)), _stream()), "uvx_grad_accumulate")


# ------------------------------------------------------------------------------------------ decode step (a13)
def gemv(x: torch.Tensor, w: torch.Tensor, residual: Optional[torch.Tensor] = None, out: Optional[torch.Tensor] = None,
         out_dtype=BF16, norm: Optional[tuple] = None, swiglu: bool = False) -> torch.Tensor:
    """y = x @ w.T (+ residual) for x [B <= 8, K]: weight-streaming matrix-vector kernel (no tensor cores).  Fused prologues of the
    decode step: ``norm=(weight, eps)`` -> y = RMSNorm(x) @ w.T; ``swiglu=True`` -> x is [B, 2K] = gate | up and
    y = (act_fn(gate) * up) @ w.T - both bit-identical to the separate kernels."""
    _cuda(x, BF16, "x"), _cuda(w, BF16, "w")
    B = x.shape[0]
    K = x.shape[1] // 2 if swiglu else x.shape[1]
    N = w.shape[0]
    if norm is not None or swiglu:
        if (200 * 1024) // (2 * K) < B or B > 8:            # (the fused form has no slab loop)
            x = rmsnorm(x, norm[0], norm[1]) if norm is not None else globals()["swiglu"](x, gate_first=True)
            return gemv(x, w, residual=residual, out=out, out_dtype=out_dtype)
        if out is None:
            out = torch.empty(B, N, dtype=out_dtype, device=x.device)
        check(lib().uvx_gemv_fused_bf16(x.data_ptr(), B, x.stride(0), w.data_ptr(), w.stride(0), N, K, _p(residual),
                                        residual.stride(0) if residual is not None else 0, out.data_ptr(), out.stride(0),
                                        int(out.dtype == torch.float32), norm[0].data_ptr() if norm is not None else None,
                                        float(norm[1]) if norm is not None else 0.0, int(swiglu), _stream()), "uvx_gemv_fused_bf16")
        return out
    if out is None:
        out = torch.empty(B, N, dtype=out_dtype, device=x.device)
    slab = max(1, min(8, (200 * 1024) // (2 * K)))      # rows whose activations fit the kernel's shared memory
    for b0 in range(0, B, slab):
        nb = min(slab, B - b0)
        xs, os_ = x[b0:b0 + nb], out[b0:b0 + nb]
        rs = residual[b0:b0 + nb] if residual is not None else None
        check(lib().uvx_gemv_bf16(xs.data_ptr(), nb, x.stride(0), w.data_ptr(), w.stride(0), N, K, _p(rs),
                                  residual.stride(0) if residual is not None else 0, os_.data_ptr(), out.stride(0),
                                  int(out.dtype == torch.float32), _stream()), "uvx_gemv_bf16")
    return out


def kv_append(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor, Hq: int, Hkv: int,
              D: int) -> None:
    """qkv [B, (Hq+2Hkv)*D] -> k_cache / v_cache [B, S_max, Hkv, D] at positions[b] (device int32)."""
    B = qkv.shape[0]
    check(lib().uvx_kv_append(qkv.data_ptr(), qkv.stride(0), Hq * D, (Hq + Hkv) * D, Hkv * D, k_cache.data_ptr(),
                              v_cache.data_ptr(), k_cache.stride(0), positions.data_ptr(), B, _stream()), "uvx_kv_append")


def rope_kv_append_(qkv: torch.Tensor, Hq: int, Hkv: int, D: int, cos: torch.Tensor, sin: torch.Tensor, rope_positions: torch.Tensor,
                    k_cache: torch.Tensor, v_cache: torch.Tensor, positions: torch.Tensor) -> None:
    """``rope_`` (per-row positions) + ``kv_append`` in one launch: the decode step's q / k rotation and cache append."""
    B = qkv.shape[0]
    check(lib().uvx_rope_kv_append(qkv.data_ptr(), B, qkv.stride(0), Hq, Hkv, D, cos.data_ptr(), sin.data_ptr(), rope_positions.data_ptr(),
                                   k_cache.data_ptr(), v_cache.data_ptr(), k_cache.stride(0), positions.data_ptr(), _stream()),
          "uvx_rope_kv_append")


def rope_kv_append_map_(qkv: torch.Tensor, Hq: int, Hkv: int, D: int, cos: torch.Tensor, sin: torch.Tensor,
                        rope_positions: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, cache_row: torch.Tensor,
                        positions: torch.Tensor, kv_scale: Optional[torch.Tensor] = None) -> None:
    """``rope_kv_append_`` with a per-row map: row r is rotated at rope_positions[r] and appended to cache row cache_row[r] at
    positions[r], or not appended when cache_row[r] < 0 (all three [rows] int32 on the device).  A float8_e4m3fn cache (the
    FP8 paged pool) takes ``kv_scale`` [2] fp32 and stores the k / v rows quantized (``uvx_rope_kv_append_map_fp8``)."""
    _cuda(qkv, BF16, "qkv")
    fp8 = _is_fp8_kv(k_cache, v_cache, "k_cache / v_cache")
    sc = _kv_scale(kv_scale, fp8, (2,), "kv_scale")
    R = qkv.shape[0]
    for t, name in ((rope_positions, "rope_positions"), (cache_row, "cache_row"), (positions, "positions")):
        _rows(t, torch.int32, R, name)
    args = (qkv.data_ptr(), R, qkv.stride(0), Hq, Hkv, D, cos.data_ptr(), sin.data_ptr(), rope_positions.data_ptr(), k_cache.data_ptr(),
            v_cache.data_ptr(), k_cache.stride(0), cache_row.data_ptr(), positions.data_ptr())
    if fp8:
        check(lib().uvx_rope_kv_append_map_fp8(*args, sc, _stream()), "uvx_rope_kv_append_map_fp8")
    else:
        check(lib().uvx_rope_kv_append_map(*args, _stream()), "uvx_rope_kv_append_map")


def add_i32_(a: torch.Tensor, b: Optional[torch.Tensor], delta: int) -> None:
    check(lib().uvx_add_i32(a.data_ptr(), _p(b), a.numel(), delta, _stream()), "uvx_add_i32")


def kv_write(qkv: torch.Tensor, k_cache: torch.Tensor, v_cache: torch.Tensor, B: int, S: int, past: int, Hq: int, Hkv: int,
             D: int) -> None:
    """Prefill rows [B*S, (Hq+2Hkv)*D] -> k_cache / v_cache [B, S_max, Hkv, D] at positions past .. past+S-1."""
    check(lib().uvx_kv_write(qkv.data_ptr(), qkv.stride(0), Hq * D, (Hq + Hkv) * D, Hkv * D, k_cache.data_ptr(), v_cache.data_ptr(),
                             k_cache.stride(0), B, S, past, _stream()), "uvx_kv_write")


def repetition_penalty_(logits: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, penalty: float,
                        scratch: torch.Tensor) -> torch.Tensor:
    _cuda(logits, torch.float32, "logits"), _cuda(seq, torch.int64, "seq"), _cuda(cur_len, torch.int32, "cur_len")
    B, V = logits.shape
    check(lib().uvx_repetition_penalty(logits.data_ptr(), B, V, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(), float(penalty),
                                       scratch.data_ptr(), _stream()), "uvx_repetition_penalty")
    return logits


CUTOFFS_OFF = (0.0, 1.0, 0.0, 0.0)   # (min_p, typical_p, epsilon, eta) with every cut-off off: uvx_cutoffs' encoding


def sampling_cutoffs(min_p=None, typical_p=None, epsilon_cutoff=None, eta_cutoff=None) -> tuple:
    """``generate()``'s four cut-off arguments -> the (min_p, typical_p, epsilon, eta) tuple the kernels read, off = (0, 1, 0, 0).
    The checks of transformers' warper constructors: ``min_p`` outside [0, 1] and ``typical_p`` <= 0 raise ValueError (NaN
    too); ``typical_p`` >= 1 is off, and ``epsilon_cutoff`` / ``eta_cutoff`` outside (0, 1) are off, as HF only adds those
    warpers for such values."""
    mp, tp, eps, eta = CUTOFFS_OFF
    if min_p is not None:
        mp = float(min_p)
        if not 0.0 <= mp <= 1.0:                                   # NaN fails too
            raise ValueError(f"`min_p` has to be a float in the [0, 1] interval, but is {min_p}")
    if typical_p is not None:
        tp = float(typical_p)
        if not tp > 0.0:
            raise ValueError(f"`typical_p` has to be a float > 0, but is {typical_p}")
        tp = min(tp, 1.0)
    if epsilon_cutoff is not None and 0.0 < float(epsilon_cutoff) < 1.0:
        eps = float(epsilon_cutoff)
    if eta_cutoff is not None and 0.0 < float(eta_cutoff) < 1.0:
        eta = float(eta_cutoff)
    return (mp, tp, eps, eta)


def cutoffs_on(cutoffs) -> bool:
    """Whether a (min_p, typical_p, epsilon, eta) tuple has a cut-off on (None: off)."""
    if cutoffs is None:
        return False
    mp, tp, eps, eta = (float(v) for v in cutoffs)
    return mp > 0.0 or tp < 1.0 or eps > 0.0 or eta > 0.0


def sample(logits: torch.Tensor, temperature: float, top_k: int, u: torch.Tensor, step_idx: Optional[torch.Tensor] = None,
           out: Optional[torch.Tensor] = None, top_p: float = 1.0, cutoffs=None) -> torch.Tensor:
    """logits [B, V] fp32, u [steps, B] (or [B]) uniforms in [0, 1) -> sampled ids [B] int64.  ``top_p < 1`` adds nucleus
    filtering after the top-k cut (``uvx_sample_top_p``); ``top_p >= 1`` is plain ``uvx_sample``.  ``cutoffs`` =
    (min_p, typical_p, epsilon, eta) with one of them on adds those cuts after top-p (``uvx_sample_cutoffs``)."""
    _cuda(logits, torch.float32, "logits"), _cuda(u, torch.float32, "u")
    B, V = logits.shape
    if out is None:
        out = torch.empty(B, dtype=torch.int64, device=logits.device)
    u_stride = u.stride(0) if u.dim() == 2 else 0
    if cutoffs_on(cutoffs):
        check(lib().uvx_sample_cutoffs(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p),
                                       _lib.Cutoffs(*(float(v) for v in cutoffs)), u.data_ptr(), _p(step_idx), u_stride,
                                       out.data_ptr(), _stream()), "uvx_sample_cutoffs")
    elif top_p >= 1.0:
        check(lib().uvx_sample(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), u.data_ptr(), _p(step_idx), u_stride,
                               out.data_ptr(), _stream()), "uvx_sample")
    else:
        check(lib().uvx_sample_top_p(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p), u.data_ptr(),
                                     _p(step_idx), u_stride, out.data_ptr(), _stream()), "uvx_sample_top_p")
    return out


def token_finish(tok: torch.Tensor, done: torch.Tensor, eos_ids: Optional[torch.Tensor], pad_id: int, seq: Optional[torch.Tensor],
                 cur_len: torch.Tensor, step_idx: Optional[torch.Tensor] = None, bumps: tuple = (),
                 all_done: Optional[torch.Tensor] = None, stop: Optional[tuple] = None) -> None:
    """``uvx_token_finish``; ``stop`` = (hit [B] int32, fin_len [B] int32): ``uvx_token_finish_stop``, where a row with hit[b]
    finishes too and a row finishing in this step gets fin_len[b] = its length."""
    _cuda(tok, torch.int64, "tok"), _cuda(done, torch.int32, "done")
    b = list(bumps) + [None] * (3 - len(bumps))
    args = (tok.data_ptr(), done.data_ptr(), _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(), int(pad_id), _p(seq),
            seq.stride(0) if seq is not None else 0, cur_len.data_ptr(), _p(step_idx), _p(b[0]), _p(b[1]), _p(b[2]), _p(all_done),
            tok.numel())
    if stop is None:
        check(lib().uvx_token_finish(*args, _stream()), "uvx_token_finish")
        return
    B = tok.numel()
    hit, fin_len = _rows(stop[0], torch.int32, B, "hit"), _rows(stop[1], torch.int32, B, "fin_len")
    check(lib().uvx_token_finish_stop(*args, hit.data_ptr(), fin_len.data_ptr(), _stream()), "uvx_token_finish_stop")


# ------------------------------------------------------------------------------------------ continuous batching (slots)
def _rows(t: torch.Tensor, dtype, B: int, name: str) -> torch.Tensor:
    """A contiguous per-row device array [B] of ``dtype``."""
    _cuda(t, dtype, name)
    if t.shape != (B,) or not t.is_contiguous():
        raise ValueError(f"{name} must be a contiguous [{B}] tensor, got {tuple(t.shape)}")
    return t


def _seq_rows(t: torch.Tensor, dtype, B: int, name: str) -> torch.Tensor:
    """A [B, W] device tensor with unit column stride (its row stride is passed to the kernel)."""
    _cuda(t, dtype, name)
    if t.dim() != 2 or t.shape[0] != B or t.stride(1) != 1:
        raise ValueError(f"{name} must be [{B}, W] with unit column stride, got {tuple(t.shape)} strides {t.stride()}")
    return t


def sample_slots(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor, u: torch.Tensor,
                 n_new: torch.Tensor, active: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """Per-row pick of ``uvx_sample_slots``: logits [B, V] fp32, temperature / top_p [B] fp32, top_k [B] int32, u [B, W] fp32
    (row b reads u[b, n_new[b]]), n_new / active [B] int32 -> out [B] int64 (inactive rows untouched)."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _rows(temperature, torch.float32, B, "temperature"), _rows(top_k, torch.int32, B, "top_k"), _rows(top_p, torch.float32, B, "top_p")
    _rows(n_new, torch.int32, B, "n_new"), _rows(active, torch.int32, B, "active"), _rows(out, torch.int64, B, "out")
    _seq_rows(u, torch.float32, B, "u")
    check(lib().uvx_sample_slots(logits.data_ptr(), B, V, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), u.data_ptr(),
                                 u.stride(0), n_new.data_ptr(), active.data_ptr(), out.data_ptr(), _stream()), "uvx_sample_slots")
    return out


def _cutoff_rows(cutoffs: torch.Tensor, S: int) -> torch.Tensor:
    """A contiguous per-slot cut-off array [S, 4] fp32 on the device: (min_p, typical_p, epsilon, eta), off = (0, 1, 0, 0)."""
    _cuda(cutoffs, torch.float32, "cutoffs")
    if cutoffs.shape != (S, 4) or not cutoffs.is_contiguous():
        raise ValueError(f"cutoffs must be a contiguous [{S}, 4] tensor, got {tuple(cutoffs.shape)}")
    return cutoffs


def sample_slots_cutoffs(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                         cutoffs: torch.Tensor, u: torch.Tensor, n_new: torch.Tensor, active: torch.Tensor,
                         out: torch.Tensor) -> torch.Tensor:
    """``uvx_sample_slots_cutoffs``: ``sample_slots`` with row b's cut-offs cutoffs[b] ([B, 4] fp32, off = (0, 1, 0, 0))."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _rows(temperature, torch.float32, B, "temperature"), _rows(top_k, torch.int32, B, "top_k"), _rows(top_p, torch.float32, B, "top_p")
    _rows(n_new, torch.int32, B, "n_new"), _rows(active, torch.int32, B, "active"), _rows(out, torch.int64, B, "out")
    _seq_rows(u, torch.float32, B, "u"), _cutoff_rows(cutoffs, B)
    check(lib().uvx_sample_slots_cutoffs(logits.data_ptr(), B, V, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(),
                                         cutoffs.data_ptr(), u.data_ptr(), u.stride(0), n_new.data_ptr(), active.data_ptr(),
                                         out.data_ptr(), _stream()), "uvx_sample_slots_cutoffs")
    return out


def repetition_penalty_slots_(logits: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, penalty: torch.Tensor,
                              active: torch.Tensor, scratch: torch.Tensor) -> torch.Tensor:
    """HF's repetition penalty on each active row b with penalty[b] over seq[b, :cur_len[b]], in place on logits [B, V] fp32;
    scratch is fp32 [B, >= seq.stride(0)]."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _seq_rows(seq, torch.int64, B, "seq")
    _rows(cur_len, torch.int32, B, "cur_len"), _rows(penalty, torch.float32, B, "penalty"), _rows(active, torch.int32, B, "active")
    _seq_rows(scratch, torch.float32, B, "scratch")
    if scratch.stride(0) < seq.stride(0) or scratch.shape[1] < seq.shape[1]:
        raise ValueError("scratch rows must be at least as long as the seq rows")
    if scratch.stride(0) != seq.stride(0):
        raise ValueError("scratch and seq must share a row stride")
    check(lib().uvx_repetition_penalty_slots(logits.data_ptr(), B, V, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(), penalty.data_ptr(),
                                             active.data_ptr(), scratch.data_ptr(), _stream()), "uvx_repetition_penalty_slots")
    return logits


def slot_finish(tok: torch.Tensor, done: torch.Tensor, eos_ids: Optional[torch.Tensor], seq: torch.Tensor, cur_len: torch.Tensor,
                n_new: torch.Tensor, max_new: torch.Tensor, active: torch.Tensor, pos: torch.Tensor, lens: torch.Tensor,
                rope_pos: torch.Tensor, n_open: torch.Tensor, hit: Optional[torch.Tensor] = None) -> None:
    """``uvx_slot_finish``: tok [B] int64, seq [B, W] int64, every other per-row array [B] int32, eos_ids int64 or None,
    n_open [1] int32 (the count of active rows still open).  ``hit`` [B] int32: ``uvx_slot_finish_stop`` (a hit finishes the
    row as an EOS id does)."""
    B = tok.numel()
    _rows(tok, torch.int64, B, "tok"), _seq_rows(seq, torch.int64, B, "seq")
    for t, name in ((done, "done"), (cur_len, "cur_len"), (n_new, "n_new"), (max_new, "max_new"), (active, "active"), (pos, "pos"),
                    (lens, "lens"), (rope_pos, "rope_pos")):
        _rows(t, torch.int32, B, name)
    _rows(n_open, torch.int32, 1, "n_open")
    if eos_ids is not None:
        _cuda(eos_ids, torch.int64, "eos_ids")
    args = (tok.data_ptr(), done.data_ptr(), _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(), seq.data_ptr(), seq.stride(0),
            cur_len.data_ptr(), n_new.data_ptr(), max_new.data_ptr(), active.data_ptr(), pos.data_ptr(), lens.data_ptr(),
            rope_pos.data_ptr(), n_open.data_ptr(), B)
    if hit is None:
        check(lib().uvx_slot_finish(*args, _stream()), "uvx_slot_finish")
    else:
        check(lib().uvx_slot_finish_stop(*args, _rows(hit, torch.int32, B, "hit").data_ptr(), _stream()), "uvx_slot_finish_stop")


# ------------------------------------------------------------------------------------------ log-probabilities
LOGPROBS_MAX = 20   # alternatives per token (kLogprobsMax in generate.cu)


def token_logprobs(logits: torch.Tensor, tok: torch.Tensor, n_top: torch.Tensor, dst: torch.Tensor, out_lp: torch.Tensor,
                   out_ids: Optional[torch.Tensor] = None, out_top: Optional[torch.Tensor] = None) -> None:
    """``uvx_token_logprobs``: raw logits [B, V] fp32, chosen tokens [B] int64, n_top / dst [B] int32 -> at index dst[b] of
    row b: out_lp [B, cap] fp32 = log_softmax(logits[b])[tok[b]], out_ids [B, cap, n_max] int64 / out_top [B, cap, n_max] fp32 =
    the n_top[b] largest entries (value desc, index asc) and their log-probs.  Rows with n_top < 0 are not touched."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _rows(tok, torch.int64, B, "tok"), _rows(n_top, torch.int32, B, "n_top"), _rows(dst, torch.int32, B, "dst")
    _cuda(out_lp, torch.float32, "out_lp")
    if out_lp.dim() != 2 or out_lp.shape[0] != B or not out_lp.is_contiguous():
        raise ValueError(f"out_lp must be a contiguous [{B}, cap] tensor, got {tuple(out_lp.shape)}")
    cap = out_lp.shape[1]
    n_max = 0
    if out_ids is not None or out_top is not None:
        _cuda(out_ids, torch.int64, "out_ids"), _cuda(out_top, torch.float32, "out_top")
        n_max = out_ids.shape[-1]
        for t, name in ((out_ids, "out_ids"), (out_top, "out_top")):
            if t.shape != (B, cap, n_max) or not t.is_contiguous():
                raise ValueError(f"{name} must be a contiguous [{B}, {cap}, n_max] tensor, got {tuple(t.shape)}")
    check(lib().uvx_token_logprobs(logits.data_ptr(), B, V, tok.data_ptr(), n_top.data_ptr(), dst.data_ptr(), cap, n_max,
                                   out_lp.data_ptr(), _p(out_ids), _p(out_top), _stream()), "uvx_token_logprobs")


def record_scores(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, step_idx: torch.Tensor,
                  scores: Optional[torch.Tensor] = None, raw: Optional[torch.Tensor] = None, cutoffs=None) -> None:
    """``uvx_record_scores``: logits [B, V] fp32 -> at step s = step_idx[0] of the [steps, B, V] fp32 buffers, raw[s] = the
    logits as given and scores[s] = HF's processed scores (temperature <= 0: the logits; else x / temperature on the entries the
    sampler keeps with top_k / top_p and, when on, the (min_p, typical_p, epsilon, eta) ``cutoffs``; -inf elsewhere)."""
    _cuda(logits, torch.float32, "logits"), _cuda(step_idx, torch.int32, "step_idx")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    steps = None
    for t, name in ((scores, "scores"), (raw, "raw")):
        if t is not None:
            _cuda(t, torch.float32, name)
            if t.dim() != 3 or t.shape[1:] != (B, V) or not t.is_contiguous() or (steps is not None and t.shape[0] != steps):
                raise ValueError(f"{name} must be a contiguous [steps, {B}, {V}] tensor, got {tuple(t.shape)}")
            steps = t.shape[0]
    if steps is None:
        raise ValueError("record_scores needs scores, raw or both")
    if cutoffs_on(cutoffs):
        check(lib().uvx_record_scores_cutoffs(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p),
                                              _lib.Cutoffs(*(float(v) for v in cutoffs)), step_idx.data_ptr(), steps, _p(scores),
                                              _p(raw), _stream()), "uvx_record_scores_cutoffs")
        return
    check(lib().uvx_record_scores(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p), step_idx.data_ptr(),
                                  steps, _p(scores), _p(raw), _stream()), "uvx_record_scores")


def record_scores_rows(logits: torch.Tensor, temperature: float, top_k: int, top_p: float, idx: torch.Tensor,
                       scores: Optional[torch.Tensor] = None, raw: Optional[torch.Tensor] = None, cutoffs=None) -> None:
    """``uvx_record_scores_rows``: ``record_scores`` with per-row destinations - row b of logits [B, V] fp32 goes to index
    s = idx[b] ([B] int32) of the [steps, V] fp32 buffers (nothing when s is outside [0, steps)).  ``cutoffs`` as in
    ``record_scores`` (``uvx_record_scores_rows_cutoffs``)."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _rows(idx, torch.int32, B, "idx")
    steps = None
    for t, name in ((scores, "scores"), (raw, "raw")):
        if t is not None:
            _cuda(t, torch.float32, name)
            if t.dim() != 2 or t.shape[1] != V or not t.is_contiguous() or (steps is not None and t.shape[0] != steps):
                raise ValueError(f"{name} must be a contiguous [steps, {V}] tensor, got {tuple(t.shape)}")
            steps = t.shape[0]
    if steps is None:
        raise ValueError("record_scores_rows needs scores, raw or both")
    if cutoffs_on(cutoffs):
        check(lib().uvx_record_scores_rows_cutoffs(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p),
                                                   _lib.Cutoffs(*(float(v) for v in cutoffs)), idx.data_ptr(), steps, _p(scores),
                                                   _p(raw), _stream()), "uvx_record_scores_rows_cutoffs")
        return
    check(lib().uvx_record_scores_rows(logits.data_ptr(), B, V, float(temperature), int(top_k or 0), float(top_p), idx.data_ptr(),
                                       steps, _p(scores), _p(raw), _stream()), "uvx_record_scores_rows")


# ------------------------------------------------------------------------------------------ prompt lookup
LOOKUP_MAX_K = 31   # drafts per step (kLookupMaxK in generate.cu): k + 1 rows within the decode-form GEMM's 32


def repetition_penalty_rows_(logits: torch.Tensor, seq: torch.Tensor, lens: torch.Tensor, penalty: float,
                             scratch: torch.Tensor) -> torch.Tensor:
    """``uvx_repetition_penalty_rows``: HF's repetition penalty on row b of logits [B, V] fp32 over seq[b, :lens[b]], in place.
    seq [B, W] int64 with unit column stride and any row stride (0: the rows share one sequence, e.g. ``s.expand(B, -1)``),
    lens [B] int32, scratch fp32 [B, >= W] with its own rows."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    B, V = logits.shape
    _seq_rows(seq, torch.int64, B, "seq"), _rows(lens, torch.int32, B, "lens"), _seq_rows(scratch, torch.float32, B, "scratch")
    if scratch.shape[1] < seq.shape[1] or (B > 1 and scratch.stride(0) < scratch.shape[1]):
        raise ValueError("scratch must have its own row of at least seq.shape[1] entries per row")
    if not float(penalty) > 0.0:
        raise ValueError(f"penalty must be > 0, got {penalty}")
    check(lib().uvx_repetition_penalty_rows(logits.data_ptr(), B, V, seq.data_ptr(), seq.stride(0), lens.data_ptr(), float(penalty),
                                            scratch.data_ptr(), scratch.stride(0), _stream()), "uvx_repetition_penalty_rows")
    return logits


def _constraint_table(table, settings: Optional[int]):
    """(cfg, ids, end, bias, kind) of ``constraints.LogitsConstraints.tables``: one setting (``settings`` None: cfg [4], the
    rest [T]) or ``settings`` of them (cfg [settings, 4], the rest [settings, T]), contiguous -> (pointers, T)."""
    cfg, ids, end, bias, kind = table
    lead = () if settings is None else (settings,)
    _cuda(cfg, torch.int32, "cfg")
    if tuple(cfg.shape) != lead + (4,) or not cfg.is_contiguous():
        raise ValueError(f"cfg must be a contiguous {lead + (4,)} tensor, got {tuple(cfg.shape)}")
    T = ids.shape[-1]
    for t, dt, name in ((ids, torch.int64, "ids"), (end, torch.int32, "end"), (bias, torch.float32, "bias"),
                        (kind, torch.int32, "kind")):
        _cuda(t, dt, name)
        if tuple(t.shape) != lead + (T,) or not t.is_contiguous() or T < 1:
            raise ValueError(f"{name} must be a contiguous {lead + (T,)} tensor (T >= 1), got {tuple(t.shape)}")
    return (cfg.data_ptr(), ids.data_ptr(), end.data_ptr(), bias.data_ptr(), kind.data_ptr()), T


def _logits_rows(logits: torch.Tensor):
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [B, V] tensor")
    return logits.shape


def logits_constraints_(logits: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, table) -> torch.Tensor:
    """``uvx_logits_constraints``: the token constraints of one setting ``table`` on every row b of logits [B, V] fp32 over
    seq[b, :cur_len[0]], in place (before the repetition penalty)."""
    B, V = _logits_rows(logits)
    _seq_rows(seq, torch.int64, B, "seq"), _rows(cur_len, torch.int32, 1, "cur_len")
    p, _ = _constraint_table(table, None)
    check(lib().uvx_logits_constraints(logits.data_ptr(), B, V, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(), *p, _stream()),
          "uvx_logits_constraints")
    return logits


def logits_constraints_slots_(logits: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, active: torch.Tensor,
                              table) -> torch.Tensor:
    """``uvx_logits_constraints_slots``: active row b with its own setting b of ``table`` (cfg [B, 4], the rest [B, T]) over
    seq[b, :cur_len[b]], in place."""
    B, V = _logits_rows(logits)
    _seq_rows(seq, torch.int64, B, "seq"), _rows(cur_len, torch.int32, B, "cur_len"), _rows(active, torch.int32, B, "active")
    p, T = _constraint_table(table, B)
    check(lib().uvx_logits_constraints_slots(logits.data_ptr(), B, V, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(),
                                             active.data_ptr(), *p, T, _stream()), "uvx_logits_constraints_slots")
    return logits


def logits_constraints_rows_(logits: torch.Tensor, seq: torch.Tensor, lens: torch.Tensor, table) -> torch.Tensor:
    """``uvx_logits_constraints_rows``: one setting on row b over seq[b, :lens[b]] (seq's row stride may be 0: one shared
    sequence), in place."""
    R, V = _logits_rows(logits)
    _seq_rows(seq, torch.int64, R, "seq"), _rows(lens, torch.int32, R, "lens")
    p, _ = _constraint_table(table, None)
    check(lib().uvx_logits_constraints_rows(logits.data_ptr(), R, V, seq.data_ptr(), seq.stride(0), lens.data_ptr(), *p, _stream()),
          "uvx_logits_constraints_rows")
    return logits


def logits_constraints_rows_map_(logits: torch.Tensor, seq: torch.Tensor, active: torch.Tensor, row_slot: torch.Tensor,
                                 row_len: torch.Tensor, row_idx: torch.Tensor, table) -> torch.Tensor:
    """``uvx_logits_constraints_rows_map``: row r with slot s = row_slot[r]'s setting over seq[s, :row_len[r]]; rows of inactive
    slots or with row_idx[r] < 0 untouched.  seq [slots, W], active [slots], table of ``slots`` settings, row arrays [R]."""
    R, V = _logits_rows(logits)
    S = seq.shape[0]
    _seq_rows(seq, torch.int64, S, "seq"), _rows(active, torch.int32, S, "active")
    for t, name in ((row_slot, "row_slot"), (row_len, "row_len"), (row_idx, "row_idx")):
        _rows(t, torch.int32, R, name)
    p, T = _constraint_table(table, S)
    check(lib().uvx_logits_constraints_rows_map(logits.data_ptr(), R, V, seq.data_ptr(), seq.stride(0), active.data_ptr(),
                                                row_slot.data_ptr(), row_len.data_ptr(), row_idx.data_ptr(), *p, T, _stream()),
          "uvx_logits_constraints_rows_map")
    return logits


# ------------------------------------------------------------------------------------------ stop strings
from .stop_strings import HEADER as STOP_HEADER     # noqa: E402  (the table header's words, kStopHdr in generate.cu)


def _stop_table(tab: torch.Tensor, rows: Optional[int] = None) -> torch.Tensor:
    """A packed stop-string table (``stop_strings.StopStrings``): int32 [W] (one) or [rows, W] (one per slot), contiguous."""
    _cuda(tab, torch.int32, "stop table")
    if not tab.is_contiguous() or (rows is None and tab.dim() != 1) or (rows is not None and (tab.dim() != 2 or tab.shape[0] != rows)):
        raise ValueError(f"the stop table must be a contiguous int32 {'[W]' if rows is None else f'[{rows}, W]'} tensor, got "
                         f"{tuple(tab.shape)}")
    if tab.shape[-1] < STOP_HEADER:
        raise ValueError(f"a stop table holds at least its {STOP_HEADER}-word header")
    return tab


def stop_strings(tok: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, table: torch.Tensor, hit: torch.Tensor) -> torch.Tensor:
    """``uvx_stop_strings``: hit[b] = whether candidate tok[b] after seq[b, :cur_len[0]] ends a stop string of ``table``."""
    B = tok.numel()
    _rows(tok, torch.int64, B, "tok"), _seq_rows(seq, torch.int64, B, "seq"), _rows(hit, torch.int32, B, "hit")
    _rows(cur_len, torch.int32, 1, "cur_len"), _stop_table(table)
    check(lib().uvx_stop_strings(tok.data_ptr(), B, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(), table.data_ptr(), hit.data_ptr(),
                                 _stream()), "uvx_stop_strings")
    return hit


def stop_strings_beam(cand_i: torch.Tensor, V: int, num_beams: int, run_seq: torch.Tensor, cur_len: torch.Tensor,
                      table: torch.Tensor, hit: torch.Tensor) -> torch.Tensor:
    """``uvx_stop_strings_beam``: candidate c of prompt b (cand_i [B, K] int64 = parent beam * V + token) after its parent's
    running sequence run_seq[b * num_beams + parent, :cur_len[0]] -> hit [B * K] int32."""
    _cuda(cand_i, torch.int64, "cand_i")
    if cand_i.dim() != 2 or not cand_i.is_contiguous():
        raise ValueError("cand_i must be a contiguous [B, K] tensor")
    B, K = cand_i.shape
    _seq_rows(run_seq, torch.int64, B * int(num_beams), "run_seq"), _rows(cur_len, torch.int32, 1, "cur_len")
    _rows(hit, torch.int32, B * K, "hit"), _stop_table(table)
    check(lib().uvx_stop_strings_beam(cand_i.data_ptr(), B, int(num_beams), K, int(V), run_seq.data_ptr(), run_seq.stride(0),
                                      cur_len.data_ptr(), table.data_ptr(), hit.data_ptr(), _stream()), "uvx_stop_strings_beam")
    return hit


def stop_strings_slots(tok: torch.Tensor, seq: torch.Tensor, cur_len: torch.Tensor, active: torch.Tensor, table: torch.Tensor,
                       hit: torch.Tensor) -> torch.Tensor:
    """``uvx_stop_strings_slots``: active row b after seq[b, :cur_len[b]] with its own table[b] ([B, W] int32); inactive rows'
    hit untouched."""
    B = tok.numel()
    _rows(tok, torch.int64, B, "tok"), _seq_rows(seq, torch.int64, B, "seq"), _rows(hit, torch.int32, B, "hit")
    _rows(cur_len, torch.int32, B, "cur_len"), _rows(active, torch.int32, B, "active"), _stop_table(table, B)
    check(lib().uvx_stop_strings_slots(tok.data_ptr(), B, seq.data_ptr(), seq.stride(0), cur_len.data_ptr(), active.data_ptr(),
                                       table.data_ptr(), table.stride(0), hit.data_ptr(), _stream()), "uvx_stop_strings_slots")
    return hit


def stop_strings_rows(tok: torch.Tensor, seq: torch.Tensor, lens: torch.Tensor, table: torch.Tensor, hit: torch.Tensor) -> torch.Tensor:
    """``uvx_stop_strings_rows``: row r after seq[r, :lens[r]] (seq's row stride may be 0: one shared sequence), one table."""
    R = tok.numel()
    _rows(tok, torch.int64, R, "tok"), _rows(lens, torch.int32, R, "lens"), _rows(hit, torch.int32, R, "hit"), _stop_table(table)
    _cuda(seq, torch.int64, "seq")
    if seq.dim() != 2 or seq.shape[0] != R or seq.stride(1) != 1:
        raise ValueError(f"seq must be [{R}, W] with unit column stride (row stride 0 allowed), got {tuple(seq.shape)}")
    check(lib().uvx_stop_strings_rows(tok.data_ptr(), R, seq.data_ptr(), seq.stride(0), lens.data_ptr(), table.data_ptr(), hit.data_ptr(),
                                      _stream()), "uvx_stop_strings_rows")
    return hit


def stop_strings_rows_map(tok: torch.Tensor, seq: torch.Tensor, active: torch.Tensor, row_slot: torch.Tensor, row_len: torch.Tensor,
                          row_idx: torch.Tensor, table: torch.Tensor, hit: torch.Tensor) -> torch.Tensor:
    """``uvx_stop_strings_rows_map``: row r of slot s = row_slot[r] after seq[s, :row_len[r]] with table[s]; rows of inactive
    slots or with row_idx[r] < 0 untouched."""
    R, S = tok.numel(), active.numel()
    _rows(tok, torch.int64, R, "tok"), _seq_rows(seq, torch.int64, S, "seq"), _rows(active, torch.int32, S, "active")
    for t, name in ((row_slot, "row_slot"), (row_len, "row_len"), (row_idx, "row_idx"), (hit, "hit")):
        _rows(t, torch.int32, R, name)
    _stop_table(table, S)
    check(lib().uvx_stop_strings_rows_map(tok.data_ptr(), R, seq.data_ptr(), seq.stride(0), active.data_ptr(), row_slot.data_ptr(),
                                          row_len.data_ptr(), row_idx.data_ptr(), table.data_ptr(), table.stride(0), hit.data_ptr(),
                                          _stream()), "uvx_stop_strings_rows_map")
    return hit


def lookup_draft(seq: torch.Tensor, cur_len: torch.Tensor, n_new: torch.Tensor, max_new: int, k: int, n: int,
                 eos_ids: Optional[torch.Tensor], done: torch.Tensor, tok: torch.Tensor, n_draft: torch.Tensor, pos: torch.Tensor,
                 lens: torch.Tensor, rope_pos: torch.Tensor, pen_len: torch.Tensor, idx: torch.Tensor) -> None:
    """``uvx_lookup_draft`` (include/uvx.h): prompt-lookup drafts for the sequence seq [W] int64 (its first cur_len[0] tokens)
    -> the k + 1 fed tokens tok [k + 1] int64, n_draft [1], the per-row pos / lens / rope_pos / pen_len / idx [k + 1] int32, and
    the drafts into seq[cur_len : cur_len + n_draft].  cur_len / n_new / done are [1] int32 device counters."""
    if not 1 <= int(k) <= LOOKUP_MAX_K:
        raise ValueError(f"k must be in [1, {LOOKUP_MAX_K}], got {k}")
    if int(n) < 1:
        raise ValueError(f"n must be >= 1, got {n}")
    if int(max_new) < 1:
        raise ValueError(f"max_new must be >= 1, got {max_new}")
    _cuda(seq, torch.int64, "seq")
    if seq.dim() != 1 or not seq.is_contiguous():
        raise ValueError("seq must be a contiguous [W] tensor")
    R = int(k) + 1
    for t, name in ((cur_len, "cur_len"), (n_new, "n_new"), (done, "done"), (n_draft, "n_draft")):
        _rows(t, torch.int32, 1, name)
    _rows(tok, torch.int64, R, "tok")
    for t, name in ((pos, "pos"), (lens, "lens"), (rope_pos, "rope_pos"), (pen_len, "pen_len"), (idx, "idx")):
        _rows(t, torch.int32, R, name)
    if eos_ids is not None:
        _cuda(eos_ids, torch.int64, "eos_ids")
    check(lib().uvx_lookup_draft(seq.data_ptr(), cur_len.data_ptr(), n_new.data_ptr(), int(max_new), int(k), int(n), _p(eos_ids),
                                 0 if eos_ids is None else eos_ids.numel(), done.data_ptr(), tok.data_ptr(), n_draft.data_ptr(),
                                 pos.data_ptr(), lens.data_ptr(), rope_pos.data_ptr(), pen_len.data_ptr(), idx.data_ptr(), _stream()),
          "uvx_lookup_draft")


def lookup_accept(pick: torch.Tensor, tok: torch.Tensor, n_draft: torch.Tensor, eos_ids: Optional[torch.Tensor], seq: torch.Tensor,
                  cur_len: torch.Tensor, n_new: torch.Tensor, max_new: int, done: torch.Tensor, step: Optional[torch.Tensor] = None,
                  accepted: Optional[torch.Tensor] = None, hit: Optional[torch.Tensor] = None) -> None:
    """``uvx_lookup_accept`` (include/uvx.h): picks [R] int64 of the rows that fed tok [R] int64 (R >= n_draft[0] + 1) -> the
    agreeing prefix plus one token appended to seq [W] int64 at cur_len[0]; cur_len / n_new / done [1] int32 advance.  With
    ``accepted`` ([steps] int32) and ``step`` ([1] int32) the step's accepted draft count is logged at step[0].  ``hit`` [R]
    int32: ``uvx_lookup_accept_stop``, the accept cut at the first row with a stop-string hit."""
    R = pick.numel()
    if not 1 <= R <= LOOKUP_MAX_K + 1:
        raise ValueError(f"pick must hold 1..{LOOKUP_MAX_K + 1} rows, got {R}")
    _rows(pick, torch.int64, R, "pick"), _rows(tok, torch.int64, R, "tok")
    _cuda(seq, torch.int64, "seq")
    if seq.dim() != 1 or not seq.is_contiguous():
        raise ValueError("seq must be a contiguous [W] tensor")
    for t, name in ((n_draft, "n_draft"), (cur_len, "cur_len"), (n_new, "n_new"), (done, "done")):
        _rows(t, torch.int32, 1, name)
    if (step is None) != (accepted is None):
        raise ValueError("step and accepted go together")
    if accepted is not None:
        _rows(step, torch.int32, 1, "step")
        _cuda(accepted, torch.int32, "accepted")
        if accepted.dim() != 1 or not accepted.is_contiguous():
            raise ValueError("accepted must be a contiguous [steps] tensor")
    if int(max_new) < 1:
        raise ValueError(f"max_new must be >= 1, got {max_new}")
    if eos_ids is not None:
        _cuda(eos_ids, torch.int64, "eos_ids")
    args = (pick.data_ptr(), tok.data_ptr(), n_draft.data_ptr(), _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(),
            seq.data_ptr(), cur_len.data_ptr(), n_new.data_ptr(), int(max_new), _p(step), _p(accepted),
            0 if accepted is None else accepted.numel(), done.data_ptr())
    if hit is None:
        check(lib().uvx_lookup_accept(*args, _stream()), "uvx_lookup_accept")
    else:
        check(lib().uvx_lookup_accept_stop(*args, _rows(hit, torch.int32, R, "hit").data_ptr(), _stream()), "uvx_lookup_accept_stop")


# ------------------------------------------------------------------------------------------ prompt lookup in slots
def lookup_draft_slots(seq: torch.Tensor, token: torch.Tensor, cur_len: torch.Tensor, n_new: torch.Tensor, max_new: torch.Tensor,
                       k: torch.Tensor, n: torch.Tensor, done: torch.Tensor, active: torch.Tensor, prefilling: torch.Tensor,
                       pos: torch.Tensor, lens: torch.Tensor, rope_pos: torch.Tensor, K: int, eos_ids: Optional[torch.Tensor],
                       tok: torch.Tensor, n_draft: torch.Tensor, row_pos: torch.Tensor, row_lens: torch.Tensor, row_rope: torch.Tensor,
                       pen_len: torch.Tensor, idx: torch.Tensor, row_slot: torch.Tensor, cache_row: torch.Tensor) -> None:
    """``uvx_lookup_draft_slots`` (include/uvx.h): the drafts of every slot and the R = slots * (K + 1) rows of a lookup step.
    seq [slots, W] int64, token [slots] int64 and the other per-slot arrays [slots] int32 in; tok [R] int64, n_draft [slots],
    row_pos / row_lens / row_rope / pen_len / idx / row_slot / cache_row [R] int32 out."""
    S = cur_len.shape[0]
    if not 1 <= int(K) <= LOOKUP_MAX_K:
        raise ValueError(f"K must be in [1, {LOOKUP_MAX_K}], got {K}")
    R = S * (int(K) + 1)
    _seq_rows(seq, torch.int64, S, "seq"), _rows(token, torch.int64, S, "token")
    for t, name in ((cur_len, "cur_len"), (n_new, "n_new"), (max_new, "max_new"), (k, "k"), (n, "n"), (done, "done"),
                    (active, "active"), (prefilling, "prefilling"), (pos, "pos"), (lens, "lens"), (rope_pos, "rope_pos"),
                    (n_draft, "n_draft")):
        _rows(t, torch.int32, S, name)
    _rows(tok, torch.int64, R, "tok")
    for t, name in ((row_pos, "row_pos"), (row_lens, "row_lens"), (row_rope, "row_rope"), (pen_len, "pen_len"), (idx, "idx"),
                    (row_slot, "row_slot"), (cache_row, "cache_row")):
        _rows(t, torch.int32, R, name)
    if eos_ids is not None:
        _cuda(eos_ids, torch.int64, "eos_ids")
    check(lib().uvx_lookup_draft_slots(seq.data_ptr(), seq.stride(0), token.data_ptr(), cur_len.data_ptr(), n_new.data_ptr(),
                                       max_new.data_ptr(), k.data_ptr(), n.data_ptr(), done.data_ptr(), active.data_ptr(),
                                       prefilling.data_ptr(), pos.data_ptr(), lens.data_ptr(), rope_pos.data_ptr(), S, int(K),
                                       _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(), tok.data_ptr(), n_draft.data_ptr(),
                                       row_pos.data_ptr(), row_lens.data_ptr(), row_rope.data_ptr(), pen_len.data_ptr(), idx.data_ptr(),
                                       row_slot.data_ptr(), cache_row.data_ptr(), _stream()), "uvx_lookup_draft_slots")


def lookup_accept_slots(pick: torch.Tensor, tok: torch.Tensor, n_draft: torch.Tensor, K: int, eos_ids: Optional[torch.Tensor],
                        seq: torch.Tensor, token: torch.Tensor, done: torch.Tensor, cur_len: torch.Tensor, n_new: torch.Tensor,
                        max_new: torch.Tensor, active: torch.Tensor, pos: torch.Tensor, lens: torch.Tensor, rope_pos: torch.Tensor,
                        accepted: torch.Tensor, n_open: torch.Tensor, hit: Optional[torch.Tensor] = None) -> None:
    """``uvx_lookup_accept_slots`` (include/uvx.h): picks [R] int64 of the rows that fed tok [R] -> each open slot's agreeing
    drafts plus one token appended to seq [slots, W] int64 with ``uvx_slot_finish``'s bookkeeping; accepted [slots] += m.
    ``hit`` [R] int32: ``uvx_lookup_accept_slots_stop``, each slot's accept cut at its first row with a stop-string hit."""
    S = cur_len.shape[0]
    if not 1 <= int(K) <= LOOKUP_MAX_K:
        raise ValueError(f"K must be in [1, {LOOKUP_MAX_K}], got {K}")
    R = S * (int(K) + 1)
    _rows(pick, torch.int64, R, "pick"), _rows(tok, torch.int64, R, "tok")
    _seq_rows(seq, torch.int64, S, "seq"), _rows(token, torch.int64, S, "token")
    for t, name in ((n_draft, "n_draft"), (done, "done"), (cur_len, "cur_len"), (n_new, "n_new"), (max_new, "max_new"),
                    (active, "active"), (pos, "pos"), (lens, "lens"), (rope_pos, "rope_pos"), (accepted, "accepted")):
        _rows(t, torch.int32, S, name)
    _rows(n_open, torch.int32, 1, "n_open")
    if eos_ids is not None:
        _cuda(eos_ids, torch.int64, "eos_ids")
    args = (pick.data_ptr(), tok.data_ptr(), n_draft.data_ptr(), S, int(K), _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(),
            seq.data_ptr(), seq.stride(0), token.data_ptr(), done.data_ptr(), cur_len.data_ptr(), n_new.data_ptr(),
            max_new.data_ptr(), active.data_ptr(), pos.data_ptr(), lens.data_ptr(), rope_pos.data_ptr(), accepted.data_ptr(),
            n_open.data_ptr())
    if hit is None:
        check(lib().uvx_lookup_accept_slots(*args, _stream()), "uvx_lookup_accept_slots")
    else:
        check(lib().uvx_lookup_accept_slots_stop(*args, _rows(hit, torch.int32, R, "hit").data_ptr(), _stream()),
              "uvx_lookup_accept_slots_stop")


def sample_rows(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor, u: torch.Tensor,
                active: torch.Tensor, row_slot: torch.Tensor, row_idx: torch.Tensor, out: torch.Tensor) -> torch.Tensor:
    """``uvx_sample_rows``: ``sample_slots`` per row r of logits [R, V] with slot row_slot[r]'s settings (per-slot arrays [slots],
    u [slots, W]) and its uniform at row_idx[r] -> out [R] int64 (rows with row_idx < 0 or an inactive slot untouched)."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [R, V] tensor")
    R, V = logits.shape
    S = temperature.shape[0]
    _rows(temperature, torch.float32, S, "temperature"), _rows(top_k, torch.int32, S, "top_k"), _rows(top_p, torch.float32, S, "top_p")
    _rows(active, torch.int32, S, "active"), _seq_rows(u, torch.float32, S, "u")
    _rows(row_slot, torch.int32, R, "row_slot"), _rows(row_idx, torch.int32, R, "row_idx"), _rows(out, torch.int64, R, "out")
    check(lib().uvx_sample_rows(logits.data_ptr(), R, V, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(), u.data_ptr(),
                                u.stride(0), active.data_ptr(), row_slot.data_ptr(), row_idx.data_ptr(), out.data_ptr(), _stream()),
          "uvx_sample_rows")
    return out


def sample_rows_cutoffs(logits: torch.Tensor, temperature: torch.Tensor, top_k: torch.Tensor, top_p: torch.Tensor,
                        cutoffs: torch.Tensor, u: torch.Tensor, active: torch.Tensor, row_slot: torch.Tensor, row_idx: torch.Tensor,
                        out: torch.Tensor) -> torch.Tensor:
    """``uvx_sample_rows_cutoffs``: ``sample_rows`` with slot row_slot[r]'s cut-offs (cutoffs [slots, 4] fp32)."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [R, V] tensor")
    R, V = logits.shape
    S = temperature.shape[0]
    _rows(temperature, torch.float32, S, "temperature"), _rows(top_k, torch.int32, S, "top_k"), _rows(top_p, torch.float32, S, "top_p")
    _rows(active, torch.int32, S, "active"), _seq_rows(u, torch.float32, S, "u"), _cutoff_rows(cutoffs, S)
    _rows(row_slot, torch.int32, R, "row_slot"), _rows(row_idx, torch.int32, R, "row_idx"), _rows(out, torch.int64, R, "out")
    check(lib().uvx_sample_rows_cutoffs(logits.data_ptr(), R, V, temperature.data_ptr(), top_k.data_ptr(), top_p.data_ptr(),
                                        cutoffs.data_ptr(), u.data_ptr(), u.stride(0), active.data_ptr(), row_slot.data_ptr(),
                                        row_idx.data_ptr(), out.data_ptr(), _stream()), "uvx_sample_rows_cutoffs")
    return out


def repetition_penalty_rows_map_(logits: torch.Tensor, seq: torch.Tensor, penalty: torch.Tensor, active: torch.Tensor,
                                 row_slot: torch.Tensor, row_len: torch.Tensor, row_idx: torch.Tensor,
                                 scratch: torch.Tensor) -> torch.Tensor:
    """``uvx_repetition_penalty_rows_map``: HF's repetition penalty on row r of logits [R, V] fp32 with slot s = row_slot[r]'s
    penalty over seq[s, :row_len[r]] (seq [slots, W] int64), in place; scratch fp32 [R, >= W] sharing seq's row stride."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [R, V] tensor")
    R, V = logits.shape
    S = penalty.shape[0]
    _seq_rows(seq, torch.int64, S, "seq"), _rows(penalty, torch.float32, S, "penalty"), _rows(active, torch.int32, S, "active")
    for t, name in ((row_slot, "row_slot"), (row_len, "row_len"), (row_idx, "row_idx")):
        _rows(t, torch.int32, R, name)
    _seq_rows(scratch, torch.float32, R, "scratch")
    if scratch.stride(0) != seq.stride(0) or scratch.shape[1] < seq.shape[1]:
        raise ValueError("scratch and seq must share a row stride")
    check(lib().uvx_repetition_penalty_rows_map(logits.data_ptr(), R, V, seq.data_ptr(), seq.stride(0), penalty.data_ptr(),
                                                active.data_ptr(), row_slot.data_ptr(), row_len.data_ptr(), row_idx.data_ptr(),
                                                scratch.data_ptr(), _stream()), "uvx_repetition_penalty_rows_map")
    return logits


def token_logprobs_rows(logits: torch.Tensor, tok: torch.Tensor, n_top: torch.Tensor, row_slot: torch.Tensor, dst: torch.Tensor,
                        out_lp: torch.Tensor, out_ids: Optional[torch.Tensor] = None, out_top: Optional[torch.Tensor] = None) -> None:
    """``uvx_token_logprobs_rows``: ``token_logprobs`` per row r of logits [R, V] with slot s = row_slot[r]'s n_top[s], written to
    slot s's outputs (out_lp [slots, cap], out_ids / out_top [slots, cap, n_max]) at index dst[r] (< 0: nothing)."""
    _cuda(logits, torch.float32, "logits")
    if logits.dim() != 2 or not logits.is_contiguous():
        raise ValueError("logits must be a contiguous [R, V] tensor")
    R, V = logits.shape
    S = n_top.shape[0]
    _rows(tok, torch.int64, R, "tok"), _rows(n_top, torch.int32, S, "n_top"), _rows(row_slot, torch.int32, R, "row_slot")
    _rows(dst, torch.int32, R, "dst")
    _cuda(out_lp, torch.float32, "out_lp")
    if out_lp.dim() != 2 or out_lp.shape[0] != S or not out_lp.is_contiguous():
        raise ValueError(f"out_lp must be a contiguous [{S}, cap] tensor, got {tuple(out_lp.shape)}")
    cap = out_lp.shape[1]
    n_max = 0
    if out_ids is not None or out_top is not None:
        _cuda(out_ids, torch.int64, "out_ids"), _cuda(out_top, torch.float32, "out_top")
        n_max = out_ids.shape[-1]
        for t, name in ((out_ids, "out_ids"), (out_top, "out_top")):
            if t.shape != (S, cap, n_max) or not t.is_contiguous():
                raise ValueError(f"{name} must be a contiguous [{S}, {cap}, n_max] tensor, got {tuple(t.shape)}")
    check(lib().uvx_token_logprobs_rows(logits.data_ptr(), R, V, tok.data_ptr(), n_top.data_ptr(), row_slot.data_ptr(), dst.data_ptr(),
                                        cap, n_max, out_lp.data_ptr(), _p(out_ids), _p(out_top), _stream()), "uvx_token_logprobs_rows")


# ------------------------------------------------------------------------------------------ beam search
BEAM_MAX = 8        # beams per prompt (kBeamMax in generate.cu)
BEAM_MAX_K = 64     # candidates per prompt, max(2, 1 + n_eos) * num_beams


def log_softmax(x: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """[R, V] fp32 -> log_softmax over each row, fp32 (``out`` may be ``x``)."""
    _cuda(x, torch.float32, "x")
    R, V = x.shape
    if out is None:
        out = torch.empty_like(x)
    check(lib().uvx_log_softmax(x.data_ptr(), out.data_ptr(), R, V, _stream()), "uvx_log_softmax")
    return out


def beam_select(logprobs: torch.Tensor, run_score: torch.Tensor, num_beams: int, k: int, scratch=None, out=None):
    """logprobs [B*nb, V] fp32, run_score [B*nb] fp32 -> (scores [B, k] fp32, flat ids [B, k] int64 = beam * V + token): the
    k largest logprobs + run_score per prompt, descending, equal values in flat-index order."""
    _cuda(logprobs, torch.float32, "logprobs"), _cuda(run_score, torch.float32, "run_score")
    R, V = logprobs.shape
    B = R // num_beams
    dev = logprobs.device
    if scratch is None:
        scratch = (torch.empty(R * k, dtype=torch.float32, device=dev), torch.empty(R * k, dtype=torch.int64, device=dev))
    if out is None:
        out = (torch.empty(B, k, dtype=torch.float32, device=dev), torch.empty(B, k, dtype=torch.int64, device=dev))
    check(lib().uvx_beam_select(logprobs.data_ptr(), B, num_beams, V, run_score.data_ptr(), k, scratch[0].data_ptr(),
                                scratch[1].data_ptr(), out[0].data_ptr(), out[1].data_ptr(), _stream()), "uvx_beam_select")
    return out


def beam_update(cand_s: torch.Tensor, cand_i: torch.Tensor, V: int, num_beams: int, eos_ids: Optional[torch.Tensor], max_new: int,
                len_div: torch.Tensor, early_stopping: int, lp_positive: bool, state: dict, counters: dict, bumps: tuple = (),
                hit: Optional[torch.Tensor] = None) -> None:
    """``uvx_beam_update`` on the candidates of ``beam_select``.  ``state`` holds the device tensors run_score, run_seq,
    pool_seq, pool_score, pool_len, pool_fin, parent, tok, heur, flags, ticket; ``counters`` cur_len, step_idx, done.
    ``hit`` [B * K] int32 (``stop_strings_beam``): ``uvx_beam_update_stop``, a candidate with a hit finishes."""
    B, K = cand_s.shape
    s, c = state, counters
    b = list(bumps) + [None] * (3 - len(bumps))
    args = (cand_s.data_ptr(), cand_i.data_ptr(), B, num_beams, K, V, _p(eos_ids), 0 if eos_ids is None else eos_ids.numel(),
            int(max_new), len_div.data_ptr(), int(early_stopping), int(bool(lp_positive)), s["run_score"].data_ptr(),
            s["run_seq"].data_ptr(), s["pool_seq"].data_ptr(), s["run_seq"].stride(0), s["pool_score"].data_ptr(),
            s["pool_len"].data_ptr(), s["pool_fin"].data_ptr(), s["parent"].data_ptr(), s["tok"].data_ptr(), s["heur"].data_ptr(),
            s["flags"].data_ptr(), s["ticket"].data_ptr(), c["cur_len"].data_ptr(), c["step_idx"].data_ptr(), _p(b[0]), _p(b[1]),
            _p(b[2]), c["done"].data_ptr())
    if hit is None:
        check(lib().uvx_beam_update(*args, _stream()), "uvx_beam_update")
    else:
        check(lib().uvx_beam_update_stop(*args, _rows(hit, torch.int32, B * K, "hit").data_ptr(), _stream()), "uvx_beam_update_stop")


def kv_reorder_(k_cache: torch.Tensor, v_cache: torch.Tensor, parent: torch.Tensor, n_pos: torch.Tensor, num_beams: int) -> None:
    """k / v caches [L, B*nb, S_max, Hkv, D] bf16: row r <- row parent[r] (int32, same prompt) at positions [0, n_pos[0]), in place."""
    _cuda(k_cache, BF16, "k_cache"), _cuda(v_cache, BF16, "v_cache"), _cuda(parent, torch.int32, "parent")
    _cuda(n_pos, torch.int32, "n_pos")
    if not (k_cache.is_contiguous() and v_cache.is_contiguous() and k_cache.shape == v_cache.shape):
        raise ValueError("kv_reorder_ needs two contiguous caches of one shape")
    L, R, S_max = k_cache.shape[:3]
    row_elems = k_cache[0, 0, 0].numel()
    check(lib().uvx_kv_reorder(k_cache.data_ptr(), v_cache.data_ptr(), L, R // num_beams, num_beams, S_max, row_elems,
                               parent.data_ptr(), n_pos.data_ptr(), _stream()), "uvx_kv_reorder")
