/* libuvx - C ABI of the H100-native Ultravox audio->LLM hot path.
 *
 * The reference (fixie-ai/ultravox @ 648efe7f) has NO native / FFI boundary: its hot path is Python over
 * transformers/torch.  This header is therefore the boundary a maintainer would bind from
 * `ultravox/model/ultravox_model.py` / `ultravox_processing.py` with ctypes (see INTEGRATION.md); every entry
 * cites the reference (or third-party) function whose arithmetic it replaces.  `ref:` = /root/reference,
 * `hf:` = transformers (4.51.3 pinned by the reference; same formulas in 5.5.0).
 *
 * Conventions
 *   - plain pointers + sizes only; all pointers are DEVICE pointers unless named host_*;
 *   - bf16 tensors are passed as `const void*` / `void*` (2-byte elements, row-major);
 *   - every call is asynchronous on `stream` (a cudaStream_t), allocates nothing and performs no host
 *     synchronisation.  Process-wide state: immutable per-device tables (twiddles, mel filters) built once on
 *     first use, and the uvx_debug_* tuning hooks (tile / split / pipeline-isolation overrides - process
 *     globals, for benchmarking only: leave them at their defaults in production).  The split-K workspace is
 *     the CALLER's buffer (uvx_gemm_args.workspace): one workspace per stream if GEMMs run concurrently;
 *   - returns 0 on success, a negative UVX_ERR_* otherwise; `uvx_last_error()` gives the message
 *     (thread-local).  Argument validation that the reference does in Python stays in Python.
 */
#ifndef UVX_H_
#define UVX_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UVX_ABI_VERSION 1

#define UVX_OK 0
#define UVX_ERR_ARG (-1)   /* bad shape / alignment / null pointer */
#define UVX_ERR_CUDA (-2)  /* CUDA runtime / driver error (launch failure, tensor-map encode, ...) */
#define UVX_ERR_WS (-3)    /* workspace too small */

typedef void* uvx_stream_t; /* cudaStream_t */

int uvx_abi_version(void);
const char* uvx_last_error(void);
/* number of kernels this library has launched in the calling process (bench.py's "gpu_launches") */
int64_t uvx_launch_count(void);

/* ---------------------------------------------------------------------------------------------
 * a1 / K1-K3  log-mel front end.
 * Replaces WhisperFeatureExtractor._torch_extract_fbank_features (hf:models/whisper/
 * feature_extraction_whisper.py:135-164; call site ref:ultravox/model/ultravox_processing.py:295-303):
 * reflect-pad 200, 400-point periodic-hann STFT with hop 160, last frame dropped, |.|^2, slaney mel
 * filterbank (n_mels 80 or 128), log10(max(.,1e-10)), per-clip max-8 floor, (x+4)/4.
 *   wave      [B, L] fp32, L % 160 == 0 (zero-padded by the host like the extractor does)
 *   out_f32   [B, n_mels, T] fp32, T = L/160 (the reference's `audio_values` layout) or NULL
 *   out_tm    [B, T + 2, n_mels] bf16 time-major with one zero row before and after each clip (the
 *             layout the conv stem consumes, see uvx_gemm_bf16) or NULL
 *   workspace >= uvx_logmel_workspace(B, L, n_mels) bytes                                            */
size_t uvx_logmel_workspace(int64_t B, int64_t L, int n_mels);
int uvx_logmel(const float* wave, int64_t B, int64_t L, int n_mels, float* out_f32, void* out_tm,
               void* workspace, size_t workspace_bytes, uvx_stream_t stream);

/* host-only helper: writes the dense [201, n_mels] fp32 slaney filterbank the library uses (no GPU needed) */
int uvx_debug_mel_filters(int n_mels, float* host_dense);

/* `audio_values` [N, n_mels, T] fp32 (as produced by the reference processor / collator, any padding
 * content) -> bf16 time-major [N, T + 2, n_mels] with zero guard rows.  Replaces the
 * `audio_values.to(dtype)` cast of ref:ultravox/model/ultravox_model.py:382-385.                      */
int uvx_mel_to_timemajor(const float* mel, int64_t N, int n_mels, int64_t T, void* out_tm, uvx_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Dense contraction on the Hopper tensor cores (TMA -> smem ring -> wgmma -> fp32 registers -> epilogue).
 *   C[row(b,m), n] = act( alpha * sum_k A[b,m,k] * W[n,k] + bias[n] ) + R[b,m,n]
 * A is addressed as A + b*a_batch_stride + m*a_row_stride + k (elements), which lets the same kernel run
 *   - every nn.Linear of the path (hf:models/whisper/modeling_whisper.py:279-335,403-408;
 *     hf:models/llama/modeling_llama.py:171-184,262-288; ref:ultravox/model/ultravox_model.py:793-799),
 *   - conv1 / conv2 of the Whisper stem as implicit GEMMs over the time-major padded activation
 *     (ref:ultravox/model/ultravox_model.py:893-894): row m of clip b is the 3*C contiguous elements
 *     starting at frame stride*m of the guard-padded buffer, W is the conv weight re-laid as [C_out, 3*C_in].
 * Output rows: c_row_map ? c_row_map[b*a_rows+m] (negative = drop) : b*c_batch_rows + m + c_row_offset.
 * R (optional) is addressed R + b*r_batch_stride + m*r_row_stride + n: residual stream (whisper/llama) or the
 * positional embedding added after GELU (ref :896-899, r_batch_stride = 0).
 * Requirements: K % 8 == 0, N % 64 == 0, strides % 8 == 0, 16-byte aligned bases.
 * Split-K partial sums are reduced in a fixed order by a second kernel: results are deterministic.
 * Calls with a_batch == 1, a_rows <= 32 (decode batches), a plain bf16 output (no SwiGLU), row-major or 128-row weights and a
 * workspace of at least a_rows*N*4 bytes run the DECODE FORM: 128 weight rows on the wgmma M dimension, the tokens on N, split-K
 * over the weight stream (default; UVX_GEMM_WS=0 / uvx_debug_gemm_ws(0, ., .): never).  UVX_GEMM_WS=1 additionally runs calls
 * with 33..256 rows and N % 128 == 0 as a single pass over 128-wide tiles (no split-K).                                         */
enum { UVX_ACT_NONE = 0, UVX_ACT_GELU = 1, UVX_ACT_SWIGLU = 2 };
enum { UVX_DT_BF16 = 0, UVX_DT_F32 = 1 };
enum { UVX_TILE_PLAIN = 0, UVX_TILE_ROPE_PAIRS = 1, UVX_TILE_GATE_UP_8 = 8, UVX_TILE_GATE_UP_16 = 16 };   /* uvx_tile_weight interleave */
enum { UVX_GEMM_W_STATIC = 4 };   /* uvx_gemm_args.flags bit 2 */

typedef struct uvx_gemm_args {
  const void* A;            /* bf16 */
  int64_t a_batch, a_rows, K;
  int64_t a_row_stride, a_batch_stride;
  const void* W;            /* bf16 [N, K] row-major (nn.Linear layout) */
  int64_t N, w_row_stride;
  void* C;                  /* bf16 or f32 */
  int64_t c_row_stride, c_batch_rows, c_row_offset;
  const int32_t* c_row_map; /* optional */
  const void* bias;         /* bf16 [N] or NULL */
  const void* R;            /* bf16 or NULL */
  int64_t r_row_stride, r_batch_stride;
  float alpha;
  int32_t act;              /* UVX_ACT_* */
  int32_t out_dtype;        /* UVX_DT_* */
  void* workspace;          /* optional, 256-byte aligned scratch: enables split-K when the tile count cannot fill   */
  int64_t workspace_bytes;  /* the SMs (fp32 partial sums [splits][rows][N]; contents on entry do not matter).       */
  const void* norm_w;       /* optional: also emit norm_out[row,:] = norm_w * bf16(C[row,:] * rsqrt(mean(C^2) + eps)),  */
  void* norm_out;           /* the LlamaRMSNorm that follows o_proj / down_proj (hf:modeling_llama.py:53-67, 321-329),  */
  float norm_eps;           /* fused into the split-K reduction when there is one.  bf16 [rows, N], plain row order.    */
  /* ---- round 2 (all optional, zero = off) -------------------------------------------------------------------------
   * w_tiled = R (64 / 128 / 208 / 256): W points at the pre-tiled image [ceil(N/R)][K/64][R][64] of the [N, K] weight (rows past
   *   N zero) instead of the row-major matrix, so every k-block of a tile is ONE contiguous R*128-byte run of DRAM (the weight
   *   stream of the LLM prefill is HBM-bound; see uvx_tile_weight).  The kernel then uses R-wide tiles.
   * act = UVX_ACT_SWIGLU (needs an interleaved gate|up image: w_tiled = 128 with interleave = 16 - 16 gate rows | 16 up rows per
   *   32-row quarter - or another width with interleave = 8 - 8 gate rows alternating with the 8 up rows of the same features): the epilogue writes C[row, f] = silu(gate_f) * up_f for the N/2 features
   *   (LlamaMLP act_fn(gate_proj(x)) * up_proj(x), hf:modeling_llama.py:183) - the [rows, N] intermediate never reaches HBM.
   * rope_cos/rope_sin [max_pos, 64] fp32 (+ rope_positions / rope_rows_per_seq / rope_pos_offset as in uvx_rope): tiles whose
   *   first column is < rope_cols (= (Hq + Hkv) * 128) are rotated in the epilogue (hf:modeling_llama.py:124-168, head_dim 128).  */
  int32_t w_tiled;
  int32_t rope_cols;
  const float* rope_cos;
  const float* rope_sin;
  const int32_t* rope_positions;
  int64_t rope_rows_per_seq, rope_pos_offset;
  int32_t flags;            /* bit 1: never take the single-pass form for this call (bit 0 is accepted and ignored).
                             * bit 2 (UVX_GEMM_W_STATIC): W is not written by any kernel that may still be running when this call
                             *   starts - kernels launched with programmatic dependent launch begin before the previous kernel has
                             *   finished, and its predecessor may be running too.  The call may then start its weight stream before
                             *   waiting for the previous kernel.  Set it only for weights nothing in the stream writes (frozen
                             *   pre-tiled images), never where weights change in-stream (adapter merges, training steps).        */
  int32_t w_perm;           /* row order inside the tiles of a w_tiled = 128 image: 0 = plain, 1 = UVX_TILE_ROPE_PAIRS          */
} uvx_gemm_args;

/* Contracts of uvx_gemm_bf16 (pinned per element by tests/test_gemm_gpu.py):
 *  - workspace: its contents on entry do not matter.  Every partial sum the reduce reads was written by the same call, so a
 *    workspace full of NaN gives the same bits as a zeroed one.
 *  - accumulation: fp32, K summed in k-block order within a split and the splits summed in split order; the tile width, the
 *    cluster shape, the grid and the epilogue form (registers or the staged shared-memory tile) never change a bit.
 *  - epilogue rounding order (plain): v = acc * alpha, v += bias, v = GELU(v), v += R, all in fp32, then ONE round-to-nearest-even
 *    to bf16 at the store (fp32 output: no rounding).  The fused SwiGLU rounds gate * alpha and up * alpha to bf16, silu(gate)
 *    to bf16, and the product once more; the fused RoPE rounds the projection to bf16 and rotates it in fp32 with every
 *    product and sum rounded (o1 = x1 cos - x2 sin, o2 = x2 cos + x1 sin, no FMA), then rounds once; the fused RMSNorm writes
 *    norm_out = norm_w * bf16(bf16(C) * rsqrt(mean(bf16(C)^2) + eps)), the bits uvx_rmsnorm gives on the finished rows.
 *  - GELU: the split-K reduce evaluates it with erff (gelu_erf); the direct, staged and decode-form epilogues use the
 *    Abramowitz-Stegun 7.1.26 form with ex2 / rcp approximations (|error| <= 7.5e-8 |x| plus fp32 roundings).  The same call can
 *    therefore differ in its low bits between split counts, and so between configurations that pick different split counts. */
int uvx_gemm_bf16(const uvx_gemm_args* args, uvx_stream_t stream);
/* tuning hook: force tile config MT*1000+BN (MT in {1,2}, BN in {64,128,208,256}; 0 = heuristic) and split-K count (0 = heuristic) */
int uvx_debug_gemm_override(int cfg, int splits);
/* tuning hook: cap the shared-memory ring depth of uvx_gemm_bf16 (0 = as deep as fits) */
int uvx_debug_gemm_stages(int n);
/* tuning hook of the weight-streaming forms: enable (0 = never, 1 = decode form + single-pass form, 2 = decode form only; -1 =
 * UVX_GEMM_WS env, default 2), `mode` (ignored), upper bound on the persistent grid of every uvx_gemm_bf16 launch (0 = one CTA per SM) */
int uvx_debug_gemm_ws(int enable, int mode, int grid);
/* tuning hook: the staged epilogue of the tensor-bound calls (more than 256 rows or a batch; plain bias / GELU / residual epilogue,
 * no row map, one split, 128 x 64 or 128 x 128 tiles): the output tile goes through shared memory and leaves by TMA store, the
 * residual is loaded by TMA ahead of the epilogue.  -1 (default) or > 0 = staged wherever it applies, 0 = register epilogue
 * everywhere.  Never changes the result bits. */
int uvx_debug_gemm_tma_store(int on);
/* tuning hook: the split ring.  Calls whose rows one m-tile covers (one batch, <= 256 rows, tiles at most 128 wide, no
 * thread-block cluster cutting the A box) may stream W through a ring of their own, beside a ring of A boxes that hold only the
 * rows that exist.  0 = one ring of A + W stages for every call; n >= 2 = split rings with n activation slots (at most 8) for
 * every such call; -1 (default) = split rings with 5 activation slots where that leaves the W ring deeper than the one ring.
 * uvx_debug_gemm_stages caps the weight ring.  Never changes the result bits. */
int uvx_debug_gemm_split_ring(int a_stages);
/* hooks of tuning knobs the Hopper kernel does not have (phase timestamps, L2 prefetch distance, pipeline isolation): accepted
 * for ABI compatibility, no effect */
int uvx_debug_gemm_times(void* dev_buf);
int uvx_debug_gemm_pf(int pf);
int uvx_debug_gemm_ws_times(void* dev_buf);
/* W [N, K] bf16 row-major (row stride w_row_stride) -> the pre-tiled image uvx_gemm_args.w_tiled = R reads:
 * out[t][kb][r][0:64] = W[row(t, r), kb*64 : kb*64+64], zero where row >= N.  interleave = 0: row(t, r) = t*R + r.
 * interleave = 8 (fused gate|up, N = 2*F, R % 16 == 0): r = 16*g + j -> gate feature t*R/2 + 8g + j (j < 8) = W row of that
 * feature, or the up row F + t*R/2 + 8g + (j-8) (j >= 8).  interleave = 16 (R = 128): r = 32q + j ->
 * gate feature 64t + 16q + j (j < 16) or the up row of feature 64t + 16q + (j - 16).  interleave = 1 (UVX_TILE_ROPE_PAIRS, R = 128 =
 * head_dim): r = 32q + j -> row 128t + 16q + j (j < 16) or its rotation partner 128t + 64 + 16q + (j - 16).  out: ceil(N/R) * (K/64) * R * 64 bf16 elements.                 */
int uvx_tile_weight(const void* W, int64_t N, int64_t K, int64_t w_row_stride, int32_t R, int32_t interleave, void* out,
                    uvx_stream_t stream);
/* tuning hook: thread-block cluster of uvx_gemm_bf16, cm tiles along M x cn along N sharing their A / W boxes by TMA multicast
 * ((0, 0) = heuristic: clusters for calls of <= 256 rows and one batch unless UVX_GEMM_CLUSTER=0; (1, 1) = none).  An axis whose
 * tile count it does not divide falls back to 1.  The cluster shape never changes the result bits. */
int uvx_debug_gemm_cluster(int cm, int cn);
/* accepted for ABI compatibility, no effect */
int uvx_debug_gemm_mode(int mode);

/* ---------------------------------------------------------------------------------------------
 * Row-wise normalisations (fp32 statistics, bf16 in/out).
 * uvx_layernorm: nn.LayerNorm(eps 1e-5) of the Whisper encoder (hf:modeling_whisper.py:393,403;
 *                ref:ultravox_model.py:980).
 * uvx_rmsnorm:   LlamaRMSNorm (hf:models/llama/modeling_llama.py:53-67) and the projector RMSNorm
 *                (ref:ultravox_model.py:733-736): y = w * bf16(x * rsqrt(mean(x^2) + eps)).
 *                `valid_per_group`/`group_rows` implement StackAudioFrames (ref :722-730) without a copy:
 *                rows are grouped `group_rows` per clip; row t of a clip only has
 *                clamp(valid_elems - t*cols, 0, cols) real elements, the rest read as zero.
 *                Pass group_rows = 0 for a plain matrix.                                               */
int uvx_layernorm(const void* x, const void* w, const void* b, void* y, int64_t rows, int64_t cols,
                  int64_t x_row_stride, float eps, uvx_stream_t stream);
int uvx_rmsnorm(const void* x, const void* w, void* y, int64_t rows, int64_t cols, int64_t x_row_stride,
                int64_t group_rows, int64_t group_stride, int64_t valid_elems, float eps, uvx_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Fused softmax(QK^T*scale + mask)V, flash style, fp32 softmax, bf16 in/out.
 *   Whisper encoder self-attention (hf:modeling_whisper.py:215-238,305-349): non-causal, keys >= kv_len[b]
 *   masked (ref:ultravox_model.py:915-926), optional block-causal streaming mask (ref :834-863,928-936);
 *   Llama attention (hf:modeling_llama.py:199-289): causal, grouped-query.
 * q[b, i, h, :] = q + b*q_bs + i*q_rs + h*D  (same for k, v with h / (Hq/Hkv), and o).
 * Visible keys of sequence b: [clamp(kv_start[b], 0, end), end) with end = clamp(kv_len[b], 0, Skv), further cut by the causal
 * and block rules.  Key / value rows outside that range (left padding, rows from kv_len on, a cache's rows from Skv on) may
 * hold anything, NaN and Inf included: they change no output bit.  A query that sees no key (inside the left padding of a
 * causal call, or kv_len[b] <= kv_start[b]) writes an output row of exactly 0 and lse = -inf (the log of an empty sum).   */
typedef struct uvx_attn_args {
  const void *q, *k, *v;
  void* o;
  int64_t B, Hq, Hkv, Sq, Skv, D;   /* D in {64, 128} */
  int64_t q_rs, q_bs, k_rs, k_bs, v_rs, v_bs, o_rs, o_bs;
  const int32_t* kv_len;            /* [B] or NULL (= Skv) */
  int32_t causal;                   /* query i sees keys j <= i + (Skv - Sq) */
  int32_t block;                    /* >0: block-causal, query i sees keys j with j/block <= i/block */
  float scale;
  float* lse;                       /* optional [B, Hq, Sq] fp32: log-sum-exp of the scaled scores (training) */
  const int32_t* kv_start;          /* optional [B]: keys j < kv_start[b] are masked - left-padded batches              */
                                    /* (ref collator ultravox_processing.py:53-63; hf masking_utils padding mask)       */
} uvx_attn_args;
int uvx_attention(const uvx_attn_args* args, uvx_stream_t stream);
/* calls with >= 16 queries run on the TMA + wgmma kernel (attention_wg.cu), single-token decode steps on mma.sync (attention.cu).
 * Tuning hook: 0 forces mma.sync everywhere, 1 = default, -1 = UVX_ATTN_TC env. */
int uvx_debug_attn_tc(int on);
/* Whisper-encoder entry (head_dim 64, Sq == Skv, non-causal + key-length / block-causal masks), same kernel as uvx_attention: qkv is the fused projection [B*S, row_stride] with head h's q / k / v at columns q_col + 64h, k_col + 64h,
 * v_col + 64h; output o[b*S + i, 64h .. 64h+63] (row stride o_rs).  Same math as uvx_attention.                      */
int uvx_attention_enc_tc(const void* qkv, int64_t row_stride, int64_t B, int64_t S, int64_t H, int64_t q_col, int64_t k_col,
                         int64_t v_col, void* o, int64_t o_rs, const int32_t* kv_len, int32_t block, float scale,
                         uvx_stream_t stream);
/* Device-indexed causal attention of a prompt chunk against a slot KV cache (chunked prefill inside the captured decode step of
 * continuous batching, ultravox_b200/engine.py).  The q side is a->B sequences of a->Sq queries as in uvx_attention; k / v
 * cover the whole cache [kv_batch, Skv = S_max, Hkv, D] (batch strides k_bs / v_bs), so the tensor maps never change between
 * graph replays.  Query batch b reads cache row kv_row[b] and has past[b] keys before its first query: query i sees keys
 * j <= i + past[b], j < kv_len[b] (a->kv_len required, normally past + valid queries).  Same kernel, tile schedule, masks
 * and arithmetic as the wgmma path of uvx_attention (bit-identical to it on a cache row with Skv = past + Sq, Sq >= 16);
 * cache rows other than kv_row[b] and keys from kv_len[b] on may hold anything, NaN included.  Requires causal = 1,
 * block = 0, kv_start = NULL, lse = NULL; kv_row / past / kv_len are read on the device, so they may change between replays. */
int uvx_attention_indexed(const uvx_attn_args* a, int64_t kv_batch, const int32_t* kv_row, const int32_t* past,
                          uvx_stream_t stream);
/* Paged KV cache (continuous batching with conversation sessions, ultravox_b200/engine.py PagedSlotDecodeEngine): one layer of the
 * K / V pool is [n_pages, 64, Hkv, D]; a page holds 64 positions, exactly one key tile of both attention kernels, so the same
 * keys meet in the same order and the results are bit-identical to the contiguous forms.  table [rows, table_stride] int32:
 * key tile t of table row b is page table[b * table_stride + t].  Only entries of tiles below the key bound are read (entries past a
 * sequence's pages may hold -1).
 * uvx_attention_paged          uvx_attention on the mma.sync kernel with K / V read through the table: a->k / a->v point at the
 *                              pool layer, k_rs / v_rs are the row strides inside a page and k_bs / v_bs = 64 rows (the page
 *                              stride); batch row b uses table row b; a->kv_len required; Skv bounds the keys (<= 64 *
 *                              table_stride).  Bit-identical to uvx_attention on a contiguous cache holding the same rows, for
 *                              calls that take its mma.sync kernel.  Requires kv_start = NULL, lse = NULL, block = 0, causal only
 *                              with Sq = 1.
 * uvx_attention_indexed_paged  uvx_attention_indexed with kv_row[b] a table row: the K / V tensor maps cover the pool layer
 *                              (n_pages pages) as {D, Hkv, 64, n_pages}, key tile t is loaded from page table[kv_row[b] *
 *                              table_stride + t].  Same restrictions; bit-identical to uvx_attention_indexed.                 */
int uvx_attention_paged(const uvx_attn_args* a, const int32_t* table, int64_t table_stride, uvx_stream_t stream);
int uvx_attention_indexed_paged(const uvx_attn_args* a, int64_t n_pages, const int32_t* table, int64_t table_stride,
                                const int32_t* kv_row, const int32_t* past, uvx_stream_t stream);

/* FP8 (e4m3) paged KV pool: the same pool layout with 1-byte elements (strides in elements = bytes; torch.float8_e4m3fn), one fp32
 * scale for K and one for V per layer, kv_scales [L, 2] (positive, finite), read on the device so captured graphs stay valid.
 *   quantize   (every write into the pool):  q = cvt.rn.satfinite.e4m3(float(x) / s), IEEE fp32 division.  NaN stays NaN (stored
 *              as 0x7F whatever its sign); +-Inf and anything beyond +-448 become +-448 (host reference, equal up to the sign of
 *              NaN: (x.float() / s).clamp(-448, 448).to(float8_e4m3fn)).
 *   dequantize (every read from the pool):   x = bf16_rn(float(q) * s); after it every kernel does the arithmetic of its bf16 twin.
 * Bytes 0x7F / 0xFF are NaN: keys outside the key bound never reach O (zero-filled / zeroed as in the bf16 kernels).
 * uvx_attention_paged_fp8          uvx_attention_paged over an e4m3 pool layer, kv_scale = that layer's [K, V] scales.  Bit-identical
 *                                  to uvx_attention_paged on a bf16 pool holding the dequantized values.  k_rs / v_rs % 16 == 0.
 * uvx_attention_indexed_paged_fp8  uvx_attention_indexed_paged over an e4m3 pool layer (bf16 wgmma MMAs on the dequantized tiles);
 *                                  bit-identical to uvx_attention_indexed_paged on a bf16 pool holding the dequantized values.  */
int uvx_attention_paged_fp8(const uvx_attn_args* a, const int32_t* table, int64_t table_stride, const float* kv_scale,
                            uvx_stream_t stream);
int uvx_attention_indexed_paged_fp8(const uvx_attn_args* a, int64_t n_pages, const int32_t* table, int64_t table_stride,
                                    const int32_t* kv_row, const int32_t* past, const float* kv_scale, uvx_stream_t stream);

/* Row-mapped decode attention (the prompt-lookup slot step, ultravox_b200/engine.py SlotDecodeEngine): several query rows read
 * the keys of one slot.  Query row b (a->B rows, Sq = 1) reads cache row kv_row[b] (int32 [B], read on the device) instead of
 * row b, and the keys [0, kv_len[b]) of it; everything else is the unmapped call on the mma.sync kernel, so each row is bit-identical
 * to uvx_attention / uvx_attention_paged / uvx_attention_paged_fp8 of that row against that cache row.  Requires a->kv_len,
 * Sq = 1, kv_start = NULL, lse = NULL, block = 0; kv_row[b] must address a row that exists (a->k + kv_row[b] * k_bs, or a table row).
 * uvx_attention_rows            contiguous cache [rows, S_max, Hkv, D] through the strides of a.
 * uvx_attention_paged_rows      uvx_attention_paged with table row kv_row[b].
 * uvx_attention_paged_fp8_rows  uvx_attention_paged_fp8 with table row kv_row[b].                                             */
int uvx_attention_rows(const uvx_attn_args* a, const int32_t* kv_row, uvx_stream_t stream);
int uvx_attention_paged_rows(const uvx_attn_args* a, const int32_t* table, int64_t table_stride, const int32_t* kv_row,
                             uvx_stream_t stream);
int uvx_attention_paged_fp8_rows(const uvx_attn_args* a, const int32_t* table, int64_t table_stride, const float* kv_scale,
                                 const int32_t* kv_row, uvx_stream_t stream);

/* RoPE on the q and k sections of a fused [rows, (Hq + 2*Hkv) * D] projection, in place
 * (hf:modeling_llama.py:124-168; cos/sin tables [max_pos, D/2] fp32 built by the host exactly like
 * LlamaRotaryEmbedding incl. llama3 scaling, hf:modeling_rope_utils.py:550-626).
 * position of row r = positions ? positions[r] : pos_offset + (r % rows_per_seq); with positions, rows_per_seq and
 * pos_offset are not read.  Every row is rotated, pad rows too: the caller gives them a position inside the tables
 * (generate() gives position 0, where cos = 1 and sin = 0, so a pad row keeps its bits).  The v section is not touched. */
int uvx_rope(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
             const float* sin_tab, const int32_t* positions, int64_t rows_per_seq, int64_t pos_offset,
             uvx_stream_t stream);

/* out[r, j] = silu(gate) * lin where for x[r, 0:2H]:
 *   gate_first = 0: lin = x[:, j], gate = x[:, H + j]   (ref SwiGLU, ultravox_model.py:739-742)
 *   gate_first = 1: gate = x[:, j], lin = x[:, H + j]   (llama MLP act(gate)*up, hf:modeling_llama.py:183) */
int uvx_swiglu(const void* x, void* out, int64_t rows, int64_t H, int64_t x_row_stride, int gate_first,
               uvx_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * a11 + a5 (K14 + K15): token-embedding gather fused with the audio splice, sync-free and bit-exact.
 * uvx_splice_plan builds src[b*S + s] = (row of audio_embeds) or -1 from the reference's index vectors
 *   (ref:ultravox_model.py:259-275,390-394: chunks in batch order, later chunks overwrite earlier ones);
 *   audio_embeds rows are a*tok_stride + j, j < audio_token_len[a].
 * uvx_embed_splice writes out[b, s, :] = src >= 0 ? audio_embeds[src] : embed_tokens[input_ids[b, s]].  */
int uvx_splice_plan(const int64_t* start_idx, const int32_t* tok_len, const int64_t* audio_batch_size,
                    int64_t n_chunks, int64_t B, int64_t S, int64_t tok_stride, int32_t* src,
                    uvx_stream_t stream);
int uvx_embed_splice(const int64_t* input_ids, const void* embed_tokens, int64_t vocab, const void* audio_embeds,
                     const int32_t* src, int64_t rows, int64_t d, void* out, uvx_stream_t stream);

/* Last-position LM head: logits[b, v] = sum_k h[b, k] * W[v, k] (bf16 x bf16 -> f32), HBM-streaming GEMV
 * (hf:modeling_llama.py:485-491 with logits_to_keep = 1), and greedy argmax (first maximal index, like
 * torch.argmax; ref:ultravox/inference/infer.py:319-328 greedy path).  uvx_argmax takes finite or -inf logits
 * (a row that is all -inf gives 0, as torch.argmax does); NaN is out of contract.                        */
int uvx_lm_head(const void* h, int64_t B, int64_t h_row_stride, const void* W, int64_t V, int64_t d,
                float* logits, uvx_stream_t stream);
int uvx_argmax(const float* logits, int64_t B, int64_t V, int64_t* out_idx, uvx_stream_t stream);

/* a13 decode step (ref:ultravox/model/ultravox_model.py:398-426 -> HF greedy generate): with one token per stream every
 * linear layer is a weight-streaming matrix-vector product, y[b, n] = sum_k x[b, k] W[n, k] (+ R[b, n]), 1 <= B <= 8.   */
int uvx_gemv_bf16(const void* x, int64_t B, int64_t x_row_stride, const void* W, int64_t w_row_stride, int64_t N, int64_t K,
                  const void* R, int64_t r_row_stride, void* out, int64_t o_row_stride, int out_f32, uvx_stream_t stream);
/* copy this step's k / v sections of the fused projection into the static KV cache at positions[b] (device index, so
 * the decode step is capturable in a CUDA graph); cache layout [B, S_max, kv_width]                                    */
int uvx_kv_append(const void* qkv, int64_t row_stride, int64_t k_col, int64_t v_col, int64_t kv_width, void* k_cache,
                  void* v_cache, int64_t cache_batch_stride, const int32_t* positions, int64_t B, uvx_stream_t stream);
/* Decode-step fusions (one CUDA graph per step, ultravox_b200/engine.py): uvx_gemv_bf16 with a fused prologue on the B activation rows -
 * norm_w != NULL: LlamaRMSNorm (bit-identical to uvx_rmsnorm followed by uvx_gemv_bf16), swiglu = 1: the row is [gate | up] of width
 * 2K and the kernel consumes act_fn(gate) * up (bit-identical to uvx_swiglu(gate_first = 1) + uvx_gemv_bf16) - and RoPE on q / k +
 * KV-cache append in one launch (same bits as uvx_rope + uvx_kv_append).                                                       */
int uvx_gemv_fused_bf16(const void* x, int64_t B, int64_t x_row_stride, const void* W, int64_t w_row_stride, int64_t N, int64_t K,
                        const void* R, int64_t r_row_stride, void* out, int64_t o_row_stride, int out_f32, const void* norm_w,
                        float norm_eps, int swiglu, uvx_stream_t stream);
int uvx_rope_kv_append(void* qkv, int64_t B, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab, const float* sin_tab,
                       const int32_t* rope_positions, void* k_cache, void* v_cache, int64_t cache_batch_stride,
                       const int32_t* positions, uvx_stream_t stream);
/* uvx_rope_kv_append with a per-row map (the mixed decode + prompt-chunk step): row r is rotated at rope_positions[r] and,
 * when cache_row[r] >= 0, its k / v go to cache row cache_row[r] at positions[r]; cache_row[r] < 0 writes nothing (q and k are
 * still rotated in qkv).  Same bits as uvx_rope_kv_append for the rows it writes; shares its kernel body.                    */
int uvx_rope_kv_append_map(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                           const float* sin_tab, const int32_t* rope_positions, void* k_cache, void* v_cache,
                           int64_t cache_batch_stride, const int32_t* cache_row, const int32_t* positions, uvx_stream_t stream);
/* uvx_rope_kv_append_map into an e4m3 cache (the FP8 paged pool, see uvx_attention_paged_fp8): q / k in qkv get the same bits as
 * uvx_rope_kv_append_map; the stored k / v are the bf16 rows it would store, quantized with kv_scale[0] / kv_scale[1] (this layer's
 * K and V scales).  Rows with cache_row[r] < 0 write nothing.                                                                   */
int uvx_rope_kv_append_map_fp8(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                               const float* sin_tab, const int32_t* rope_positions, void* k_cache, void* v_cache,
                               int64_t cache_batch_stride, const int32_t* cache_row, const int32_t* positions, const float* kv_scale,
                               uvx_stream_t stream);
/* a[i] += delta (and b[i] += delta when b != NULL): advances the device-side positions / lengths after each step     */
int uvx_add_i32(int32_t* a, int32_t* b, int64_t n, int32_t delta, uvx_stream_t stream);
/* prefill counterpart of uvx_kv_append: rows b*S + s of the fused projection -> cache[b, past + s] (k and v sections),
 * what DynamicCache.update does for the prompt (hf:cache_utils.py; call site hf:modeling_llama.py:262-273)           */
int uvx_kv_write(const void* qkv, int64_t row_stride, int64_t k_col, int64_t v_col, int64_t kv_width, void* k_cache,
                 void* v_cache, int64_t cache_batch_stride, int64_t B, int64_t S, int64_t past, uvx_stream_t stream);

/* The rest of one `GenerationMixin` step (ref:ultravox/model/ultravox_model.py:398-426 -> hf:generation/utils.py _sample),
 * with every per-step scalar read from DEVICE memory so that a whole decode step replays from one CUDA graph:
 * uvx_repetition_penalty  scores of tokens already in seq[b, 0:cur_len[0]] are divided (positive) / multiplied (negative)
 *                         by `penalty`, each distinct token once (hf:generation/logits_process.py
 *                         RepetitionPenaltyLogitsProcessor; the reference pipeline enables 1.1, ref ultravox_pipeline.py:95-113);
 *                         scratch: [B, seq_stride] fp32.
 * uvx_sample              out[b] ~ softmax(logits[b] / temperature) restricted to the top_k largest logits (top_k <= 0: all),
 *                         by inverse CDF on the uniform u[step_idx[0] * u_stride + b] (step_idx NULL = 0): the do_sample branch of
 *                         ref:ultravox/inference/infer.py:319-328.  Deterministic given u.  The pick always has positive
 *                         mass (never a -inf logit); a row with no mass (all -inf) gives 0, as uvx_argmax does.  -0.0 and
 *                         +0.0 are one value for the top-k cut and the tie groups below.
 * uvx_sample_top_p        uvx_sample with nucleus filtering after the top-k cut, in HF's order (hf:generation/logits_process.py
 *                         TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper): with P = softmax(logits[b] / temperature)
 *                         over the top-k survivors, token i stays iff sum_{j: x_j <= x_i} P_j > 1 - top_p, and the largest logit
 *                         always stays (min_tokens_to_keep = 1, so top_p = 0 is the argmax).  The draw is the inverse CDF of P
 *                         renormalised over the kept tokens, on the same u as uvx_sample.  0 <= top_p <= 1 (else UVX_ERR_ARG);
 *                         top_p = 1 is uvx_sample bit for bit.  V <= 2^24.  Ties: equal logits are kept or dropped as one group,
 *                         whereas HF's unstable sort may split a tie group that straddles the cut - the one intended difference.
 *                         The masses are summed in 64-bit fixed point (2^-40 resolution), so the result is deterministic given u.
 * uvx_token_finish        tok[b] = done[b] ? pad_id : tok[b]; seq[b, cur_len[0]] = tok[b]; done[b] |= tok[b] in eos_ids;
 *                         cur_len[0]++, step_idx[0]++ (if given), bump{0,1,2}[b]++ (if given: cache slot / visible keys / RoPE
 *                         position); all_done[0] = all(done).                                                                 */
int uvx_repetition_penalty(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                           float penalty, float* scratch, uvx_stream_t stream);
int uvx_sample(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, const float* u, const int32_t* step_idx,
               int64_t u_stride, int64_t* out_idx, uvx_stream_t stream);
int uvx_sample_top_p(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p, const float* u,
                     const int32_t* step_idx, int64_t u_stride, int64_t* out_idx, uvx_stream_t stream);
int uvx_token_finish(int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int64_t* seq,
                     int64_t seq_stride, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1, int32_t* bump2,
                     int32_t* all_done, int64_t B, uvx_stream_t stream);

/* Continuous batching (ultravox_b200/engine.py SlotDecodeEngine): B decode rows ("slots") that each carry their own request, so
 * every per-request scalar is a device array [B] and rows with active[b] == 0 are idle.
 * uvx_sample_slots              active rows only: temperature[b] <= 0 -> out[b] = uvx_argmax of the row (first maximal index, an
 *                               all -inf row gives 0); otherwise out[b] = uvx_sample (top_p[b] >= 1) or uvx_sample_top_p
 *                               (top_p[b] < 1) of the row with temperature[b], top_k[b], top_p[b] and the uniform
 *                               u[b * u_stride + n_new[b]] - bit for bit the pick those entries make.  Inactive rows are not written.
 * uvx_repetition_penalty_slots  uvx_repetition_penalty on active rows with penalty[b] != 1, over seq[b, 0:cur_len[b]], scratch
 *                               [B, seq_stride] fp32.
 * uvx_slot_finish               for each active row that is not done: seq[b, cur_len[b]] = tok[b]; cur_len[b]++, n_new[b]++;
 *                               done[b] = tok[b] in eos_ids or n_new[b] >= max_new[b]; pos / lens / rope_pos [b]++ only if the
 *                               row is still open.  Done and inactive rows are frozen (their decode KV writes stay at one
 *                               position).  n_open[0] = number of active rows still open.                                         */
int uvx_sample_slots(const float* logits, int64_t B, int64_t V, const float* temperature, const int32_t* top_k, const float* top_p,
                     const float* u, int64_t u_stride, const int32_t* n_new, const int32_t* active, int64_t* out_idx,
                     uvx_stream_t stream);
int uvx_repetition_penalty_slots(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                                 const float* penalty, const int32_t* active, float* scratch, uvx_stream_t stream);
int uvx_slot_finish(const int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride,
                    int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active, int32_t* pos, int32_t* lens,
                    int32_t* rope_pos, int32_t* n_open, int64_t B, uvx_stream_t stream);

/* Log-probabilities and scores of a decode step, written on the device at an index read from device memory (no host sync, so
 * they sit inside the captured step).
 * uvx_token_logprobs  per row b with n_top[b] >= 0 (rows with n_top[b] < 0 are not touched), on the RAW logits row x:
 *                     lse = m + log(sum exp(x - m)) (m = max x) and, at d = dst[b] (0 <= d < cap, else nothing is written):
 *                     out_lp[b * cap + d] = x[tok[b]] - lse (torch.log_softmax(x)[tok], the OpenAI-style `logprobs` of the
 *                     chosen token); for n = min(n_top[b], n_max) > 0, out_ids / out_top[(b * cap + d) * n_max + i], i < n, are
 *                     the n largest entries by (value desc, index asc) - a tie at the n-th place goes to the lower index, as in
 *                     uvx_beam_select - with their x - lse (`top_logprobs`); entries i >= n are not written.  0 <= n_max <= 20.
 *                     One CTA per row with fixed-order reductions: a row's bits depend on its own logits only.
 * uvx_record_scores   at s = step_idx[0] (nothing when s is outside [0, steps)): raw[s, b, :] = logits[b] (HF's `output_logits`;
 *                     call it before uvx_repetition_penalty, which rewrites the logits in place) and scores[s, b, :] = HF's
 *                     processed scores (`output_scores`, hf:generation/utils.py _sample) of the penalised logits: for
 *                     temperature <= 0 (greedy: HF adds no warper) the row itself, otherwise TemperatureLogitsWarper ->
 *                     TopKLogitsWarper -> TopPLogitsWarper: x / temperature (IEEE division) on the entries uvx_sample /
 *                     uvx_sample_top_p draw from with the same temperature, top_k and top_p (a tie group, -0.0 == +0.0,
 *                     kept or dropped whole), -inf elsewhere, so a sampled token always has a finite score.  scores / raw are [steps, B, V] fp32; either may be NULL.  V <= 2^24. */
int uvx_token_logprobs(const float* logits, int64_t B, int64_t V, const int64_t* tok, const int32_t* n_top, const int32_t* dst,
                       int64_t cap, int32_t n_max, float* out_lp, int64_t* out_ids, float* out_top, uvx_stream_t stream);
int uvx_record_scores(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                      const int32_t* step_idx, int64_t steps, float* scores, float* raw, uvx_stream_t stream);

/* Prompt lookup decoding (ultravox_b200/engine.py LookupDecodeEngine; hf:generation/candidate_generator.py
 * PromptLookupCandidateGenerator and hf:generation/utils.py _assisted_decoding, transformers 5.5): one decode step feeds k + 1
 * positions of ONE sequence seq[0:cur_len] (its last token not yet fed) - the last token and up to k drafts - and keeps the
 * picks that agree with the drafts.  All state is on the device ([1] int32 counters), so the step is one graph.
 * uvx_lookup_draft           one CTA.  Drafts: for n-gram sizes g = min(n, L - 1) .. 1 (L = cur_len[0]) the leftmost earlier
 *                            occurrence of seq[L - g, L) followed by at least one token; the continuation seq[e, min(e + k, L))
 *                            of the first size that has one, cut before its first EOS (an EOS first: no drafts, no further
 *                            search) and to d <= max_new - n_new[0] - 1 (so n_new + d + 1 <= max_new); none when done[0].
 *                            Writes tok[0..k] (tok[0] = seq[L - 1], tok[1..d] the drafts, tok[d + 1..k] = seq[L - 1]),
 *                            n_draft[0] = d, and for row i <= k: pos = rope_pos = L - 1 + i, lens = pen_len = L + i,
 *                            idx = n_new + i; the drafts also go to seq[L, L + d).  1 <= k <= 31, n >= 1.
 * uvx_lookup_accept          one warp; nothing once done[0].  m = the number of leading i < d with pick[i] == tok[i + 1]; appends
 *                            pick[0..m] at seq[cur_len], cur_len and n_new grow by m + 1, done[0] = pick[m] in eos_ids or
 *                            n_new >= max_new.  With accepted (int32 [steps]): accepted[step[0]] = m (when inside), step[0]++.
 * uvx_repetition_penalty_rows  uvx_repetition_penalty on row b over seq[b * seq_stride, 0:len[b]] with row b's own scratch
 *                            [b * scratch_stride, ...]: seq_stride 0 lets the rows share one sequence.
 * uvx_record_scores_rows     uvx_record_scores with per-row destinations: row b at s = idx[b] of scores / raw [steps, V] fp32
 *                            (nothing when s is outside [0, steps)).                                                          */
int uvx_lookup_draft(int64_t* seq, const int32_t* cur_len, const int32_t* n_new, int32_t max_new, int32_t k, int32_t n,
                     const int64_t* eos_ids, int32_t n_eos, const int32_t* done, int64_t* tok, int32_t* n_draft, int32_t* pos,
                     int32_t* lens, int32_t* rope_pos, int32_t* pen_len, int32_t* idx, uvx_stream_t stream);
int uvx_lookup_accept(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, const int64_t* eos_ids, int32_t n_eos,
                      int64_t* seq, int32_t* cur_len, int32_t* n_new, int32_t max_new, int32_t* step, int32_t* accepted, int32_t steps,
                      int32_t* done, uvx_stream_t stream);
int uvx_repetition_penalty_rows(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* len,
                                float penalty, float* scratch, int64_t scratch_stride, uvx_stream_t stream);
int uvx_record_scores_rows(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                           const int32_t* idx, int64_t steps, float* scores, float* raw, uvx_stream_t stream);

/* Sampling cut-offs after top-k / top-p, in HF's order (hf:generation/logits_process.py, transformers 5.5, min_tokens_to_keep = 1):
 * TemperatureLogitsWarper -> TopKLogitsWarper -> TopPLogitsWarper -> MinPLogitsWarper -> TypicalLogitsWarper ->
 * EpsilonLogitsWarper -> EtaLogitsWarper, each on the survivors of the one before.  With P = softmax(x / temperature) over the
 * current survivors and H = -sum P log P:
 *   min_p      keep P_i >= min_p * max P (the maximum always stays).  0 <= min_p <= 1; 0 is off.
 *   typical_p  d_i = |-log P_i - H|; with the survivors sorted by d ascending, keep d_i <= the d of the first one whose cumulative
 *              P reaches typical_p.  This may drop the row maximum.  0 < typical_p; >= 1 is off.
 *   epsilon    keep P_i >= epsilon, and the largest survivor's tie group.  0 <= epsilon < 1; 0 is off.
 *   eta        keep P_i >= min(eta, sqrt(eta) * exp(-H)), and the largest survivor's tie group.  0 <= eta < 1; 0 is off.
 * Arguments outside those ranges (NaN included) give UVX_ERR_ARG.  Ties: a tie group (equal logits, -0.0 == +0.0) is kept or
 * dropped whole at every cut, which HF's per-element comparisons also do.  The kept set is a band lo <= key <= hi of the
 * sampler's order-preserving float keys; the masses are 64-bit fixed point (2^-40) and the entropy a fixed-order float64 sum,
 * so the band, and the pick given u, depend on the row and its settings alone.  V <= 2^24.  Each cut-off that is on costs
 * one to six more passes over the row; with every cut-off off each entry below is its plain form bit for bit.
 * uvx_sample_cutoffs              uvx_sample_top_p, then the cut-offs; the draw is the inverse CDF over the kept band on u.
 * uvx_record_scores_cutoffs       uvx_record_scores with the cut-offs: x / temperature exactly where uvx_sample_cutoffs can
 *                                 pick, -inf elsewhere (greedy, temperature <= 0, ignores them as HF does).
 * uvx_record_scores_rows_cutoffs  uvx_record_scores_rows with the cut-offs.
 * uvx_sample_slots_cutoffs        uvx_sample_slots with slot b's cut-offs at cutoffs[4 b .. 4 b + 4) = (min_p, typical_p, epsilon,
 *                                 eta) fp32 on the device, off encoded as (0, 1, 0, 0); a row with every cut-off off makes the
 *                                 pick uvx_sample_slots makes, bit for bit.  Values are not checked on the device: the caller
 *                                 writes them in range.
 * uvx_sample_rows_cutoffs         uvx_sample_rows with slot row_slot[r]'s cut-offs, as above.                                   */
typedef struct uvx_cutoffs {
  float min_p, typical_p, epsilon, eta;
} uvx_cutoffs;
int uvx_sample_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p, uvx_cutoffs cutoffs,
                       const float* u, const int32_t* step_idx, int64_t u_stride, int64_t* out_idx, uvx_stream_t stream);
int uvx_record_scores_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                              uvx_cutoffs cutoffs, const int32_t* step_idx, int64_t steps, float* scores, float* raw,
                              uvx_stream_t stream);
int uvx_record_scores_rows_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                   uvx_cutoffs cutoffs, const int32_t* idx, int64_t steps, float* scores, float* raw,
                                   uvx_stream_t stream);
int uvx_sample_slots_cutoffs(const float* logits, int64_t B, int64_t V, const float* temperature, const int32_t* top_k,
                             const float* top_p, const float* cutoffs, const float* u, int64_t u_stride, const int32_t* n_new,
                             const int32_t* active, int64_t* out_idx, uvx_stream_t stream);
int uvx_sample_rows_cutoffs(const float* logits, int64_t R, int64_t V, const float* temperature, const int32_t* top_k,
                            const float* top_p, const float* cutoffs, const float* u, int64_t u_stride, const int32_t* active,
                            const int32_t* row_slot, const int32_t* row_idx, int64_t* out_idx, uvx_stream_t stream);

/* Prompt lookup inside the slot step (ultravox_b200/engine.py SlotDecodeEngine with prompt_lookup_num_tokens = K): slot s owns
 * the R = slots * (K + 1) step rows r = s * (K + 1) + i, i <= K.  Per-slot arrays are [slots]; per-row arrays are [R]; seq is
 * [slots, seq_stride] int64.
 * uvx_lookup_draft_slots       one CTA per slot: the drafts of uvx_lookup_draft on seq[s, 0:cur_len[s]] with k[s] (<= K, 0 = none),
 *                              n[s], n_new[s], max_new[s] - searched only when active[s], !done[s] and !prefilling[s] - written to
 *                              seq[s, L, L + d) and n_draft[s] = d.  Row 0 of the slot feeds tok = token[s] at row_pos / row_lens /
 *                              row_rope = pos[s] / lens[s] / rope_pos[s] (the slot's row of a plain step); row i in 1..d feeds
 *                              draft i - 1 at pos[s] + i, lens[s] + i, rope_pos[s] + i; rows past d feed token[s] at row 0's values.
 *                              pen_len = L + i and idx = n_new[s] + i for rows i <= d, idx = -1 past them; row_slot = s;
 *                              cache_row = s for rows 1..d and for row 0 unless the slot is done or prefilling, else -1 (no
 *                              K / V write).  1 <= K <= 31.
 * uvx_lookup_accept_slots      for each active slot that is not done: uvx_lookup_accept's m over its rows (pick[r], tok[r + 1])
 *                              appended at seq[s, cur_len[s]]; cur_len / n_new += m + 1; done = the last pick is an EOS id or
 *                              n_new >= max_new; pos / lens / rope_pos += m + 1 while the slot stays open (m when it finishes) - what
 *                              m + 1 uvx_slot_finish calls leave; token[s] = the last pick; accepted[s] += m.  Done and inactive
 *                              slots are untouched.  n_open[0] = active slots still open.  One warp per slot.
 * uvx_sample_rows              uvx_sample_slots per row r with slot s = row_slot[r]'s temperature / top_k / top_p, active[s] and the
 *                              uniform u[s * u_stride + row_idx[r]]; rows with row_idx[r] < 0 or an inactive slot are not written.
 *                              Bit for bit the pick uvx_sample_slots makes for slot s with n_new[s] = row_idx[r].
 * uvx_repetition_penalty_rows_map  uvx_repetition_penalty_slots per row r with slot s = row_slot[r]'s penalty and active flag over
 *                              seq[s, 0:row_len[r]], scratch [R, seq_stride] fp32 (row r's own); rows with row_idx[r] < 0 skipped.
 * uvx_token_logprobs_rows      uvx_token_logprobs per row r with n_top[s], s = row_slot[r], written to slot s's outputs
 *                              (out_lp[s * cap + dst[r]], ...); dst[r] < 0 writes nothing.                                      */
int uvx_lookup_draft_slots(int64_t* seq, int64_t seq_stride, const int64_t* token, const int32_t* cur_len, const int32_t* n_new,
                           const int32_t* max_new, const int32_t* k, const int32_t* n, const int32_t* done, const int32_t* active,
                           const int32_t* prefilling, const int32_t* pos, const int32_t* lens, const int32_t* rope_pos, int64_t slots,
                           int32_t K, const int64_t* eos_ids, int32_t n_eos, int64_t* tok, int32_t* n_draft, int32_t* row_pos,
                           int32_t* row_lens, int32_t* row_rope, int32_t* pen_len, int32_t* idx, int32_t* row_slot,
                           int32_t* cache_row, uvx_stream_t stream);
int uvx_lookup_accept_slots(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, int64_t slots, int32_t K,
                            const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride, int64_t* token, int32_t* done,
                            int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active, int32_t* pos,
                            int32_t* lens, int32_t* rope_pos, int32_t* accepted, int32_t* n_open, uvx_stream_t stream);
int uvx_sample_rows(const float* logits, int64_t R, int64_t V, const float* temperature, const int32_t* top_k, const float* top_p,
                    const float* u, int64_t u_stride, const int32_t* active, const int32_t* row_slot, const int32_t* row_idx,
                    int64_t* out_idx, uvx_stream_t stream);
int uvx_repetition_penalty_rows_map(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride, const float* penalty,
                                    const int32_t* active, const int32_t* row_slot, const int32_t* row_len, const int32_t* row_idx,
                                    float* scratch, uvx_stream_t stream);
int uvx_token_logprobs_rows(const float* logits, int64_t R, int64_t V, const int64_t* tok, const int32_t* n_top,
                            const int32_t* row_slot, const int32_t* dst, int64_t cap, int32_t n_max, float* out_lp, int64_t* out_ids,
                            float* out_top, uvx_stream_t stream);

/* Token constraints (hf:generation/logits_process.py SequenceBias -> NoRepeatNGram -> NoBadWords -> MinLength / MinNewTokens
 * -> SuppressTokens -> SuppressTokensAtBegin, transformers 5.5), one launch in place on fp32 logits rows, run BEFORE the
 * repetition penalty: every processor but the sequence bias adds or sets -inf, which the penalty maps to itself (NaN and +inf
 * too), so the result equals HF's up to the sign of zero (HF adds its all-row bias tensor, +0 where no entry matches, to every
 * column, which turns a -0.0 score into +0.0; here only the tokens with entries are written).  A setting is cfg int32[4] = (n, min_len, begin_len, n_ent) plus a packed table of n_ent
 * entries: entry j is the ids ids[end[j - 1] .. end[j]) (end[-1] = 0, at least one id), int64 ids, int32 end, fp32 bias[j] and
 * int32 kind[j] (UVX_CK_*).  Its last id is its target token t; the others are the prefix that the last ids of the sequence
 * must equal for the entry to match (an entry longer than L never matches).  All entries of one t are consecutive, in HF's
 * order: sequence-bias entries (the single-token one first, then dict order), bad words, sets.  Per row with sequence seq[0:L]:
 *   x[t] = ((x[t] + sum of matching UVX_CK_BIAS) + sum of matching UVX_CK_BAD), each sum in fp32 from 0 and added only when t
 *          has entries of that kind; then x[t] = -inf if a matching entry is UVX_CK_SUPPRESS, UVX_CK_BEGIN with L == begin_len,
 *          or UVX_CK_MIN_LEN with L < min_len;
 *   then (n >= 1 and L + 1 >= n) x[seq[e]] = -inf for every e in [n - 1, L) with seq[e - n + 1 .. e - 1] == seq[L - n + 1 .. L - 1].
 * seq is never read at or past L.  Every form runs 1024 threads per row.
 * uvx_logits_constraints           B rows, row b over seq[b * seq_stride, 0:cur_len[0]], one setting.
 * uvx_logits_constraints_slots     active rows b over seq[b, 0:cur_len[b]] with setting b (cfg + 4 b, table at b * tab_stride).
 * uvx_logits_constraints_rows      row b over seq[b * seq_stride, 0:len[b]] (seq_stride 0: one shared sequence), one setting.
 * uvx_logits_constraints_rows_map  row r of slot s = row_slot[r] (active[s], row_idx[r] >= 0; others untouched) over
 *                                  seq[s, 0:row_len[r]] with setting s.                                                          */
#define UVX_CK_BIAS 0      /* sequence_bias: add */
#define UVX_CK_BAD 1       /* bad_words_ids: add (bias -inf) */
#define UVX_CK_SUPPRESS 2  /* suppress_tokens: set -inf */
#define UVX_CK_BEGIN 3     /* begin_suppress_tokens: set -inf when L == begin_len */
#define UVX_CK_MIN_LEN 4   /* EOS under min_length / min_new_tokens: set -inf when L < min_len */
int uvx_logits_constraints(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                           const int32_t* cfg, const int64_t* ids, const int32_t* end, const float* bias, const int32_t* kind,
                           uvx_stream_t stream);
int uvx_logits_constraints_slots(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                                 const int32_t* active, const int32_t* cfg, const int64_t* ids, const int32_t* end, const float* bias,
                                 const int32_t* kind, int64_t tab_stride, uvx_stream_t stream);
int uvx_logits_constraints_rows(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride, const int32_t* len,
                                const int32_t* cfg, const int64_t* ids, const int32_t* end, const float* bias, const int32_t* kind,
                                uvx_stream_t stream);
int uvx_logits_constraints_rows_map(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride,
                                    const int32_t* active, const int32_t* row_slot, const int32_t* row_len, const int32_t* row_idx,
                                    const int32_t* cfg, const int64_t* ids, const int32_t* end, const float* bias, const int32_t* kind,
                                    int64_t tab_stride, uvx_stream_t stream);

/* Stop strings (hf:generation/stopping_criteria.py StopStringCriteria, transformers 5.5), checked on the device after the pick,
 * so a row that completes a stop string finishes inside the captured step.  The table is HF's precompute in sparse form, int32:
 *   [0] n_ent  [1] n_stop  [2] mvp (max_valid_positions)  [3] mvel (max_valid_end_lens)  [4] W_max (longest string, characters)
 *   [5, 5 + n_stop)  the target lengths;  then ids [n_ent], ascending: the tokens with an entry other than -1 outside HF's
 *   length column;  then their HF rows [n_ent][rw], rw = n_stop * (mvp + mvel) + 1: the valid positions of string s at
 *   s * mvp, its end overlaps at n_stop * mvp + s * mvel, the token's length last.  n_ent = 0: no stop strings (hit 0).
 * Rule for one row with x = (the L preceding tokens, the candidate): W = min(W_max, L + 1); for each string s and each end
 * overlap e > 0 of the candidate, c = e, hit if c >= |s|; then for j = 1 .. W - 1 with y = x[L - j]: stop this chain unless c
 * is one of y's valid positions for s, else c += len(y), hit if c >= |s|.  Ids outside the table have no entries.  hit[r] is
 * 1 or 0.  seq is never read at or past L.  One warp per row (32 threads): the lanes walk the chains, the window is looked up
 * 32 tokens at a time (binary search over ids).
 * uvx_stop_strings           B rows, row b's candidate tok[b] after seq[b * seq_stride, 0:cur_len[0]], one table.
 * uvx_stop_strings_slots     active rows b after seq[b, 0:cur_len[b]] with table b (tab + b * tab_stride); inactive rows untouched.
 * uvx_stop_strings_rows      row r after seq[r * seq_stride, 0:len[r]] (seq_stride 0: one shared sequence), one table.
 * uvx_stop_strings_rows_map  row r of slot s = row_slot[r] (active[s], row_idx[r] >= 0; others untouched) after
 *                            seq[s, 0:row_len[r]] with table s.
 * uvx_stop_strings_beam      beam search: row r = b * K + c is candidate c of prompt b (cand_i [B, K] of uvx_beam_select),
 *                            token cand_i[r] % V after run_seq[b * nb + cand_i[r] / V, 0:cur_len[0]] (its parent's running
 *                            sequence, read before uvx_beam_update rewrites it), one table; hit [B * K].
 * Finishing forms that honour hit (each one the entry without _stop when hit is all zero, same bits):
 * uvx_token_finish_stop         uvx_token_finish; a row not yet done with hit[b] finishes too (its token kept, later ones pad), and a
 *                               row that finishes in this step (EOS or hit) gets fin_len[b] = cur_len[0] + 1 (its length then).
 * uvx_slot_finish_stop          uvx_slot_finish; hit[b] finishes the row as an EOS id would.
 * uvx_lookup_accept_stop        uvx_lookup_accept with m cut at the first i <= m with hit[i]; a hit at the last kept pick finishes.
 * uvx_lookup_accept_slots_stop  uvx_lookup_accept_slots with the same cut over the slot's rows hit[s * (K + 1) + i].
 * uvx_beam_update_stop          uvx_beam_update where candidate c of prompt b also hits the stopping criteria when
 *                               hit[b * K + c] (HF _beam_search's next_token_hits_stopping_criteria with StopStringCriteria).          */
int uvx_stop_strings(const int64_t* tok, int64_t B, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len, const int32_t* tab,
                     int32_t* hit, uvx_stream_t stream);
int uvx_stop_strings_slots(const int64_t* tok, int64_t B, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                           const int32_t* active, const int32_t* tab, int64_t tab_stride, int32_t* hit, uvx_stream_t stream);
int uvx_stop_strings_rows(const int64_t* tok, int64_t R, const int64_t* seq, int64_t seq_stride, const int32_t* len, const int32_t* tab,
                          int32_t* hit, uvx_stream_t stream);
int uvx_stop_strings_rows_map(const int64_t* tok, int64_t R, const int64_t* seq, int64_t seq_stride, const int32_t* active,
                              const int32_t* row_slot, const int32_t* row_len, const int32_t* row_idx, const int32_t* tab,
                              int64_t tab_stride, int32_t* hit, uvx_stream_t stream);
int uvx_stop_strings_beam(const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V, const int64_t* run_seq,
                          int64_t seq_stride, const int32_t* cur_len, const int32_t* tab, int32_t* hit, uvx_stream_t stream);
int uvx_beam_update_stop(const float* cand_s, const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V, const int64_t* eos_ids,
                         int32_t n_eos, int32_t max_new, const float* len_div, int32_t early_stopping, int32_t lp_positive,
                         float* run_score, int64_t* run_seq, int64_t* pool_seq, int64_t seq_stride, float* pool_score,
                         int32_t* pool_len, int32_t* pool_fin, int32_t* parent, int64_t* tok, int32_t* heur, int32_t* flags,
                         uint32_t* ticket, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1, int32_t* bump2,
                         int32_t* done, const int32_t* hit, uvx_stream_t stream);
int uvx_token_finish_stop(int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int64_t* seq,
                          int64_t seq_stride, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1, int32_t* bump2,
                          int32_t* all_done, int64_t B, const int32_t* hit, int32_t* fin_len, uvx_stream_t stream);
int uvx_slot_finish_stop(const int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride,
                         int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active, int32_t* pos, int32_t* lens,
                         int32_t* rope_pos, int32_t* n_open, int64_t B, const int32_t* hit, uvx_stream_t stream);
int uvx_lookup_accept_stop(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, const int64_t* eos_ids, int32_t n_eos,
                           int64_t* seq, int32_t* cur_len, int32_t* n_new, int32_t max_new, int32_t* step, int32_t* accepted,
                           int32_t steps, int32_t* done, const int32_t* hit, uvx_stream_t stream);
int uvx_lookup_accept_slots_stop(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, int64_t slots, int32_t K,
                                 const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride, int64_t* token, int32_t* done,
                                 int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active, int32_t* pos,
                                 int32_t* lens, int32_t* rope_pos, int32_t* accepted, int32_t* n_open, const int32_t* hit,
                                 uvx_stream_t stream);

/* Beam search (hf:generation/utils.py _beam_search, transformers 5.5, and the helpers above it), one decode step as four
 * launches that read every per-step scalar from device memory.  B prompts, nb <= 8 beams each: row r = b * nb + j.
 * uvx_log_softmax   out[r] = log_softmax(in[r]) in fp32 (in == out allowed).  Beam search scores log-probs; the repetition
 *                   penalty (uvx_repetition_penalty on the running sequences) then applies to these, not to the logits.
 * uvx_beam_select   per prompt, the K (1 <= K <= 64, K <= V) largest a[b, j * V + v] = logprobs[r, v] + run_score[r] (one
 *                   fp32 add), sorted descending: out_s[b, :K] the values, out_i[b, :K] the flat index j * V + v.
 *                   row_s / row_i [B * nb * K] are scratch (the per-row top K, merged per prompt).
 * uvx_beam_update   one CTA per prompt on the K candidates (K = max(2, 1 + n_eos) * nb): a candidate hits the stopping criteria
 *                   if its token is in eos_ids or step_idx[0] + 1 >= max_new; the next running beams are the top nb of
 *                   score + hit * -1e9 (run_score, tok, parent = the source row, run_seq rows gathered by parent and extended at
 *                   cur_len[0]); the finished pool (pool_seq / pool_score / pool_len = generated length / pool_fin) keeps the top
 *                   nb of itself merged with score / len_div[step_idx + 1] + the -1e9 masks (early_stopping 1 and a full pool,
 *                   heur[b] cleared, not a top-nb finisher).  heur[b] &= the early-stop heuristic (early_stopping 0 = False,
 *                   1 = True, 2 = "never"; lp_positive = length_penalty > 0), evaluated at the new length with the divisor
 *                   len_div[len] = fp32(double(len) ** length_penalty).  The last prompt's CTA writes done[0] = !(loop
 *                   condition over the batch), advances cur_len[0] and step_idx[0] and resets ticket[0] (0 before the first
 *                   launch); bump{0,1,2}[r]++ (if given).  flags [B] is scratch.  While done[0] is set a launch changes nothing
 *                   but parent, which becomes the identity.  All scores are fp32 in HF's operation order.
 * uvx_kv_reorder    k / v caches [L, B * nb, S_max, row_elems] bf16 (contiguous): row r <- row parent[r] (parent in the same
 *                   prompt) at positions [0, n_pos[0]), in place, for every layer in one launch.  A row whose parent is itself
 *                   is not written, and is read only when another beam descends from it; positions >= n_pos[0] are untouched.
 *                   With parent[b * nb + j] = b * nb it broadcasts each prompt's prefilled row to its beams.
 * Ties: where two values are exactly equal (in both selections and in the pool merge) the lower flat / candidate / merged
 * index ranks first.  torch.topk leaves that order unspecified; in a search it matters only at a top-k cut.               */
int uvx_log_softmax(const float* in, float* out, int64_t rows, int64_t V, uvx_stream_t stream);
int uvx_beam_select(const float* logprobs, int64_t B, int32_t nb, int64_t V, const float* run_score, int32_t K, float* row_s,
                    int64_t* row_i, float* out_s, int64_t* out_i, uvx_stream_t stream);
int uvx_beam_update(const float* cand_s, const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V, const int64_t* eos_ids,
                    int32_t n_eos, int32_t max_new, const float* len_div, int32_t early_stopping, int32_t lp_positive,
                    float* run_score, int64_t* run_seq, int64_t* pool_seq, int64_t seq_stride, float* pool_score, int32_t* pool_len,
                    int32_t* pool_fin, int32_t* parent, int64_t* tok, int32_t* heur, int32_t* flags, uint32_t* ticket,
                    int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1, int32_t* bump2, int32_t* done,
                    uvx_stream_t stream);
int uvx_kv_reorder(void* k_cache, void* v_cache, int64_t L, int64_t B, int32_t nb, int64_t S_max, int64_t row_elems,
                   const int32_t* parent, const int32_t* n_pos, uvx_stream_t stream);

/* Paged KV cache bookkeeping (pages of 64 positions, see uvx_attention_paged).
 * uvx_kv_page_map    for each of `rows` step rows: cache_row[r] < 0, or r < n_frozen and frozen[r] != 0 (optional, e.g. the
 *                    slots' done flags: a finished row that is still fed must not overwrite the last position its conversation
 *                    keeps) -> page_out[r] = -1, off_out[r] = 0 (no table read); otherwise page_out[r] = table[cache_row[r] * table_stride + pos[r] / 64], off_out[r] = pos[r] % 64.
 *                    uvx_rope_kv_append_map then appends into a pool layer viewed as [n_pages, 64, Hkv, D] with
 *                    cache_row = page_out and positions = off_out.  Everything is read on the device (graph-capturable).
 * uvx_kv_pages_copy  bit-exact copy of positions [p0, p1) of every layer, K and V, between a contiguous one-row cache (layer
 *                    l, position p at l * row_layer_stride + p * row_elems) and the pool (page pages[p / 64], row p % 64, at
 *                    l * pool_layer_stride + (page * 64 + p % 64) * row_elems), 16-byte accesses, one launch.  to_pages = 1:
 *                    row -> pages (scatter); 0: pages -> row (gather).  `pages` (device) lists the pages of positions 0, 64,
 *                    128, ...; nothing outside [p0, p1) is written.                                                       */
int uvx_kv_page_map(const int32_t* table, int64_t table_stride, const int32_t* cache_row, const int32_t* pos, const int32_t* frozen,
                    int64_t n_frozen, int64_t rows, int32_t* page_out, int32_t* off_out, uvx_stream_t stream);
int uvx_kv_pages_copy(void* k_row, void* v_row, int64_t row_layer_stride, void* k_pool, void* v_pool, int64_t pool_layer_stride,
                      int64_t L, int64_t row_elems, const int32_t* pages, int64_t p0, int64_t p1, int32_t to_pages,
                      uvx_stream_t stream);
/* uvx_kv_pages_copy between a bf16 one-row cache and an e4m3 pool (see uvx_attention_paged_fp8): to_pages = 1 quantizes, 0
 * dequantizes, with layer l's scales kv_scales[2 l] (K) / kv_scales[2 l + 1] (V).  row_elems and both layer strides % 16 == 0;
 * nothing outside [p0, p1) is written.                                                                                          */
int uvx_kv_pages_copy_fp8(void* k_row, void* v_row, int64_t row_layer_stride, void* k_pool, void* v_pool, int64_t pool_layer_stride,
                          int64_t L, int64_t row_elems, const int32_t* pages, int64_t p0, int64_t p1, int32_t to_pages,
                          const float* kv_scales, uvx_stream_t stream);
/* uvx_kv_pages_move  whole pages between two pools, byte for byte, every layer, K and V, one launch: page src_pages[j] of the
 *                    source -> page dst_pages[j] of the destination for j < n (both lists int32 on the device; the caller keeps
 *                    the ids inside each pool and the destination ids distinct).  Layer l of a pool starts at
 *                    l * *_layer_stride bytes, page p at p * page_bytes within it; nothing else is written.  The element type
 *                    is not read (a bf16 and an e4m3 pool move alike; an e4m3 pool's scales do not change).  Exception to
 *                    the DEVICE-pointer convention: each of the four bases may instead be pinned / registered host memory
 *                    mapped at the same address (the SMs read / write it over PCIe, no staging buffer); anything else (a
 *                    pageable host pointer) returns UVX_ERR_ARG before any launch (cudaPointerGetAttributes).  16-byte
 *                    aligned bases, page_bytes and layer strides % 16 == 0, n >= 0 (0 launches nothing).  Not meant for
 *                    graph capture: the serving scheduler calls it between replays, on the stream of every other kernel
 *                    that touches either pool.                                                                            */
int uvx_kv_pages_move(const void* src_k, const void* src_v, int64_t src_layer_stride, void* dst_k, void* dst_v,
                      int64_t dst_layer_stride, int64_t L, int64_t page_bytes, const int32_t* src_pages, const int32_t* dst_pages,
                      int64_t n, uvx_stream_t stream);

/* Shifted causal-LM cross entropy (hf:loss/loss_utils.py:28-67; called through LlamaForCausalLM.forward(labels=)
 * from ref:ultravox/model/ultravox_model.py:328-334).  logits [B*S, V] fp32 (row_stride elements), labels [B, S]
 * un-shifted (the shift and the ignore_index padding happen inside).  row_loss/row_lse [B*S] are kept for the
 * backward; out_loss2[0] = mean loss over non-ignored positions, out_loss2[1] = their count.  shift = 1 is the
 * HF convention above; shift = 0 takes labels[row] as is (rows pre-gathered by the caller).               */
int uvx_ce_loss(const float* logits, int64_t row_stride, const int64_t* labels, int64_t B, int64_t S, int64_t V,
                int64_t ignore_index, int shift, float* row_loss, float* row_lse, float* out_loss2, uvx_stream_t stream);

/* a15: KL distillation loss of ref:ultravox/model/ultravox_model.py:202-257 (the reference's default training loss):
 * F.kl_div(log_softmax(student / T), softmax(teacher / T), "batchmean") on the prediction rows + eot_loss_weight x the
 * same on the EOT rows.  Rows are pre-gathered ([R, V] fp32 each) and carry a weight row_w[r] (1/#pred, plus
 * eot_weight/#eot on EOT rows): out_loss[0] = sum_r row_w[r] * KL_r.  uvx_kl_bwd gives d/d(student logits) in bf16.  */
int uvx_kl_loss(const float* student, const float* teacher, int64_t row_stride, int64_t R, int64_t V, float temperature,
                const float* row_w, float* row_kl, float* lse_s, float* lse_t, float* out_loss, uvx_stream_t stream);
int uvx_kl_bwd(const float* student, const float* teacher, int64_t row_stride, int64_t R, int64_t V, float temperature,
               const float* row_w, const float* lse_s, const float* lse_t, float grad_scale, void* dlogits,
               uvx_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * a14: adapter backward (encoder + LLM frozen: ref apply_lora r=0, ultravox_model.py:690-709).  These are the
 * pieces torch.autograd runs for the reference between `loss.backward()` and the projector weights; dense
 * contractions reuse uvx_gemm_bf16 (dgrad against pre-transposed weights, wgrad against transposed activations). */
int uvx_rope_bwd(void* dqkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                 const float* sin_tab, const int32_t* positions, int64_t rows_per_seq, int64_t pos_offset,
                 uvx_stream_t stream);
/* dQ/dK/dV of uvx_attention; `a` is the forward's argument struct (with a->lse filled by the forward), o the
 * forward output, dout its gradient (same strides as o); delta_ws is [B, Hq, Sq] fp32 scratch.               */
int uvx_attention_bwd(const uvx_attn_args* a, const void* o, const void* dout, void* dq, void* dk, void* dv,
                      int64_t dq_rs, int64_t dq_bs, int64_t dk_rs, int64_t dk_bs, int64_t dv_rs, int64_t dv_bs,
                      float* delta_ws, uvx_stream_t stream);
int uvx_transpose_bf16(const void* in, int64_t rows, int64_t cols, int64_t in_row_stride, void* out,
                       int64_t out_row_stride, uvx_stream_t stream);
/* dx = dres + d(rmsnorm)/dx . dy (dx may be NULL), dw[cols] += sum_rows dy * xhat (fp32, dw may be NULL);
 * dy / dres / dx are dense [rows, cols].  group_* as in uvx_rmsnorm; in stack mode dx is written in the stacked
 * layout [rows, cols] (the frames of a group in order, the zero tail of the last row included), which the
 * projector backward views as [N, group_rows * stack, C] to get d(encoder output).                          */
int uvx_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, float* dw,
                    int64_t rows, int64_t cols, int64_t x_row_stride, int64_t group_rows, int64_t group_stride,
                    int64_t valid_elems, float eps, uvx_stream_t stream);
/* LayerNorm data gradient (+ optional residual-branch gradient dres): dx = LN'(x)^T dy + dres; the norm's weight / bias are frozen
 * (encoder backward of LoRA training, hf:modeling_whisper.py:403-440).  cols %% 8 == 0, <= 2048.                                */
int uvx_layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int64_t rows, int64_t cols,
                      float eps, uvx_stream_t stream);
/* erf-form GELU on bf16 (training keeps fc1's pre-activation) and its derivative: dx = dy * (Phi(x) + x phi(x)); n %% 8 == 0 */
int uvx_gelu(const void* x, void* y, int64_t n, uvx_stream_t stream);
int uvx_gelu_bwd(const void* x, const void* dy, void* dx, int64_t n, uvx_stream_t stream);
int uvx_swiglu_bwd(const void* x, const void* dout, void* dx, int64_t rows, int64_t H, int64_t x_row_stride,
                   int gate_first, uvx_stream_t stream);
/* dlogits (bf16 [B*S, V]) of uvx_ce_loss: (softmax - onehot) * grad_scale / count on valid rows, 0 elsewhere. */
int uvx_ce_bwd(const float* logits, int64_t row_stride, const int64_t* labels, int64_t B, int64_t S, int64_t V,
               int64_t ignore_index, int shift, const float* row_lse, const float* loss2, float grad_scale,
               void* dlogits, uvx_stream_t stream);
/* out[i, :] = idx[i] >= 0 ? src[idx[i], :] : 0  (gradient of the splice: rows of d(inputs_embeds) -> d(audio_embeds)) */
int uvx_gather_rows(const void* src, const int32_t* idx, int64_t rows, int64_t d, void* out, uvx_stream_t stream);
/* inverse of the splice table: inv[audio_row] = position (b*S+s) it was spliced to, or -1                     */
int uvx_splice_inverse(const int32_t* src, int64_t n_pos, int32_t* inv, int64_t n_audio_rows, uvx_stream_t stream);
/* AdamW on bf16 parameters with fp32 gradient / moments (torch.optim.AdamW semantics, ref meta_config.yaml:27) */
int uvx_adamw(void* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
              float weight_decay, int64_t step, float grad_scale, uvx_stream_t stream);
int uvx_cast_f32_bf16(const float* in, void* out, int64_t n, uvx_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * a14: the optimizer step of the released recipes (HF Trainer, ref train.py:250-307): global-norm gradient clipping
 * (torch.nn.utils.clip_grad_norm_, max_grad_norm), AdamW (adamw_torch) with a learning-rate schedule read from a device
 * table, and gradient accumulation over micro-batches.  Every trained tensor of a step (the projector's flat buffer, the
 * encoder-LoRA A / Bq / Bk) goes through one launch per entry, described by a tensor list passed by value at launch time.
 * Entry i: numel[i] > 0 elements; the pointers an entry reads are named below, the others are ignored.  Tensors of one
 * list must not overlap.  Vector accesses are used where a tensor's pointers are 16-byte (fp32) / 8-byte (bf16) aligned.  */
#define UVX_TL_MAX 8
typedef struct uvx_tensor_list {
  int64_t count;                /* 1 .. UVX_TL_MAX                                                                 */
  int64_t numel[UVX_TL_MAX];
  const float* g[UVX_TL_MAX];   /* fp32 gradients                                                                  */
  float* acc[UVX_TL_MAX];       /* fp32 gradient accumulators (uvx_grad_accumulate)                                */
  void* p[UVX_TL_MAX];          /* bf16 parameters (uvx_adamw_multi)                                               */
  float* m[UVX_TL_MAX];         /* fp32 first / second moments (uvx_adamw_multi)                                   */
  float* v[UVX_TL_MAX];
} uvx_tensor_list;

/* Size of the workspace of uvx_grad_norm_clip: UVX_NORM_BLOCKS fp64 block partials + a 4-byte ticket.                  */
#define UVX_NORM_BLOCKS 1024
#define UVX_NORM_WS_BYTES (8 * UVX_NORM_BLOCKS + 8)

/* uvx_grad_norm_clip   reads g[i].  norm = || scale[0] * g ||_2 over all tensors of the list, where each element is first
 *                      rounded to fp32 as fl(g * scale[0]) (the gradient the reference would hold after the all-reduce mean
 *                      and the 1 / accumulation-steps loss division), squared and summed in fp64.  Deterministic: a fixed
 *                      grid of UVX_NORM_BLOCKS blocks, a fixed per-thread order, fp64 block partials, and the last block to
 *                      finish (ticket in the workspace) sums the partials in index order; the result depends on the inputs
 *                      only.  norm_coef[0] = fp32(sqrt(sum)); norm_coef[1] = coef = min(max_norm / (norm + 1e-6), 1) in
 *                      fp32 as torch.nn.utils.clip_grad_norm_ computes it (error_if_nonfinite=False; the division is
 *                      torch's reciprocal-then-multiply): a NaN norm gives a NaN
 *                      coef, an Inf norm coef 0; max_norm <= 0 means no clipping, coef = 1 (the norm is still written).
 *                      If step is not NULL the same final block does step[0] += 1 (int64, device) and writes
 *                      lr[0] = lr_table[min(step[0], table_len) - 1] (the lr of the optimizer step about to run).
 *                      workspace: UVX_NORM_WS_BYTES bytes, zero before the first call; the last block resets the ticket,
 *                      so calls (and graph replays) may follow each other on one stream without re-initialisation.
 *                      Nothing is read from the host but the list and max_norm: the call is graph-capturable.
 * uvx_adamw_multi      reads g[i], p[i], m[i], v[i]; writes p, m, v.  torch.optim.AdamW (decoupled weight decay,
 *                      adamw_torch) with lr = lr[0], step = step[0] (>= 1), coef = coef[0] (NULL = 1) and scale = scale[0]
 *                      read from device memory: effective gradient fl(fl(g * scale) * coef); p *= 1 - lr * wd;
 *                      m = lerp(m, g, 1 - beta1); v = beta2 v + (1 - beta2) g^2; p -= (lr / bc1) * m / (sqrt(v) / sqrt(bc2) + eps)
 *                      with bc = 1 - beta ** step, the scalars formed in double from the device values and rounded to
 *                      fp32 where torch's foreach implementation rounds them.  Moments fp32, parameters bf16
 *                      (round-to-nearest once per step).  A NaN gradient makes its own elements NaN; a NaN coef makes every
 *                      element NaN, as torch's clip + step does.  Elementwise: deterministic.
 * uvx_grad_accumulate  reads g[i]; acc[i] = g[i] if assign else acc[i] + g[i] (fp32), the micro-batch accumulation of a
 *                      gradient-accumulation step.  acc may not alias g.  Deterministic.                                */
int uvx_grad_norm_clip(const uvx_tensor_list* tl, const float* scale, float max_norm, void* workspace, float* norm_coef,
                       int64_t* step, const float* lr_table, int64_t table_len, float* lr, uvx_stream_t stream);
int uvx_adamw_multi(const uvx_tensor_list* tl, const float* lr, const int64_t* step, const float* coef, const float* scale,
                    double beta1, double beta2, double eps, double weight_decay, uvx_stream_t stream);
int uvx_grad_accumulate(const uvx_tensor_list* tl, int32_t assign, uvx_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* UVX_H_ */
