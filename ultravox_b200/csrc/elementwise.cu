// HBM-bound glue kernels of the hot path: RoPE, SwiGLU, mel re-layout, embedding gather + audio splice.
// All use 128-bit accesses where the layout allows and are pure index / elementwise work (no tensor cores).
#include "uvx_common.cuh"

namespace uvx {

// ------------------------------------------------------------------------------------------- RoPE
// one thread handles 8 consecutive dims j..j+7 (j < D/2) of one (row, head): loads x[j..] and x[j+D/2..]
__global__ void rope_kernel(bf16* __restrict__ qkv, int64_t rows, int64_t row_stride, int heads_rot, int D,
                            const float* __restrict__ cos_tab, const float* __restrict__ sin_tab,
                            const int32_t* __restrict__ positions, int64_t rows_per_seq, int64_t pos_offset, float sgn) {
  pdl_trigger();
  pdl_wait();
  const int half = D / 2;
  const int vec_per_head = half / 8;
  const int64_t total = rows * heads_rot * vec_per_head;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int jv = (int)(idx % vec_per_head);
    const int h = (int)((idx / vec_per_head) % heads_rot);
    const int64_t r = idx / ((int64_t)vec_per_head * heads_rot);
    const int64_t pos = positions ? (int64_t)positions[r] : pos_offset + (r % rows_per_seq);
    bf16* base = qkv + r * row_stride + (int64_t)h * D + jv * 8;
    float x1[8], x2[8], c[8], s[8], o1[8], o2[8];
    unpack8(*reinterpret_cast<const bf16x8*>(base), x1);
    unpack8(*reinterpret_cast<const bf16x8*>(base + half), x2);
    const float4* cp = reinterpret_cast<const float4*>(cos_tab + pos * half + jv * 8);
    const float4* sp = reinterpret_cast<const float4*>(sin_tab + pos * half + jv * 8);
    *reinterpret_cast<float4*>(c) = cp[0];
    *reinterpret_cast<float4*>(c + 4) = cp[1];
    *reinterpret_cast<float4*>(s) = sp[0];
    *reinterpret_cast<float4*>(s + 4) = sp[1];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      // x*cos + rotate_half(x)*sin (first half: -x2, second half: +x1); sgn = -1 applies the transposed rotation (backward)
      rope_pair(x1[e], x2[e], c[e], sgn * s[e], o1[e], o2[e]);
    }
    *reinterpret_cast<bf16x8*>(base) = pack8(o1);
    *reinterpret_cast<bf16x8*>(base + half) = pack8(o2);
  }
}

// ------------------------------------------------------------------------------------------- SwiGLU
__global__ void swiglu_kernel(const bf16* __restrict__ x, bf16* __restrict__ out, int64_t rows, int64_t H,
                              int64_t x_row_stride, int gate_first) {
  pdl_trigger();
  pdl_wait();
  const int64_t vec_per_row = H / 8;
  const int64_t total = rows * vec_per_row;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / vec_per_row, j = (idx % vec_per_row) * 8;
    float a[8], g[8], o[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + r * x_row_stride + j), a);
    unpack8(*reinterpret_cast<const bf16x8*>(x + r * x_row_stride + H + j), g);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float gate = gate_first ? a[e] : g[e];
      const float lin = gate_first ? g[e] : a[e];
      // torch: silu(gate) is rounded to bf16 before the multiply
      o[e] = __bfloat162float(__float2bfloat16_rn(silu(gate))) * lin;
    }
    *reinterpret_cast<bf16x8*>(out + r * H + j) = pack8(o);
  }
}

// --------------------------------------------------------------------- mel [N, C, T] f32 -> [N, T+2, C] bf16
// 32x32 shared-memory transpose tile; guard rows t = -1 and t = T are zeroed by the same kernel.
__global__ void mel_to_tm_kernel(const float* __restrict__ mel, int n_mels, int64_t T, bf16* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float tile[32][33];
  const int64_t n = blockIdx.z;
  const int64_t t0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const float* src = mel + n * n_mels * T;
  bf16* dst = out + n * (T + 2) * n_mels;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i;
    const int64_t t = t0 + threadIdx.x;
    tile[i][threadIdx.x] = (c < n_mels && t < T) ? src[(int64_t)c * T + t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int64_t t = t0 + i;
    const int c = c0 + threadIdx.x;
    if (t < T && c < n_mels) dst[(t + 1) * n_mels + c] = __float2bfloat16_rn(tile[threadIdx.x][i]);
  }
  if (blockIdx.x == 0 && threadIdx.y == 0) {
    const int c = c0 + threadIdx.x;
    if (c < n_mels) {
      dst[c] = __float2bfloat16_rn(0.f);
      dst[(T + 1) * n_mels + c] = __float2bfloat16_rn(0.f);
    }
  }
}

// --------------------------------------------------------------------------------- splice plan
// Single CTA.  Chunks are applied in batch order with a barrier in between, so overlapping ranges resolve
// exactly like the reference's sequential slice assignments.
__global__ void splice_plan_kernel(const int64_t* __restrict__ start_idx, const int32_t* __restrict__ tok_len,
                                   const int64_t* __restrict__ audio_batch_size, int64_t n_chunks, int64_t B, int64_t S,
                                   int64_t tok_stride, int32_t* __restrict__ src) {
  pdl_trigger();
  pdl_wait();
  for (int64_t i = threadIdx.x; i < B * S; i += blockDim.x) src[i] = -1;
  __syncthreads();
  int64_t a = 0;
  for (int64_t b = 0; b < B; ++b) {
    const int64_t cnt = audio_batch_size[b];
    for (int64_t c = 0; c < cnt && a < n_chunks; ++c, ++a) {
      const int64_t s = start_idx[a];
      const int64_t n = tok_len[a];
      for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
        const int64_t pos = s + j;
        if (pos >= 0 && pos < S) src[b * S + pos] = (int32_t)(a * tok_stride + j);
      }
      __syncthreads();
    }
  }
}

// one warp per output row; 16-byte copies
__global__ void embed_splice_kernel(const int64_t* __restrict__ ids, const bf16* __restrict__ table, int64_t vocab,
                                    const bf16* __restrict__ audio, const int32_t* __restrict__ src, int64_t rows,
                                    int64_t d, bf16* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int32_t a = src ? src[row] : -1;
  const bf16* from;
  if (a >= 0) {
    from = audio + (int64_t)a * d;
  } else {
    int64_t id = ids[row];
    id = id < 0 ? 0 : (id >= vocab ? vocab - 1 : id);
    from = table + id * d;
  }
  const uint4* s4 = reinterpret_cast<const uint4*>(from);
  uint4* d4 = reinterpret_cast<uint4*>(out + row * d);
  for (int64_t i = lane; i < d / 8; i += 32) d4[i] = s4[i];
}

// --------------------------------------------------------------------------------- decode-step helpers
// Append this step's (post-RoPE) k and v rows of the fused projection to the static KV cache at positions[b].
__global__ void kv_append_kernel(const bf16* __restrict__ qkv, int64_t row_stride, int k_col, int v_col, int kv_width,
                                 bf16* __restrict__ k_cache, bf16* __restrict__ v_cache, int64_t cache_batch_stride,
                                 const int32_t* __restrict__ positions, int64_t B) {
  pdl_trigger();
  pdl_wait();
  const int vec = kv_width / 8;
  const int64_t total = B * vec * 2;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int which = (int)(idx / (B * vec));
    const int64_t rem = idx % (B * vec);
    const int64_t b = rem / vec;
    const int j = (int)(rem % vec);
    const bf16* src = qkv + b * row_stride + (which ? v_col : k_col) + j * 8;
    bf16* dst = (which ? v_cache : k_cache) + b * cache_batch_stride + (int64_t)positions[b] * kv_width + j * 8;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
  }
}


// The two row-local steps between the q|k|v projection and the attention: RoPE on the q and k heads (in place, same arithmetic
// as rope_kernel) and the append of the rotated k and of v to the static KV cache.  Row b goes to cache row b at positions[b]
// (kMap = false: the decode step), or to cache row cache_row[b] at positions[b], nowhere when cache_row[b] < 0 (kMap = true:
// the mixed decode + prompt-chunk step of continuous batching).  q and k are rotated either way.
template <bool kMap>
__device__ __forceinline__ void rope_kv_append_body(bf16* __restrict__ qkv, int64_t row_stride, int Hq, int Hkv, int D,
                                                    const float* __restrict__ cos_tab, const float* __restrict__ sin_tab,
                                                    const int32_t* __restrict__ rope_pos, bf16* __restrict__ k_cache,
                                                    bf16* __restrict__ v_cache, int64_t cache_batch_stride,
                                                    const int32_t* __restrict__ positions, const int32_t* __restrict__ cache_row,
                                                    int64_t B) {
  const int half = D / 2;
  const int vec_per_head = half / 8;
  const int heads = Hq + 2 * Hkv;
  const int kv_width = Hkv * D;
  const int64_t total = B * heads * vec_per_head;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int jv = (int)(idx % vec_per_head);
    const int h = (int)((idx / vec_per_head) % heads);
    const int64_t b = idx / ((int64_t)vec_per_head * heads);
    bf16* base = qkv + b * row_stride + (int64_t)h * D + jv * 8;
    const int64_t crow = kMap ? (int64_t)cache_row[b] : b;
    const int64_t slot = (int64_t)positions[b];
    if (h >= Hq + Hkv) {   // v head: copy both halves
      if (kMap && crow < 0) continue;
      bf16* dst = v_cache + crow * cache_batch_stride + slot * kv_width + (int64_t)(h - Hq - Hkv) * D + jv * 8;
      *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(base);
      *reinterpret_cast<uint4*>(dst + half) = *reinterpret_cast<const uint4*>(base + half);
      continue;
    }
    const int64_t pos = (int64_t)rope_pos[b];
    float x1[8], x2[8], c[8], sn[8], o1[8], o2[8];
    unpack8(*reinterpret_cast<const bf16x8*>(base), x1);
    unpack8(*reinterpret_cast<const bf16x8*>(base + half), x2);
    const float4* cp = reinterpret_cast<const float4*>(cos_tab + pos * half + jv * 8);
    const float4* sp = reinterpret_cast<const float4*>(sin_tab + pos * half + jv * 8);
    *reinterpret_cast<float4*>(c) = cp[0];
    *reinterpret_cast<float4*>(c + 4) = cp[1];
    *reinterpret_cast<float4*>(sn) = sp[0];
    *reinterpret_cast<float4*>(sn + 4) = sp[1];
#pragma unroll
    for (int e = 0; e < 8; ++e) rope_pair(x1[e], x2[e], c[e], sn[e], o1[e], o2[e]);
    const bf16x8 p1 = pack8(o1), p2 = pack8(o2);
    *reinterpret_cast<bf16x8*>(base) = p1;
    *reinterpret_cast<bf16x8*>(base + half) = p2;
    if (h >= Hq && (!kMap || crow >= 0)) {         // k head: the rotated row also goes to the cache
      bf16* dst = k_cache + crow * cache_batch_stride + slot * kv_width + (int64_t)(h - Hq) * D + jv * 8;
      *reinterpret_cast<bf16x8*>(dst) = p1;
      *reinterpret_cast<bf16x8*>(dst + half) = p2;
    }
  }
}

__global__ void rope_kv_append_kernel(bf16* __restrict__ qkv, int64_t row_stride, int Hq, int Hkv, int D,
                                      const float* __restrict__ cos_tab, const float* __restrict__ sin_tab,
                                      const int32_t* __restrict__ rope_pos, bf16* __restrict__ k_cache, bf16* __restrict__ v_cache,
                                      int64_t cache_batch_stride, const int32_t* __restrict__ positions, int64_t B) {
  pdl_trigger();
  pdl_wait();
  rope_kv_append_body<false>(qkv, row_stride, Hq, Hkv, D, cos_tab, sin_tab, rope_pos, k_cache, v_cache, cache_batch_stride, positions,
                             nullptr, B);
}

__global__ void rope_kv_append_map_kernel(bf16* __restrict__ qkv, int64_t row_stride, int Hq, int Hkv, int D,
                                          const float* __restrict__ cos_tab, const float* __restrict__ sin_tab,
                                          const int32_t* __restrict__ rope_pos, bf16* __restrict__ k_cache, bf16* __restrict__ v_cache,
                                          int64_t cache_batch_stride, const int32_t* __restrict__ cache_row,
                                          const int32_t* __restrict__ positions, int64_t B) {
  pdl_trigger();
  pdl_wait();
  rope_kv_append_body<true>(qkv, row_stride, Hq, Hkv, D, cos_tab, sin_tab, rope_pos, k_cache, v_cache, cache_batch_stride, positions,
                            cache_row, B);
}

__global__ void add_i32_kernel(int32_t* __restrict__ a, int32_t* __restrict__ b2, int64_t n, int32_t delta) {
  pdl_trigger();
  pdl_wait();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
    a[i] += delta;
    if (b2) b2[i] += delta;
  }
}

// W [N, K] row-major -> pre-tiled image [ceil(N/R)][K/64][R][64] (see include/uvx.h: uvx_tile_weight); 16 bytes per thread.
__global__ void tile_weight_kernel(const bf16* __restrict__ W, int64_t N, int64_t K, int64_t w_row_stride, int R, int interleave,
                                   bf16* __restrict__ out, int64_t total_vec) {
  const int64_t num_kb = K / 64;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total_vec; idx += (int64_t)gridDim.x * blockDim.x) {
    const int c8 = (int)(idx % 8);
    const int64_t rowi = idx / 8;                 // (t * num_kb + kb) * R + r
    const int r = (int)(rowi % R);
    const int64_t tk = rowi / R;
    const int64_t kb = tk % num_kb, t = tk / num_kb;
    int64_t src_row;
    if (interleave == 8) {
      const int64_t F = N / 2;
      const int g = r / 16, j = r % 16;
      const int64_t f = t * (R / 2) + (int64_t)g * 8 + (j & 7);
      src_row = f < F ? (j < 8 ? f : F + f) : -1;
    } else if (interleave == 16) {
      // 128-row image, fused gate|up: every 32-row quarter of a tile holds 16 gate rows then the 16 up rows of the
      // same features, so the partner of a row sits in the same TMEM lane quarter (= the same epilogue warp)
      const int64_t F = N / 2;
      const int qq = r >> 5, j = r & 31;
      const int64_t f = t * (R / 2) + qq * 16 + (j & 15);
      src_row = f < F ? (j < 16 ? f : F + f) : -1;
    } else if (interleave == 1) {
      // pair-permuted 128-row image, fused RoPE (head_dim 128 = one tile): quarter qq holds head columns 16 qq .. 16 qq + 15, then their
      // rotation partners 64 + 16 qq ..
      const int qq = r >> 5, j = r & 31;
      src_row = t * R + (j < 16 ? qq * 16 + j : 64 + qq * 16 + (j - 16));
      if (src_row >= N) src_row = -1;
    } else {
      src_row = t * R + r;
      if (src_row >= N) src_row = -1;
    }
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (src_row >= 0) v = *reinterpret_cast<const uint4*>(W + src_row * w_row_stride + kb * 64 + c8 * 8);
    reinterpret_cast<uint4*>(out)[idx] = v;
  }
}

}  // namespace uvx

extern "C" int uvx_tile_weight(const void* W, int64_t N, int64_t K, int64_t w_row_stride, int32_t R, int32_t interleave, void* out,
                               uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(W && out && N >= 1 && K >= 64 && K % 64 == 0 && w_row_stride % 8 == 0, "uvx_tile_weight: K %% 64 == 0 required");
  UVX_REQUIRE(R == 64 || R == 128 || R == 208 || R == 256, "uvx_tile_weight: R must be 64 / 128 / 208 / 256");
  UVX_REQUIRE(interleave == 0 || (interleave == 8 && R % 16 == 0 && N % 16 == 0) || (interleave == 16 && R == 128 && N % 32 == 0) ||
                  (interleave == 1 && R == 128 && N % 128 == 0),
              "uvx_tile_weight: interleave must be 0, 8 (8 gate | 8 up rows), 16 (R = 128: 16 gate | 16 up rows per 32) or 1 (R = 128: RoPE pairs)");
  const int64_t n_tiles = (N + R - 1) / R;
  const int64_t total_vec = n_tiles * (K / 64) * R * 8;
  int64_t blocks = (total_vec + 255) / 256;
  if (blocks > 148 * 32) blocks = 148 * 32;
  launch_k(tile_weight_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const bf16*)W, N, K, w_row_stride, (int)R,
           (int)interleave, (bf16*)out, total_vec);
  return check_launch("tile_weight_kernel");
}

static int rope_launch(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                       const float* sin_tab, const int32_t* positions, int64_t rows_per_seq, int64_t pos_offset, float sgn,
                       uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && cos_tab && sin_tab, "uvx_rope: null pointer");
  UVX_REQUIRE(D % 16 == 0 && row_stride % 8 == 0 && rows_per_seq > 0, "uvx_rope: D %% 16 == 0 required");
  if (rows == 0) return UVX_OK;
  const int64_t total = rows * (Hq + Hkv) * (D / 16);
  const int threads = 256;
  const int64_t blocks = (total + threads - 1) / threads;
  launch_k(rope_kernel, dim3((unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks)), dim3(threads), 0, (cudaStream_t)stream, (bf16*)qkv, rows, row_stride, Hq + Hkv, D, cos_tab, sin_tab, positions, rows_per_seq, pos_offset, sgn);
  return check_launch("rope_kernel");
}

extern "C" int uvx_rope(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                        const float* sin_tab, const int32_t* positions, int64_t rows_per_seq, int64_t pos_offset,
                        uvx_stream_t stream) {
  return rope_launch(qkv, rows, row_stride, Hq, Hkv, D, cos_tab, sin_tab, positions, rows_per_seq, pos_offset, 1.f, stream);
}

extern "C" int uvx_rope_bwd(void* dqkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                            const float* sin_tab, const int32_t* positions, int64_t rows_per_seq, int64_t pos_offset,
                            uvx_stream_t stream) {
  return rope_launch(dqkv, rows, row_stride, Hq, Hkv, D, cos_tab, sin_tab, positions, rows_per_seq, pos_offset, -1.f, stream);
}

extern "C" int uvx_swiglu(const void* x, void* out, int64_t rows, int64_t H, int64_t x_row_stride, int gate_first,
                          uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && out, "uvx_swiglu: null pointer");
  UVX_REQUIRE(H % 8 == 0 && x_row_stride % 8 == 0, "uvx_swiglu: H %% 8 == 0 required");
  if (rows == 0) return UVX_OK;
  const int64_t total = rows * (H / 8);
  const int threads = 256;
  const int64_t blocks = (total + threads - 1) / threads;
  launch_k(swiglu_kernel, dim3((unsigned)(blocks > 148 * 16 ? 148 * 16 : blocks)), dim3(threads), 0, (cudaStream_t)stream, (const bf16*)x, (bf16*)out, rows, H, x_row_stride, gate_first);
  return check_launch("swiglu_kernel");
}

extern "C" int uvx_mel_to_timemajor(const float* mel, int64_t N, int n_mels, int64_t T, void* out_tm, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(mel && out_tm, "uvx_mel_to_timemajor: null pointer");
  UVX_REQUIRE(N > 0 && T > 0 && n_mels > 0 && N < 65536, "uvx_mel_to_timemajor: bad shape");
  dim3 grid((unsigned)((T + 31) / 32), (unsigned)((n_mels + 31) / 32), (unsigned)N), block(32, 8);
  launch_k(mel_to_tm_kernel, dim3(grid), dim3(block), 0, (cudaStream_t)stream, mel, n_mels, T, (bf16*)out_tm);
  return check_launch("mel_to_tm_kernel");
}

extern "C" int uvx_splice_plan(const int64_t* start_idx, const int32_t* tok_len, const int64_t* audio_batch_size,
                               int64_t n_chunks, int64_t B, int64_t S, int64_t tok_stride, int32_t* src,
                               uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(src && B > 0 && S > 0, "uvx_splice_plan: bad arguments");
  UVX_REQUIRE(n_chunks == 0 || (start_idx && tok_len && audio_batch_size), "uvx_splice_plan: null index vectors");
  launch_k(splice_plan_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, start_idx, tok_len, audio_batch_size, n_chunks, B, S, tok_stride, src);
  return check_launch("splice_plan_kernel");
}

extern "C" int uvx_embed_splice(const int64_t* input_ids, const void* embed_tokens, int64_t vocab, const void* audio_embeds,
                                const int32_t* src, int64_t rows, int64_t d, void* out, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(input_ids && embed_tokens && out, "uvx_embed_splice: null pointer");
  UVX_REQUIRE(d % 8 == 0, "uvx_embed_splice: d %% 8 == 0 required");
  UVX_REQUIRE(!src || audio_embeds, "uvx_embed_splice: src without audio_embeds");
  if (rows == 0) return UVX_OK;
  const int warps = 8;
  launch_k(embed_splice_kernel, dim3((unsigned)((rows + warps - 1) / warps)), dim3(warps * 32), 0, (cudaStream_t)stream, input_ids, (const bf16*)embed_tokens, vocab, (const bf16*)audio_embeds, src, rows, d, (bf16*)out);
  return check_launch("embed_splice_kernel");
}

extern "C" int uvx_kv_append(const void* qkv, int64_t row_stride, int64_t k_col, int64_t v_col, int64_t kv_width, void* k_cache,
                             void* v_cache, int64_t cache_batch_stride, const int32_t* positions, int64_t B, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && k_cache && v_cache && positions && B >= 1, "uvx_kv_append: bad arguments");
  UVX_REQUIRE(kv_width % 8 == 0 && row_stride % 8 == 0 && k_col % 8 == 0 && v_col % 8 == 0 && cache_batch_stride % 8 == 0,
              "uvx_kv_append: alignment");
  const int64_t total = B * (kv_width / 8) * 2;
  launch_k(kv_append_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, (const bf16*)qkv, row_stride, (int)k_col, (int)v_col, (int)kv_width, (bf16*)k_cache, (bf16*)v_cache, cache_batch_stride, positions, B);
  return check_launch("kv_append_kernel");
}


extern "C" int uvx_rope_kv_append(void* qkv, int64_t B, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                                  const float* sin_tab, const int32_t* rope_positions, void* k_cache, void* v_cache,
                                  int64_t cache_batch_stride, const int32_t* positions, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && cos_tab && sin_tab && rope_positions && k_cache && v_cache && positions, "uvx_rope_kv_append: null pointer");
  UVX_REQUIRE(D % 16 == 0 && row_stride % 8 == 0 && cache_batch_stride % 8 == 0 && B >= 1, "uvx_rope_kv_append: alignment");
  const int64_t total = B * (Hq + 2 * Hkv) * (D / 16);
  launch_k(rope_kv_append_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, (bf16*)qkv, row_stride, Hq,
           Hkv, D, cos_tab, sin_tab, rope_positions, (bf16*)k_cache, (bf16*)v_cache, cache_batch_stride, positions, B);
  return check_launch("rope_kv_append_kernel");
}

extern "C" int uvx_rope_kv_append_map(void* qkv, int64_t rows, int64_t row_stride, int Hq, int Hkv, int D, const float* cos_tab,
                                      const float* sin_tab, const int32_t* rope_positions, void* k_cache, void* v_cache,
                                      int64_t cache_batch_stride, const int32_t* cache_row, const int32_t* positions,
                                      uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && cos_tab && sin_tab && rope_positions && k_cache && v_cache && cache_row && positions,
              "uvx_rope_kv_append_map: null pointer");
  UVX_REQUIRE(D % 16 == 0 && row_stride % 8 == 0 && cache_batch_stride % 8 == 0 && rows >= 1, "uvx_rope_kv_append_map: alignment");
  const int64_t total = rows * (Hq + 2 * Hkv) * (D / 16);
  launch_k(rope_kv_append_map_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, (bf16*)qkv, row_stride,
           Hq, Hkv, D, cos_tab, sin_tab, rope_positions, (bf16*)k_cache, (bf16*)v_cache, cache_batch_stride, cache_row, positions, rows);
  return check_launch("rope_kv_append_map_kernel");
}

extern "C" int uvx_add_i32(int32_t* a, int32_t* b, int64_t n, int32_t delta, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(a && n >= 1, "uvx_add_i32: bad arguments");
  launch_k(add_i32_kernel, dim3((unsigned)((n + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, a, b, n, delta);
  return check_launch("add_i32_kernel");
}
