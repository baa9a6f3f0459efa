// Last-position LM head as an HBM-streaming GEMV (V x d bf16 weights read exactly once, 128-bit no-allocate
// loads, fp32 accumulate, warp-shuffle reduction) + greedy argmax.
#include "uvx_common.cuh"

namespace uvx {

static constexpr int kLmWarps = 8;
static constexpr int kLmMaxB = 8;

// each warp owns vocabulary rows v = warp_global, warp_global + total_warps, ...; h (B x d) sits in shared memory
template <int B>
__global__ void __launch_bounds__(kLmWarps * 32) lm_head_kernel(const bf16* __restrict__ h, int64_t h_row_stride,
                                                                const bf16* __restrict__ W, int64_t V, int64_t d,
                                                                float* __restrict__ logits) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ uint8_t lm_smem[];
  bf16* hs = reinterpret_cast<bf16*>(lm_smem);  // [B][d]
  for (int64_t i = threadIdx.x; i < (int64_t)B * d / 8; i += blockDim.x) {
    const int64_t b = i / (d / 8), j = i % (d / 8);
    reinterpret_cast<uint4*>(hs)[i] = *reinterpret_cast<const uint4*>(h + b * h_row_stride + j * 8);
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t)blockIdx.x * kLmWarps + (threadIdx.x >> 5);
  const int64_t total_warps = (int64_t)gridDim.x * kLmWarps;
  const int nvec = (int)(d / 8);
  for (int64_t v = warp_global; v < V; v += total_warps) {
    const bf16* wr = W + v * d;
    float acc[B];
#pragma unroll
    for (int b = 0; b < B; ++b) acc[b] = 0.f;
#pragma unroll 4
    for (int j = lane; j < nvec; j += 32) {
      const uint4 raw = ld_nc_v4(wr + (int64_t)j * 8);
      float wv[8];
      unpack8(*reinterpret_cast<const bf16x8*>(&raw), wv);
#pragma unroll
      for (int b = 0; b < B; ++b) {
        float hv[8];
        unpack8(*reinterpret_cast<const bf16x8*>(hs + (int64_t)b * d + (int64_t)j * 8), hv);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[b] = fmaf(wv[e], hv[e], acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < B; ++b) {
      const float s = warp_sum(acc[b]);
      if (lane == 0) logits[(int64_t)b * V + v] = s;
    }
  }
}

__global__ void __launch_bounds__(1024) argmax_kernel(const float* __restrict__ logits, int64_t V, int64_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sv[32];
  __shared__ int64_t si[32];
  const float* row = logits + (int64_t)blockIdx.x * V;
  float best = -INFINITY;
  int64_t bi = INT64_MAX;
  const int64_t v4 = ((uintptr_t)row % 16 == 0) ? V / 4 : 0;  // 128-bit loads over the aligned body
  for (int64_t i = threadIdx.x; i < v4; i += blockDim.x) {
    const float4 t = reinterpret_cast<const float4*>(row)[i];
    const float xs[4] = {t.x, t.y, t.z, t.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      // within a thread indices grow monotonically: strict > keeps the first maximum.  A thread's first element is always taken,
      // so a -inf element still carries its index and a row that is all -inf resolves to 0 below, as torch.argmax does.
      if (xs[e] > best || bi == INT64_MAX) {
        best = xs[e];
        bi = i * 4 + e;
      }
    }
  }
  for (int64_t i = v4 * 4 + threadIdx.x; i < V; i += blockDim.x) {
    const float x = row[i];
    if (x > best || (x == best && i < bi)) {
      best = x;
      bi = i;
    }
  }
  // Finite or -inf logits only: NaN handling is out of contract (torch would return the NaN position).
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
    if (ob > best || (ob == best && oi < bi)) {
      best = ob;
      bi = oi;
    }
  }
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) {
    sv[w] = best;
    si[w] = bi;
  }
  __syncthreads();
  if (w == 0) {
    best = sv[lane];
    bi = si[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int64_t oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ob > best || (ob == best && oi < bi)) {
        best = ob;
        bi = oi;
      }
    }
    if (lane == 0) out[blockIdx.x] = bi;
  }
}

// Small-batch linear layer (decode, M <= 8): y[b, n] = sum_k x[b, k] W[n, k] (+ R[b, n]); same streaming structure as the
// LM head - no tensor cores, every weight byte read once at HBM rate.
template <int B>
__global__ void __launch_bounds__(kLmWarps * 32) gemv_kernel(const bf16* __restrict__ x, int64_t x_row_stride,
                                                             const bf16* __restrict__ W, int64_t w_row_stride, int64_t N,
                                                             int64_t K, const bf16* __restrict__ R, int64_t r_row_stride,
                                                             void* __restrict__ out, int64_t o_row_stride, int out_f32,
                                                             const bf16* __restrict__ norm_w, float norm_eps, int swiglu) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ uint8_t lm_smem[];
  __shared__ float red[32];
  bf16* xs = reinterpret_cast<bf16*>(lm_smem);  // [B][K]
  // Fused prologues of the decode step (every CTA stages the B activation rows anyway): act_fn(gate) * up of the row [gate | up]
  // (LlamaMLP, same rounding as uvx_swiglu), or LlamaRMSNorm of the row (same rounding AND the same fp32 summation order as
  // uvx_rmsnorm: 256 threads, element j = thread + 256 i, block_sum) - two launches per layer less, bit-identical results.
  for (int64_t i = threadIdx.x; i < (int64_t)B * K / 8; i += blockDim.x) {
    const int64_t b = i / (K / 8), j = i % (K / 8);
    if (swiglu) {
      float g[8], u[8], o[8];
      unpack8(*reinterpret_cast<const bf16x8*>(x + b * x_row_stride + j * 8), g);
      unpack8(*reinterpret_cast<const bf16x8*>(x + b * x_row_stride + K + j * 8), u);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = __bfloat162float(__float2bfloat16_rn(silu(g[e]))) * u[e];
      reinterpret_cast<bf16x8*>(xs)[i] = pack8(o);
    } else {
      reinterpret_cast<uint4*>(xs)[i] = *reinterpret_cast<const uint4*>(x + b * x_row_stride + j * 8);
    }
  }
  __syncthreads();
  if (norm_w) {
    const int nv = (int)(K / 8);
    for (int b = 0; b < B; ++b) {
      bf16* xr = xs + (int64_t)b * K;
      float sq = 0.f;
      for (int j = threadIdx.x; j < nv; j += blockDim.x) {
        float v[8];
        unpack8(reinterpret_cast<const bf16x8*>(xr)[j], v);
#pragma unroll
        for (int e = 0; e < 8; ++e) sq += v[e] * v[e];
      }
      const float rstd = rsqrtf(block_sum(sq, red) / (float)K + norm_eps);
      for (int j = threadIdx.x; j < nv; j += blockDim.x) {
        float v[8], wv[8], o[8];
        unpack8(reinterpret_cast<const bf16x8*>(xr)[j], v);
        unpack8(*reinterpret_cast<const bf16x8*>(norm_w + (int64_t)j * 8), wv);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = wv[e] * __bfloat162float(__float2bfloat16_rn(v[e] * rstd));
        reinterpret_cast<bf16x8*>(xr)[j] = pack8(o);
      }
    }
    __syncthreads();
  }
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t)blockIdx.x * kLmWarps + (threadIdx.x >> 5);
  const int64_t total_warps = (int64_t)gridDim.x * kLmWarps;
  const int nvec = (int)(K / 8);
  for (int64_t n = warp_global; n < N; n += total_warps) {
    const bf16* wr = W + n * w_row_stride;
    float acc[B];
#pragma unroll
    for (int b = 0; b < B; ++b) acc[b] = 0.f;
#pragma unroll 4
    for (int j = lane; j < nvec; j += 32) {
      const uint4 raw = ld_nc_v4(wr + (int64_t)j * 8);
      float wv[8];
      unpack8(*reinterpret_cast<const bf16x8*>(&raw), wv);
#pragma unroll
      for (int b = 0; b < B; ++b) {
        float hv[8];
        unpack8(*reinterpret_cast<const bf16x8*>(xs + (int64_t)b * K + (int64_t)j * 8), hv);
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[b] = fmaf(wv[e], hv[e], acc[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < B; ++b) {
      float sres = warp_sum(acc[b]);
      if (lane == 0) {
        if (R) sres += __bfloat162float(R[(int64_t)b * r_row_stride + n]);
        if (out_f32) reinterpret_cast<float*>(out)[(int64_t)b * o_row_stride + n] = sres;
        else reinterpret_cast<bf16*>(out)[(int64_t)b * o_row_stride + n] = __float2bfloat16_rn(sres);
      }
    }
  }
}

template <int B>
static int launch_gemv(const bf16* x, int64_t xs, const bf16* W, int64_t ws, int64_t N, int64_t K, const bf16* R, int64_t rs,
                       void* out, int64_t os, int out_f32, cudaStream_t st, const bf16* norm_w = nullptr, float norm_eps = 0.f,
                       int swiglu = 0) {
  const size_t smem = (size_t)B * K * 2;
  static bool attr = false;
  if (!attr && smem > 48 * 1024) {
    cudaFuncSetAttribute(gemv_kernel<B>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr = true;
  }
  int64_t blocks = (N + kLmWarps - 1) / kLmWarps;
  if (blocks > 148 * 8) blocks = 148 * 8;
  launch_k(gemv_kernel<B>, dim3((unsigned)blocks), dim3(kLmWarps * 32), smem, st, x, xs, W, ws, N, K, R, rs, out, os, out_f32, norm_w, norm_eps, swiglu);
  return check_launch("gemv_kernel");
}

template <int B>
static int launch_lm(const bf16* h, int64_t hs, const bf16* W, int64_t V, int64_t d, float* logits, cudaStream_t st) {
  const size_t smem = (size_t)B * d * 2;
  static bool attr = false;
  if (!attr && smem > 48 * 1024) {
    cudaFuncSetAttribute(lm_head_kernel<B>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    attr = true;
  }
  int64_t blocks = (V + kLmWarps - 1) / kLmWarps;
  if (blocks > 148 * 8) blocks = 148 * 8;
  launch_k(lm_head_kernel<B>, dim3((unsigned)blocks), dim3(kLmWarps * 32), smem, st, h, hs, W, V, d, logits);
  return check_launch("lm_head_kernel");
}

}  // namespace uvx

extern "C" int uvx_lm_head(const void* h, int64_t B, int64_t h_row_stride, const void* W, int64_t V, int64_t d,
                           float* logits, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(h && W && logits, "uvx_lm_head: null pointer");
  UVX_REQUIRE(d % 8 == 0 && h_row_stride % 8 == 0 && B >= 1, "uvx_lm_head: d %% 8 == 0 required");
  UVX_REQUIRE((size_t)kLmMaxB * d * 2 <= 200 * 1024, "uvx_lm_head: hidden size too large");
  cudaStream_t st = (cudaStream_t)stream;
  const bf16* hp = (const bf16*)h;
  float* lp = logits;
  // batches larger than kLmMaxB are processed in slabs (weights re-read once per slab)
  while (B > 0) {
    const int64_t nb = B > kLmMaxB ? kLmMaxB : B;
    int rc;
    switch (nb) {
      case 1: rc = launch_lm<1>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 2: rc = launch_lm<2>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 3: rc = launch_lm<3>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 4: rc = launch_lm<4>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 5: rc = launch_lm<5>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 6: rc = launch_lm<6>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      case 7: rc = launch_lm<7>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
      default: rc = launch_lm<8>(hp, h_row_stride, (const bf16*)W, V, d, lp, st); break;
    }
    if (rc) return rc;
    hp += nb * h_row_stride;
    lp += nb * V;
    B -= nb;
  }
  return UVX_OK;
}

extern "C" int uvx_gemv_bf16(const void* x, int64_t B, int64_t x_row_stride, const void* W, int64_t w_row_stride, int64_t N,
                             int64_t K, const void* R, int64_t r_row_stride, void* out, int64_t o_row_stride, int out_f32,
                             uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && W && out, "uvx_gemv_bf16: null pointer");
  UVX_REQUIRE(B >= 1 && B <= kLmMaxB && K % 8 == 0 && x_row_stride % 8 == 0 && w_row_stride % 8 == 0,
              "uvx_gemv_bf16: 1 <= B <= %d and K %% 8 == 0 required", kLmMaxB);
  UVX_REQUIRE((size_t)B * K * 2 <= 200 * 1024, "uvx_gemv_bf16: B * K too large for shared memory (split the batch)");
  cudaStream_t st = (cudaStream_t)stream;
  const bf16 *xp = (const bf16*)x, *wp = (const bf16*)W, *rp = (const bf16*)R;
  switch (B) {
    case 1: return launch_gemv<1>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 2: return launch_gemv<2>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 3: return launch_gemv<3>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 4: return launch_gemv<4>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 5: return launch_gemv<5>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 6: return launch_gemv<6>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    case 7: return launch_gemv<7>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
    default: return launch_gemv<8>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st);
  }
}

extern "C" int uvx_gemv_fused_bf16(const void* x, int64_t B, int64_t x_row_stride, const void* W, int64_t w_row_stride, int64_t N,
                                   int64_t K, const void* R, int64_t r_row_stride, void* out, int64_t o_row_stride, int out_f32,
                                   const void* norm_w, float norm_eps, int swiglu, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && W && out, "uvx_gemv_fused_bf16: null pointer");
  UVX_REQUIRE(B >= 1 && B <= kLmMaxB && K % 8 == 0 && x_row_stride % 8 == 0 && w_row_stride % 8 == 0,
              "uvx_gemv_fused_bf16: 1 <= B <= %d and K %% 8 == 0 required", kLmMaxB);
  UVX_REQUIRE((size_t)B * K * 2 <= 200 * 1024, "uvx_gemv_fused_bf16: B * K too large for shared memory (split the batch)");
  cudaStream_t st = (cudaStream_t)stream;
  UVX_REQUIRE(!(norm_w && swiglu), "uvx_gemv_fused_bf16: one prologue at a time");
  const bf16 *xp = (const bf16*)x, *wp = (const bf16*)W, *rp = (const bf16*)R, *nw = (const bf16*)norm_w;
  switch (B) {
    case 1: return launch_gemv<1>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 2: return launch_gemv<2>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 3: return launch_gemv<3>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 4: return launch_gemv<4>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 5: return launch_gemv<5>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 6: return launch_gemv<6>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    case 7: return launch_gemv<7>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
    default: return launch_gemv<8>(xp, x_row_stride, wp, w_row_stride, N, K, rp, r_row_stride, out, o_row_stride, out_f32, st, nw, norm_eps, swiglu);
  }
}

extern "C" int uvx_argmax(const float* logits, int64_t B, int64_t V, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && out_idx && B >= 1 && V >= 1, "uvx_argmax: bad arguments");
  launch_k(argmax_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, out_idx);
  return check_launch("argmax_kernel");
}
