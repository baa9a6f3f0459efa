// Shared device/host helpers for libuvx (sm_90a, H100).
#pragma once
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/uvx.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ < 900)
#error "libuvx is written for sm_90a (H100)"
#endif

namespace uvx {

// ---- error reporting -------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int check_launch(const char* what);  // cudaGetLastError -> UVX_ERR_CUDA + message

#define UVX_REQUIRE(cond, ...)                 \
  do {                                         \
    if (!(cond)) {                             \
      ::uvx::set_error(__VA_ARGS__);           \
      return UVX_ERR_ARG;                      \
    }                                          \
  } while (0)

typedef __nv_bfloat16 bf16;

// ---- programmatic dependent launch (PDL) -------------------------------------------------------
// Every kernel on the inference path is launched with the programmatic-stream-serialization attribute and starts with
// pdl_trigger() (let the next kernel's CTAs be scheduled as soon as SM resources free up) followed - after its
// input-independent set-up - by pdl_wait() (all memory of the preceding grids is complete and visible).  Inside a CUDA
// graph this turns the kernel->kernel edges into programmatic edges: launch latency, barrier init, TMEM allocation and
// descriptor prefetch of kernel N+1 overlap the tail of kernel N.  On by default since round 2 (UVX_PDL=0 disables it; the
// griddepcontrol.* instructions are no-ops then): the GEMM additionally requests the weight boxes of its first ring round before
// the wait.  Round 1 (no early loads) had measured 10.86 ms per prefill step with PDL vs 10.47 ms without.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}

// launch with a thread-block cluster of `cluster_x` CTAs along x (grid.x must be a multiple of it)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, unsigned cluster_x,
                                    Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = cluster_x;
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  return cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...);
}
#endif

// ---- small device helpers --------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum for blockDim.x <= 1024 (multiple of 32); `red` is >= 32 floats of shared memory
__device__ __forceinline__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[w] = v;
  __syncthreads();
  float t = (lane < nw) ? red[lane] : 0.f;
  return warp_sum(t);
}

struct __align__(16) bf16x8 {
  __nv_bfloat162 v[4];
};

__device__ __forceinline__ void unpack8(const bf16x8& p, float* f) {
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    float2 t = __bfloat1622float2(p.v[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}
__device__ __forceinline__ bf16x8 pack8(const float* f) {
  bf16x8 p;
#pragma unroll
  for (int i = 0; i < 4; ++i) p.v[i] = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
  return p;
}

// ---- FP8 (e4m3) paged KV pool (include/uvx.h): quantize q = cvt.rn.satfinite.e4m3(x / s) with IEEE fp32 division (NaN stays
// NaN, as 0x7F: the division returns the canonical NaN; +-Inf and |x / s| > 448 become +-448), dequantize
// x = bf16_rn(float(q) * s).  Element i of a packed group sits in byte i.
__device__ __forceinline__ uint32_t e4m3x2_quant(float lo, float hi, float s) {
  uint16_t r;
  asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(__fdiv_rn(hi, s)), "f"(__fdiv_rn(lo, s)));
  return r;
}
__device__ __forceinline__ uint2 e4m3x8_quant(const float* f, float s) {
  return make_uint2(e4m3x2_quant(f[0], f[1], s) | e4m3x2_quant(f[2], f[3], s) << 16,
                    e4m3x2_quant(f[4], f[5], s) | e4m3x2_quant(f[6], f[7], s) << 16);
}
// two e4m3 (bytes 0, 1 of q) -> packed bf16x2; e4m3 -> f16 is exact
__device__ __forceinline__ uint32_t e4m3x2_dequant(uint32_t q, float s) {
  uint32_t h;
  asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(h) : "h"((uint16_t)q));
  const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&h));
  __nv_bfloat162 b = __floats2bfloat162_rn(f.x * s, f.y * s);
  return *reinterpret_cast<uint32_t*>(&b);
}
// 16 e4m3 -> 16 bf16 (lo: elements 0..7, hi: 8..15)
__device__ __forceinline__ void e4m3x16_dequant(const uint4 q, float s, uint4& lo, uint4& hi) {
  lo = make_uint4(e4m3x2_dequant(q.x, s), e4m3x2_dequant(q.x >> 16, s), e4m3x2_dequant(q.y, s), e4m3x2_dequant(q.y >> 16, s));
  hi = make_uint4(e4m3x2_dequant(q.z, s), e4m3x2_dequant(q.z >> 16, s), e4m3x2_dequant(q.w, s), e4m3x2_dequant(q.w >> 16, s));
}

// streaming 128-bit global load that does not allocate in L1 (weights are read once)
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f)); }
// GELU(x) = x * Phi(x) with Phi from the Abramowitz-Stegun 7.1.26 erfc form (|error in erf| <= 1.5e-7, i.e. fp32-level for a
// bf16 result): one rcp + one ex2 + 8 FMA instead of erff's two divergent branches - the fc1 epilogue is issue-bound.
__device__ __forceinline__ float gelu_fast(float x) {
  const float z = fabsf(x) * 0.70710678118654752440f;
  float t, ex;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.0f)));   // 1 ulp-class, argument in [1, inf)
  float pl = fmaf(1.061405429f, t, -1.453152027f);
  pl = fmaf(pl, t, 1.421413741f);
  pl = fmaf(pl, t, -0.284496736f);
  pl = fmaf(pl, t, 0.254829592f);
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(ex) : "f"(-1.4426950408889634f * z * z));
  const float half_erfc = 0.5f * pl * t * ex;  // 0.5 * erfc(|x| / sqrt 2)
  return x * (x >= 0.f ? 1.0f - half_erfc : half_erfc);
}
__device__ __forceinline__ float silu(float x) { return x / (1.0f + expf(-x)); }
// x * sigmoid(x) with one ex2.approx and one rcp.approx (relative error ~2^-21, far below the bf16 rounding that follows): the
// fused gate|up epilogue evaluates 21k of these per CTA on four warps, where expf + a true division cost ~10 us of exposed tail
__device__ __forceinline__ float silu_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(-1.4426950408889634f * x));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return x * r;
}
// RoPE pair rotation with the rounding spelled out (no FMA contraction), shared by uvx_rope and the fused q|k|v epilogue so that
// both produce the same bits: o1 = x1 cos - x2 sin, o2 = x2 cos + x1 sin
__device__ __forceinline__ void rope_pair(float x1, float x2, float c, float s, float& o1, float& o2) {
  o1 = __fsub_rn(__fmul_rn(x1, c), __fmul_rn(x2, s));
  o2 = __fadd_rn(__fmul_rn(x2, c), __fmul_rn(x1, s));
}

}  // namespace uvx
