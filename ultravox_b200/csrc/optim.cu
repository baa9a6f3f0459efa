// Optimizer step of adapter training (a14): global-norm gradient clipping, multi-tensor AdamW with every per-step scalar
// (step, lr, clip coefficient, gradient scale) read from device memory, and micro-batch gradient accumulation.  One launch
// per entry covers every trained tensor (uvx_tensor_list, passed by value), so the norm + clip + AdamW sequence is two
// launches with no host value that changes between steps (graph-capturable).
#include "uvx_common.cuh"

namespace uvx {

static constexpr int kNormThreads = 256;
static constexpr int kOptThreads = 256;
static constexpr unsigned kOptBlocks = 148 * 8;

__device__ __forceinline__ bool aligned16(const void* p) { return ((uintptr_t)p & 15) == 0; }
__device__ __forceinline__ bool aligned8(const void* p) { return ((uintptr_t)p & 7) == 0; }

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
// fixed-order block sum (kNormThreads threads); the result is valid in thread 0
__device__ __forceinline__ double block_sum_f64(double v, double* red) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  v = warp_sum_f64(v);
  if (lane == 0) red[w] = v;
  __syncthreads();
  double t = 0.0;
  if (w == 0) {
    t = lane < kNormThreads / 32 ? red[lane] : 0.0;
    t = warp_sum_f64(t);
  }
  __syncthreads();
  return t;
}

__device__ __forceinline__ double sq_scaled(float g, float s) {
  const double x = (double)__fmul_rn(g, s);
  return x * x;
}

// ---------------------------------------------------------------------------------------------- || scale * g ||_2 + clip
__global__ void __launch_bounds__(kNormThreads) grad_norm_clip_kernel(uvx_tensor_list tl, const float* scale_p, float max_norm,
                                                                      double* partials, unsigned* ticket, float* norm_coef,
                                                                      int64_t* step, const float* lr_table, int64_t table_len,
                                                                      float* lr) {
  __shared__ double red[kNormThreads / 32];
  __shared__ bool last;
  const float s = scale_p[0];
  const int64_t tid = (int64_t)blockIdx.x * kNormThreads + threadIdx.x, nthr = (int64_t)gridDim.x * kNormThreads;
  double acc = 0.0;
  for (int t = 0; t < tl.count; ++t) {
    const float* g = tl.g[t];
    const int64_t n = tl.numel[t];
    const int64_t n4 = aligned16(g) ? n / 4 : 0;
    const float4* g4 = reinterpret_cast<const float4*>(g);
    for (int64_t i = tid; i < n4; i += nthr) {
      const float4 x = __ldg(g4 + i);
      acc += sq_scaled(x.x, s) + sq_scaled(x.y, s) + sq_scaled(x.z, s) + sq_scaled(x.w, s);
    }
    for (int64_t i = 4 * n4 + tid; i < n; i += nthr) acc += sq_scaled(__ldg(g + i), s);
  }
  acc = block_sum_f64(acc, red);
  if (threadIdx.x == 0) {
    partials[blockIdx.x] = acc;
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  double tot = 0.0;
  for (unsigned b = threadIdx.x; b < gridDim.x; b += kNormThreads) tot += __ldcg(partials + b);
  tot = block_sum_f64(tot, red);
  if (threadIdx.x == 0) {
    const float norm = (float)sqrt(tot);
    float coef = 1.f;
    if (max_norm > 0.f) {
      // torch evaluates max_norm / (norm + 1e-6) as (norm + 1e-6).reciprocal() * max_norm
      const float c = __fmul_rn(__frcp_rn(__fadd_rn(norm, 1e-6f)), max_norm);
      coef = c > 1.f ? 1.f : c;  // torch.clamp(max=1): a NaN coefficient stays NaN
    }
    norm_coef[0] = norm;
    norm_coef[1] = coef;
    if (step) {
      const int64_t st = step[0] + 1;
      step[0] = st;
      const int64_t k = st < table_len ? st : table_len;
      lr[0] = lr_table[(k < 1 ? 1 : k) - 1];
    }
    *ticket = 0u;
  }
}

// ---------------------------------------------------------------------------------------------- multi-tensor AdamW
struct AdamScalars {
  float s, coef, decay, w1, b2, w2, bc2_sqrt, eps, neg_step_size;
};

__device__ __forceinline__ void adam_elem(float g, float& p, float& m, float& v, const AdamScalars& k) {
  const float gi = __fmul_rn(__fmul_rn(g, k.s), k.coef);
  p = __fmul_rn(p, k.decay);
  m = __fadd_rn(m, __fmul_rn(k.w1, __fsub_rn(gi, m)));  // torch lerp, weight 1 - beta1 < 0.5
  v = __fadd_rn(__fmul_rn(v, k.b2), __fmul_rn(__fmul_rn(k.w2, gi), gi));
  const float denom = __fadd_rn(__fdiv_rn(sqrtf(v), k.bc2_sqrt), k.eps);
  p = __fadd_rn(p, __fmul_rn(k.neg_step_size, __fdiv_rn(m, denom)));
}

__global__ void __launch_bounds__(kOptThreads) adamw_multi_kernel(uvx_tensor_list tl, const float* lr_p, const int64_t* step_p,
                                                                  const float* coef_p, const float* scale_p, double beta1,
                                                                  double beta2, double eps, double wd) {
  // per-step scalars exactly as torch's _multi_tensor_adam forms them (python doubles, cast to fp32 by the foreach ops)
  const double lr = (double)lr_p[0], st = (double)step_p[0];
  const double bc1 = 1.0 - pow(beta1, st), bc2 = 1.0 - pow(beta2, st);
  AdamScalars k;
  k.s = scale_p[0];
  k.coef = coef_p ? coef_p[0] : 1.f;
  k.decay = (float)(1.0 - lr * wd);
  k.w1 = (float)(1.0 - beta1);
  k.b2 = (float)beta2;
  k.w2 = (float)(1.0 - beta2);
  k.bc2_sqrt = (float)sqrt(bc2);
  k.eps = (float)eps;
  k.neg_step_size = (float)(-(lr / bc1));
  const int64_t tid = (int64_t)blockIdx.x * kOptThreads + threadIdx.x, nthr = (int64_t)gridDim.x * kOptThreads;
  for (int t = 0; t < tl.count; ++t) {
    const float* g = tl.g[t];
    bf16* p = (bf16*)tl.p[t];
    float *m = tl.m[t], *v = tl.v[t];
    const int64_t n = tl.numel[t];
    const int64_t n4 = (aligned16(g) && aligned16(m) && aligned16(v) && aligned8(p)) ? n / 4 : 0;
    for (int64_t i = tid; i < n4; i += nthr) {
      const float4 g4 = reinterpret_cast<const float4*>(g)[i];
      float4 m4 = reinterpret_cast<float4*>(m)[i], v4 = reinterpret_cast<float4*>(v)[i];
      const uint2 pr = reinterpret_cast<const uint2*>(p)[i];
      const float2 p01 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pr.x));
      const float2 p23 = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&pr.y));
      float q[4] = {p01.x, p01.y, p23.x, p23.y};
      adam_elem(g4.x, q[0], m4.x, v4.x, k);
      adam_elem(g4.y, q[1], m4.y, v4.y, k);
      adam_elem(g4.z, q[2], m4.z, v4.z, k);
      adam_elem(g4.w, q[3], m4.w, v4.w, k);
      reinterpret_cast<float4*>(m)[i] = m4;
      reinterpret_cast<float4*>(v)[i] = v4;
      uint2 pw;
      *reinterpret_cast<__nv_bfloat162*>(&pw.x) = __floats2bfloat162_rn(q[0], q[1]);
      *reinterpret_cast<__nv_bfloat162*>(&pw.y) = __floats2bfloat162_rn(q[2], q[3]);
      reinterpret_cast<uint2*>(p)[i] = pw;
    }
    for (int64_t i = 4 * n4 + tid; i < n; i += nthr) {
      float q = __bfloat162float(p[i]), mi = m[i], vi = v[i];
      adam_elem(g[i], q, mi, vi, k);
      m[i] = mi;
      v[i] = vi;
      p[i] = __float2bfloat16_rn(q);
    }
  }
}

// ---------------------------------------------------------------------------------------------- acc (+)= g
__global__ void __launch_bounds__(kOptThreads) grad_accumulate_kernel(uvx_tensor_list tl, int assign) {
  const int64_t tid = (int64_t)blockIdx.x * kOptThreads + threadIdx.x, nthr = (int64_t)gridDim.x * kOptThreads;
  for (int t = 0; t < tl.count; ++t) {
    const float* g = tl.g[t];
    float* a = tl.acc[t];
    const int64_t n = tl.numel[t];
    const int64_t n4 = (aligned16(g) && aligned16(a)) ? n / 4 : 0;
    for (int64_t i = tid; i < n4; i += nthr) {
      const float4 x = reinterpret_cast<const float4*>(g)[i];
      float4 y = x;
      if (!assign) {
        y = reinterpret_cast<float4*>(a)[i];
        y.x = __fadd_rn(y.x, x.x), y.y = __fadd_rn(y.y, x.y), y.z = __fadd_rn(y.z, x.z), y.w = __fadd_rn(y.w, x.w);
      }
      reinterpret_cast<float4*>(a)[i] = y;
    }
    for (int64_t i = 4 * n4 + tid; i < n; i += nthr) a[i] = assign ? g[i] : __fadd_rn(a[i], g[i]);
  }
}

static int check_list(const uvx_tensor_list* tl, bool g, bool acc, bool pmv, const char* what) {
  UVX_REQUIRE(tl && tl->count >= 1 && tl->count <= UVX_TL_MAX, "%s: tensor list count must be 1..%d", what, UVX_TL_MAX);
  for (int64_t i = 0; i < tl->count; ++i) {
    UVX_REQUIRE(tl->numel[i] > 0, "%s: tensor %lld is empty", what, (long long)i);
    UVX_REQUIRE(!g || tl->g[i], "%s: g[%lld] is NULL", what, (long long)i);
    UVX_REQUIRE(!acc || (tl->acc[i] && tl->acc[i] != tl->g[i]), "%s: acc[%lld] is NULL or aliases g", what, (long long)i);
    UVX_REQUIRE(!pmv || (tl->p[i] && tl->m[i] && tl->v[i]), "%s: p / m / v[%lld] is NULL", what, (long long)i);
  }
  return UVX_OK;
}

}  // namespace uvx

extern "C" int uvx_grad_norm_clip(const uvx_tensor_list* tl, const float* scale, float max_norm, void* workspace, float* norm_coef,
                                  int64_t* step, const float* lr_table, int64_t table_len, float* lr, uvx_stream_t stream) {
  using namespace uvx;
  if (int rc = check_list(tl, true, false, false, "uvx_grad_norm_clip")) return rc;
  UVX_REQUIRE(scale && workspace && norm_coef, "uvx_grad_norm_clip: scale, workspace and norm_coef are required");
  UVX_REQUIRE(!step || (lr_table && table_len >= 1 && lr), "uvx_grad_norm_clip: step needs lr_table (table_len >= 1) and lr");
  double* partials = (double*)workspace;
  unsigned* ticket = (unsigned*)(partials + UVX_NORM_BLOCKS);
  grad_norm_clip_kernel<<<UVX_NORM_BLOCKS, kNormThreads, 0, (cudaStream_t)stream>>>(*tl, scale, max_norm, partials, ticket, norm_coef,
                                                                                    step, lr_table, table_len, lr);
  return check_launch("grad_norm_clip_kernel");
}

extern "C" int uvx_adamw_multi(const uvx_tensor_list* tl, const float* lr, const int64_t* step, const float* coef, const float* scale,
                               double beta1, double beta2, double eps, double weight_decay, uvx_stream_t stream) {
  using namespace uvx;
  if (int rc = check_list(tl, true, false, true, "uvx_adamw_multi")) return rc;
  UVX_REQUIRE(lr && step && scale, "uvx_adamw_multi: lr, step and scale are required");
  adamw_multi_kernel<<<kOptBlocks, kOptThreads, 0, (cudaStream_t)stream>>>(*tl, lr, step, coef, scale, beta1, beta2, eps, weight_decay);
  return check_launch("adamw_multi_kernel");
}

extern "C" int uvx_grad_accumulate(const uvx_tensor_list* tl, int32_t assign, uvx_stream_t stream) {
  using namespace uvx;
  if (int rc = check_list(tl, true, true, false, "uvx_grad_accumulate")) return rc;
  grad_accumulate_kernel<<<kOptBlocks, kOptThreads, 0, (cudaStream_t)stream>>>(*tl, assign);
  return check_launch("grad_accumulate_kernel");
}
