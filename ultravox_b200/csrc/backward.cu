// Backward-side HBM-bound kernels of the adapter-training path (SURVEY.md 8a-14): everything autograd would run
// between the loss and the projector weights, except the dense contractions (uvx_gemm_bf16) and attention
// (attention_bwd.cu).  Encoder and LLM are frozen (ref apply_lora r=0, ultravox_model.py:690-709), so only data
// gradients flow through the LLM and only the four projector tensors receive weight gradients.
#include "uvx_common.cuh"

namespace uvx {

// ------------------------------------------------------------------------------------- bf16 2-D transpose
__global__ void transpose_kernel(const bf16* __restrict__ in, int64_t rows, int64_t cols, int64_t in_rs,
                                 bf16* __restrict__ out, int64_t out_rs) {
  __shared__ bf16 tile[64][66];
  const int64_t r0 = (int64_t)blockIdx.y * 64, c0 = (int64_t)blockIdx.x * 64;
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int64_t r = r0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x) {
      const int64_t c = c0 + j;
      tile[i][j] = (r < rows && c < cols) ? in[r * in_rs + c] : __float2bfloat16_rn(0.f);
    }
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 64; i += blockDim.y) {
    const int64_t c = c0 + i;
    for (int j = threadIdx.x; j < 64; j += blockDim.x) {
      const int64_t r = r0 + j;
      if (r < rows && c < cols) out[c * out_rs + r] = tile[j][i];
    }
  }
}

// ------------------------------------------------------------------------------------- RMSNorm backward
// y = w * bf16(x * rstd); dx = rstd * (g - xhat * mean(g * xhat)) with g = dy * w, xhat = x * rstd.
// Optional: dres is added to dx (residual-stream gradient), dw[cols] += sum_rows dy * xhat (fp32 atomics, one per
// column per CTA of kRowsPerCta rows).  Stack mode as in rmsnorm_kernel (elements past `valid` are zero); dx is stacked.
static constexpr int kNbThreads = 256;
static constexpr int kNbMaxVec = 5;  // up to 256*5*8 = 10240 columns
static constexpr int kRowsPerCta = 8;

__global__ void __launch_bounds__(kNbThreads) rmsnorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                                 const bf16* __restrict__ w, const bf16* __restrict__ dres,
                                                                 bf16* __restrict__ dx, float* __restrict__ dw, int64_t rows,
                                                                 int64_t cols, int64_t x_row_stride, int64_t group_rows,
                                                                 int64_t group_stride, int64_t valid_elems, float eps) {
  __shared__ float red[32];
  const int nvec = (int)(cols / 8);
  float dwacc[kNbMaxVec][8];
#pragma unroll
  for (int i = 0; i < kNbMaxVec; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) dwacc[i][e] = 0.f;
  for (int rr = 0; rr < kRowsPerCta; ++rr) {
    const int64_t row = (int64_t)blockIdx.x * kRowsPerCta + rr;
    if (row >= rows) break;
    const bf16* xr;
    int64_t valid = cols;
    if (group_rows > 0) {
      const int64_t g = row / group_rows, t = row % group_rows;
      xr = x + g * group_stride + t * cols;
      valid = valid_elems - t * cols;
      valid = valid < 0 ? 0 : (valid > cols ? cols : valid);
    } else {
      xr = x + row * x_row_stride;
    }
    float xv[kNbMaxVec][8], gv[kNbMaxVec][8];
    float sq = 0.f;
#pragma unroll
    for (int i = 0; i < kNbMaxVec; ++i) {
      const int j = threadIdx.x + i * kNbThreads;
      if (j < nvec) {
        if ((int64_t)j * 8 < valid) {
          unpack8(*reinterpret_cast<const bf16x8*>(xr + (int64_t)j * 8), xv[i]);
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e) xv[i][e] = 0.f;
        }
#pragma unroll
        for (int e = 0; e < 8; ++e) sq += xv[i][e] * xv[i][e];
      }
    }
    const float rstd = rsqrtf(block_sum(sq, red) / (float)cols + eps);
    float dot = 0.f;
#pragma unroll
    for (int i = 0; i < kNbMaxVec; ++i) {
      const int j = threadIdx.x + i * kNbThreads;
      if (j < nvec) {
        float dyv[8], wv[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dy + row * cols + (int64_t)j * 8), dyv);
        unpack8(*reinterpret_cast<const bf16x8*>(w + (int64_t)j * 8), wv);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float xhat = xv[i][e] * rstd;
          gv[i][e] = dyv[e] * wv[e];
          dot += gv[i][e] * xhat;
          dwacc[i][e] += dyv[e] * xhat;
          xv[i][e] = xhat;
        }
      }
    }
    const float mean_dot = block_sum(dot, red) / (float)cols;
    if (dx) {
#pragma unroll
      for (int i = 0; i < kNbMaxVec; ++i) {
        const int j = threadIdx.x + i * kNbThreads;
        if (j < nvec) {
          float o[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) o[e] = rstd * (gv[i][e] - xv[i][e] * mean_dot);
          if (dres) {
            float rv[8];
            unpack8(*reinterpret_cast<const bf16x8*>(dres + row * cols + (int64_t)j * 8), rv);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] += rv[e];
          }
          *reinterpret_cast<bf16x8*>(dx + row * cols + (int64_t)j * 8) = pack8(o);
        }
      }
    }
  }
  if (dw) {
#pragma unroll
    for (int i = 0; i < kNbMaxVec; ++i) {
      const int j = threadIdx.x + i * kNbThreads;
      if (j < nvec) {
#pragma unroll
        for (int e = 0; e < 8; ++e) atomicAdd(dw + (int64_t)j * 8 + e, dwacc[i][e]);
      }
    }
  }
}

// ------------------------------------------------------------------------------------- SwiGLU backward
__global__ void swiglu_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dout, bf16* __restrict__ dxo,
                                  int64_t rows, int64_t H, int64_t x_row_stride, int gate_first) {
  const int64_t vec_per_row = H / 8;
  const int64_t total = rows * vec_per_row;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / vec_per_row, j = (idx % vec_per_row) * 8;
    float a[8], g[8], d[8], da[8], dg[8];
    unpack8(*reinterpret_cast<const bf16x8*>(x + r * x_row_stride + j), a);
    unpack8(*reinterpret_cast<const bf16x8*>(x + r * x_row_stride + H + j), g);
    unpack8(*reinterpret_cast<const bf16x8*>(dout + r * H + j), d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float gate = gate_first ? a[e] : g[e];
      const float lin = gate_first ? g[e] : a[e];
      const float sg = 1.f / (1.f + expf(-gate));
      const float dl = d[e] * gate * sg;                                   // d/dlin   = silu(gate)
      const float dgt = d[e] * lin * sg * (1.f + gate * (1.f - sg));       // d/dgate  = lin * silu'(gate)
      if (gate_first) { da[e] = dgt; dg[e] = dl; } else { da[e] = dl; dg[e] = dgt; }
    }
    *reinterpret_cast<bf16x8*>(dxo + r * 2 * H + j) = pack8(da);
    *reinterpret_cast<bf16x8*>(dxo + r * 2 * H + H + j) = pack8(dg);
  }
}


// ------------------------------------------------------------------------------------- LayerNorm backward (data gradient)
// y = (x - mean) * rstd * w + b  ->  dx = rstd * (g - mean(g) - xhat * mean(g * xhat)),  g = dy * w  (+ dres: the gradient that
// bypasses the norm on the residual branch).  One warp per row, values in registers (cols <= 2048: the Whisper encoder's d_model).
// Used by the encoder backward of LoRA training (ref:ultravox_model.py:690-709; hf:modeling_whisper.py:403-440); the norm's own
// weight / bias are frozen there, so no dw / db.
static constexpr int kLnbVec = 8;
__global__ void __launch_bounds__(128) layernorm_bwd_kernel(const bf16* __restrict__ dy, const bf16* __restrict__ x,
                                                            const bf16* __restrict__ w, const bf16* __restrict__ dres,
                                                            bf16* __restrict__ dx, int64_t rows, int64_t cols, float eps) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int nvec = (int)(cols / 8);
  float xv[kLnbVec][8], gv[kLnbVec][8];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < kLnbVec; ++i) {
    const int j = lane + i * 32;
    if (j < nvec) {
      unpack8(*reinterpret_cast<const bf16x8*>(x + row * cols + (int64_t)j * 8), xv[i]);
#pragma unroll
      for (int e = 0; e < 8; ++e) s += xv[i][e];
    }
  }
  const float mean = warp_sum(s) / (float)cols;
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kLnbVec; ++i) {
    const int j = lane + i * 32;
    if (j < nvec) {
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        xv[i][e] -= mean;
        sq += xv[i][e] * xv[i][e];
      }
    }
  }
  const float rstd = rsqrtf(warp_sum(sq) / (float)cols + eps);
  float sg = 0.f, sgx = 0.f;
#pragma unroll
  for (int i = 0; i < kLnbVec; ++i) {
    const int j = lane + i * 32;
    if (j < nvec) {
      float dyv[8], wv[8];
      unpack8(*reinterpret_cast<const bf16x8*>(dy + row * cols + (int64_t)j * 8), dyv);
      unpack8(*reinterpret_cast<const bf16x8*>(w + (int64_t)j * 8), wv);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        xv[i][e] *= rstd;                 // xhat
        gv[i][e] = dyv[e] * wv[e];
        sg += gv[i][e];
        sgx += gv[i][e] * xv[i][e];
      }
    }
  }
  const float mg = warp_sum(sg) / (float)cols, mgx = warp_sum(sgx) / (float)cols;
#pragma unroll
  for (int i = 0; i < kLnbVec; ++i) {
    const int j = lane + i * 32;
    if (j < nvec) {
      float o[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = rstd * (gv[i][e] - mg - xv[i][e] * mgx);
      if (dres) {
        float rv[8];
        unpack8(*reinterpret_cast<const bf16x8*>(dres + row * cols + (int64_t)j * 8), rv);
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] += rv[e];
      }
      *reinterpret_cast<bf16x8*>(dx + row * cols + (int64_t)j * 8) = pack8(o);
    }
  }
}

// ------------------------------------------------------------------------------------- GELU (erf form) forward / backward
// Training keeps the pre-activation of fc1 (the inference path fuses GELU into the GEMM epilogue and never stores it).
__global__ void gelu_kernel(const bf16* __restrict__ x, bf16* __restrict__ y, int64_t nvec) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float v[8];
    unpack8(reinterpret_cast<const bf16x8*>(x)[i], v);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = gelu_erf(v[e]);
    reinterpret_cast<bf16x8*>(y)[i] = pack8(v);
  }
}
// d/dx [x * Phi(x)] = Phi(x) + x * phi(x)
__global__ void gelu_bwd_kernel(const bf16* __restrict__ x, const bf16* __restrict__ dy, bf16* __restrict__ dx, int64_t nvec) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float v[8], d[8];
    unpack8(reinterpret_cast<const bf16x8*>(x)[i], v);
    unpack8(reinterpret_cast<const bf16x8*>(dy)[i], d);
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float cdf = 0.5f * (1.0f + erff(v[e] * 0.70710678118654752440f));
      const float pdf = 0.3989422804014327f * expf(-0.5f * v[e] * v[e]);
      d[e] *= cdf + v[e] * pdf;
    }
    reinterpret_cast<bf16x8*>(dx)[i] = pack8(d);
  }
}

// ------------------------------------------------------------------------------------- CE backward
// dlogits[r, v] = (softmax(logits[r])[v] - [v == label_r]) / count for rows with a valid (shifted) label, else 0.
__global__ void __launch_bounds__(512) ce_bwd_kernel(const float* __restrict__ logits, int64_t row_stride,
                                                    const int64_t* __restrict__ labels, int64_t S, int64_t V,
                                                    int64_t ignore_index, int shift, const float* __restrict__ row_lse,
                                                    const float* __restrict__ loss2, float grad_scale, bf16* __restrict__ dlogits) {
  const int64_t row = blockIdx.x;
  const int64_t b = row / S, s = row % S;
  const int64_t label = shift ? ((s + 1 < S) ? labels[b * S + s + 1] : ignore_index) : labels[row];
  const bool valid = label != ignore_index && label >= 0 && label < V;
  const float inv = valid ? grad_scale / loss2[1] : 0.f;
  const float lse = row_lse[row];
  const float* x = logits + row * row_stride;
  bf16* d = dlogits + row * V;
  for (int64_t i = (int64_t)threadIdx.x * 8; i < V; i += (int64_t)blockDim.x * 8) {
    float o[8];
    if (i + 7 < V) {
      const float4 v0 = *reinterpret_cast<const float4*>(x + i), v1 = *reinterpret_cast<const float4*>(x + i + 4);
      const float xs[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = valid ? (expf(xs[e] - lse) - ((i + e) == label ? 1.f : 0.f)) * inv : 0.f;
      *reinterpret_cast<bf16x8*>(d + i) = pack8(o);
    } else {
      for (int64_t j = i; j < V; ++j)
        d[j] = __float2bfloat16_rn(valid ? (expf(x[j] - lse) - (j == label ? 1.f : 0.f)) * inv : 0.f);
    }
  }
}

// ------------------------------------------------------------------------------------- row gather / splice inverse
__global__ void gather_rows_kernel(const bf16* __restrict__ src, const int32_t* __restrict__ idx, int64_t rows, int64_t d,
                                   bf16* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int32_t s = idx[row];
  uint4* d4 = reinterpret_cast<uint4*>(out + row * d);
  if (s >= 0) {
    const uint4* s4 = reinterpret_cast<const uint4*>(src + (int64_t)s * d);
    for (int64_t i = lane; i < d / 8; i += 32) d4[i] = s4[i];
  } else {
    for (int64_t i = lane; i < d / 8; i += 32) d4[i] = make_uint4(0, 0, 0, 0);
  }
}

__global__ void splice_inverse_kernel(const int32_t* __restrict__ src, int64_t n_pos, int32_t* __restrict__ inv, int64_t n_audio) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_audio; i += (int64_t)gridDim.x * blockDim.x) inv[i] = -1;
  // grid-wide ordering is not needed: a second launch phase would be cleaner, so the init runs in its own launch
}
__global__ void splice_inverse_fill_kernel(const int32_t* __restrict__ src, int64_t n_pos, int32_t* __restrict__ inv) {
  for (int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; p < n_pos; p += (int64_t)gridDim.x * blockDim.x) {
    const int32_t r = src[p];
    if (r >= 0) inv[r] = (int32_t)p;  // each audio row is spliced to at most one position
  }
}

// ------------------------------------------------------------------------------------- AdamW (fp32 state, bf16 params)
__global__ void adamw_kernel(bf16* __restrict__ p, const float* __restrict__ g, float* __restrict__ m, float* __restrict__ v,
                             int64_t n, float lr, float b1, float b2, float eps, float wd, float bc1, float bc2, float gscale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float gi = g[i] * gscale;
    float pi = __bfloat162float(p[i]);
    pi *= 1.f - lr * wd;  // decoupled weight decay (torch.optim.AdamW)
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / sqrtf(bc2) + eps;
    pi -= (lr / bc1) * (mi / denom);
    p[i] = __float2bfloat16_rn(pi);
  }
}

__global__ void cast_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __float2bfloat16_rn(in[i]);
}

static inline unsigned grid_for(int64_t total, int threads) {
  int64_t b = (total + threads - 1) / threads;
  return (unsigned)(b > 148 * 16 ? 148 * 16 : (b < 1 ? 1 : b));
}

}  // namespace uvx

extern "C" int uvx_transpose_bf16(const void* in, int64_t rows, int64_t cols, int64_t in_row_stride, void* out,
                                  int64_t out_row_stride, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(in && out && rows > 0 && cols > 0, "uvx_transpose_bf16: bad arguments");
  dim3 grid((unsigned)((cols + 63) / 64), (unsigned)((rows + 63) / 64)), block(32, 8);
  UVX_REQUIRE(grid.y < 65536, "uvx_transpose_bf16: too many rows");
  transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>((const bf16*)in, rows, cols, in_row_stride, (bf16*)out, out_row_stride);
  return check_launch("transpose_kernel");
}

extern "C" int uvx_rmsnorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, float* dw,
                               int64_t rows, int64_t cols, int64_t x_row_stride, int64_t group_rows, int64_t group_stride,
                               int64_t valid_elems, float eps, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(dy && x && w && (dx || dw), "uvx_rmsnorm_bwd: null pointer");
  UVX_REQUIRE(cols % 8 == 0 && cols <= kNbThreads * kNbMaxVec * 8 && x_row_stride % 8 == 0, "uvx_rmsnorm_bwd: cols %% 8, <= %d",
              kNbThreads * kNbMaxVec * 8);
  if (rows == 0) return UVX_OK;
  rmsnorm_bwd_kernel<<<(unsigned)((rows + kRowsPerCta - 1) / kRowsPerCta), kNbThreads, 0, (cudaStream_t)stream>>>(
      (const bf16*)dy, (const bf16*)x, (const bf16*)w, (const bf16*)dres, (bf16*)dx, dw, rows, cols, x_row_stride, group_rows,
      group_stride, valid_elems, eps);
  return check_launch("rmsnorm_bwd_kernel");
}

extern "C" int uvx_swiglu_bwd(const void* x, const void* dout, void* dx, int64_t rows, int64_t H, int64_t x_row_stride,
                              int gate_first, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && dout && dx && H % 8 == 0 && x_row_stride % 8 == 0, "uvx_swiglu_bwd: bad arguments");
  if (rows == 0) return UVX_OK;
  swiglu_bwd_kernel<<<grid_for(rows * (H / 8), 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)dout, (bf16*)dx,
                                                                                     rows, H, x_row_stride, gate_first);
  return check_launch("swiglu_bwd_kernel");
}


extern "C" int uvx_layernorm_bwd(const void* dy, const void* x, const void* w, const void* dres, void* dx, int64_t rows, int64_t cols,
                                 float eps, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(dy && x && w && dx, "uvx_layernorm_bwd: null pointer");
  UVX_REQUIRE(cols % 8 == 0 && cols <= 32 * kLnbVec * 8, "uvx_layernorm_bwd: cols must be a multiple of 8 and <= %d", 32 * kLnbVec * 8);
  if (rows == 0) return UVX_OK;
  layernorm_bwd_kernel<<<(unsigned)((rows + 3) / 4), 128, 0, (cudaStream_t)stream>>>((const bf16*)dy, (const bf16*)x, (const bf16*)w,
                                                                                     (const bf16*)dres, (bf16*)dx, rows, cols, eps);
  return check_launch("layernorm_bwd_kernel");
}

extern "C" int uvx_gelu(const void* x, void* y, int64_t n, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && y && n % 8 == 0, "uvx_gelu: n %% 8 == 0 required");
  if (n == 0) return UVX_OK;
  gelu_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (bf16*)y, n / 8);
  return check_launch("gelu_kernel");
}

extern "C" int uvx_gelu_bwd(const void* x, const void* dy, void* dx, int64_t n, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(x && dy && dx && n % 8 == 0, "uvx_gelu_bwd: n %% 8 == 0 required");
  if (n == 0) return UVX_OK;
  gelu_bwd_kernel<<<grid_for(n / 8, 256), 256, 0, (cudaStream_t)stream>>>((const bf16*)x, (const bf16*)dy, (bf16*)dx, n / 8);
  return check_launch("gelu_bwd_kernel");
}

extern "C" int uvx_ce_bwd(const float* logits, int64_t row_stride, const int64_t* labels, int64_t B, int64_t S, int64_t V,
                          int64_t ignore_index, int shift, const float* row_lse, const float* loss2, float grad_scale,
                          void* dlogits, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && labels && row_lse && loss2 && dlogits, "uvx_ce_bwd: null pointer");
  UVX_REQUIRE(V % 8 == 0 && row_stride % 4 == 0, "uvx_ce_bwd: V %% 8 == 0 required");
  ce_bwd_kernel<<<(unsigned)(B * S), 512, 0, (cudaStream_t)stream>>>(logits, row_stride, labels, S, V, ignore_index, shift, row_lse,
                                                                     loss2, grad_scale, (bf16*)dlogits);
  return check_launch("ce_bwd_kernel");
}

extern "C" int uvx_gather_rows(const void* src, const int32_t* idx, int64_t rows, int64_t d, void* out, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(src && idx && out && d % 8 == 0, "uvx_gather_rows: bad arguments");
  if (rows == 0) return UVX_OK;
  gather_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>((const bf16*)src, idx, rows, d, (bf16*)out);
  return check_launch("gather_rows_kernel");
}

extern "C" int uvx_splice_inverse(const int32_t* src, int64_t n_pos, int32_t* inv, int64_t n_audio_rows, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(src && inv && n_pos > 0 && n_audio_rows > 0, "uvx_splice_inverse: bad arguments");
  splice_inverse_kernel<<<grid_for(n_audio_rows, 256), 256, 0, (cudaStream_t)stream>>>(src, n_pos, inv, n_audio_rows);
  int rc = check_launch("splice_inverse_kernel");
  if (rc) return rc;
  splice_inverse_fill_kernel<<<grid_for(n_pos, 256), 256, 0, (cudaStream_t)stream>>>(src, n_pos, inv);
  return check_launch("splice_inverse_fill_kernel");
}

extern "C" int uvx_adamw(void* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2, float eps,
                         float weight_decay, int64_t step, float grad_scale, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(p && g && m && v && n > 0 && step >= 1, "uvx_adamw: bad arguments");
  const float bc1 = 1.f - powf(beta1, (float)step), bc2 = 1.f - powf(beta2, (float)step);
  adamw_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>((bf16*)p, g, m, v, n, lr, beta1, beta2, eps, weight_decay, bc1,
                                                                   bc2, grad_scale);
  return check_launch("adamw_kernel");
}

extern "C" int uvx_cast_f32_bf16(const float* in, void* out, int64_t n, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(in && out && n > 0, "uvx_cast_f32_bf16: bad arguments");
  cast_f32_bf16_kernel<<<grid_for(n, 256), 256, 0, (cudaStream_t)stream>>>(in, (bf16*)out, n);
  return check_launch("cast_f32_bf16_kernel");
}
