// Decode-loop helpers (a13): everything `GenerationMixin.generate` does between two LLM steps, as kernels that read their
// step state from device memory so the whole step can sit in one CUDA graph (no host sync per token):
//   uvx_kv_write            prefill: k / v sections of the fused projection -> the static KV cache (replaces two strided copies)
//   uvx_repetition_penalty  hf:generation/logits_process.py RepetitionPenaltyLogitsProcessor (ref ultravox_pipeline.py:95-113)
//   uvx_sample              temperature / top-k multinomial sampling (ref:ultravox/inference/infer.py:319-328: do_sample when
//                           temperature > 0; hf:generation/utils.py _sample: softmax(logits / T) -> multinomial)
//   uvx_sample_top_p        the same with nucleus (top-p) filtering after top-k (hf:generation/logits_process.py TopPLogitsWarper)
//   uvx_token_finish        EOS / pad bookkeeping of the finished rows, append to `sequences`, advance positions
#include "uvx_common.cuh"

namespace uvx {

__global__ void kv_write_kernel(const bf16* __restrict__ qkv, int64_t row_stride, int k_col, int v_col, int kv_width,
                                bf16* __restrict__ k_cache, bf16* __restrict__ v_cache, int64_t cache_batch_stride, int64_t B,
                                int64_t S, int64_t past) {
  pdl_trigger();
  pdl_wait();
  const int vec = kv_width / 8;
  const int64_t per = B * S * vec;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < 2 * per; idx += (int64_t)gridDim.x * blockDim.x) {
    const int which = (int)(idx / per);
    const int64_t rem = idx % per;
    const int64_t row = rem / vec;  // b * S + s
    const int j = (int)(rem % vec);
    const int64_t b = row / S, s = row % S;
    const bf16* src = qkv + row * row_stride + (which ? v_col : k_col) + j * 8;
    bf16* dst = (which ? v_cache : k_cache) + b * cache_batch_stride + (past + s) * kv_width + j * 8;
    *reinterpret_cast<uint4*>(dst) = *reinterpret_cast<const uint4*>(src);
  }
}

// One CTA per row.  HF gathers the ORIGINAL scores of every token already in the sequence, rescales them and scatters them
// back, so a token that occurs several times is penalised once: read phase, barrier, write phase (duplicates write the same value).
__global__ void __launch_bounds__(1024) rep_penalty_kernel(float* __restrict__ logits, int64_t V, const int64_t* __restrict__ seq,
                                                          int64_t seq_stride, const int32_t* __restrict__ cur_len, float penalty,
                                                          float* __restrict__ scratch) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  const int n = *cur_len;
  float* row = logits + b * V;
  const int64_t* sq = seq + b * seq_stride;
  float* sc = scratch + b * seq_stride;
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t t = sq[i];
    sc[i] = (t >= 0 && t < V) ? row[t] : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += blockDim.x) {
    const int64_t t = sq[i];
    if (t >= 0 && t < V) {
      const float x = sc[i];
      row[t] = x < 0.f ? x * penalty : x / penalty;
    }
  }
}

__device__ __forceinline__ uint32_t f2key(float f) {  // order-preserving float -> uint map
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// One CTA (1024 threads) per row: max, optional exact k-th-largest threshold by 4-pass radix select on the float keys,
// (TOP_P) optional nucleus threshold by a 4-pass radix select on probability mass, sum of exp((x - max) / T) over the kept
// entries, then the inverse-CDF pick for the uniform u: thread t owns the contiguous chunk [t*c, (t+1)*c), a block scan of
// the chunk sums finds the chunk, a serial walk finds the index.  Deterministic for a given u (the host draws u from a
// seeded torch generator).  sample_kernel<false> is uvx_sample; top_p is read only by sample_kernel<true>.
constexpr float kMassOne = 1099511627776.f;  // 2^40: fixed-point unit of the top-p mass (sum <= V * 2^40 < 2^64 for V <= 2^24)

template <bool TOP_P>  // (1024, 1): lets ptxas use the 64 registers a lone 1024-thread CTA may have (the top-p form uses 56)
__global__ void __launch_bounds__(1024, 1) sample_kernel(const float* __restrict__ logits, int64_t V, float inv_temp, int top_k,
                                                     float top_p, const float* __restrict__ u_all,
                                                     const int32_t* __restrict__ step_idx, int64_t u_stride,
                                                     int64_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ float chunk_base[32];
  __shared__ int win_thread;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t b = blockIdx.x;
  const float* row = logits + b * V;
  // ---- max
  float mx = -INFINITY;
  for (int64_t i = tid; i < V; i += 1024) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = warp_max(red[lane]);
  __syncthreads();
  // ---- top-k threshold (keys >= thr_key are kept); top_k <= 0 or >= V keeps everything
  uint32_t thr_key = 0u;
  if (top_k > 0 && (int64_t)top_k < V) {
    if (tid == 0) { sel_prefix = 0u; sel_remaining = (uint32_t)top_k; }
    for (int pass = 3; pass >= 0; --pass) {
      if (tid < 256) hist[tid] = 0u;
      __syncthreads();
      const uint32_t prefix = sel_prefix;
      const uint32_t hi_mask = pass == 3 ? 0u : (0xFFFFFFFFu << ((pass + 1) * 8));
      for (int64_t i = tid; i < V; i += 1024) {
        const uint32_t k = f2key(row[i]);
        if ((k & hi_mask) == (prefix & hi_mask)) atomicAdd(&hist[(k >> (pass * 8)) & 255u], 1u);
      }
      __syncthreads();
      if (tid == 0) {
        uint32_t rem = sel_remaining;
        int d = 255;
        for (; d > 0; --d) {
          if (hist[d] >= rem) break;
          rem -= hist[d];
        }
        sel_prefix = prefix | ((uint32_t)d << (pass * 8));
        sel_remaining = rem;
      }
      __syncthreads();
    }
    thr_key = sel_prefix;
  }
  if constexpr (TOP_P) {
    // ---- top-p threshold over the top-k survivors (HF TopPLogitsWarper after TopKLogitsWarper): with m_i = exp((x_i - max) / T),
    // the smallest key v such that the mass of the keys <= v exceeds (1 - top_p) * (total mass); keys >= v are kept.  Radix
    // select from the top byte down: a 256-bin mass histogram of the keys that match the prefix, scanned upward from the mass
    // carried below the prefix.  Masses are 64-bit fixed point (kMassOne = 1), so the atomics are order-free and the result
    // deterministic; a tie group has one key and is kept or dropped whole.  Entries whose mass rounds to 0 never cross the
    // threshold and are skipped.  target <= total - 1 makes the maximum (mass exactly kMassOne) always kept: top_p = 0 -> argmax.
    __shared__ unsigned long long mhist[256];
    __shared__ unsigned long long p_below, p_target;
    __shared__ uint32_t p_prefix;
    if (tid == 0) { p_prefix = 0u; p_below = 0ull; p_target = 0ull; }
    for (int pass = 3; pass >= 0; --pass) {
      if (tid < 256) mhist[tid] = 0ull;
      __syncthreads();
      const uint32_t prefix = p_prefix;
      const uint32_t hi_mask = pass == 3 ? 0u : (0xFFFFFFFFu << ((pass + 1) * 8));
      // a per-thread cache of 4 (bin, mass) slots in registers: without top-k most of the row carries mass, and the first pass
      // puts it in the few top-byte bins its exponents span, where shared atomics would serialise on a handful of addresses
      uint32_t cb[4] = {~0u, ~0u, ~0u, ~0u};
      unsigned long long cs[4] = {0ull, 0ull, 0ull, 0ull};
      constexpr int kLoads = 8;  // independent loads in flight per thread: one at a time, a pass is bound by L2 latency
      for (int64_t base = tid; base < V; base += 1024 * kLoads) {
        float xs[kLoads];
#pragma unroll
        for (int j = 0; j < kLoads; ++j) {
          const int64_t i = base + (int64_t)j * 1024;
          xs[j] = i < V ? row[i] : -INFINITY;
        }
#pragma unroll
        for (int j = 0; j < kLoads; ++j) {
          const float x = xs[j];
          const uint32_t k = f2key(x);
          if (base + (int64_t)j * 1024 >= V || k < thr_key || (k & hi_mask) != (prefix & hi_mask)) continue;
          const unsigned long long m = __float2ull_rn(__expf((x - mx) * inv_temp) * kMassOne);
          if (m == 0ull) continue;
          const uint32_t bin = (k >> (pass * 8)) & 255u;
          bool held = false;
#pragma unroll
          for (int s = 0; s < 4; ++s)
            if (!held && cb[s] == bin) { cs[s] += m; held = true; }
#pragma unroll
          for (int s = 0; s < 4; ++s)
            if (!held && cs[s] == 0ull) { cb[s] = bin; cs[s] = m; held = true; }
          if (!held) atomicAdd(&mhist[bin], m);
        }
      }
#pragma unroll
      for (int s = 0; s < 4; ++s)
        if (cs[s] != 0ull) atomicAdd(&mhist[cb[s]], cs[s]);
      __syncthreads();
      if (w == 0) {  // lane l scans bins [8l, 8l + 8)
        unsigned long long s = 0ull;
#pragma unroll
        for (int j = 0; j < 8; ++j) s += mhist[lane * 8 + j];
        unsigned long long incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned long long t = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += t;
        }
        if (pass == 3) {  // the first pass sees every survivor: its histogram total is the whole mass
          const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
          if (lane == 0 && total > 0ull) {
            const unsigned long long t = (unsigned long long)((1.0 - (double)top_p) * (double)total);
            p_target = t < total - 1ull ? t : total - 1ull;
          }
          __syncwarp();
        }
        const unsigned long long below = p_below, target = p_target;
        const unsigned hit = __ballot_sync(0xffffffffu, below + incl > target);
        if (hit != 0u && lane == __ffs(hit) - 1) {  // no hit only for a row without mass (all -inf): no top-p cut
          unsigned long long acc = below + incl - s;
          int d = lane * 8;
          for (; d < lane * 8 + 7; ++d) {
            if (acc + mhist[d] > target) break;
            acc += mhist[d];
          }
          p_prefix = prefix | ((uint32_t)d << (pass * 8));
          p_below = acc;
        }
      }
      __syncthreads();
    }
    thr_key = max(thr_key, p_prefix);
  }
  // ---- chunk sums
  const int64_t c = (V + 1023) / 1024;
  const int64_t lo = (int64_t)tid * c, hi = lo + c < V ? lo + c : V;
  float local = 0.f;
  for (int64_t i = lo; i < hi; ++i) {
    const float x = row[i];
    if (f2key(x) >= thr_key) local += __expf((x - mx) * inv_temp);
  }
  // inclusive scan over the 1024 chunk sums
  float incl = local;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) red[w] = incl;
  __syncthreads();
  if (w == 0) {
    float v = red[lane], s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const float t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    chunk_base[lane] = s - v;  // exclusive prefix of the warp totals
    if (lane == 31) red[0] = s;  // grand total (red[] is dead: every warp has read it)
  }
  if (tid == 0) win_thread = -1;
  __syncthreads();
  const float total = red[0];
  const float excl = chunk_base[w] + incl - local;
  const float u = u_all[(int64_t)(step_idx ? *step_idx : 0) * u_stride + b];
  const float target = fminf(u, 0.99999994f) * total;
  if (local > 0.f && target >= excl && target < excl + local) atomicMax(&win_thread, tid);
  __syncthreads();
  int wt = win_thread;
  if (wt < 0) {
    // rounding at a chunk edge: fall back to the last chunk with mass at or before the target
    if (local > 0.f && excl <= target) atomicMax(&win_thread, tid);
    __syncthreads();
    wt = win_thread;
  }
  if (tid == (wt < 0 ? 0 : wt)) {
    float acc = excl;
    int64_t pick = -1, last = -1;
    for (int64_t i = lo; i < hi; ++i) {
      const float x = row[i];
      if (f2key(x) < thr_key) continue;
      last = i;
      acc += __expf((x - mx) * inv_temp);
      if (acc > target) { pick = i; break; }
    }
    if (pick < 0) pick = last >= 0 ? last : 0;
    out[b] = pick;
  }
}

// One CTA: rows that already produced an EOS emit pad_id (HF semantics), the token is appended to `sequences`, rows whose token
// is an EOS become finished, every counter in `bump` advances by one, all_done[0] = (every row finished).
__global__ void token_finish_kernel(int64_t* __restrict__ tok, int32_t* __restrict__ done, const int64_t* __restrict__ eos,
                                    int n_eos, int64_t pad_id, int64_t* __restrict__ seq, int64_t seq_stride,
                                    int32_t* __restrict__ cur_len, int32_t* __restrict__ step_idx, int32_t* __restrict__ bump0,
                                    int32_t* __restrict__ bump1, int32_t* __restrict__ bump2, int32_t* __restrict__ all_done,
                                    int64_t B) {
  pdl_trigger();
  pdl_wait();
  __shared__ int any_open;
  if (threadIdx.x == 0) any_open = 0;
  __syncthreads();
  const int n = *cur_len;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    int64_t t = tok[b];
    int d = done[b];
    if (d) t = pad_id;
    tok[b] = t;
    if (seq) seq[b * seq_stride + n] = t;
    for (int e = 0; e < n_eos; ++e) d |= (t == eos[e]);
    done[b] = d;
    if (!d) atomicOr(&any_open, 1);
    if (bump0) bump0[b] += 1;
    if (bump1) bump1[b] += 1;
    if (bump2) bump2[b] += 1;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    *cur_len = n + 1;
    if (step_idx) *step_idx += 1;
    if (all_done) *all_done = any_open ? 0 : 1;
  }
}

}  // namespace uvx

extern "C" int uvx_kv_write(const void* qkv, int64_t row_stride, int64_t k_col, int64_t v_col, int64_t kv_width, void* k_cache,
                            void* v_cache, int64_t cache_batch_stride, int64_t B, int64_t S, int64_t past, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && k_cache && v_cache && B >= 1 && S >= 1 && past >= 0, "uvx_kv_write: bad arguments");
  UVX_REQUIRE(kv_width % 8 == 0 && row_stride % 8 == 0 && k_col % 8 == 0 && v_col % 8 == 0 && cache_batch_stride % 8 == 0,
              "uvx_kv_write: alignment");
  const int64_t total = 2 * B * S * (kv_width / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 148 * 8) blocks = 148 * 8;
  launch_k(kv_write_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const bf16*)qkv, row_stride, (int)k_col,
           (int)v_col, (int)kv_width, (bf16*)k_cache, (bf16*)v_cache, cache_batch_stride, B, S, past);
  return check_launch("kv_write_kernel");
}

extern "C" int uvx_repetition_penalty(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                      const int32_t* cur_len, float penalty, float* scratch, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && cur_len && scratch && B >= 1 && V >= 1 && penalty > 0.f, "uvx_repetition_penalty: bad arguments");
  launch_k(rep_penalty_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, cur_len, penalty,
           scratch);
  return check_launch("rep_penalty_kernel");
}

extern "C" int uvx_sample(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, const float* u,
                          const int32_t* step_idx, int64_t u_stride, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && u && out_idx && B >= 1 && V >= 1 && temperature > 0.f, "uvx_sample: bad arguments");
  launch_k(sample_kernel<false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature, (int)top_k,
           1.0f, u, step_idx, u_stride, out_idx);
  return check_launch("sample_kernel");
}

extern "C" int uvx_sample_top_p(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                const float* u, const int32_t* step_idx, int64_t u_stride, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && u && out_idx && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && temperature > 0.f && top_p >= 0.f &&
                  top_p <= 1.f,
              "uvx_sample_top_p: bad arguments");
  if (top_p >= 1.f) return uvx_sample(logits, B, V, temperature, top_k, u, step_idx, u_stride, out_idx, stream);
  launch_k(sample_kernel<true>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature, (int)top_k,
           top_p, u, step_idx, u_stride, out_idx);
  return check_launch("sample_kernel_top_p");
}

extern "C" int uvx_token_finish(int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int64_t* seq,
                                int64_t seq_stride, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1,
                                int32_t* bump2, int32_t* all_done, int64_t B, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && cur_len && B >= 1 && (n_eos == 0 || eos_ids), "uvx_token_finish: bad arguments");
  launch_k(token_finish_kernel, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, pad_id, seq, seq_stride,
           cur_len, step_idx, bump0, bump1, bump2, all_done, B);
  return check_launch("token_finish_kernel");
}
