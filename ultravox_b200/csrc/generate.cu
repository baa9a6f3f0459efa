// Decode-loop helpers (a13): everything `GenerationMixin.generate` does between two LLM steps, as kernels that read their
// step state from device memory so the whole step can sit in one CUDA graph (no host sync per token):
//   uvx_kv_write            prefill: k / v sections of the fused projection -> the static KV cache (replaces two strided copies)
//   uvx_repetition_penalty  hf:generation/logits_process.py RepetitionPenaltyLogitsProcessor (ref ultravox_pipeline.py:95-113)
//   uvx_sample              temperature / top-k multinomial sampling (ref:ultravox/inference/infer.py:319-328: do_sample when
//                           temperature > 0; hf:generation/utils.py _sample: softmax(logits / T) -> multinomial)
//   uvx_sample_top_p        the same with nucleus (top-p) filtering after top-k (hf:generation/logits_process.py TopPLogitsWarper)
//   uvx_token_finish        EOS / pad bookkeeping of the finished rows, append to `sequences`, advance positions
//   uvx_sample_slots        continuous batching: per-row greedy / sampled pick with each row's own settings and uniform
//   uvx_repetition_penalty_slots   the repetition penalty with each row's own penalty and length
//   uvx_slot_finish         per-row append / budget / EOS bookkeeping; finished and idle rows stay frozen
//   uvx_log_softmax         beam search scores: log_softmax over each logits row (hf:generation/utils.py _beam_search)
//   uvx_beam_select         the top K of (log-prob + running beam score) over each prompt's nb * V continuations
//   uvx_beam_update         running beams, finished-hypothesis pool, early-stop heuristic and loop condition of one step
//   uvx_kv_reorder          in-place gather of the KV cache rows by parent beam (and the prefill broadcast to the beams)
//   uvx_kv_page_map         paged KV cache: (table row, position) of each step row -> (page, offset) for the mapped RoPE + append
//   uvx_kv_pages_copy       paged KV cache: positions of a contiguous one-row cache <-> their pages, all layers, K and V
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

// The body is sample_row, shared with uvx_sample_slots: TOP_P = 0 never runs the nucleus pass, 1 always does, 2 does when the
// row's top_p < 1 (the per-row form of uvx_sample_top_p routing top_p >= 1 to uvx_sample).  The caller's CTA handles one row.
template <int TOP_P>
__device__ __forceinline__ void sample_row(const float* __restrict__ row, int64_t V, float inv_temp, int top_k, float top_p,
                                           const float* __restrict__ u_all, const int32_t* __restrict__ step_idx, int64_t u_stride,
                                           int64_t col, int64_t* __restrict__ out_ptr) {
  __shared__ float red[32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ float chunk_base[32];
  __shared__ int win_thread;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
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
  if (TOP_P == 1 || (TOP_P == 2 && top_p < 1.f)) {
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
  const float u = u_all[(int64_t)(step_idx ? *step_idx : 0) * u_stride + col];
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
    *out_ptr = pick;
  }
}

template <bool TOP_P>  // (1024, 1): lets ptxas use the 64 registers a lone 1024-thread CTA may have (the top-p form uses 56)
__global__ void __launch_bounds__(1024, 1) sample_kernel(const float* __restrict__ logits, int64_t V, float inv_temp, int top_k,
                                                     float top_p, const float* __restrict__ u_all,
                                                     const int32_t* __restrict__ step_idx, int64_t u_stride,
                                                     int64_t* __restrict__ out) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  sample_row<TOP_P ? 1 : 0>(logits + b * V, V, inv_temp, top_k, top_p, u_all, step_idx, u_stride, b, out + b);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Continuous batching: a fixed set of decode rows ("slots"), each with its own request state.  The state written by the
// preceding kernel (or by the host between graph replays) is read through plain pointers, as in the beam kernels below.

// One CTA per row: first index of the row maximum (uvx_argmax's rule: an all -inf row gives 0).
__device__ __forceinline__ void argmax_row(const float* row, int64_t V, int64_t* out_ptr) {
  __shared__ float red[32];
  __shared__ unsigned long long ired[32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float mx = -INFINITY;
  for (int64_t i = tid; i < V; i += 1024) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = warp_max(red[lane]);
  unsigned long long first = ~0ull;
  for (int64_t i = tid; i < V; i += 1024)
    if (row[i] == mx) { first = (unsigned long long)i; break; }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long t = __shfl_xor_sync(0xffffffffu, first, o);
    first = t < first ? t : first;
  }
  if (lane == 0) ired[w] = first;
  __syncthreads();
  if (w == 0) {
    first = ired[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long t = __shfl_xor_sync(0xffffffffu, first, o);
      first = t < first ? t : first;
    }
    if (lane == 0) *out_ptr = (int64_t)first;
  }
}

// One CTA per row: inactive rows are left alone; temperature <= 0 takes the argmax, otherwise sample_row with the row's own
// settings and the uniform u[row * u_stride + n_new[row]].
__global__ void __launch_bounds__(1024, 1) sample_slots_kernel(const float* logits, int64_t V, const float* temperature,
                                                               const int32_t* top_k, const float* top_p, const float* u,
                                                               int64_t u_stride, const int32_t* n_new, const int32_t* active,
                                                               int64_t* out) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  if (!active[b]) return;
  const float t = temperature[b];
  const float* row = logits + b * V;
  if (!(t > 0.f)) {
    argmax_row(row, V, out + b);
    return;
  }
  sample_row<2>(row, V, __frcp_rn(t), top_k[b], top_p[b], u + b * u_stride, n_new + b, 1, 0, out + b);
}

// One CTA per row: uvx_repetition_penalty's rule with the row's own penalty over seq[b, 0:cur_len[b]]; inactive rows and
// penalty 1 are skipped.
__global__ void __launch_bounds__(1024) rep_penalty_slots_kernel(float* logits, int64_t V, const int64_t* seq, int64_t seq_stride,
                                                                 const int32_t* cur_len, const float* penalty, const int32_t* active,
                                                                 float* __restrict__ scratch) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  if (!active[b]) return;
  const float pen = penalty[b];
  if (pen == 1.f) return;
  const int n = cur_len[b];
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
      row[t] = x < 0.f ? x * pen : x / pen;
    }
  }
}

// One CTA: for each active, unfinished row append tok at seq[b, cur_len[b]], advance cur_len / n_new, finish on an EOS id or
// at the budget, and advance pos / lens / rope_pos only while the row stays open.  n_open[0] = active rows still open.
__global__ void slot_finish_kernel(const int64_t* tok, int32_t* done, const int64_t* __restrict__ eos, int n_eos, int64_t* seq,
                                   int64_t seq_stride, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                                   int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* n_open, int64_t B) {
  pdl_trigger();
  pdl_wait();
  __shared__ int open;
  if (threadIdx.x == 0) open = 0;
  __syncthreads();
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    if (!active[b] || done[b]) continue;
    const int64_t t = tok[b];
    const int n = cur_len[b];
    seq[b * seq_stride + n] = t;
    cur_len[b] = n + 1;
    const int k = n_new[b] + 1;
    n_new[b] = k;
    int d = k >= max_new[b];
    for (int e = 0; e < n_eos; ++e) d |= (t == eos[e]);
    done[b] = d;
    if (!d) {
      pos[b] += 1;
      lens[b] += 1;
      rope_pos[b] += 1;
      atomicAdd(&open, 1);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *n_open = open;
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

// ---------------------------------------------------------------------------------------------------------------------------
// Beam search (hf:generation/utils.py _beam_search and the helpers above it).  Row r = b * nb + j is beam j of prompt b.
// Inputs written by the preceding kernel are plain (not const __restrict__) pointers: nvcc may hoist a read-only (.nc)
// load above griddepcontrol.wait, and under PDL that reads the previous kernel's output before it is complete.
constexpr int kBeamMax = 8;     // beams per prompt
constexpr int kBeamMaxK = 64;   // candidates per prompt, K = max(2, 1 + n_eos) * nb
constexpr int kSeqChunk = 128;  // token positions staged per round by beam_update_kernel

// One CTA per row: y = (x - max) - log(sum exp(x - max)), in fp32 (in == out allowed).
__global__ void __launch_bounds__(1024) log_softmax_kernel(const float* in, float* out, int64_t V) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const float* x = in + (int64_t)blockIdx.x * V;
  float* y = out + (int64_t)blockIdx.x * V;
  float mx = -INFINITY;
  for (int64_t i = tid; i < V; i += 1024) mx = fmaxf(mx, x[i]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = warp_max(red[lane]);
  __syncthreads();
  float s = 0.f;
  for (int64_t i = tid; i < V; i += 1024) s += expf(x[i] - mx);
  s = warp_sum(s);
  if (lane == 0) red[w] = s;
  __syncthreads();
  const float lse = logf(warp_sum(red[lane]));
  for (int64_t i = tid; i < V; i += 1024) y[i] = (x[i] - mx) - lse;
}

// One CTA (1024 threads) per row: the K largest of lp[r, v] + run_score[r] (one fp32 add, as HF adds the running score),
// sorted by (value desc, v asc).  The K-th largest key comes from the 4-pass radix select of sample_kernel; the keys above it
// (fewer than K) are appended in any order, the missing ones are taken from the keys equal to it in index order (thread t
// owns the chunk [t*c, (t+1)*c), an exclusive scan of the per-chunk counts ranks them), and the K survivors are sorted by
// rank.  out_i holds the prompt-flat index j * V + v.
__global__ void __launch_bounds__(1024, 1) beam_row_topk_kernel(const float* lp, int64_t V, const float* run_score, int nb, int K,
                                                                float* __restrict__ out_s, int64_t* __restrict__ out_i) {
  pdl_trigger();
  pdl_wait();
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ int n_gt;
  __shared__ int scan[32];
  __shared__ float s_val[kBeamMaxK];
  __shared__ int64_t s_idx[kBeamMaxK];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t r = blockIdx.x;
  const float* row = lp + r * V;
  const float sc = run_score[r];
  if (tid == 0) { sel_prefix = 0u; sel_remaining = (uint32_t)K; n_gt = 0; }
  for (int pass = 3; pass >= 0; --pass) {
    if (tid < 256) hist[tid] = 0u;
    __syncthreads();
    const uint32_t prefix = sel_prefix;
    const uint32_t hi_mask = pass == 3 ? 0u : (0xFFFFFFFFu << ((pass + 1) * 8));
    for (int64_t i = tid; i < V; i += 1024) {
      const uint32_t k = f2key(row[i] + sc);
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
  const uint32_t thr = sel_prefix;
  const int need_eq = (int)sel_remaining;  // keys equal to thr to take; K - need_eq keys lie above it
  for (int64_t i = tid; i < V; i += 1024) {
    const float x = row[i] + sc;
    if (f2key(x) > thr) {
      const int s = atomicAdd(&n_gt, 1);
      s_val[s] = x;
      s_idx[s] = i;
    }
  }
  const int64_t c = (V + 1023) / 1024;
  const int64_t lo = (int64_t)tid * c, hi = lo + c < V ? lo + c : V;
  int cnt = 0;
  for (int64_t i = lo; i < hi; ++i) cnt += f2key(row[i] + sc) == thr;
  int incl = cnt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, incl, o);
    if (lane >= o) incl += t;
  }
  if (lane == 31) scan[w] = incl;
  __syncthreads();
  if (w == 0) {
    const int v = scan[lane];
    int s = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += t;
    }
    scan[lane] = s - v;
  }
  __syncthreads();
  int rank = scan[w] + incl - cnt;
  const int base = K - need_eq;
  for (int64_t i = lo; i < hi && rank < need_eq; ++i) {
    const float x = row[i] + sc;
    if (f2key(x) == thr) {
      s_val[base + rank] = x;
      s_idx[base + rank] = i;
      ++rank;
    }
  }
  __syncthreads();
  if (tid < K) {
    const float x = s_val[tid];
    const int64_t ix = s_idx[tid];
    int pos = 0;
    for (int m = 0; m < K; ++m) pos += s_val[m] > x || (s_val[m] == x && s_idx[m] < ix);
    out_s[r * K + pos] = x;
    out_i[r * K + pos] = (r % nb) * V + ix;
  }
}

// One CTA per prompt: the top K of its nb row lists (nb * K entries), by (value desc, flat index asc).
__global__ void __launch_bounds__(kBeamMax * kBeamMaxK) beam_merge_kernel(const float* row_s, const int64_t* row_i, int nb, int K,
                                                                          float* __restrict__ out_s, int64_t* __restrict__ out_i) {
  pdl_trigger();
  pdl_wait();
  __shared__ float sv[kBeamMax * kBeamMaxK];
  __shared__ int64_t si[kBeamMax * kBeamMaxK];
  const int64_t b = blockIdx.x;
  const int n = nb * K;
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    sv[t] = row_s[b * n + t];
    si[t] = row_i[b * n + t];
  }
  __syncthreads();
  for (int t = threadIdx.x; t < n; t += blockDim.x) {
    const float x = sv[t];
    const int64_t ix = si[t];
    int pos = 0;
    for (int m = 0; m < n; ++m) pos += sv[m] > x || (sv[m] == x && si[m] < ix);
    if (pos < K) {
      out_s[b * K + pos] = x;
      out_i[b * K + pos] = ix;
    }
  }
}

// One CTA per prompt: steps d-g of one _beam_search iteration on the K sorted candidates of uvx_beam_select.  Every fp32
// operation is HF's, in HF's order; top-k ties are broken towards the lower index.  The last CTA to finish (ticket) folds the
// per-prompt flags into the loop condition and advances the step counters.  With done[0] set nothing changes except parent,
// which becomes the identity (so the uvx_kv_reorder that follows is a no-op).
__global__ void __launch_bounds__(256) beam_update_kernel(
    const float* cand_s, const int64_t* cand_i, int64_t V, int nb, int K, const int64_t* __restrict__ eos,
    int n_eos, int max_new, const float* __restrict__ len_div, int early_stopping, int lp_positive, float* __restrict__ run_score,
    int64_t* __restrict__ run_seq, int64_t* __restrict__ pool_seq, int64_t seq_stride, float* __restrict__ pool_score,
    int32_t* __restrict__ pool_len, int32_t* __restrict__ pool_fin, int32_t* __restrict__ parent, int64_t* __restrict__ tok,
    int32_t* __restrict__ heur, int32_t* __restrict__ flags, uint32_t* __restrict__ ticket, int32_t* __restrict__ cur_len,
    int32_t* __restrict__ step_idx, int32_t* __restrict__ bump0, int32_t* __restrict__ bump1, int32_t* __restrict__ bump2,
    int32_t* __restrict__ done, int64_t B) {
  pdl_trigger();
  pdl_wait();
  __shared__ float rsc[kBeamMaxK], psc[kBeamMaxK];  // running-selection / pool-merge scores of the candidates
  __shared__ int cj[kBeamMaxK], chit[kBeamMaxK];
  __shared__ int64_t ct[kBeamMaxK];
  __shared__ float old_ps[kBeamMax];
  __shared__ int old_pl[kBeamMax], old_pf[kBeamMax];
  __shared__ int run_src[kBeamMax], pool_src[kBeamMax];
  __shared__ int64_t stage[2 * kBeamMax * kSeqChunk];
  const int tid = threadIdx.x;
  const int64_t b = blockIdx.x, r0 = b * nb;
  if (*done) {
    if (tid < nb) parent[r0 + tid] = (int32_t)(r0 + tid);
    return;
  }
  const int n = *cur_len, gen = *step_idx + 1;  // HF: cur_len = n, the candidates' generated length cur_len + 1 - prompt = gen
  const int heur_old = heur[b];
  if (tid < nb) {
    old_ps[tid] = pool_score[r0 + tid];
    old_pl[tid] = pool_len[r0 + tid];
    old_pf[tid] = pool_fin[r0 + tid];
  }
  __syncthreads();
  int full = early_stopping == 1;  // beams_in_batch_are_full
  for (int j = 0; j < nb; ++j) full &= old_pf[j] != 0;
  if (tid < K) {
    const float s = cand_s[b * K + tid];
    const int64_t idx = cand_i[b * K + tid];
    const int64_t t = idx % V;
    int hit = gen >= max_new;  // MaxLengthCriteria: cur_len + 1 >= prompt + max_new_tokens
    for (int e = 0; e < n_eos; ++e) hit |= t == eos[e];
    cj[tid] = (int)(idx / V);
    ct[tid] = t;
    chit[tid] = hit;
    rsc[tid] = s + (hit ? -1.0e9f : -0.0f);  // _get_running_beams_for_next_iteration
    const int did = hit && tid < nb;         // _update_finished_beams: only the top nb may finish
    float p = s / len_div[gen];
    p = p + (full ? -1.0e9f : -0.0f);
    p = p + (heur_old ? -0.0f : -1.0e9f);
    p = p + (did ? -0.0f : -1.0e9f);
    psc[tid] = p;
  }
  __syncthreads();
  if (tid < K) {
    const float x = rsc[tid];
    int pos = 0;
    for (int m = 0; m < K; ++m) pos += rsc[m] > x || (rsc[m] == x && m < tid);
    if (pos < nb) run_src[pos] = tid;
  }
  if (tid < nb + K) {  // merged pool: old entries [0, nb), then the K candidates
    const float x = tid < nb ? old_ps[tid] : psc[tid - nb];
    int pos = 0;
    for (int m = 0; m < nb + K; ++m) {
      const float y = m < nb ? old_ps[m] : psc[m - nb];
      pos += y > x || (y == x && m < tid);
    }
    if (pos < nb) pool_src[pos] = tid;
  }
  __syncthreads();
  // sequences [0, n): every new row is a copy of an old running or pool row of this prompt, staged through shared memory
  for (int c0 = 0; c0 < n; c0 += kSeqChunk) {
    const int len = min(kSeqChunk, n - c0);
    for (int e = tid; e < nb * len; e += blockDim.x) {
      const int j = e / len, p = e % len;
      stage[j * kSeqChunk + p] = run_seq[(r0 + j) * seq_stride + c0 + p];
      stage[(nb + j) * kSeqChunk + p] = pool_seq[(r0 + j) * seq_stride + c0 + p];
    }
    __syncthreads();
    for (int e = tid; e < nb * len; e += blockDim.x) {
      const int i = e / len, p = e % len;
      const int m = pool_src[i];
      run_seq[(r0 + i) * seq_stride + c0 + p] = stage[cj[run_src[i]] * kSeqChunk + p];
      pool_seq[(r0 + i) * seq_stride + c0 + p] = m < nb ? stage[(nb + m) * kSeqChunk + p] : stage[cj[m - nb] * kSeqChunk + p];
    }
    __syncthreads();
  }
  if (tid < nb) {
    const int k = run_src[tid], m = pool_src[tid];
    run_seq[(r0 + tid) * seq_stride + n] = ct[k];
    run_score[r0 + tid] = rsc[k];
    parent[r0 + tid] = (int32_t)(r0 + cj[k]);
    tok[r0 + tid] = ct[k];
    if (m < nb) {  // an older hypothesis ends before position n
      pool_score[r0 + tid] = old_ps[m];
      pool_len[r0 + tid] = old_pl[m];
      pool_fin[r0 + tid] = old_pf[m];
    } else {
      pool_seq[(r0 + tid) * seq_stride + n] = ct[m - nb];
      pool_score[r0 + tid] = psc[m - nb];
      pool_len[r0 + tid] = gen;
      pool_fin[r0 + tid] = chit[m - nb] && m - nb < nb;
    }
    if (bump0) bump0[r0 + tid] += 1;
    if (bump1) bump1[r0 + tid] += 1;
    if (bump2) bump2[r0 + tid] += 1;
  }
  if (tid == 0) {
    // _check_early_stop_heuristic at cur_len + 1 on the new running scores and pool
    float worst = INFINITY;
    int all_fin = 1;
    for (int i = 0; i < nb; ++i) {
      const int m = pool_src[i];
      worst = fminf(worst, m < nb ? old_ps[m] : psc[m - nb]);
      all_fin &= m < nb ? old_pf[m] != 0 : (chit[m - nb] && m - nb < nb);
    }
    const int best_len = (early_stopping == 2 && lp_positive) ? max_new : gen;
    const float best = rsc[run_src[0]] / len_div[best_len];
    int improvable = 0;
    for (int i = 0; i < nb; ++i) {
      const int m = pool_src[i];
      const int fin = m < nb ? old_pf[m] != 0 : (chit[m - nb] && m - nb < nb);
      improvable |= best > (fin ? worst : -1.0e9f);
    }
    const int h = heur_old && improvable;
    heur[b] = h;
    int all_hit = 1;
    for (int k = 0; k < K; ++k) all_hit &= chit[k];
    flags[b] = h | (all_fin << 1) | (all_hit << 2);
    __threadfence();
    if (atomicAdd(ticket, 1u) == (uint32_t)(B - 1)) {  // last prompt: _beam_search_has_unfinished_sequences over the batch
      __threadfence();
      int any_h = 0, every_fin = 1, every_hit = 1;
      for (int64_t q = 0; q < B; ++q) {
        const int f = ((volatile int32_t*)flags)[q];
        any_h |= f & 1;
        every_fin &= (f >> 1) & 1;
        every_hit &= (f >> 2) & 1;
      }
      const int open = any_h && !(every_fin && early_stopping == 1) && !every_hit;
      *done = open ? 0 : 1;
      *cur_len = n + 1;
      *step_idx = gen;
      *ticket = 0u;
    }
  }
}

// k / v [L, G * nb, S_max, row_elems] bf16.  Tiles (layer, prompt, P positions) are spread over the grid; each stages the
// rows of its prompt that some other beam descends from, synchronises, then rewrites every beam whose parent is another row.
// A tile owns its positions of its prompt's rows, so duplicates, swaps and cycles need no scratch copy of the cache.
__global__ void __launch_bounds__(256) kv_reorder_kernel(bf16* k, bf16* v, int64_t L, int64_t G, int nb, int64_t S_max,
                                                         int64_t row_elems, const int32_t* parent, const int32_t* n_pos, int P) {
  pdl_trigger();
  pdl_wait();
  extern __shared__ uint4 kv_stage[];  // [nb][k, v][P * row_elems / 8]
  __shared__ int par[kBeamMax], need[kBeamMax];
  const int tid = threadIdx.x;
  const int n = *n_pos;
  const int64_t slices = (n + P - 1) / P;
  const int64_t tiles = L * G * slices;
  const int64_t vec = row_elems / 8;
  const int64_t row_vec = S_max * vec;
  const int64_t slot = (int64_t)P * vec;
  uint4* K4 = reinterpret_cast<uint4*>(k);
  uint4* V4 = reinterpret_cast<uint4*>(v);
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t s = tile % slices, g = (tile / slices) % G, l = tile / (slices * G);
    const int64_t row0 = l * G * nb + g * nb;
    if (tid < nb) par[tid] = parent[g * nb + tid] - (int32_t)(g * nb);
    __syncthreads();
    if (tid < nb) {
      int nd = 0;
      for (int c = 0; c < nb; ++c) nd |= c != tid && par[c] == tid;
      need[tid] = nd;
    }
    __syncthreads();
    const int64_t p0 = s * P;
    const int64_t cnt = (p0 + P < n ? (int64_t)P : n - p0) * vec;
    for (int j = 0; j < nb; ++j) {
      if (!need[j]) continue;
      const int64_t src = (row0 + j) * row_vec + p0 * vec;
      for (int64_t e = tid; e < cnt; e += blockDim.x) {
        kv_stage[(2 * j) * slot + e] = K4[src + e];
        kv_stage[(2 * j + 1) * slot + e] = V4[src + e];
      }
    }
    __syncthreads();
    for (int c = 0; c < nb; ++c) {
      const int p = par[c];
      if (p == c) continue;
      const int64_t dst = (row0 + c) * row_vec + p0 * vec;
      for (int64_t e = tid; e < cnt; e += blockDim.x) {
        K4[dst + e] = kv_stage[(2 * p) * slot + e];
        V4[dst + e] = kv_stage[(2 * p + 1) * slot + e];
      }
    }
    __syncthreads();
  }
}

static constexpr int kPageRows = 64;  // positions per KV page = keys per attention tile

// (cache_row[r], pos[r]) -> (page_out[r], off_out[r]) through the page table; cache_row < 0 or a frozen row -> (-1, 0), nothing
// is looked up
__global__ void kv_page_map_kernel(const int32_t* __restrict__ table, int64_t table_stride, const int32_t* __restrict__ cache_row,
                                   const int32_t* __restrict__ pos, const int32_t* __restrict__ frozen, int64_t n_frozen,
                                   int32_t* __restrict__ page_out, int32_t* __restrict__ off_out, int64_t rows) {
  pdl_trigger();
  pdl_wait();
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= rows) return;
  const int cr = cache_row[r];
  if (cr < 0 || (r < n_frozen && frozen[r])) {
    page_out[r] = -1;
    off_out[r] = 0;
    return;
  }
  const int p = pos[r];
  page_out[r] = table[(int64_t)cr * table_stride + p / kPageRows];
  off_out[r] = p % kPageRows;
}

// 16-byte vectors of positions [p0, p1) of every layer, K and V: row cache [L][S_max][row_elems] <-> pool [L][n_pages][64][row_elems]
__global__ void __launch_bounds__(256) kv_pages_copy_kernel(uint4* __restrict__ k_row, uint4* __restrict__ v_row, int64_t row_layer_vec,
                                                            uint4* __restrict__ k_pool, uint4* __restrict__ v_pool,
                                                            int64_t pool_layer_vec, int64_t L, int64_t vec,
                                                            const int32_t* __restrict__ pages, int64_t p0, int64_t n, int to_pages) {
  pdl_trigger();
  pdl_wait();
  const int64_t per_layer = n * vec;
  const int64_t total = 2 * L * per_layer;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int which = (int)(i / (L * per_layer));
    const int64_t rem = i % (L * per_layer);
    const int64_t l = rem / per_layer, e = rem % per_layer;
    const int64_t p = p0 + e / vec, c = e % vec;
    const int64_t pg = pages[p / kPageRows];
    const int64_t ri = l * row_layer_vec + p * vec + c;
    const int64_t pi = l * pool_layer_vec + (pg * kPageRows + p % kPageRows) * vec + c;
    uint4* row = which ? v_row : k_row;
    uint4* pool = which ? v_pool : k_pool;
    if (to_pages)
      pool[pi] = row[ri];
    else
      row[ri] = pool[pi];
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

extern "C" int uvx_sample_slots(const float* logits, int64_t B, int64_t V, const float* temperature, const int32_t* top_k,
                                const float* top_p, const float* u, int64_t u_stride, const int32_t* n_new, const int32_t* active,
                                int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && temperature && top_k && top_p && u && n_new && active && out_idx && B >= 1 && V >= 1 &&
                  V <= (int64_t)1 << 24 && u_stride >= 0,
              "uvx_sample_slots: bad arguments");
  launch_k(sample_slots_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, temperature, top_k, top_p, u,
           u_stride, n_new, active, out_idx);
  return check_launch("sample_slots_kernel");
}

extern "C" int uvx_repetition_penalty_slots(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                            const int32_t* cur_len, const float* penalty, const int32_t* active, float* scratch,
                                            uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && cur_len && penalty && active && scratch && B >= 1 && V >= 1,
              "uvx_repetition_penalty_slots: bad arguments");
  launch_k(rep_penalty_slots_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, cur_len,
           penalty, active, scratch);
  return check_launch("rep_penalty_slots_kernel");
}

extern "C" int uvx_slot_finish(const int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t* seq,
                               int64_t seq_stride, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                               int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* n_open, int64_t B, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && seq && cur_len && n_new && max_new && active && pos && lens && rope_pos && n_open && B >= 1 &&
                  n_eos >= 0 && (n_eos == 0 || eos_ids),
              "uvx_slot_finish: bad arguments");
  launch_k(slot_finish_kernel, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, seq, seq_stride, cur_len,
           n_new, max_new, active, pos, lens, rope_pos, n_open, B);
  return check_launch("slot_finish_kernel");
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

extern "C" int uvx_log_softmax(const float* in, float* out, int64_t rows, int64_t V, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(in && out && rows >= 1 && V >= 1, "uvx_log_softmax: bad arguments");
  launch_k(log_softmax_kernel, dim3((unsigned)rows), dim3(1024), 0, (cudaStream_t)stream, in, out, V);
  return check_launch("log_softmax_kernel");
}

extern "C" int uvx_beam_select(const float* logprobs, int64_t B, int32_t nb, int64_t V, const float* run_score, int32_t K,
                               float* row_s, int64_t* row_i, float* out_s, int64_t* out_i, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logprobs && run_score && row_s && row_i && out_s && out_i && B >= 1 && nb >= 1 && nb <= kBeamMax && K >= 1 &&
                  K <= kBeamMaxK && V >= K && V <= ((int64_t)1 << 40),
              "uvx_beam_select: bad arguments (1 <= nb <= %d, 1 <= K <= min(%d, V))", kBeamMax, kBeamMaxK);
  launch_k(beam_row_topk_kernel, dim3((unsigned)(B * nb)), dim3(1024), 0, (cudaStream_t)stream, logprobs, V, run_score, (int)nb, (int)K,
           row_s, row_i);
  if (int rc = check_launch("beam_row_topk_kernel")) return rc;
  launch_k(beam_merge_kernel, dim3((unsigned)B), dim3(kBeamMax * kBeamMaxK), 0, (cudaStream_t)stream, (const float*)row_s,
           (const int64_t*)row_i, (int)nb, (int)K, out_s, out_i);
  return check_launch("beam_merge_kernel");
}

extern "C" int uvx_beam_update(const float* cand_s, const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V,
                               const int64_t* eos_ids, int32_t n_eos, int32_t max_new, const float* len_div, int32_t early_stopping,
                               int32_t lp_positive, float* run_score, int64_t* run_seq, int64_t* pool_seq, int64_t seq_stride,
                               float* pool_score, int32_t* pool_len, int32_t* pool_fin, int32_t* parent, int64_t* tok,
                               int32_t* heur, int32_t* flags, uint32_t* ticket, int32_t* cur_len, int32_t* step_idx, int32_t* bump0,
                               int32_t* bump1, int32_t* bump2, int32_t* done, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(cand_s && cand_i && len_div && run_score && run_seq && pool_seq && pool_score && pool_len && pool_fin && parent && tok &&
                  heur && flags && ticket && cur_len && step_idx && done && B >= 1 && nb >= 1 && nb <= kBeamMax && K >= nb &&
                  K <= kBeamMaxK && V >= 1 && (n_eos == 0 || eos_ids) && n_eos >= 0 && max_new >= 1 && early_stopping >= 0 &&
                  early_stopping <= 2,
              "uvx_beam_update: bad arguments");
  launch_k(beam_update_kernel, dim3((unsigned)B), dim3(256), 0, (cudaStream_t)stream, cand_s, cand_i, V, (int)nb, (int)K, eos_ids,
           (int)n_eos, (int)max_new, len_div, (int)early_stopping, (int)lp_positive, run_score, run_seq, pool_seq, seq_stride,
           pool_score, pool_len, pool_fin, parent, tok, heur, flags, ticket, cur_len, step_idx, bump0, bump1, bump2, done, B);
  return check_launch("beam_update_kernel");
}

extern "C" int uvx_kv_reorder(void* k_cache, void* v_cache, int64_t L, int64_t B, int32_t nb, int64_t S_max, int64_t row_elems,
                              const int32_t* parent, const int32_t* n_pos, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(k_cache && v_cache && parent && n_pos && L >= 1 && B >= 1 && nb >= 1 && nb <= kBeamMax && S_max >= 1 && row_elems >= 8 &&
                  row_elems % 8 == 0,
              "uvx_kv_reorder: bad arguments");
  const int64_t per_pos = (int64_t)nb * 2 * row_elems * 2;  // staged bytes per position: nb rows of k and v
  int64_t P = 32768 / per_pos;  // (the static 64 bytes of the kernel count towards the 48 KB default as well)
  P = P < 1 ? 1 : (P > 64 ? 64 : P);
  const size_t smem = (size_t)(P * per_pos);
  UVX_REQUIRE(smem <= 227 * 1024, "uvx_kv_reorder: %lld-element rows do not fit in shared memory", (long long)row_elems);
  if (smem > 40 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(kv_reorder_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    UVX_REQUIRE(e == cudaSuccess, "uvx_kv_reorder: %s", cudaGetErrorString(e));
  }
  const int64_t tiles = L * B * ((S_max + P - 1) / P);
  const int64_t blocks = tiles < 132 * 6 ? tiles : 132 * 6;
  launch_k(kv_reorder_kernel, dim3((unsigned)blocks), dim3(256), smem, (cudaStream_t)stream, (bf16*)k_cache, (bf16*)v_cache, L, B,
           (int)nb, S_max, row_elems, parent, n_pos, (int)P);
  return check_launch("kv_reorder_kernel");
}

extern "C" int uvx_kv_page_map(const int32_t* table, int64_t table_stride, const int32_t* cache_row, const int32_t* pos,
                               const int32_t* frozen, int64_t n_frozen, int64_t rows, int32_t* page_out, int32_t* off_out,
                               uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(table && cache_row && pos && page_out && off_out && rows >= 1 && table_stride >= 1 && n_frozen >= 0 &&
                  n_frozen <= rows && (frozen || n_frozen == 0),
              "uvx_kv_page_map: bad arguments");
  launch_k(kv_page_map_kernel, dim3((unsigned)((rows + 255) / 256)), dim3(256), 0, (cudaStream_t)stream, table, table_stride, cache_row,
           pos, frozen, n_frozen, page_out, off_out, rows);
  return check_launch("kv_page_map_kernel");
}

extern "C" int uvx_kv_pages_copy(void* k_row, void* v_row, int64_t row_layer_stride, void* k_pool, void* v_pool, int64_t pool_layer_stride,
                                 int64_t L, int64_t row_elems, const int32_t* pages, int64_t p0, int64_t p1, int32_t to_pages,
                                 uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(k_row && v_row && k_pool && v_pool && pages && L >= 1, "uvx_kv_pages_copy: null pointer");
  UVX_REQUIRE(row_elems >= 8 && row_elems % 8 == 0 && row_layer_stride % 8 == 0 && pool_layer_stride % 8 == 0 && p0 >= 0 && p1 >= p0 &&
                  p1 * row_elems <= row_layer_stride,
              "uvx_kv_pages_copy: bad shape");
  UVX_REQUIRE(((uintptr_t)k_row | (uintptr_t)v_row | (uintptr_t)k_pool | (uintptr_t)v_pool) % 16 == 0,
              "uvx_kv_pages_copy: base pointers must be 16-byte aligned");
  if (p1 == p0) return UVX_OK;
  const int64_t total = 2 * L * (p1 - p0) * (row_elems / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_k(kv_pages_copy_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (uint4*)k_row, (uint4*)v_row,
           row_layer_stride / 8, (uint4*)k_pool, (uint4*)v_pool, pool_layer_stride / 8, L, row_elems / 8, pages, p0, p1 - p0,
           (int)to_pages);
  return check_launch("kv_pages_copy_kernel");
}
