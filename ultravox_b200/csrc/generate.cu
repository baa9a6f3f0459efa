// Decode-loop helpers (a13): everything `GenerationMixin.generate` does between two LLM steps, as kernels that read their
// step state from device memory so the whole step can sit in one CUDA graph (no host sync per token):
//   uvx_kv_write            prefill: k / v sections of the fused projection -> the static KV cache (replaces two strided copies)
//   uvx_repetition_penalty  hf:generation/logits_process.py RepetitionPenaltyLogitsProcessor (ref ultravox_pipeline.py:95-113)
//   uvx_sample              temperature / top-k multinomial sampling (ref:ultravox/inference/infer.py:319-328: do_sample when
//                           temperature > 0; hf:generation/utils.py _sample: softmax(logits / T) -> multinomial)
//   uvx_sample_top_p        the same with nucleus (top-p) filtering after top-k (hf:generation/logits_process.py TopPLogitsWarper)
//   uvx_sample_cutoffs      the same with min_p / typical_p / epsilon / eta cut-offs after top-p (MinP, Typical, Epsilon, Eta
//                           LogitsWarper); _slots_cutoffs / _rows_cutoffs with each slot's own cut-offs
//   uvx_token_finish        EOS / pad bookkeeping of the finished rows, append to `sequences`, advance positions
//   uvx_sample_slots        continuous batching: per-row greedy / sampled pick with each row's own settings and uniform
//   uvx_repetition_penalty_slots   the repetition penalty with each row's own penalty and length
//   uvx_repetition_penalty_rows    the repetition penalty with each row's own length and scratch (rows may share a sequence)
//   uvx_logits_constraints  sequence bias, n-gram ban, bad words, min length, suppression (hf:generation/logits_process.py),
//                           before the penalty; _slots / _rows / _rows_map with the penalty's per-row forms
//   uvx_lookup_draft        prompt lookup: n-gram search over the sequence, the k + 1 fed tokens and their positions
//   uvx_lookup_accept       prompt lookup: the picks that agree with the drafts, appended; counters, budget / EOS, the log
//   uvx_slot_finish         per-row append / budget / EOS bookkeeping; finished and idle rows stay frozen
//   uvx_log_softmax         beam search scores: log_softmax over each logits row (hf:generation/utils.py _beam_search)
//   uvx_beam_select         the top K of (log-prob + running beam score) over each prompt's nb * V continuations
//   uvx_beam_update         running beams, finished-hypothesis pool, early-stop heuristic and loop condition of one step
//   uvx_kv_reorder          in-place gather of the KV cache rows by parent beam (and the prefill broadcast to the beams)
//   uvx_kv_page_map         paged KV cache: (table row, position) of each step row -> (page, offset) for the mapped RoPE + append
//   uvx_kv_pages_copy       paged KV cache: positions of a contiguous one-row cache <-> their pages, all layers, K and V
//   uvx_kv_pages_move       paged KV cache: whole pages between two pools (device <-> pinned host), all layers, K and V, raw bytes
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

// Order-preserving float -> uint map.  A negative float maps to -bits (mod 2^32) rather than ~bits, which puts -0.0 on the key
// of +0.0 (0x80000000): the two compare equal, so a top-k cut, a top-p tie group and the (value desc, index asc) order of
// uvx_token_logprobs treat them as one value.  The same instruction count as ~bits.
__device__ __forceinline__ uint32_t f2key(float f) {
  const uint32_t u = __float_as_uint(f);
  return (u & 0x80000000u) ? 0u - u : (u | 0x80000000u);
}

// One CTA (1024 threads) per row: max, optional exact k-th-largest threshold by 4-pass radix select on the float keys,
// (TOP_P) optional nucleus threshold by a 4-pass radix select on probability mass, sum of exp((x - max) / T) over the kept
// entries, then the inverse-CDF pick for the uniform u: thread t owns the contiguous chunk [t*c, (t+1)*c), a block scan of
// the chunk sums finds the chunk, a serial walk finds the index.  Deterministic for a given u (the host draws u from a
// seeded torch generator).  sample_kernel<false> is uvx_sample; top_p is read only by sample_kernel<true>.
constexpr float kMassOne = 1099511627776.f;  // 2^40: fixed-point unit of the top-p mass (sum <= V * 2^40 < 2^64 for V <= 2^24)

// The k-th largest f2key of a row (1 <= k <= V) by a 4-pass radix select from the top byte down: afterwards sel_prefix is that
// key and sel_remaining the number of entries equal to it that rank among the k largest (the rest of the k lie above it).
// Every thread of the CTA (1024) calls it; hist [256] and the two scalars are the caller's shared memory.
__device__ __forceinline__ void radix_select_kth(const float* __restrict__ row, int64_t V, uint32_t k_th, uint32_t* hist,
                                                 uint32_t& sel_prefix, uint32_t& sel_remaining) {
  const int tid = threadIdx.x;
  if (tid == 0) { sel_prefix = 0u; sel_remaining = k_th; }
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
}

// The row maximum (mx) and the key threshold of the set a sampled pick draws from: entries with f2key(x) >= the returned key
// are kept (top-k, then top-p as below).  Shared by sample_row and uvx_record_scores, so a recorded score is finite exactly
// where the sampler can pick.  TOP_P = 0 never runs the nucleus pass, 1 always does, 2 does when the row's top_p < 1 (the
// per-row form of uvx_sample_top_p routing top_p >= 1 to uvx_sample).
struct ThresholdSmem {  // keep_threshold's shared memory, declared by the caller (sample_row keeps its own declaration order)
  float* red;                                     // [32]
  uint32_t* hist;                                 // [256]
  uint32_t *sel_prefix, *sel_remaining;
  unsigned long long* mhist;                      // [256]
  unsigned long long *p_below, *p_target;
  uint32_t* p_prefix;
};

// Mass-weighted radix select over the entries in_set(x, key_of(x)) accepts, keyed by key_of(x): the smallest key v such that the mass of the
// entries with key <= v exceeds target_of(total mass), total > 0 (0 when no entry has mass: the caller then makes no cut).  From
// the top byte down: a 256-bin mass histogram of the keys that match the prefix, scanned upward from the mass carried below the
// prefix.  Masses m = exp((x - max) / T) are 64-bit fixed point (kMassOne = 1), so the atomics are order-free and the result
// deterministic; equal keys share a bin and are counted or passed over whole.  Entries whose mass rounds to 0 never cross the
// threshold and are skipped.  The typical cut (keys = deviation from the mean log-mass).  It is keep_threshold's top-p pass
// with the key, the set and the target as parameters; keep_threshold keeps its own copy because routing it through this one
// changes the SASS of uvx_sample_top_p and uvx_record_scores (+32 instructions of scheduling) for no change in what they do.
template <class KeyOf, class InSet, class TargetOf>
__device__ __forceinline__ uint32_t mass_select(const float* __restrict__ row, int64_t V, float mx, float inv_temp, KeyOf key_of,
                                                InSet in_set, TargetOf target_of, const ThresholdSmem& sm) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  unsigned long long* mhist = sm.mhist;
  unsigned long long& p_below = *sm.p_below;
  unsigned long long& p_target = *sm.p_target;
  uint32_t& p_prefix = *sm.p_prefix;
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
        const uint32_t k = key_of(x);
        if (base + (int64_t)j * 1024 >= V || !in_set(x, k) || (k & hi_mask) != (prefix & hi_mask)) continue;
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
      if (pass == 3) {  // the first pass sees every entry of the set: its histogram total is the whole mass
        const unsigned long long total = __shfl_sync(0xffffffffu, incl, 31);
        if (lane == 0 && total > 0ull) p_target = target_of(total);
        __syncwarp();
      }
      const unsigned long long below = p_below, target = p_target;
      const unsigned hit = __ballot_sync(0xffffffffu, below + incl > target);
      if (hit != 0u && lane == __ffs(hit) - 1) {  // no hit only for a set without mass (all -inf)
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
  return p_prefix;
}

template <int TOP_P>
__device__ __forceinline__ uint32_t keep_threshold(const float* __restrict__ row, int64_t V, float inv_temp, int top_k, float top_p,
                                                   ThresholdSmem sm, float& mx_out) {
  float* red = sm.red;
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  // ---- max
  float mx = -INFINITY;
  for (int64_t i = tid; i < V; i += 1024) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = warp_max(red[lane]);
  __syncthreads();
  mx_out = mx;
  // ---- top-k threshold (keys >= thr_key are kept); top_k <= 0 or >= V keeps everything
  uint32_t thr_key = 0u;
  if (top_k > 0 && (int64_t)top_k < V) {
    radix_select_kth(row, V, (uint32_t)top_k, sm.hist, *sm.sel_prefix, *sm.sel_remaining);
    thr_key = *sm.sel_prefix;
  }
  if (TOP_P == 1 || (TOP_P == 2 && top_p < 1.f)) {
    // ---- top-p threshold over the top-k survivors (HF TopPLogitsWarper after TopKLogitsWarper): with m_i = exp((x_i - max) / T),
    // the smallest key v such that the mass of the keys <= v exceeds (1 - top_p) * (total mass); keys >= v are kept.  Radix
    // select from the top byte down: a 256-bin mass histogram of the keys that match the prefix, scanned upward from the mass
    // carried below the prefix.  Masses are 64-bit fixed point (kMassOne = 1), so the atomics are order-free and the result
    // deterministic; a tie group has one key and is kept or dropped whole.  Entries whose mass rounds to 0 never cross the
    // threshold and are skipped.  target <= total - 1 makes the maximum (mass exactly kMassOne) always kept: top_p = 0 -> argmax.
    unsigned long long* mhist = sm.mhist;
    unsigned long long& p_below = *sm.p_below;
    unsigned long long& p_target = *sm.p_target;
    uint32_t& p_prefix = *sm.p_prefix;
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
  return thr_key;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Sampling cut-offs after top-k / top-p (hf:generation/logits_process.py MinPLogitsWarper, TypicalLogitsWarper,
// EpsilonLogitsWarper, EtaLogitsWarper, in that order, min_tokens_to_keep = 1).  Each acts on the survivors of the one before;
// every one is on only when its value is (the host encodes off as min_p 0, typical 1, epsilon 0, eta 0).  The kept set is a band
// lo <= f2key(x) <= hi: min_p, epsilon and eta raise lo, typical can also lower hi (it may drop the row maximum).
struct Cutoffs {
  float min_p, typical_p, epsilon, eta;
};

__device__ __forceinline__ bool cutoffs_on(const Cutoffs& cf) {
  return cf.min_p > 0.f || cf.typical_p < 1.f || cf.epsilon > 0.f || cf.eta > 0.f;
}

struct CutoffSmem {  // the cut-off stage's shared memory, besides ThresholdSmem's
  double* dred;      // [32]
  unsigned long long* zsum;
  uint32_t *klo, *khi;
};

// Z = sum of the fixed-point masses over the band (integer atomics: order-free) and, when S is wanted, S = sum m * a with
// a = (x - max) / T in float64, reduced in a fixed order (per-thread stride, warp butterfly, warp 0 over the 32 partials), so the
// value depends on the row alone.  Entries of mass 0 add nothing (HF's 0 * log 0 = 0).
template <bool kWithS>
__device__ __forceinline__ void band_moments(const float* __restrict__ row, int64_t V, float mx, float inv_temp, uint32_t lo,
                                             uint32_t hi, const CutoffSmem& cs, unsigned long long& Z, double& S) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  if (tid == 0) *cs.zsum = 0ull;
  __syncthreads();
  unsigned long long z = 0ull;
  double s = 0.0;
  for (int64_t i = tid; i < V; i += 1024) {
    const float x = row[i];
    const uint32_t k = f2key(x);
    if (k < lo || k > hi) continue;
    const float a = (x - mx) * inv_temp;
    const float m = __expf(a);
    if (!(m > 0.f)) continue;
    z += __float2ull_rn(m * kMassOne);
    if (kWithS) s += (double)m * (double)a;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) z += __shfl_xor_sync(0xffffffffu, z, o);
  if (lane == 0 && z) atomicAdd(cs.zsum, z);
  if (kWithS) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) cs.dred[w] = s;
  }
  __syncthreads();
  Z = *cs.zsum;
  if (kWithS) {
    s = cs.dred[lane];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    S = s;
  }
  __syncthreads();
}

// The smallest key in the band whose fp32 mass __expf((x - max) / T) is >= mt (~0u when none is): a lower cut that keeps tie
// groups whole, as equal keys have equal masses.  Integer atomicMin: order-free.
__device__ __forceinline__ uint32_t band_min_key(const float* __restrict__ row, int64_t V, float mx, float inv_temp, uint32_t lo,
                                                 uint32_t hi, float mt, const CutoffSmem& cs) {
  if (threadIdx.x == 0) *cs.klo = ~0u;
  __syncthreads();
  uint32_t best = ~0u;
  for (int64_t i = threadIdx.x; i < V; i += 1024) {
    const float x = row[i];
    const uint32_t k = f2key(x);
    if (k >= lo && k <= hi && k < best && __expf((x - mx) * inv_temp) >= mt) best = k;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
  if ((threadIdx.x & 31) == 0 && best != ~0u) atomicMin(cs.klo, best);
  __syncthreads();
  const uint32_t r = *cs.klo;
  __syncthreads();
  return r;
}

// The cut-offs over the band [lo, hi] left by top-k / top-p (hi = ~0u).  With p = m / Z over the current survivors:
//  min_p:     keep m >= min_p (m_max = 1: p >= min_p * max p).
//  typical:   d = |-log p - H| = |a - S / Z|; the smallest deviation key D whose cumulative mass (by d ascending) reaches
//             typical_p * Z (HF's last_ind), by mass_select over deviation keys; keep d <= D, converted to the key band it spans
//             (d is V-shaped in x, so {d <= D} is an interval of keys).
//  epsilon:   keep m >= epsilon * Z, and the band's top key (the largest survivor's tie group).
//  eta:       keep m >= min(epsilon, sqrt(eta) exp(-H)) * Z, H = log Z - S / Z, and the band's top key.
// A band without mass (an all -inf row) is left as it is.  Every value that decides a cut is a fixed-point sum, a fixed-order
// float64 sum or an integer atomic: the band depends on the row and its settings alone.
__device__ __forceinline__ void cutoff_band(const float* __restrict__ row, int64_t V, float mx, float inv_temp, const Cutoffs& cf,
                                            const ThresholdSmem& sm, const CutoffSmem& cs, uint32_t& lo, uint32_t& hi) {
  const int tid = threadIdx.x;
  if (!(mx > -INFINITY)) return;
  if (cf.min_p > 0.f) {
    const uint32_t k = band_min_key(row, V, mx, inv_temp, lo, hi, cf.min_p, cs);
    if (k != ~0u) lo = max(lo, k);
  }
  if (cf.typical_p < 1.f) {
    unsigned long long Z;
    double S;
    band_moments<true>(row, V, mx, inv_temp, lo, hi, cs, Z, S);
    if (Z > 0ull) {
      const float c = (float)(S / ((double)Z / (double)kMassOne));
      const uint32_t blo = lo, bhi = hi;
      const auto dkey = [mx, inv_temp, c](float x) { return __float_as_uint(fabsf((x - mx) * inv_temp - c)); };
      const float tp = cf.typical_p;
      const uint32_t D = mass_select(
          row, V, mx, inv_temp, dkey,
          [blo, bhi](float x, uint32_t) {
            const uint32_t k = f2key(x);
            return k >= blo && k <= bhi;
          },
          [tp](unsigned long long total) {  // mass(d <= D) >= typical_p * Z: the first sorted cumulative mass not < typical_p
            const double want = ceil((double)tp * (double)total);
            const unsigned long long t = want >= 1.0 ? (unsigned long long)want - 1ull : 0ull;
            return t < total - 1ull ? t : total - 1ull;
          },
          sm);
      if (tid == 0) { *cs.klo = ~0u; *cs.khi = 0u; }
      __syncthreads();
      uint32_t kl = ~0u, kh = 0u;
      for (int64_t i = tid; i < V; i += 1024) {
        const float x = row[i];
        const uint32_t k = f2key(x);
        if (k >= blo && k <= bhi && __expf((x - mx) * inv_temp) > 0.f && dkey(x) <= D) { kl = min(kl, k); kh = max(kh, k); }
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        kl = min(kl, __shfl_xor_sync(0xffffffffu, kl, o));
        kh = max(kh, __shfl_xor_sync(0xffffffffu, kh, o));
      }
      if ((tid & 31) == 0 && kl != ~0u) { atomicMin(cs.klo, kl); atomicMax(cs.khi, kh); }
      __syncthreads();
      if (*cs.klo != ~0u) { lo = *cs.klo; hi = *cs.khi; }
      __syncthreads();
    }
  }
  // the band's top key: the row maximum's while typical has not lowered hi
  const uint32_t top = hi == ~0u ? f2key(mx) : hi;
  if (cf.epsilon > 0.f) {
    unsigned long long Z;
    double S;
    band_moments<false>(row, V, mx, inv_temp, lo, hi, cs, Z, S);
    const uint32_t k = band_min_key(row, V, mx, inv_temp, lo, hi, (float)((double)cf.epsilon * ((double)Z / (double)kMassOne)), cs);
    lo = max(lo, min(k, top));
  }
  if (cf.eta > 0.f) {
    unsigned long long Z;
    double S;
    band_moments<true>(row, V, mx, inv_temp, lo, hi, cs, Z, S);
    const double z = (double)Z / (double)kMassOne;
    const double H = log(z) - S / z;
    const double e = (double)cf.eta;
    const uint32_t k = band_min_key(row, V, mx, inv_temp, lo, hi, (float)(fmin(e, sqrt(e) * exp(-H)) * z), cs);
    lo = max(lo, min(k, top));
  }
}

// keep_threshold, then (CUT = 1 always, 2 when the row has a cut-off on, 0 never) cutoff_band: the kept set is lo <= key <= hi.
// CUT = 0 is keep_threshold itself with hi = ~0u.
template <int TOP_P, int CUT>
__device__ __forceinline__ uint32_t keep_band(const float* __restrict__ row, int64_t V, float inv_temp, int top_k, float top_p,
                                              const Cutoffs& cf, ThresholdSmem sm, const CutoffSmem& cs, float& mx, uint32_t& hi) {
  uint32_t lo = keep_threshold<TOP_P>(row, V, inv_temp, top_k, top_p, sm, mx);
  hi = ~0u;
  if (CUT == 1 || (CUT == 2 && cutoffs_on(cf))) cutoff_band(row, V, mx, inv_temp, cf, sm, cs, lo, hi);
  return lo;
}

// The body of sample_kernel, shared with uvx_sample_slots (TOP_P as in keep_threshold, CUT as in keep_band).  The caller's CTA
// handles one row.
template <int TOP_P, int CUT>
__device__ __forceinline__ void sample_row(const float* __restrict__ row, int64_t V, float inv_temp, int top_k, float top_p,
                                           const Cutoffs& cf, const float* __restrict__ u_all, const int32_t* __restrict__ step_idx,
                                           int64_t u_stride, int64_t col, int64_t* __restrict__ out_ptr) {
  __shared__ float red[32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ float chunk_base[32];
  __shared__ int win_thread;
  __shared__ unsigned long long mhist[256];
  __shared__ unsigned long long p_below, p_target;
  __shared__ uint32_t p_prefix;
  CutoffSmem cs{};
  if constexpr (CUT != 0) {
    __shared__ double dred[32];
    __shared__ unsigned long long zsum;
    __shared__ uint32_t klo, khi;
    cs = {dred, &zsum, &klo, &khi};
  }
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  float mx;
  uint32_t thr_hi;
  const uint32_t thr_key = keep_band<TOP_P, CUT>(row, V, inv_temp, top_k, top_p, cf,
                                                 {red, hist, &sel_prefix, &sel_remaining, mhist, &p_below, &p_target, &p_prefix}, cs,
                                                 mx, thr_hi);
  // ---- chunk sums
  const int64_t c = (V + 1023) / 1024;
  const int64_t lo = (int64_t)tid * c, hi = lo + c < V ? lo + c : V;
  float local = 0.f;
  for (int64_t i = lo; i < hi; ++i) {
    const float x = row[i];
    const uint32_t k = f2key(x);
    if (k >= thr_key && k <= thr_hi) local += __expf((x - mx) * inv_temp);
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
    // The walk re-adds the chunk's masses onto excl, which rounds differently from excl + local: a target in the top ulps
    // of the chunk (or past it, wt < 0) can outrun it.  The pick is then the chunk's last entry with positive mass - never a
    // kept entry of mass 0 (a -inf logit, or one __expf flushes to 0).  A row without mass (all -inf: NaN masses) gives 0.
    float acc = excl;
    int64_t pick = -1, last = -1;
    for (int64_t i = lo; i < hi; ++i) {
      const float x = row[i];
      const uint32_t k = f2key(x);
      if (k < thr_key || k > thr_hi) continue;
      const float m = __expf((x - mx) * inv_temp);
      if (m > 0.f) last = i;
      acc += m;
      if (acc > target) { pick = i; break; }
    }
    if (pick < 0) pick = last >= 0 ? last : 0;
    *out_ptr = pick;
  }
}

// (1024, 1): lets ptxas use the 64 registers a lone 1024-thread CTA may have (the top-p form uses 56).  CUT: uvx_sample_cutoffs
// (cf read only then; appended last so the other forms keep their parameter layout).
template <bool TOP_P, bool CUT>
__global__ void __launch_bounds__(1024, 1) sample_kernel(const float* __restrict__ logits, int64_t V, float inv_temp, int top_k,
                                                     float top_p, const float* __restrict__ u_all,
                                                     const int32_t* __restrict__ step_idx, int64_t u_stride,
                                                     int64_t* __restrict__ out, Cutoffs cf) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  sample_row<TOP_P ? 1 : 0, CUT ? 1 : 0>(logits + b * V, V, inv_temp, top_k, top_p, cf, u_all, step_idx, u_stride, b, out + b);
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
// Row-mapped form (row_slot != NULL, uvx_sample_rows): row b takes slot s = row_slot[b]'s settings and the uniform
// u[s * u_stride + row_idx[b]]; rows with row_idx[b] < 0 are left alone.
// CUT (uvx_sample_slots_cutoffs / uvx_sample_rows_cutoffs): slot s's cut-offs are cut[4 s .. 4 s + 4) = (min_p, typical_p,
// epsilon, eta); a row whose cut-offs are all off takes the path of CUT = false.
template <bool CUT>
__global__ void __launch_bounds__(1024, 1) sample_slots_kernel(const float* logits, int64_t V, const float* temperature,
                                                               const int32_t* top_k, const float* top_p, const float* u,
                                                               int64_t u_stride, const int32_t* n_new, const int32_t* active,
                                                               int64_t* out, const int32_t* row_slot, const int32_t* row_idx,
                                                               const float* cut) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  const int64_t s = row_slot ? row_slot[b] : b;
  const int32_t* step = row_slot ? row_idx + b : n_new + s;
  if (!active[s] || *step < 0) return;
  const float t = temperature[s];
  const float* row = logits + b * V;
  if (!(t > 0.f)) {
    argmax_row(row, V, out + b);
    return;
  }
  Cutoffs cf{0.f, 1.f, 0.f, 0.f};
  if (CUT) cf = {cut[4 * s], cut[4 * s + 1], cut[4 * s + 2], cut[4 * s + 3]};
  sample_row<2, CUT ? 2 : 0>(row, V, __frcp_rn(t), top_k[s], top_p[s], cf, u + s * u_stride, step, 1, 0, out + b);
}

// uvx_repetition_penalty's rule on one row (the caller's CTA) with penalty pen over sq[0:n], staging the original scores in
// sc[0:n].  The body of rep_penalty_slots_kernel and rep_penalty_rows_kernel.
__device__ __forceinline__ void penalty_row(float* row, int64_t V, const int64_t* sq, float* __restrict__ sc, int n, float pen) {
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

// One CTA per row: uvx_repetition_penalty's rule with the row's own penalty over seq[b, 0:cur_len[b]]; inactive rows and
// penalty 1 are skipped.
// Row-mapped form (row_slot != NULL, uvx_repetition_penalty_rows_map): row b takes slot s = row_slot[b]'s penalty over
// seq[s, 0:row_len[b]] with its own scratch row b; rows with row_idx[b] < 0 are skipped.
__global__ void __launch_bounds__(1024) rep_penalty_slots_kernel(float* logits, int64_t V, const int64_t* seq, int64_t seq_stride,
                                                                 const int32_t* cur_len, const float* penalty, const int32_t* active,
                                                                 float* __restrict__ scratch, const int32_t* row_slot,
                                                                 const int32_t* row_len, const int32_t* row_idx) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  const int64_t s = row_slot ? row_slot[b] : b;
  if (!active[s] || (row_slot && row_idx[b] < 0)) return;
  const float pen = penalty[s];
  if (pen == 1.f) return;
  penalty_row(logits + b * V, V, seq + s * seq_stride, scratch + b * seq_stride, row_slot ? row_len[b] : cur_len[s], pen);
}

// One CTA per row: the penalty over seq[b * seq_stride, 0:len[b]] with per-row scratch, so rows may share one sequence
// (seq_stride 0: prompt lookup checks k + 1 positions of one sequence, row i over its first len[i] tokens).
__global__ void __launch_bounds__(1024) rep_penalty_rows_kernel(float* logits, int64_t V, const int64_t* seq, int64_t seq_stride,
                                                                const int32_t* len, float penalty, float* __restrict__ scratch,
                                                                int64_t scratch_stride) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  penalty_row(logits + b * V, V, seq + b * seq_stride, scratch + b * scratch_stride, len[b], penalty);
}

// Token constraints of one row (the caller's CTA) with sequence sq[0:L] and one setting: cfg = (no_repeat_ngram_size n, min
// length, begin length, entry count) and the packed table (include/uvx.h: entry j is ids[end[j - 1] .. end[j]), its last id the
// target token; a token's entries are consecutive, in HF's order).  Phase 1: one thread per token group adds its matching
// sequence-bias entries (one fp32 sum), then its matching bad-word entries (a second sum), then applies the sets.  Phase 2 (after
// a barrier, so no logit is written by both phases at once): the n-gram bans, threads striding over the end positions e.
__device__ __forceinline__ void constrain_row(float* row, int64_t V, const int64_t* sq, int L, const int32_t* cfg,
                                              const int64_t* ids, const int32_t* end, const float* bias, const int32_t* kind) {
  const int n = cfg[0], min_len = cfg[1], begin_len = cfg[2], n_ent = cfg[3];
  for (int e = threadIdx.x; e < n_ent; e += blockDim.x) {
    const int64_t t = ids[end[e] - 1];
    if ((e > 0 && ids[end[e - 1] - 1] == t) || t < 0 || t >= V) continue;     // not its group's head
    float sb = 0.f, bw = 0.f;
    bool has_sb = false, has_bw = false, set = false;
    for (int j = e; j < n_ent; ++j) {
      const int lo = j ? end[j - 1] : 0, hi = end[j];
      if (ids[hi - 1] != t) break;
      const int k = kind[j], len = hi - lo;
      has_sb |= k == UVX_CK_BIAS;
      has_bw |= k == UVX_CK_BAD;
      if (len > L) continue;                  // longer than the sequence: skipped, as HF does
      bool match = true;
      for (int i = len - 2; i >= 0 && match; --i) match = sq[L - len + 1 + i] == ids[lo + i];
      if (!match) continue;
      if (k == UVX_CK_BIAS) sb += bias[j];
      else if (k == UVX_CK_BAD) bw += bias[j];
      else set |= k == UVX_CK_SUPPRESS || (k == UVX_CK_BEGIN && L == begin_len) || (k == UVX_CK_MIN_LEN && L < min_len);
    }
    float x = row[t];
    if (has_sb) x = x + sb;
    if (has_bw) x = x + bw;
    row[t] = set ? -INFINITY : x;
  }
  if (n < 1 || L + 1 < n) return;             // HF bans nothing while cur_len + 1 < n
  __syncthreads();
  for (int e = n - 1 + threadIdx.x; e < L; e += blockDim.x) {
    bool match = true;
    for (int i = 1; i < n && match; ++i) match = sq[e - i] == sq[L - i];
    const int64_t t = sq[e];
    if (match && t >= 0 && t < V) row[t] = -INFINITY;
  }
}

// One CTA per row b.  Slot s = row_slot ? row_slot[b] : b reads seq + s * seq_stride; its length is len[b * len_stride]; setting
// c = per_slot ? s : 0 (cfg + 4 c, the table at c * tab_stride).  Rows of an inactive slot (active given) or with row_idx[b] < 0
// (row_idx given) are skipped.  uvx_logits_constraints / _slots / _rows / _rows_map are the four argument patterns.
__global__ void __launch_bounds__(1024) logits_constraints_kernel(float* logits, int64_t V, const int64_t* seq, int64_t seq_stride,
                                                                  const int32_t* len, int64_t len_stride, const int32_t* active,
                                                                  const int32_t* row_slot, const int32_t* row_idx, const int32_t* cfg,
                                                                  int per_slot, const int64_t* ids, const int32_t* end,
                                                                  const float* bias, const int32_t* kind, int64_t tab_stride) {
  pdl_trigger();
  pdl_wait();
  const int64_t b = blockIdx.x;
  const int64_t s = row_slot ? row_slot[b] : b;
  if ((active && !active[s]) || (row_idx && row_idx[b] < 0)) return;
  const int64_t c = per_slot ? s : 0;
  const int64_t o = c * tab_stride;
  constrain_row(logits + b * V, V, seq + s * seq_stride, len[b * len_stride], cfg + 4 * c, ids + o, end + o, bias + o, kind + o);
}

// ---------------------------------------------------------------------------------------------------------------------------
// Stop strings (hf:generation/stopping_criteria.py StopStringCriteria).  The packed table (include/uvx.h): header n_ent,
// n_stop, mvp, mvel, W_max, then the n_stop target lengths, the n_ent sorted token ids and their HF rows of
// rw = n_stop * (mvp + mvel) + 1 int32 (positions of string s at s * mvp, end overlaps at n_stop * mvp + s * mvel, length last).
constexpr int kStopHdr = 5;

// Index of token t among the sorted ids[0:n], -1 when absent (ids outside the table have no entries, as HF's clamped row).
__device__ __forceinline__ int stop_find(const int32_t* ids, int n, int64_t t) {
  if (t < 0 || t > INT32_MAX) return -1;
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < t) lo = mid + 1;
    else hi = mid;
  }
  return lo < n && ids[lo] == t ? lo : -1;
}

// One warp per row r.  Slot s = row_slot ? row_slot[r] : r; the row's candidate is tok[r], preceded by
// seq[s * seq_stride, 0:L), L = len[r * len_stride]; the table is tab + (per_slot ? s * tab_stride : 0).  Beam form (beam_V > 0):
// row r is candidate r % K of prompt r / K, tok[r] = parent beam * beam_V + token, s = (r / K) * nb + tok[r] / beam_V and the
// candidate token tok[r] % beam_V.  Rows of an inactive
// slot (active given) or with row_idx[r] < 0 (row_idx given) are not written.  Lane c walks chain c = (string c / mvel, end
// overlap slot c % mvel) of the candidate, 32 chains per round; the window tokens x[L - j], j = 1 .. W - 1 (W = min(W_max,
// L + 1)), are looked up 32 at a time by the 32 lanes into shared memory, so seq is read only inside [L - W + 1, L).
__global__ void __launch_bounds__(32) stop_strings_kernel(const int64_t* tok, const int64_t* seq, int64_t seq_stride,
                                                          const int32_t* len, int64_t len_stride, const int32_t* active,
                                                          const int32_t* row_slot, const int32_t* row_idx, const int32_t* tab,
                                                          int64_t tab_stride, int per_slot, int32_t* hit, int64_t beam_V, int nb,
                                                          int K) {
  pdl_trigger();
  pdl_wait();
  __shared__ int win[32];
  const int lane = threadIdx.x;
  const int64_t r = blockIdx.x;
  int64_t t0 = tok[r];
  int64_t s = row_slot ? row_slot[r] : r;
  if (beam_V > 0) {
    s = (r / K) * nb + t0 / beam_V;
    t0 %= beam_V;
  }
  if ((active && !active[s]) || (row_idx && row_idx[r] < 0)) return;
  const int32_t* T = tab + (per_slot ? s * tab_stride : 0);
  const int n_ent = T[0], n_stop = T[1], mvp = T[2], mvel = T[3], wmax = T[4];
  const int32_t* tgt = T + kStopHdr;
  const int32_t* ids = tgt + n_stop;
  const int32_t* rows = ids + n_ent;
  const int rw = n_stop * (mvp + mvel) + 1;
  const int64_t* sq = seq + s * seq_stride;
  const int L = len[r * len_stride];
  const int W = min(wmax, L + 1);
  const int first = n_ent > 0 ? stop_find(ids, n_ent, t0) : -1;
  int found = 0;
  if (first >= 0) {
    const int n_chain = n_stop * mvel;
    for (int c0 = 0; c0 < n_chain && !found; c0 += 32) {
      const int c = c0 + lane;
      int st = -1, cv = 0;  // the chain's string (-1: dead) and the characters matched so far
      if (c < n_chain) {
        cv = rows[(int64_t)first * rw + n_stop * mvp + c];
        st = cv > 0 ? c / mvel : -1;
        found = st >= 0 && cv >= tgt[st];
      }
      for (int j0 = 1; j0 < W; j0 += 32) {
        if (__any_sync(0xffffffffu, found) || !__any_sync(0xffffffffu, st >= 0)) break;
        const int j = j0 + lane;
        win[lane] = j < W ? stop_find(ids, n_ent, sq[L - j]) : -1;
        __syncwarp();
        const int jn = min(32, W - j0);
        for (int q = 0; q < jn && st >= 0 && !found; ++q) {
          const int y = win[q];
          bool ok = false;
          if (y >= 0) {
            const int32_t* yr = rows + (int64_t)y * rw + st * mvp;
            for (int p = 0; p < mvp; ++p) ok |= yr[p] == cv;
          }
          if (!ok) {
            st = -1;
            break;
          }
          cv += rows[(int64_t)y * rw + rw - 1];
          found = cv >= tgt[st];
        }
        __syncwarp();
      }
      found = __any_sync(0xffffffffu, found);
    }
  }
  if (lane == 0) hit[r] = found;
}

// One CTA: for each active, unfinished row append tok at seq[b, cur_len[b]], advance cur_len / n_new, finish on an EOS id or
// at the budget (kStop: or on hit[b]), and advance pos / lens / rope_pos only while the row stays open.  n_open[0] = active rows
// still open.
template <bool kStop>
__global__ void slot_finish_kernel(const int64_t* tok, int32_t* done, const int64_t* __restrict__ eos, int n_eos, int64_t* seq,
                                   int64_t seq_stride, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                                   int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* n_open, int64_t B, const int32_t* hit) {
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
    if (kStop) d |= hit[b] != 0;
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
// is an EOS become finished, every counter in `bump` advances by one, all_done[0] = (every row finished).  kStop: an open row
// with hit[b] finishes too (its token kept), and a row that finishes in this step gets fin_len[b] = cur_len + 1.
template <bool kStop>
__global__ void token_finish_kernel(int64_t* __restrict__ tok, int32_t* __restrict__ done, const int64_t* __restrict__ eos,
                                    int n_eos, int64_t pad_id, int64_t* __restrict__ seq, int64_t seq_stride,
                                    int32_t* __restrict__ cur_len, int32_t* __restrict__ step_idx, int32_t* __restrict__ bump0,
                                    int32_t* __restrict__ bump1, int32_t* __restrict__ bump2, int32_t* __restrict__ all_done,
                                    int64_t B, const int32_t* hit, int32_t* fin_len) {
  pdl_trigger();
  pdl_wait();
  __shared__ int any_open;
  if (threadIdx.x == 0) any_open = 0;
  __syncthreads();
  const int n = *cur_len;
  for (int64_t b = threadIdx.x; b < B; b += blockDim.x) {
    int64_t t = tok[b];
    int d = done[b];
    const int was = d;
    if (d) t = pad_id;
    tok[b] = t;
    if (seq) seq[b * seq_stride + n] = t;
    for (int e = 0; e < n_eos; ++e) d |= (t == eos[e]);
    if (kStop) {
      if (!was) d |= hit[b] != 0;
      if (d && !was) fin_len[b] = n + 1;
    }
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
// Log-probabilities of the decode step, recorded on the device at an index the step state holds, so the step stays one graph.
constexpr int kLogprobsMax = 20;  // alternatives per token (OpenAI-style top_logprobs <= 20)

// One CTA (1024 threads) per row, skipped when n_top[b] < 0: lse = m + log(sum exp(x - m)) of the raw row, the chosen token's
// x[tok] - lse, and (n_top[b] > 0) the n_top[b] largest entries by (value desc, index asc) with their x - lse, written at
// index dst[b] of the row's [cap] (or [cap, n_max]) outputs.  The radix select of the sampler finds the n-th largest key; the
// keys above it (fewer than n) are gathered in any order, the missing ones are taken from the keys equal to it in index order
// (thread t owns the chunk [t*c, (t+1)*c), an exclusive scan of the per-chunk counts ranks them), and the n are sorted by
// rank, as in beam_row_topk_kernel.  Every reduction has a fixed order, so a row's bits depend on its logits alone.
// Row-mapped form (row_slot != NULL, uvx_token_logprobs_rows): row b takes slot s = row_slot[b]'s n_top[s] and writes slot s's
// outputs at index dst[b].
__global__ void __launch_bounds__(1024, 1) token_logprobs_kernel(const float* logits, int64_t V, const int64_t* tok,
                                                                 const int32_t* n_top, const int32_t* dst, int64_t cap, int n_max,
                                                                 float* __restrict__ out_lp, int64_t* __restrict__ out_ids,
                                                                 float* __restrict__ out_top, const int32_t* row_slot) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ int n_gt;
  __shared__ int scan[32];
  __shared__ float s_val[kLogprobsMax];
  __shared__ int64_t s_idx[kLogprobsMax];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int64_t b = blockIdx.x;
  const int64_t so = row_slot ? row_slot[b] : b;  // the output row
  const int want = n_top[so];
  const int64_t d = dst[b];
  if (want < 0 || d < 0 || d >= cap) return;
  const float* row = logits + b * V;
  float mx = -INFINITY;
  for (int64_t i = tid; i < V; i += 1024) mx = fmaxf(mx, row[i]);
  mx = warp_max(mx);
  if (lane == 0) red[w] = mx;
  __syncthreads();
  mx = warp_max(red[lane]);
  __syncthreads();
  float s = 0.f;
  for (int64_t i = tid; i < V; i += 1024) s += expf(row[i] - mx);
  s = warp_sum(s);
  if (lane == 0) red[w] = s;
  __syncthreads();
  const float lse = mx + logf(warp_sum(red[lane]));
  if (tid == 0) {
    const int64_t t = tok[b];
    out_lp[so * cap + d] = (t >= 0 && t < V) ? row[t] - lse : NAN;
  }
  int64_t kk = want < n_max ? want : n_max;
  kk = kk < V ? kk : V;
  const int K = (int)kk;
  if (K == 0) return;
  radix_select_kth(row, V, (uint32_t)K, hist, sel_prefix, sel_remaining);
  const uint32_t thr = sel_prefix;
  const int need_eq = (int)sel_remaining;  // keys equal to thr to take; K - need_eq keys lie above it
  if (tid == 0) n_gt = 0;
  __syncthreads();
  for (int64_t i = tid; i < V; i += 1024) {
    const float x = row[i];
    if (f2key(x) > thr) {
      const int j = atomicAdd(&n_gt, 1);
      s_val[j] = x;
      s_idx[j] = i;
    }
  }
  const int64_t c = (V + 1023) / 1024;
  const int64_t lo = (int64_t)tid * c, hi = lo + c < V ? lo + c : V;
  int cnt = 0;
  for (int64_t i = lo; i < hi; ++i) cnt += f2key(row[i]) == thr;
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
    int sc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, sc, o);
      if (lane >= o) sc += t;
    }
    scan[lane] = sc - v;
  }
  __syncthreads();
  int rank = scan[w] + incl - cnt;
  const int base = K - need_eq;
  for (int64_t i = lo; i < hi && rank < need_eq; ++i) {
    const float x = row[i];
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
    const int64_t o = (so * cap + d) * n_max + pos;
    out_ids[o] = ix;
    out_top[o] = x - lse;
  }
}

// One CTA (1024 threads) per row, at step s = step_idx[0] (nothing when s is outside [0, steps)): raw[s, b] = the row as given;
// scores[s, b] = the row after HF's warpers - a copy when temperature <= 0 (greedy: no warper), else x / temperature (IEEE
// division, TemperatureLogitsWarper) on the entries keep_threshold keeps (TopKLogitsWarper, TopPLogitsWarper) and -inf on the
// rest.  Either output may be NULL.
// kRows (uvx_record_scores_rows): per-row destinations instead, row b at index s = step_idx[b] of [steps, V] buffers.
// CUT (the _cutoffs forms): the band of keep_band<2, 1> with cf instead (MinP / Typical / Epsilon / EtaLogitsWarper after TopP).
template <bool kRows, bool CUT>
__global__ void __launch_bounds__(1024, 1) record_scores_kernel(const float* logits, int64_t V, float temperature, float inv_temp,
                                                                int top_k, float top_p, const int32_t* step_idx, int64_t steps,
                                                                int64_t B, float* __restrict__ scores, float* __restrict__ raw,
                                                                Cutoffs cf) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  __shared__ uint32_t hist[256];
  __shared__ uint32_t sel_prefix, sel_remaining;
  __shared__ unsigned long long mhist[256];
  __shared__ unsigned long long p_below, p_target;
  __shared__ uint32_t p_prefix;
  const int64_t b = blockIdx.x;
  const int64_t step = kRows ? step_idx[b] : *step_idx;
  if (step < 0 || step >= steps) return;
  const float* row = logits + b * V;
  const int64_t o = kRows ? step * V : (step * B + b) * V;
  if (raw)
    for (int64_t i = threadIdx.x; i < V; i += 1024) raw[o + i] = row[i];
  if (!scores) return;
  if (!(temperature > 0.f)) {
    for (int64_t i = threadIdx.x; i < V; i += 1024) scores[o + i] = row[i];
    return;
  }
  CutoffSmem cs{};
  if constexpr (CUT) {
    __shared__ double dred[32];
    __shared__ unsigned long long zsum;
    __shared__ uint32_t klo, khi;
    cs = {dred, &zsum, &klo, &khi};
  }
  float mx;
  uint32_t hi;
  const uint32_t thr = keep_band<2, CUT ? 1 : 0>(row, V, inv_temp, top_k, top_p, cf,
                                                 {red, hist, &sel_prefix, &sel_remaining, mhist, &p_below, &p_target, &p_prefix}, cs,
                                                 mx, hi);
  for (int64_t i = threadIdx.x; i < V; i += 1024) {
    const float x = row[i];
    const uint32_t k = f2key(x);
    scores[o + i] = k >= thr && k <= hi ? x / temperature : -INFINITY;
  }
}

// ---------------------------------------------------------------------------------------------------------------------------
// Prompt lookup (hf:generation/candidate_generator.py PromptLookupCandidateGenerator, transformers 5.5): one decode step checks
// k drafted positions of one sequence besides the fed token.  The sequence seq[0:cur_len] is the prompt plus the tokens
// generated so far; its last token has not been fed yet.
constexpr int kLookupMaxK = 31;  // drafts per step: k + 1 rows within the decode-form GEMM's 32

// The search and the cut, shared by lookup_draft_kernel and lookup_draft_slots_kernel (the rule is stated above
// lookup_draft_kernel): the whole CTA (1024 threads) searches seq[0:L] when `search`; returns true in warp 0 only, with d = the
// draft count (<= min(k, room)) and, in lanes < d, t = draft lane.  Needs room > 0 and min(n, L - 1) > 0 when searching.
__device__ __forceinline__ bool lookup_find(const int64_t* seq, int L, int k, int n, int room, bool search,
                                            const int64_t* __restrict__ eos, int n_eos, int* red, int& d, int64_t& t) {
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const int nmax = min(n, L - 1);
  const int64_t* tail = seq + L - 1;  // tail[-j] is the j-th token from the end
  int best = 0;
  if (search) {
    for (int e = tid + 1; e < L; e += 1024) {
      const int cap = min(nmax, e);
      int j = 0;
      while (j < cap && seq[e - 1 - j] == tail[-j]) ++j;
      best = max(best, j);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) best = max(best, __shfl_xor_sync(0xffffffffu, best, o));
  if (lane == 0) red[w] = best;
  __syncthreads();
  int g = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) g = max(g, __shfl_xor_sync(0xffffffffu, g, o));
  __syncthreads();
  int first = INT_MAX;
  if (g > 0) {
    for (int e = tid + g; e < L; e += 1024) {
      int j = 0;
      while (j < g && seq[e - 1 - j] == tail[-j]) ++j;
      if (j == g) { first = e; break; }
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  if (lane == 0) red[w] = first;
  __syncthreads();
  if (w != 0) return false;
  first = red[lane];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) first = min(first, __shfl_xor_sync(0xffffffffu, first, o));
  d = 0;
  if (g > 0) d = min(min(k, L - first), room);
  t = 0;
  bool stop = false;
  if (lane < d) {
    t = seq[first + lane];
    for (int i = 0; i < n_eos; ++i) stop |= t == eos[i];
  }
  const unsigned hit = __ballot_sync(0xffffffffu, stop);
  if (hit) d = __ffs(hit) - 1;  // drafts end before the first EOS; an EOS first means no drafts (HF looks no further)
  return true;
}

// One CTA (1024 threads).  For every continuation start e in [1, L) (L = cur_len), m(e) = the number of tokens, at most
// min(n, L - 1), that agree going back from e - 1 and from L - 1.  HF tries n-gram sizes from min(n, L - 1) down and takes
// the leftmost earlier occurrence with a non-empty continuation, so the winner is the largest size g with a match (the block
// maximum of m) at the smallest e with m(e) >= g (a block minimum).  Drafts: seq[e, min(e + k, L)), cut before the first EOS
// and to the budget (n_new + d + 1 <= max_new); none when done.  Writes the k + 1 fed tokens (row 0 the last token, rows 1..d
// the drafts, later rows the last token again), d, each row's cache position / key count / RoPE position (L - 1 + i, L + i,
// L - 1 + i), penalty length L + i and record index n_new + i, and the drafts into seq[L, L + d).
__global__ void __launch_bounds__(1024) lookup_draft_kernel(int64_t* seq, const int32_t* cur_len, const int32_t* n_new, int max_new,
                                                            int k, int n, const int64_t* __restrict__ eos, int n_eos,
                                                            const int32_t* done, int64_t* tok, int32_t* n_draft, int32_t* pos,
                                                            int32_t* lens, int32_t* rope_pos, int32_t* pen_len, int32_t* idx) {
  pdl_trigger();
  pdl_wait();
  __shared__ int red[32];
  const int lane = threadIdx.x & 31;
  const int L = *cur_len, nn = *n_new;
  const int room = max_new - nn - 1;
  const bool search = !*done && room > 0 && min(n, L - 1) > 0;
  int d;
  int64_t t;
  if (!lookup_find(seq, L, k, n, room, search, eos, n_eos, red, d, t)) return;
  if (lane < d) seq[L + lane] = t;
  const int64_t last = seq[L - 1];
  const int64_t tok_in = __shfl_up_sync(0xffffffffu, t, 1);  // lane i feeds draft i - 1
  if (lane <= k) {
    tok[lane] = (lane >= 1 && lane <= d) ? tok_in : last;
    pos[lane] = L - 1 + lane;
    lens[lane] = L + lane;
    rope_pos[lane] = L - 1 + lane;
    pen_len[lane] = L + lane;
    idx[lane] = nn + lane;
  }
  if (lane == 0) *n_draft = d;
}

// One warp: the count m of leading picks that equal the drafts; pick[0 : m + 1] are appended at seq[L] (lanes <= m), and
// whether the last of them finishes the sequence (an EOS id or the budget) is returned.  Shared by lookup_accept_kernel and
// lookup_accept_slots_kernel.  kStop: m is cut at the first row i <= m with hit[i] (a stop string ends at pick[i]), which then
// finishes the sequence.
template <bool kStop>
__device__ __forceinline__ int lookup_match(const int64_t* pick, const int64_t* tok, int d, const int64_t* __restrict__ eos, int n_eos,
                                            int64_t* seq, int L, int nn, int max_new, int& fin, const int32_t* hit) {
  const int lane = threadIdx.x & 31;
  bool miss = lane >= d || pick[lane] != tok[lane + 1];
  if (kStop) miss = miss || (lane <= d && hit[lane] != 0);
  const int m = __ffs(__ballot_sync(0xffffffffu, miss)) - 1;  // d <= 31: lane d always misses
  if (lane <= m) seq[L + lane] = pick[lane];
  const int64_t t = pick[m];
  fin = nn + m + 1 >= max_new;
  for (int i = 0; i < n_eos; ++i) fin |= t == eos[i];
  if (kStop) fin |= hit[m] != 0;
  return m;
}

// One warp.  n_matches = the leading picks that equal the drafts (pick[i] == tok[i + 1], i < d), the valid tokens are
// pick[0 : n_matches + 1] (HF _assisted_decoding): appended at seq[cur_len], cur_len and n_new advance by their count, done when
// the last is an EOS (drafts hold none, so only the last can be) or n_new reaches max_new.  accepted[step] = n_matches and step
// advances (when accepted is given).  Nothing happens once done.  kStop: lookup_match's cut at the first hit.
template <bool kStop>
__global__ void __launch_bounds__(32) lookup_accept_kernel(const int64_t* pick, const int64_t* tok, const int32_t* n_draft,
                                                           const int64_t* __restrict__ eos, int n_eos, int64_t* seq, int32_t* cur_len,
                                                           int32_t* n_new, int max_new, int32_t* step, int32_t* accepted, int steps,
                                                           int32_t* done, const int32_t* hit) {
  pdl_trigger();
  pdl_wait();
  if (*done) return;
  const int lane = threadIdx.x;
  const int L = *cur_len, nn = *n_new;
  int fin;
  const int m = lookup_match<kStop>(pick, tok, *n_draft, eos, n_eos, seq, L, nn, max_new, fin, hit);
  if (lane == 0) {
    *cur_len = L + m + 1;
    *n_new = nn + m + 1;
    *done = fin;
    if (accepted) {
      const int s = *step;
      if (s >= 0 && s < steps) accepted[s] = m;
      *step = s + 1;
    }
  }
}

// Prompt lookup inside the slot step (SlotDecodeEngine's lookup step): slot s owns rows s * (K + 1) + i, i <= K.
// One CTA (1024 threads) per slot: lookup_find over seq[s, 0:cur_len[s]] with the slot's own k[s] (<= K), n[s] and budget,
// when the slot is active, not done, not prefilling and k[s] > 0.  Row 0 feeds token[s] at the slot's pos / lens / rope_pos
// (what a plain step feeds), draft row i <= d feeds draft i - 1 at pos + i, lens + i, rope_pos + i; rows past the drafts feed
// token[s] with row 0's positions.  pen_len = cur_len + i and idx = n_new + i for row 0 and the drafts, idx = -1 past them;
// row_slot = s; cache_row = s for row 0 (-1 when the slot is done or prefilling) and the drafts, -1 past them.
__global__ void __launch_bounds__(1024) lookup_draft_slots_kernel(int64_t* seq, int64_t seq_stride, const int64_t* token,
                                                                  const int32_t* cur_len, const int32_t* n_new,
                                                                  const int32_t* max_new, const int32_t* k_slot, const int32_t* n_slot,
                                                                  const int32_t* done, const int32_t* active, const int32_t* prefilling,
                                                                  const int32_t* pos, const int32_t* lens, const int32_t* rope_pos,
                                                                  int K, const int64_t* __restrict__ eos, int n_eos, int64_t* tok,
                                                                  int32_t* n_draft, int32_t* row_pos, int32_t* row_lens,
                                                                  int32_t* row_rope, int32_t* pen_len, int32_t* idx,
                                                                  int32_t* row_slot, int32_t* cache_row) {
  pdl_trigger();
  pdl_wait();
  __shared__ int red[32];
  const int lane = threadIdx.x & 31;
  const int s = blockIdx.x;
  int64_t* sq = seq + (int64_t)s * seq_stride;
  const bool open = active[s] && !done[s] && !prefilling[s];
  const int L = cur_len[s], nn = n_new[s], ks = min(k_slot[s], K), ns = n_slot[s];
  const int room = max_new[s] - nn - 1;
  const bool search = open && ks > 0 && ns > 0 && room > 0 && min(ns, L - 1) > 0;
  int d;
  int64_t t;
  if (!lookup_find(sq, L, ks, ns, room, search, eos, n_eos, red, d, t)) return;
  if (lane < d) sq[L + lane] = t;
  const int64_t tok_in = __shfl_up_sync(0xffffffffu, t, 1);  // lane i feeds draft i - 1
  if (lane <= K) {
    const int r = s * (K + 1) + lane;
    const bool real = lane <= d;
    const int i = real ? lane : 0;
    tok[r] = (lane >= 1 && lane <= d) ? tok_in : token[s];
    row_pos[r] = pos[s] + i;
    row_lens[r] = lens[s] + i;
    row_rope[r] = rope_pos[s] + i;
    pen_len[r] = L + i;
    idx[r] = real ? nn + lane : -1;
    row_slot[r] = s;
    cache_row[r] = real && (lane > 0 || (!done[s] && !prefilling[s])) ? s : -1;
  }
  if (lane == 0) n_draft[s] = d;
}

// Warp w of one CTA takes slots w, w + warps, ...: for each active slot that is not done, lookup_match over its rows, then
// uvx_slot_finish's bookkeeping for the m + 1 tokens - cur_len / n_new += m + 1, done = the last is an EOS id or the budget is
// reached, pos / lens / rope_pos += m + 1 while the slot stays open (m when it finishes: only the last token can finish it) -
// token[s] = the last pick (fed next), accepted[s] += m.  n_open[0] = active slots still open.  kStop: the slot's rows' hits
// cut m as in lookup_accept_kernel.
template <bool kStop>
__global__ void lookup_accept_slots_kernel(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, int K,
                                           const int64_t* __restrict__ eos, int n_eos, int64_t* seq, int64_t seq_stride,
                                           int64_t* token, int32_t* done, int32_t* cur_len, int32_t* n_new, const int32_t* max_new,
                                           const int32_t* active, int32_t* pos, int32_t* lens, int32_t* rope_pos,
                                           int32_t* accepted, int32_t* n_open, int slots, const int32_t* hit) {
  pdl_trigger();
  pdl_wait();
  __shared__ int open;
  if (threadIdx.x == 0) open = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, warps = blockDim.x >> 5;
  for (int s = threadIdx.x >> 5; s < slots; s += warps) {
    if (!active[s] || done[s]) continue;
    const int64_t r0 = (int64_t)s * (K + 1);
    const int L = cur_len[s], nn = n_new[s];
    int fin;
    const int m = lookup_match<kStop>(pick + r0, tok + r0, n_draft[s], eos, n_eos, seq + s * seq_stride, L, nn, max_new[s], fin,
                                      kStop ? hit + r0 : hit);
    if (lane == 0) {
      cur_len[s] = L + m + 1;
      n_new[s] = nn + m + 1;
      done[s] = fin;
      token[s] = pick[r0 + m];
      accepted[s] += m;
      const int bump = fin ? m : m + 1;
      pos[s] += bump;
      lens[s] += bump;
      rope_pos[s] += bump;
      if (!fin) atomicAdd(&open, 1);
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) *n_open = open;
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
template <bool kStop>
__global__ void __launch_bounds__(256) beam_update_kernel(
    const float* cand_s, const int64_t* cand_i, int64_t V, int nb, int K, const int64_t* __restrict__ eos,
    int n_eos, int max_new, const float* __restrict__ len_div, int early_stopping, int lp_positive, float* __restrict__ run_score,
    int64_t* __restrict__ run_seq, int64_t* __restrict__ pool_seq, int64_t seq_stride, float* __restrict__ pool_score,
    int32_t* __restrict__ pool_len, int32_t* __restrict__ pool_fin, int32_t* __restrict__ parent, int64_t* __restrict__ tok,
    int32_t* __restrict__ heur, int32_t* __restrict__ flags, uint32_t* __restrict__ ticket, int32_t* __restrict__ cur_len,
    int32_t* __restrict__ step_idx, int32_t* __restrict__ bump0, int32_t* __restrict__ bump1, int32_t* __restrict__ bump2,
    int32_t* __restrict__ done, int64_t B, const int32_t* stop_hit) {
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
    if (kStop) hit |= stop_hit[b * K + tid] != 0;  // StopStringCriteria on the candidate's sequence
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

// 16-byte vectors of positions [p0, p1) of every layer, K and V: row cache [L][S_max][row_elems] <-> pool [L][n_pages][64][row_elems].
// kFp8: the pool is e4m3 and a vector is 16 elements (16 pool bytes, 32 row bytes), quantized into the pool / dequantized out of it
// with layer l's scales kv_scales[2 l] (K), kv_scales[2 l + 1] (V); the strides are then counted in 16-element vectors.
template <bool kFp8>
__global__ void __launch_bounds__(256) kv_pages_copy_kernel(uint4* __restrict__ k_row, uint4* __restrict__ v_row, int64_t row_layer_vec,
                                                            uint4* __restrict__ k_pool, uint4* __restrict__ v_pool,
                                                            int64_t pool_layer_vec, int64_t L, int64_t vec,
                                                            const int32_t* __restrict__ pages, int64_t p0, int64_t n, int to_pages,
                                                            const float* __restrict__ kv_scales) {
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
    if constexpr (kFp8) {
      const float s = kv_scales[2 * l + which];
      if (to_pages) {
        float f[16];
        unpack8(*reinterpret_cast<const bf16x8*>(row + 2 * ri), f);
        unpack8(*reinterpret_cast<const bf16x8*>(row + 2 * ri + 1), f + 8);
        const uint2 a = e4m3x8_quant(f, s), b = e4m3x8_quant(f + 8, s);
        pool[pi] = make_uint4(a.x, a.y, b.x, b.y);
      } else {
        e4m3x16_dequant(pool[pi], s, row[2 * ri], row[2 * ri + 1]);
      }
    } else {
      if (to_pages)
        pool[pi] = row[ri];
      else
        row[ri] = pool[pi];
    }
  }
}

// Whole pages between two pools [L][pages][page_vec] of 16-byte vectors, every layer, K and V: page src_pages[j] of the source
// -> page dst_pages[j] of the destination for j < n, raw bytes.  Either pool may be mapped pinned host memory (read / written over
// PCIe through its UVA address); the page lists are on the device.
__global__ void __launch_bounds__(256) kv_pages_move_kernel(const uint4* __restrict__ src_k, const uint4* __restrict__ src_v,
                                                            int64_t src_layer_vec, uint4* __restrict__ dst_k, uint4* __restrict__ dst_v,
                                                            int64_t dst_layer_vec, int64_t L, int64_t page_vec,
                                                            const int32_t* __restrict__ src_pages, const int32_t* __restrict__ dst_pages,
                                                            int64_t n) {
  pdl_trigger();
  pdl_wait();
  const int64_t per_layer = n * page_vec;
  const int64_t total = 2 * L * per_layer;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int which = (int)(i / (L * per_layer));
    const int64_t rem = i % (L * per_layer);
    const int64_t l = rem / per_layer, e = rem % per_layer;
    const int64_t j = e / page_vec, c = e % page_vec;
    const uint4* src = which ? src_v : src_k;
    uint4* dst = which ? dst_v : dst_k;
    dst[l * dst_layer_vec + (int64_t)dst_pages[j] * page_vec + c] = src[l * src_layer_vec + (int64_t)src_pages[j] * page_vec + c];
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
  launch_k(sample_kernel<false, false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature,
           (int)top_k, 1.0f, u, step_idx, u_stride, out_idx, Cutoffs{0.f, 1.f, 0.f, 0.f});
  return check_launch("sample_kernel");
}

extern "C" int uvx_sample_top_p(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                const float* u, const int32_t* step_idx, int64_t u_stride, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && u && out_idx && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && temperature > 0.f && top_p >= 0.f &&
                  top_p <= 1.f,
              "uvx_sample_top_p: bad arguments");
  if (top_p >= 1.f) return uvx_sample(logits, B, V, temperature, top_k, u, step_idx, u_stride, out_idx, stream);
  launch_k(sample_kernel<true, false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature,
           (int)top_k, top_p, u, step_idx, u_stride, out_idx, Cutoffs{0.f, 1.f, 0.f, 0.f});
  return check_launch("sample_kernel_top_p");
}

namespace uvx {
// The host's encoding of the four cut-offs (include/uvx.h uvx_cutoffs): min_p in [0, 1], typical_p in (0, 1] (>= 1 off),
// epsilon / eta in [0, 1) (0 off; HF also gates values outside (0, 1) off).  NaN fails every check.
static bool cutoffs_valid(const uvx_cutoffs& c) {
  return c.min_p >= 0.f && c.min_p <= 1.f && c.typical_p > 0.f && c.epsilon >= 0.f && c.epsilon < 1.f && c.eta >= 0.f &&
         c.eta < 1.f;
}
static Cutoffs cutoffs_of(const uvx_cutoffs& c) { return {c.min_p, c.typical_p < 1.f ? c.typical_p : 1.f, c.epsilon, c.eta}; }
static bool cutoffs_on_host(const uvx_cutoffs& c) { return c.min_p > 0.f || c.typical_p < 1.f || c.epsilon > 0.f || c.eta > 0.f; }
}  // namespace uvx

extern "C" int uvx_sample_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                  uvx_cutoffs cutoffs, const float* u, const int32_t* step_idx, int64_t u_stride, int64_t* out_idx,
                                  uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && u && out_idx && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && temperature > 0.f && top_p >= 0.f &&
                  top_p <= 1.f && cutoffs_valid(cutoffs),
              "uvx_sample_cutoffs: bad arguments");
  if (!cutoffs_on_host(cutoffs))
    return uvx_sample_top_p(logits, B, V, temperature, top_k, top_p, u, step_idx, u_stride, out_idx, stream);
  if (top_p < 1.f)
    launch_k(sample_kernel<true, true>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature,
             (int)top_k, top_p, u, step_idx, u_stride, out_idx, cutoffs_of(cutoffs));
  else
    launch_k(sample_kernel<false, true>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, 1.0f / temperature,
             (int)top_k, 1.0f, u, step_idx, u_stride, out_idx, cutoffs_of(cutoffs));
  return check_launch("sample_kernel_cutoffs");
}

extern "C" int uvx_sample_slots(const float* logits, int64_t B, int64_t V, const float* temperature, const int32_t* top_k,
                                const float* top_p, const float* u, int64_t u_stride, const int32_t* n_new, const int32_t* active,
                                int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && temperature && top_k && top_p && u && n_new && active && out_idx && B >= 1 && V >= 1 &&
                  V <= (int64_t)1 << 24 && u_stride >= 0,
              "uvx_sample_slots: bad arguments");
  launch_k(sample_slots_kernel<false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, temperature, top_k, top_p,
           u, u_stride, n_new, active, out_idx, (const int32_t*)nullptr, (const int32_t*)nullptr, (const float*)nullptr);
  return check_launch("sample_slots_kernel");
}

extern "C" int uvx_sample_slots_cutoffs(const float* logits, int64_t B, int64_t V, const float* temperature, const int32_t* top_k,
                                        const float* top_p, const float* cutoffs, const float* u, int64_t u_stride,
                                        const int32_t* n_new, const int32_t* active, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && temperature && top_k && top_p && cutoffs && u && n_new && active && out_idx && B >= 1 && V >= 1 &&
                  V <= (int64_t)1 << 24 && u_stride >= 0,
              "uvx_sample_slots_cutoffs: bad arguments");
  launch_k(sample_slots_kernel<true>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, temperature, top_k, top_p,
           u, u_stride, n_new, active, out_idx, (const int32_t*)nullptr, (const int32_t*)nullptr, cutoffs);
  return check_launch("sample_slots_kernel (cutoffs)");
}

extern "C" int uvx_repetition_penalty_slots(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                            const int32_t* cur_len, const float* penalty, const int32_t* active, float* scratch,
                                            uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && cur_len && penalty && active && scratch && B >= 1 && V >= 1,
              "uvx_repetition_penalty_slots: bad arguments");
  launch_k(rep_penalty_slots_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, cur_len,
           penalty, active, scratch, (const int32_t*)nullptr, (const int32_t*)nullptr, (const int32_t*)nullptr);
  return check_launch("rep_penalty_slots_kernel");
}

extern "C" int uvx_repetition_penalty_rows(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                           const int32_t* len, float penalty, float* scratch, int64_t scratch_stride,
                                           uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && len && scratch && B >= 1 && V >= 1 && penalty > 0.f && seq_stride >= 0 && scratch_stride >= 0 &&
                  (B == 1 || scratch_stride > 0),
              "uvx_repetition_penalty_rows: bad arguments");
  launch_k(rep_penalty_rows_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, len, penalty,
           scratch, scratch_stride);
  return check_launch("rep_penalty_rows_kernel");
}

extern "C" int uvx_lookup_draft(int64_t* seq, const int32_t* cur_len, const int32_t* n_new, int32_t max_new, int32_t k, int32_t n,
                                const int64_t* eos_ids, int32_t n_eos, const int32_t* done, int64_t* tok, int32_t* n_draft,
                                int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* pen_len, int32_t* idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(seq && cur_len && n_new && done && tok && n_draft && pos && lens && rope_pos && pen_len && idx &&
                  (n_eos == 0 || eos_ids) && n_eos >= 0 && max_new >= 1 && k >= 1 && k <= kLookupMaxK && n >= 1,
              "uvx_lookup_draft: bad arguments (1 <= k <= %d, n >= 1, max_new >= 1)", kLookupMaxK);
  launch_k(lookup_draft_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, seq, cur_len, n_new, (int)max_new, (int)k, (int)n,
           eos_ids, (int)n_eos, done, tok, n_draft, pos, lens, rope_pos, pen_len, idx);
  return check_launch("lookup_draft_kernel");
}

extern "C" int uvx_lookup_accept(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, const int64_t* eos_ids, int32_t n_eos,
                                 int64_t* seq, int32_t* cur_len, int32_t* n_new, int32_t max_new, int32_t* step, int32_t* accepted,
                                 int32_t steps, int32_t* done, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(pick && tok && n_draft && seq && cur_len && n_new && done && (n_eos == 0 || eos_ids) && n_eos >= 0 && max_new >= 1 &&
                  (!accepted || (step && steps >= 0)),
              "uvx_lookup_accept: bad arguments");
  launch_k(lookup_accept_kernel<false>, dim3(1), dim3(32), 0, (cudaStream_t)stream, pick, tok, n_draft, eos_ids, (int)n_eos, seq,
           cur_len, n_new, (int)max_new, step, accepted, (int)steps, done, (const int32_t*)nullptr);
  return check_launch("lookup_accept_kernel");
}

extern "C" int uvx_lookup_draft_slots(int64_t* seq, int64_t seq_stride, const int64_t* token, const int32_t* cur_len,
                                      const int32_t* n_new, const int32_t* max_new, const int32_t* k, const int32_t* n,
                                      const int32_t* done, const int32_t* active, const int32_t* prefilling, const int32_t* pos,
                                      const int32_t* lens, const int32_t* rope_pos, int64_t slots, int32_t K, const int64_t* eos_ids,
                                      int32_t n_eos, int64_t* tok, int32_t* n_draft, int32_t* row_pos, int32_t* row_lens,
                                      int32_t* row_rope, int32_t* pen_len, int32_t* idx, int32_t* row_slot, int32_t* cache_row,
                                      uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(seq && token && cur_len && n_new && max_new && k && n && done && active && prefilling && pos && lens && rope_pos && tok &&
                  n_draft && row_pos && row_lens && row_rope && pen_len && idx && row_slot && cache_row && (n_eos == 0 || eos_ids) &&
                  n_eos >= 0 && slots >= 1 && slots < 65536 && K >= 1 && K <= kLookupMaxK && seq_stride >= 1,
              "uvx_lookup_draft_slots: bad arguments (1 <= K <= %d)", kLookupMaxK);
  launch_k(lookup_draft_slots_kernel, dim3((unsigned)slots), dim3(1024), 0, (cudaStream_t)stream, seq, seq_stride, token, cur_len,
           n_new, max_new, k, n, done, active, prefilling, pos, lens, rope_pos, (int)K, eos_ids, (int)n_eos, tok, n_draft, row_pos,
           row_lens, row_rope, pen_len, idx, row_slot, cache_row);
  return check_launch("lookup_draft_slots_kernel");
}

extern "C" int uvx_lookup_accept_slots(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, int64_t slots, int32_t K,
                                       const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride, int64_t* token,
                                       int32_t* done, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                                       int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* accepted, int32_t* n_open,
                                       uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(pick && tok && n_draft && seq && token && done && cur_len && n_new && max_new && active && pos && lens && rope_pos &&
                  accepted && n_open && (n_eos == 0 || eos_ids) && n_eos >= 0 && slots >= 1 && slots < 65536 && K >= 1 &&
                  K <= kLookupMaxK,
              "uvx_lookup_accept_slots: bad arguments (1 <= K <= %d)", kLookupMaxK);
  const int warps = slots < 32 ? (int)slots : 32;
  launch_k(lookup_accept_slots_kernel<false>, dim3(1), dim3(32 * warps), 0, (cudaStream_t)stream, pick, tok, n_draft, (int)K,
           eos_ids, (int)n_eos, seq, seq_stride, token, done, cur_len, n_new, max_new, active, pos, lens, rope_pos, accepted, n_open,
           (int)slots, (const int32_t*)nullptr);
  return check_launch("lookup_accept_slots_kernel");
}

extern "C" int uvx_sample_rows(const float* logits, int64_t R, int64_t V, const float* temperature, const int32_t* top_k,
                               const float* top_p, const float* u, int64_t u_stride, const int32_t* active, const int32_t* row_slot,
                               const int32_t* row_idx, int64_t* out_idx, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && temperature && top_k && top_p && u && active && row_slot && row_idx && out_idx && R >= 1 && R < 65536 &&
                  V >= 1 && V <= (int64_t)1 << 24 && u_stride >= 0,
              "uvx_sample_rows: bad arguments");
  launch_k(sample_slots_kernel<false>, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, temperature, top_k, top_p,
           u, u_stride, (const int32_t*)nullptr, active, out_idx, row_slot, row_idx, (const float*)nullptr);
  return check_launch("sample_slots_kernel (rows)");
}

extern "C" int uvx_sample_rows_cutoffs(const float* logits, int64_t R, int64_t V, const float* temperature, const int32_t* top_k,
                                       const float* top_p, const float* cutoffs, const float* u, int64_t u_stride,
                                       const int32_t* active, const int32_t* row_slot, const int32_t* row_idx, int64_t* out_idx,
                                       uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && temperature && top_k && top_p && cutoffs && u && active && row_slot && row_idx && out_idx && R >= 1 &&
                  R < 65536 && V >= 1 && V <= (int64_t)1 << 24 && u_stride >= 0,
              "uvx_sample_rows_cutoffs: bad arguments");
  launch_k(sample_slots_kernel<true>, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, temperature, top_k, top_p,
           u, u_stride, (const int32_t*)nullptr, active, out_idx, row_slot, row_idx, cutoffs);
  return check_launch("sample_slots_kernel (rows, cutoffs)");
}

extern "C" int uvx_repetition_penalty_rows_map(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride,
                                               const float* penalty, const int32_t* active, const int32_t* row_slot,
                                               const int32_t* row_len, const int32_t* row_idx, float* scratch, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && penalty && active && row_slot && row_len && row_idx && scratch && R >= 1 && R < 65536 && V >= 1 &&
                  seq_stride >= 1,
              "uvx_repetition_penalty_rows_map: bad arguments");
  launch_k(rep_penalty_slots_kernel, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride,
           (const int32_t*)nullptr, penalty, active, scratch, row_slot, row_len, row_idx);
  return check_launch("rep_penalty_slots_kernel (rows)");
}

extern "C" int uvx_logits_constraints(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                      const int32_t* cur_len, const int32_t* cfg, const int64_t* ids, const int32_t* end,
                                      const float* bias, const int32_t* kind, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && cur_len && cfg && ids && end && bias && kind &&B >= 1 && B < 65536 && V >= 1 && seq_stride >= 0,
              "uvx_logits_constraints: bad arguments");
  launch_k(logits_constraints_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, cur_len,
           (int64_t)0, (const int32_t*)nullptr, (const int32_t*)nullptr, (const int32_t*)nullptr, cfg, 0, ids, end, bias, kind,
           (int64_t)0);
  return check_launch("logits_constraints_kernel");
}

extern "C" int uvx_logits_constraints_slots(float* logits, int64_t B, int64_t V, const int64_t* seq, int64_t seq_stride,
                                            const int32_t* cur_len, const int32_t* active, const int32_t* cfg, const int64_t* ids,
                                            const int32_t* end, const float* bias, const int32_t* kind, int64_t tab_stride,
                                            uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && cur_len && active && cfg && ids && end && bias && kind &&B >= 1 && B < 65536 && V >= 1 &&
                  seq_stride >= 1 && tab_stride >= 1,
              "uvx_logits_constraints_slots: bad arguments");
  launch_k(logits_constraints_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, cur_len,
           (int64_t)1, active, (const int32_t*)nullptr, (const int32_t*)nullptr, cfg, 1, ids, end, bias, kind, tab_stride);
  return check_launch("logits_constraints_kernel (slots)");
}

extern "C" int uvx_logits_constraints_rows(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride,
                                           const int32_t* len, const int32_t* cfg, const int64_t* ids, const int32_t* end,
                                           const float* bias, const int32_t* kind, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && len && cfg && ids && end && bias && kind &&R >= 1 && R < 65536 && V >= 1 && seq_stride >= 0,
              "uvx_logits_constraints_rows: bad arguments");
  launch_k(logits_constraints_kernel, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, len,
           (int64_t)1, (const int32_t*)nullptr, (const int32_t*)nullptr, (const int32_t*)nullptr, cfg, 0, ids, end, bias, kind,
           (int64_t)0);
  return check_launch("logits_constraints_kernel (rows)");
}

extern "C" int uvx_logits_constraints_rows_map(float* logits, int64_t R, int64_t V, const int64_t* seq, int64_t seq_stride,
                                               const int32_t* active, const int32_t* row_slot, const int32_t* row_len,
                                               const int32_t* row_idx, const int32_t* cfg, const int64_t* ids, const int32_t* end,
                                               const float* bias, const int32_t* kind, int64_t tab_stride, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && seq && active && row_slot && row_len && row_idx && cfg && ids && end && bias && kind &&R >= 1 && R < 65536 &&
                  V >= 1 && seq_stride >= 1 && tab_stride >= 1,
              "uvx_logits_constraints_rows_map: bad arguments");
  launch_k(logits_constraints_kernel, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, seq, seq_stride, row_len,
           (int64_t)1, active, row_slot, row_idx, cfg, 1, ids, end, bias, kind, tab_stride);
  return check_launch("logits_constraints_kernel (rows_map)");
}

extern "C" int uvx_slot_finish(const int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t* seq,
                               int64_t seq_stride, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                               int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* n_open, int64_t B, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && seq && cur_len && n_new && max_new && active && pos && lens && rope_pos && n_open && B >= 1 &&
                  n_eos >= 0 && (n_eos == 0 || eos_ids),
              "uvx_slot_finish: bad arguments");
  launch_k(slot_finish_kernel<false>, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, seq, seq_stride,
           cur_len, n_new, max_new, active, pos, lens, rope_pos, n_open, B, (const int32_t*)nullptr);
  return check_launch("slot_finish_kernel");
}

extern "C" int uvx_token_finish(int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int64_t* seq,
                                int64_t seq_stride, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1,
                                int32_t* bump2, int32_t* all_done, int64_t B, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && cur_len && B >= 1 && (n_eos == 0 || eos_ids), "uvx_token_finish: bad arguments");
  launch_k(token_finish_kernel<false>, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, pad_id, seq,
           seq_stride, cur_len, step_idx, bump0, bump1, bump2, all_done, B, (const int32_t*)nullptr, (int32_t*)nullptr);
  return check_launch("token_finish_kernel");
}

namespace uvx {
static int stop_strings_launch(const char* name, int64_t R, const int64_t* tok, const int64_t* seq, int64_t seq_stride,
                               const int32_t* len, int64_t len_stride, const int32_t* active, const int32_t* row_slot,
                               const int32_t* row_idx, const int32_t* tab, int64_t tab_stride, int per_slot, int32_t* hit,
                               uvx_stream_t stream) {
  UVX_REQUIRE(tok && seq && len && tab && hit && R >= 1 && R < 65536 && seq_stride >= 0 && tab_stride >= 0 &&
                  (!per_slot || tab_stride >= kStopHdr),
              "%s: bad arguments", name);
  launch_k(stop_strings_kernel, dim3((unsigned)R), dim3(32), 0, (cudaStream_t)stream, tok, seq, seq_stride, len, len_stride, active,
           row_slot, row_idx, tab, tab_stride, per_slot, hit, (int64_t)0, 0, 0);
  return check_launch(name);
}
}  // namespace uvx

extern "C" int uvx_stop_strings(const int64_t* tok, int64_t B, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                                const int32_t* tab, int32_t* hit, uvx_stream_t stream) {
  return uvx::stop_strings_launch("uvx_stop_strings", B, tok, seq, seq_stride, cur_len, 0, nullptr, nullptr, nullptr, tab, 0, 0,
                                  hit, stream);
}

extern "C" int uvx_stop_strings_slots(const int64_t* tok, int64_t B, const int64_t* seq, int64_t seq_stride, const int32_t* cur_len,
                                      const int32_t* active, const int32_t* tab, int64_t tab_stride, int32_t* hit, uvx_stream_t stream) {
  UVX_REQUIRE(active, "uvx_stop_strings_slots: bad arguments");
  return uvx::stop_strings_launch("uvx_stop_strings_slots", B, tok, seq, seq_stride, cur_len, 1, active, nullptr, nullptr, tab,
                                  tab_stride, 1, hit, stream);
}

extern "C" int uvx_stop_strings_rows(const int64_t* tok, int64_t R, const int64_t* seq, int64_t seq_stride, const int32_t* len,
                                     const int32_t* tab, int32_t* hit, uvx_stream_t stream) {
  return uvx::stop_strings_launch("uvx_stop_strings_rows", R, tok, seq, seq_stride, len, 1, nullptr, nullptr, nullptr, tab, 0, 0,
                                  hit, stream);
}

extern "C" int uvx_stop_strings_rows_map(const int64_t* tok, int64_t R, const int64_t* seq, int64_t seq_stride, const int32_t* active,
                                         const int32_t* row_slot, const int32_t* row_len, const int32_t* row_idx, const int32_t* tab,
                                         int64_t tab_stride, int32_t* hit, uvx_stream_t stream) {
  UVX_REQUIRE(active && row_slot && row_idx, "uvx_stop_strings_rows_map: bad arguments");
  return uvx::stop_strings_launch("uvx_stop_strings_rows_map", R, tok, seq, seq_stride, row_len, 1, active, row_slot, row_idx, tab,
                                  tab_stride, 1, hit, stream);
}

extern "C" int uvx_stop_strings_beam(const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V, const int64_t* run_seq,
                                     int64_t seq_stride, const int32_t* cur_len, const int32_t* tab, int32_t* hit,
                                     uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(cand_i && run_seq && cur_len && tab && hit && B >= 1 && nb >= 1 && nb <= kBeamMax && K >= 1 && K <= kBeamMaxK &&
                  V >= 1 && B * K < 65536 && seq_stride >= 1,
              "uvx_stop_strings_beam: bad arguments");
  launch_k(stop_strings_kernel, dim3((unsigned)(B * K)), dim3(32), 0, (cudaStream_t)stream, cand_i, run_seq, seq_stride, cur_len,
           (int64_t)0, (const int32_t*)nullptr, (const int32_t*)nullptr, (const int32_t*)nullptr, tab, (int64_t)0, 0, hit, V,
           (int)nb, (int)K);
  return check_launch("uvx_stop_strings_beam");
}

extern "C" int uvx_token_finish_stop(int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t pad_id, int64_t* seq,
                                     int64_t seq_stride, int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1,
                                     int32_t* bump2, int32_t* all_done, int64_t B, const int32_t* hit, int32_t* fin_len,
                                     uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && cur_len && hit && fin_len && B >= 1 && (n_eos == 0 || eos_ids), "uvx_token_finish_stop: bad arguments");
  launch_k(token_finish_kernel<true>, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, pad_id, seq,
           seq_stride, cur_len, step_idx, bump0, bump1, bump2, all_done, B, hit, fin_len);
  return check_launch("token_finish_kernel (stop)");
}

extern "C" int uvx_slot_finish_stop(const int64_t* tok, int32_t* done, const int64_t* eos_ids, int32_t n_eos, int64_t* seq,
                                    int64_t seq_stride, int32_t* cur_len, int32_t* n_new, const int32_t* max_new, const int32_t* active,
                                    int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* n_open, int64_t B, const int32_t* hit,
                                    uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(tok && done && seq && cur_len && n_new && max_new && active && pos && lens && rope_pos && n_open && hit && B >= 1 &&
                  n_eos >= 0 && (n_eos == 0 || eos_ids),
              "uvx_slot_finish_stop: bad arguments");
  launch_k(slot_finish_kernel<true>, dim3(1), dim3(128), 0, (cudaStream_t)stream, tok, done, eos_ids, (int)n_eos, seq, seq_stride,
           cur_len, n_new, max_new, active, pos, lens, rope_pos, n_open, B, hit);
  return check_launch("slot_finish_kernel (stop)");
}

extern "C" int uvx_lookup_accept_stop(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, const int64_t* eos_ids,
                                      int32_t n_eos, int64_t* seq, int32_t* cur_len, int32_t* n_new, int32_t max_new, int32_t* step,
                                      int32_t* accepted, int32_t steps, int32_t* done, const int32_t* hit, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(pick && tok && n_draft && seq && cur_len && n_new && done && hit && (n_eos == 0 || eos_ids) && n_eos >= 0 &&
                  max_new >= 1 && (!accepted || (step && steps >= 0)),
              "uvx_lookup_accept_stop: bad arguments");
  launch_k(lookup_accept_kernel<true>, dim3(1), dim3(32), 0, (cudaStream_t)stream, pick, tok, n_draft, eos_ids, (int)n_eos, seq,
           cur_len, n_new, (int)max_new, step, accepted, (int)steps, done, hit);
  return check_launch("lookup_accept_kernel (stop)");
}

extern "C" int uvx_lookup_accept_slots_stop(const int64_t* pick, const int64_t* tok, const int32_t* n_draft, int64_t slots, int32_t K,
                                            const int64_t* eos_ids, int32_t n_eos, int64_t* seq, int64_t seq_stride, int64_t* token,
                                            int32_t* done, int32_t* cur_len, int32_t* n_new, const int32_t* max_new,
                                            const int32_t* active, int32_t* pos, int32_t* lens, int32_t* rope_pos, int32_t* accepted,
                                            int32_t* n_open, const int32_t* hit, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(pick && tok && n_draft && seq && token && done && cur_len && n_new && max_new && active && pos && lens && rope_pos &&
                  accepted && n_open && hit && (n_eos == 0 || eos_ids) && n_eos >= 0 && slots >= 1 && slots < 65536 && K >= 1 &&
                  K <= kLookupMaxK,
              "uvx_lookup_accept_slots_stop: bad arguments (1 <= K <= %d)", kLookupMaxK);
  const int warps = slots < 32 ? (int)slots : 32;
  launch_k(lookup_accept_slots_kernel<true>, dim3(1), dim3(32 * warps), 0, (cudaStream_t)stream, pick, tok, n_draft, (int)K,
           eos_ids, (int)n_eos, seq, seq_stride, token, done, cur_len, n_new, max_new, active, pos, lens, rope_pos, accepted, n_open,
           (int)slots, hit);
  return check_launch("lookup_accept_slots_kernel (stop)");
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
  launch_k(beam_update_kernel<false>, dim3((unsigned)B), dim3(256), 0, (cudaStream_t)stream, cand_s, cand_i, V, (int)nb, (int)K,
           eos_ids, (int)n_eos, (int)max_new, len_div, (int)early_stopping, (int)lp_positive, run_score, run_seq, pool_seq,
           seq_stride, pool_score, pool_len, pool_fin, parent, tok, heur, flags, ticket, cur_len, step_idx, bump0, bump1, bump2,
           done, B, (const int32_t*)nullptr);
  return check_launch("beam_update_kernel");
}

extern "C" int uvx_beam_update_stop(const float* cand_s, const int64_t* cand_i, int64_t B, int32_t nb, int32_t K, int64_t V,
                                    const int64_t* eos_ids, int32_t n_eos, int32_t max_new, const float* len_div,
                                    int32_t early_stopping, int32_t lp_positive, float* run_score, int64_t* run_seq,
                                    int64_t* pool_seq, int64_t seq_stride, float* pool_score, int32_t* pool_len, int32_t* pool_fin,
                                    int32_t* parent, int64_t* tok, int32_t* heur, int32_t* flags, uint32_t* ticket,
                                    int32_t* cur_len, int32_t* step_idx, int32_t* bump0, int32_t* bump1, int32_t* bump2,
                                    int32_t* done, const int32_t* hit, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(cand_s && cand_i && len_div && run_score && run_seq && pool_seq && pool_score && pool_len && pool_fin && parent && tok &&
                  heur && flags && ticket && cur_len && step_idx && done && hit && B >= 1 && nb >= 1 && nb <= kBeamMax && K >= nb &&
                  K <= kBeamMaxK && V >= 1 && (n_eos == 0 || eos_ids) && n_eos >= 0 && max_new >= 1 && early_stopping >= 0 &&
                  early_stopping <= 2,
              "uvx_beam_update_stop: bad arguments");
  launch_k(beam_update_kernel<true>, dim3((unsigned)B), dim3(256), 0, (cudaStream_t)stream, cand_s, cand_i, V, (int)nb, (int)K,
           eos_ids, (int)n_eos, (int)max_new, len_div, (int)early_stopping, (int)lp_positive, run_score, run_seq, pool_seq,
           seq_stride, pool_score, pool_len, pool_fin, parent, tok, heur, flags, ticket, cur_len, step_idx, bump0, bump1, bump2,
           done, B, hit);
  return check_launch("beam_update_kernel (stop)");
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
  launch_k(kv_pages_copy_kernel<false>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (uint4*)k_row, (uint4*)v_row,
           row_layer_stride / 8, (uint4*)k_pool, (uint4*)v_pool, pool_layer_stride / 8, L, row_elems / 8, pages, p0, p1 - p0,
           (int)to_pages, (const float*)nullptr);
  return check_launch("kv_pages_copy_kernel");
}

extern "C" int uvx_kv_pages_copy_fp8(void* k_row, void* v_row, int64_t row_layer_stride, void* k_pool, void* v_pool,
                                     int64_t pool_layer_stride, int64_t L, int64_t row_elems, const int32_t* pages, int64_t p0, int64_t p1,
                                     int32_t to_pages, const float* kv_scales, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(k_row && v_row && k_pool && v_pool && pages && kv_scales && L >= 1, "uvx_kv_pages_copy_fp8: null pointer");
  UVX_REQUIRE(row_elems >= 16 && row_elems % 16 == 0 && row_layer_stride % 16 == 0 && pool_layer_stride % 16 == 0 && p0 >= 0 &&
                  p1 >= p0 && p1 * row_elems <= row_layer_stride,
              "uvx_kv_pages_copy_fp8: bad shape");
  UVX_REQUIRE(((uintptr_t)k_row | (uintptr_t)v_row | (uintptr_t)k_pool | (uintptr_t)v_pool) % 16 == 0,
              "uvx_kv_pages_copy_fp8: base pointers must be 16-byte aligned");
  if (p1 == p0) return UVX_OK;
  const int64_t total = 2 * L * (p1 - p0) * (row_elems / 16);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_k(kv_pages_copy_kernel<true>, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (uint4*)k_row, (uint4*)v_row,
           row_layer_stride / 16, (uint4*)k_pool, (uint4*)v_pool, pool_layer_stride / 16, L, row_elems / 16, pages, p0, p1 - p0,
           (int)to_pages, kv_scales);
  return check_launch("kv_pages_copy_kernel (fp8 pool)");
}

// Whether the kernel can dereference `p` as it is: device memory, or host memory that is pinned / registered and mapped at the
// same address (UVA).  A pageable host pointer (cudaMemoryTypeUnregistered) is refused.
static bool kv_move_addressable(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    (void)cudaGetLastError();
    return false;
  }
  if (a.type == cudaMemoryTypeDevice) return true;
  return a.type == cudaMemoryTypeHost && a.devicePointer == p;
}

extern "C" int uvx_kv_pages_move(const void* src_k, const void* src_v, int64_t src_layer_stride, void* dst_k, void* dst_v,
                                 int64_t dst_layer_stride, int64_t L, int64_t page_bytes, const int32_t* src_pages,
                                 const int32_t* dst_pages, int64_t n, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(src_k && src_v && dst_k && dst_v && src_pages && dst_pages, "uvx_kv_pages_move: null pointer");
  UVX_REQUIRE(L >= 1 && n >= 0 && page_bytes >= 16 && page_bytes % 16 == 0 && src_layer_stride % 16 == 0 && dst_layer_stride % 16 == 0,
              "uvx_kv_pages_move: bad shape (L >= 1, n >= 0, page_bytes and layer strides multiples of 16 bytes)");
  UVX_REQUIRE(((uintptr_t)src_k | (uintptr_t)src_v | (uintptr_t)dst_k | (uintptr_t)dst_v) % 16 == 0,
              "uvx_kv_pages_move: base pointers must be 16-byte aligned");
  const void* bases[4] = {src_k, src_v, dst_k, dst_v};
  for (const void* p : bases)
    UVX_REQUIRE(kv_move_addressable(p),
                "uvx_kv_pages_move: %p is neither device memory nor pinned host memory mapped into the device's address space", p);
  if (n == 0) return UVX_OK;
  const int64_t total = 2 * L * n * (page_bytes / 16);
  int64_t blocks = (total + 255) / 256;
  if (blocks > 132 * 16) blocks = 132 * 16;
  launch_k(kv_pages_move_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, (const uint4*)src_k, (const uint4*)src_v,
           src_layer_stride / 16, (uint4*)dst_k, (uint4*)dst_v, dst_layer_stride / 16, L, page_bytes / 16, src_pages, dst_pages, n);
  return check_launch("kv_pages_move_kernel");
}

extern "C" int uvx_token_logprobs(const float* logits, int64_t B, int64_t V, const int64_t* tok, const int32_t* n_top,
                                  const int32_t* dst, int64_t cap, int32_t n_max, float* out_lp, int64_t* out_ids, float* out_top,
                                  uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && tok && n_top && dst && out_lp && B >= 1 && V >= 1 && V <= ((int64_t)1 << 31) - 1 && cap >= 1 &&
                  n_max >= 0 && n_max <= kLogprobsMax && (n_max == 0 || (out_ids && out_top)),
              "uvx_token_logprobs: bad arguments (0 <= n_max <= %d)", kLogprobsMax);
  launch_k(token_logprobs_kernel, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, tok, n_top, dst, cap, (int)n_max,
           out_lp, out_ids, out_top, (const int32_t*)nullptr);
  return check_launch("token_logprobs_kernel");
}

extern "C" int uvx_token_logprobs_rows(const float* logits, int64_t R, int64_t V, const int64_t* tok, const int32_t* n_top,
                                       const int32_t* row_slot, const int32_t* dst, int64_t cap, int32_t n_max, float* out_lp,
                                       int64_t* out_ids, float* out_top, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && tok && n_top && row_slot && dst && out_lp && R >= 1 && R < 65536 && V >= 1 && V <= ((int64_t)1 << 31) - 1 &&
                  cap >= 1 && n_max >= 0 && n_max <= kLogprobsMax && (n_max == 0 || (out_ids && out_top)),
              "uvx_token_logprobs_rows: bad arguments (0 <= n_max <= %d)", kLogprobsMax);
  launch_k(token_logprobs_kernel, dim3((unsigned)R), dim3(1024), 0, (cudaStream_t)stream, logits, V, tok, n_top, dst, cap, (int)n_max,
           out_lp, out_ids, out_top, row_slot);
  return check_launch("token_logprobs_kernel (rows)");
}

extern "C" int uvx_record_scores(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                 const int32_t* step_idx, int64_t steps, float* scores, float* raw, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && step_idx && (scores || raw) && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && steps >= 1 && top_p >= 0.f &&
                  top_p <= 1.f,
              "uvx_record_scores: bad arguments");
  const float t = temperature > 0.f ? temperature : 0.f;
  launch_k(record_scores_kernel<false, false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, t,
           t > 0.f ? 1.0f / t : 0.f, (int)top_k, top_p, step_idx, steps, B, scores, raw, Cutoffs{0.f, 1.f, 0.f, 0.f});
  return check_launch("record_scores_kernel");
}

extern "C" int uvx_record_scores_rows(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                      const int32_t* idx, int64_t steps, float* scores, float* raw, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && idx && (scores || raw) && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && steps >= 1 && top_p >= 0.f &&
                  top_p <= 1.f,
              "uvx_record_scores_rows: bad arguments");
  const float t = temperature > 0.f ? temperature : 0.f;
  launch_k(record_scores_kernel<true, false>, dim3((unsigned)B), dim3(1024), 0, (cudaStream_t)stream, logits, V, t,
           t > 0.f ? 1.0f / t : 0.f, (int)top_k, top_p, idx, steps, B, scores, raw, Cutoffs{0.f, 1.f, 0.f, 0.f});
  return check_launch("record_scores_rows_kernel");
}

// The two scalar record forms with cut-offs (kRows as in record_scores_kernel); no cut-off on is the plain form.
static int record_scores_cutoffs(bool rows, const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                 uvx_cutoffs cutoffs, const int32_t* idx, int64_t steps, float* scores, float* raw,
                                 uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(logits && idx && (scores || raw) && B >= 1 && V >= 1 && V <= (int64_t)1 << 24 && steps >= 1 && top_p >= 0.f &&
                  top_p <= 1.f && cutoffs_valid(cutoffs),
              rows ? "uvx_record_scores_rows_cutoffs: bad arguments" : "uvx_record_scores_cutoffs: bad arguments");
  const float t = temperature > 0.f ? temperature : 0.f;
  if (!cutoffs_on_host(cutoffs) || !(t > 0.f))
    return rows ? uvx_record_scores_rows(logits, B, V, temperature, top_k, top_p, idx, steps, scores, raw, stream)
                : uvx_record_scores(logits, B, V, temperature, top_k, top_p, idx, steps, scores, raw, stream);
  launch_k(rows ? record_scores_kernel<true, true> : record_scores_kernel<false, true>, dim3((unsigned)B), dim3(1024), 0,
           (cudaStream_t)stream, logits, V, t, 1.0f / t, (int)top_k, top_p, idx, steps, B, scores, raw, cutoffs_of(cutoffs));
  return check_launch(rows ? "record_scores_rows_kernel (cutoffs)" : "record_scores_kernel (cutoffs)");
}

extern "C" int uvx_record_scores_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k, float top_p,
                                         uvx_cutoffs cutoffs, const int32_t* step_idx, int64_t steps, float* scores, float* raw,
                                         uvx_stream_t stream) {
  return record_scores_cutoffs(false, logits, B, V, temperature, top_k, top_p, cutoffs, step_idx, steps, scores, raw, stream);
}

extern "C" int uvx_record_scores_rows_cutoffs(const float* logits, int64_t B, int64_t V, float temperature, int32_t top_k,
                                              float top_p, uvx_cutoffs cutoffs, const int32_t* idx, int64_t steps, float* scores,
                                              float* raw, uvx_stream_t stream) {
  return record_scores_cutoffs(true, logits, B, V, temperature, top_k, top_p, cutoffs, idx, steps, scores, raw, stream);
}
