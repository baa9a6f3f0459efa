// uvx_gemm_bf16: bf16 x bf16 -> fp32 GEMM on the Hopper tensor cores (TMA + mbarrier ring + wgmma), sm_90a.
//
//   C[row(b,m), n] = act(alpha * sum_k A[b,m,k] W[n,k] + bias[n]) + R[b,m,n]
//
// Persistent, warp-specialised kernel: grid = min(#units, #SMs), each CTA walks units u = blockIdx.x + i*gridDim.x (a unit is
// one output tile, or one K range of it under split-K).  A CTA tile is (MT*128) x BN: MT in {1,2} row sub-tiles share one W
// tile (at M <= 256 - the LLM prefill - every weight byte is fetched from L2/HBM once), BN in {64,128,208,256} (208: ragged
// last column tile allowed).  At M <= 256 CTAs also run in thread-block clusters of cm x cn tiles that split the loads of the
// A box (along N) and of the W box (along M) and multicast them to their peers (pick_cluster).
//   warpgroup 0    one thread issues the TMA loads: the A box {64 k, MT*128 rows, 1 batch} and the W box {64 k, BN rows} into
//                  a deep 128B-swizzled shared-memory ring (mbarrier expect_tx); it runs ahead across unit boundaries.
//   warpgroups 1-2 consumers: warpgroup c owns rows [64c, 64c+64) of each 128-row sub-tile and issues wgmma m64 x BN x 16
//                  from shared memory with fp32 accumulators in registers, keeping one k-block of MMAs in flight while it
//                  releases the previous ring slot; then the fused epilogue (bias / GELU / residual / row remap, fused SwiGLU or
//                  RoPE) straight from the accumulator registers, or - tensor-bound calls with the plain epilogue - staged
//                  through a shared-memory tile and written by TMA store, the residual loaded into that tile by the producer.
// A is described by a 3-D tensor map (k, row, batch) with caller-chosen strides, so overlapping rows (implicit-GEMM conv over
// a time-major activation) and batch-strided inputs need no im2col copy; rows or k beyond the tensor bounds are zero-filled
// by TMA, which is how M / K tails are handled.  K is always summed in k-block order, so a result depends only on the split
// count, never on the tile width or the grid.
#include <stdlib.h>

#include "uvx_common.cuh"
#include "tc_ptx.cuh"

namespace uvx {

struct GemmParams {
  int64_t a_rows, a_batch, K, N;
  void* C;
  int64_t c_row_stride, c_batch_rows, c_row_offset;
  const int32_t* c_row_map;
  const bf16* bias;
  const bf16* R;
  int64_t r_row_stride, r_batch_stride;
  float alpha;
  int act, out_f32;
  int m_tiles;  // per batch (of MT*128 rows)
  int n_tiles, num_tiles;
  int splits, kb_per_split;  // split-K: units = num_tiles * splits
  float* ws_partial;         // [splits][a_batch * a_rows][N] fp32 partial sums (reduced by splitk_reduce_kernel)
  const bf16* norm_w;        // optional fused RMSNorm of the finished output rows: norm_out = w * bf16(C * rstd)
  bf16* norm_out;
  float norm_eps;
  int w_tiled;             // W is the pre-tiled image [n_tiles][K/64][BN][64]: every TMA box is ONE contiguous BN*128-byte run
  int w_perm;              // 128-row image in UVX_TILE_ROPE_PAIRS order: tile column 32q + j is output column 16q + j (j < 16)
                           // or 64 + 16q + (j - 16)
  int swiglu;              // 0, or the gate|up interleave of the image (8: 8 gate | 8 up rows, 16: 16 | 16); output [M, N/2]
  const float* rope_cos;   // fused RoPE (hf:modeling_llama.py:124-168) on tiles whose first column is < rope_cols, head_dim 128 == BN
  const float* rope_sin;
  const int32_t* rope_pos;
  int64_t rope_rows_per_seq, rope_pos_offset;
  int rope_cols;
  int stages;              // ring depth (split ring: depth of the weight ring)
  int a_stages;            // split ring (0: one ring of A box + W box stages): depth of the separate activation ring
  int a_box_rows;          // rows of the A box (MT*128, or round8(a_rows) for a split ring)
  int w_early;             // split ring: the weight lane issues its first ring round before griddepcontrol.wait
  int cm, cn;           // thread-block cluster of cm x cn tiles (1 x 1: no cluster); cm divides m_tiles * a_batch, cn n_tiles
  int staged_bytes;        // staged epilogue (gemm_wg_kernel<., ., true>): its output tile in shared memory, between the ring and
                           // the barriers (0: register epilogue)
  int r_bcast;             // the residual has batch stride 0: its map (tmR) has no batch dimension
};

static constexpr int kSmemTotal = 227 * 1024;
static constexpr int kMaxStages = 8;   // one ring of A + W stages, and the decode form's ring
static constexpr int kMaxWStages = 16;  // split ring: weight ring (gemm_wg_kernel's full / empty barrier arrays have this many)
static constexpr int kMaxAStages = 8;   // split ring: activation ring
static constexpr int kBarBytes = 512;   // gemm_wg_kernel's barriers: 2 x kMaxWStages + 2 + 2 x kMaxAStages mbarriers
static_assert((2 * kMaxWStages + 2 + 2 * kMaxAStages) * 8 <= kBarBytes, "barrier region");
static constexpr int kGemmThreads = 384;  // producer warpgroup + two consumer warpgroups
static constexpr int kPanelBytes = 128 * 128;  // staged output: 128 rows x 128 bytes (64 bf16 / 32 fp32 columns), 128B swizzle

template <int MT, int BN>
struct WgLayout {
  static constexpr int kABytes = MT * 128 * kBK * 2;
  static constexpr int kWBytes = BN * kBK * 2;  // BN % 8 == 0: a whole number of 1 KB swizzle atoms
  static constexpr int kStageBytes = kABytes + kWBytes;
  static constexpr int kRingMax = kSmemTotal - 1024 - kBarBytes;  // alignment slack + barriers
  static constexpr int kStages = kRingMax / kStageBytes > kMaxStages ? kMaxStages : kRingMax / kStageBytes;
  static constexpr int kAcc = BN / 2;  // fp32 accumulators per thread and 64-row sub-tile
  static_assert(kStages >= 2, "ring too shallow");
  static_assert(MT * kAcc <= 128, "accumulators must fit the register file");
};

// tile column -> output column of the tile (identity, or the pair-permuted 128-row image)
__device__ __forceinline__ int tile_col(int tc, int perm) {
  if (!perm) return tc;
  const int q = tc >> 5, j = tc & 31;
  return j < 16 ? 16 * q + j : 64 + 16 * q + (j - 16);
}

__device__ __forceinline__ int64_t out_row(const GemmParams& p, int b, int64_t m) {
  return p.c_row_map ? (int64_t)p.c_row_map[(int64_t)b * p.a_rows + m] : (int64_t)b * p.c_batch_rows + m + p.c_row_offset;
}

// fused SwiGLU row of one 64-row sub-tile (Llama MLP act(gate) * up, hf:modeling_llama.py:183): the interleaved gate|up image
// puts a feature's gate and up rows I columns apart inside the tile, so both land in this thread's registers.  Rounding order
// is the unfused path's: gate and up rounded to bf16 (what the GEMM would have stored), silu rounded to bf16, product rounded.
template <int BN, int I>
__device__ __forceinline__ void swiglu_row(const GemmParams& p, const float* a, int h, int cq, bf16* crow, int64_t n_out0) {
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    if ((8 * j) % (2 * I) >= I) continue;  // up columns are read with their gate partner
    const int64_t f = n_out0 + (8 * j / (2 * I)) * I + (8 * j) % (2 * I) + cq;
    if (f >= p.N / 2) continue;
    constexpr int kUp = I / 8;
    float o[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const float gate = __bfloat162float(__float2bfloat16_rn(a[4 * j + 2 * h + e] * p.alpha));
      const float up = __bfloat162float(__float2bfloat16_rn(a[4 * (j + kUp) + 2 * h + e] * p.alpha));
      o[e] = __bfloat162float(__float2bfloat16_rn(silu_fast(gate))) * up;
    }
    *reinterpret_cast<__nv_bfloat162*>(crow + f) = __floats2bfloat162_rn(o[0], o[1]);
  }
}

// one RoPE pair of columns (d, d + 1) and (d + 64, d + 65) of a head: x1 / x2 are the fp32 accumulators
__device__ __forceinline__ void rope_store(const GemmParams& p, float x1a, float x1b, float x2a, float x2b, int64_t pos, int d, bf16* crow) {
  const float2 cs = *reinterpret_cast<const float2*>(p.rope_cos + pos * 64 + d);
  const float2 sn = *reinterpret_cast<const float2*>(p.rope_sin + pos * 64 + d);
  float o1a, o2a, o1b, o2b;
  rope_pair(__bfloat162float(__float2bfloat16_rn(x1a * p.alpha)), __bfloat162float(__float2bfloat16_rn(x2a * p.alpha)), cs.x, sn.x, o1a, o2a);
  rope_pair(__bfloat162float(__float2bfloat16_rn(x1b * p.alpha)), __bfloat162float(__float2bfloat16_rn(x2b * p.alpha)), cs.y, sn.y, o1b, o2b);
  *reinterpret_cast<__nv_bfloat162*>(crow + d) = __floats2bfloat162_rn(o1a, o1b);
  *reinterpret_cast<__nv_bfloat162*>(crow + d + 64) = __floats2bfloat162_rn(o2a, o2b);
}

// STAGED: the staged epilogue (the output tile goes through shared memory and leaves by TMA store, the residual is loaded by TMA
// ahead of the epilogue) and no other; its own instantiation, so the register-epilogue kernels keep their register budget.
// tmC / tmR: its output and residual maps, 3-D (n, row, batch) with 128-row x 128-byte boxes.
template <int MT, int BN, bool STAGED>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wg_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmC,
               const __grid_constant__ CUtensorMap tmR, const GemmParams p) {
  using L = WgLayout<MT, BN>;
  static_assert(!STAGED || (MT == 1 && BN <= 128), "the staged epilogue is built for 128 x 64 and 128 x 128 tiles");
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);  // 128B-swizzle atoms need 1 KB alignment
  // Ring geometry.  One ring (a_stages == 0): stage s holds the A box at s * kStageBytes and the W box kABytes after it, under
  // one full and one empty barrier.  Split ring (one m-tile covers the rows of a single batch): an activation ring of a_stages
  // slots of a_box_rows * 128 bytes, then a weight ring of `stages` slots of kWBytes, each ring with its own barriers and its
  // own producer lane, so a weight load never waits for an activation slot.  The consumers' m64 MMAs still read MT * 128 rows of an
  // A slot: rows a_box_rows .. MT * 128 - 1 come from whatever follows the slot (the next A slot, or the weight ring after the
  // last one - inside the allocation).  Accumulator row r depends only on A row r, so the garbage reaches accumulator rows
  // >= a_box_rows >= a_rows alone, and every epilogue (plain, SwiGLU, RoPE, split-K partial) skips rows >= a_rows.
  // (the staged kernel and the 208 / 256-wide tiles - tensor-bound calls - never run it: their loops keep the one ring's code)
  constexpr bool kSplitRing = !STAGED && BN <= 128;
  const bool split_ring = kSplitRing && p.a_stages > 0;
  const int stages = p.stages, a_stages = split_ring ? p.a_stages : stages;
  const int a_box_bytes = p.a_box_rows * (kBK * 2);
  const int a_stride = split_ring ? a_box_bytes : L::kStageBytes, w_stride = split_ring ? L::kWBytes : L::kStageBytes;
  uint8_t* const w_ring = split_ring ? smem + a_stages * a_box_bytes : smem + L::kABytes;
  uint8_t* stage_c = smem + (split_ring ? a_stages * a_box_bytes + stages * L::kWBytes : stages * L::kStageBytes);  // staged output tile
  uint64_t* full_bar = (uint64_t*)(stage_c + p.staged_bytes);  // weight ring (one ring: the stage)
  uint64_t* empty_bar = full_bar + kMaxWStages;
  uint64_t* res_full = empty_bar + kMaxWStages;  // staged: the tile's residual box has landed in stage_c
  uint64_t* stage_free = res_full + 1;           // staged: the previous tile's TMA store has finished reading stage_c
  uint64_t* const a_full = split_ring ? stage_free + 1 : full_bar;  // activation ring (one ring: the stage's barriers)
  uint64_t* const a_empty = split_ring ? a_full + kMaxAStages : empty_bar;

  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int tiles_m_total = p.m_tiles * (int)p.a_batch;
  const int num_kb = (int)((p.K + kBK - 1) / kBK);
  // Thread-block cluster of cm x cn tiles (rank r = rm * cn + rn), walked in lockstep: the cluster takes cluster units
  // (cluster tile, split) and CTA (rm, rn) computes m-tile gm * cm + rm and n-tile gn * cn + rn of cluster tile (gm, gn) with the
  // split's k range, so every member runs the same k-blocks in the same ring order.  It loads its 1/cn share of the A box and
  // multicasts it along its row (same m-tile), and its 1/cm share of the W box to its column (same n-tile).  1 x 1 is the plain
  // persistent walk: unit u = blockIdx.x + i * gridDim.x, tiles consecutive along M.
  // the staged kernel runs without clusters (tensor-bound calls): a compile-time 1 x 1 keeps its producer within 40 registers
  const int cm = STAGED ? 1 : p.cm, cn = STAGED ? 1 : p.cn;
  const int csize = cm * cn;
  const int rank = csize > 1 ? (int)cluster_ctarank() : 0;
  const int rm = rank / cn, rn = rank % cn;
  const int cluster_tiles_m = tiles_m_total / cm;
  const int num_units = p.num_tiles / csize * p.splits;
  const int first_unit = blockIdx.x / csize, unit_step = gridDim.x / csize;

  if (threadIdx.x == 0) {
    // one arrival per consumer warp of every CTA of the cluster on each empty barrier
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8 * csize);
    }
    if (split_ring) {
      for (int s = 0; s < a_stages; ++s) {
        mbar_init(&a_full[s], 1);
        mbar_init(&a_empty[s], 8 * csize);
      }
    }
    if (STAGED) {
      mbar_init(res_full, 1);
      mbar_init(stage_free, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  // no CTA multicasts into a peer before the peer's barriers are initialised
  if (csize > 1) cluster_sync();
  else __syncthreads();
  // the weight lane of a split ring streams W (or A and W: one ring), the activation lane A
  const bool w_lane = wg == 0 && tid == 0, a_lane = split_ring && wg == 0 && tid == 32;
  // set-up above overlapped the previous kernel's tail; its outputs are visible after griddepcontrol.wait.  W no kernel that may
  // still be running writes (uvx_gemm_args.flags bit 2) is read before it: the weight lane's first ring round.
  const bool w_early = split_ring && p.w_early && w_lane;
  if (!w_early) pdl_wait();

  if (wg == 0) {
    // ---- TMA producer lanes; their warpgroup hands registers to the consumers' accumulators (128 x 40 + 256 x 232 fits the
    // 384 x 168 the CTA was launched with)
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (w_lane || a_lane) {
      const bool do_w = w_lane, do_a = split_ring ? a_lane : w_lane;
      if (do_a) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmA) : "memory");
      if (do_w) asm volatile("prefetch.tensormap [%0];" ::"l"(&tmW) : "memory");
      // slices are whole 8-row (1 KB) swizzle atoms; each lands at its own offset of the box in every CTA of the mask
      const int a_slice = p.a_box_rows / cn, w_slice = BN / cm;
      const uint16_t row_mask = (uint16_t)(((1u << cn) - 1u) << (rm * cn));
      uint16_t col_mask = 0;
      for (int j = 0; j < cm; ++j) col_mask |= (uint16_t)(1u << (j * cn + rn));
      int s = 0, sa = 0, issued = 0;
      uint32_t ph = 0, pha = 0;
      for (int unit = first_unit, tile_i = 0; unit < num_units; unit += unit_step, ++tile_i) {
        const int ctile = unit / p.splits, split = unit % p.splits;
        const int tm_idx = (ctile % cluster_tiles_m) * cm + rm;  // consecutive tiles share the W tile
        const int tn_idx = (ctile / cluster_tiles_m) * cn + rn;
        const int b = tm_idx / p.m_tiles;
        const int m0 = (tm_idx % p.m_tiles) * (MT * 128);
        const int kb_begin = split * p.kb_per_split;
        const int kb_end = min(num_kb, kb_begin + p.kb_per_split);
        // W box of k-block kb: canonical [N, K] weights -> (kb * 64, n0); pre-tiled image [tile][kb][BN][64] viewed as
        // [rows, 64] -> (0, (tn_idx * num_kb + kb) * BN): one contiguous BN * 128-byte run of DRAM
        const int wt_base = tn_idx * num_kb * BN;
        // staged epilogue with a residual: the tile's residual box is loaded into the staging tile ahead of the epilogue, after
        // the k-block `stages` before the last one.  Not earlier, since waiting for the previous tile's store to leave the staging
        // tile (the consumers signal it once this tile's first MMAs are issued) must not hold up the ring; and never before the
        // tile's first k-block is loaded, which those MMAs need.
        const int r_kb = max(kb_begin, kb_end - stages);
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          // the whole box lands in every CTA (own slices and the peers'); TMA zero fill counts toward the bytes.  One ring: the
          // weight lane loads both boxes of the stage, against one expect_tx of the stage's bytes.
          if (do_w) {
            if (w_early && issued++ == stages) pdl_wait();  // after the first ring round
            mbar_wait(&empty_bar[s], ph ^ 1u);
            mbar_expect_tx(&full_bar[s], (uint32_t)(split_ring ? L::kWBytes : L::kStageBytes));
          }
          if (do_a) {
            if (split_ring) {
              mbar_wait(&a_empty[sa], pha ^ 1u);
              mbar_expect_tx(&a_full[sa], (uint32_t)a_box_bytes);
            }
            uint8_t* da = smem + sa * a_stride + rn * a_slice * (kBK * 2);
            if (cn > 1) tma_load_3d_mc(da, &tmA, kb * kBK, m0 + rn * a_slice, b, &a_full[sa], row_mask);
            else tma_load_3d(da, &tmA, kb * kBK, m0, b, &a_full[sa]);
          }
          if (do_w) {
            uint8_t* dw = w_ring + s * w_stride + rm * w_slice * (kBK * 2);
            const int w0 = p.w_tiled ? 0 : kb * kBK;
            const int w1 = (p.w_tiled ? wt_base + kb * BN : tn_idx * BN) + rm * w_slice;
            if (cm > 1) tma_load_2d_mc(dw, &tmW, w0, w1, &full_bar[s], col_mask);
            else tma_load_2d(dw, &tmW, w0, w1, &full_bar[s]);
          }
          if (++s == stages) { s = 0; ph ^= 1u; }
          if (++sa == a_stages) { sa = 0; pha ^= 1u; }
          if (STAGED && p.R && kb == r_kb) {
            mbar_wait(stage_free, (uint32_t)(tile_i & 1) ^ 1u);
            const int n0 = tn_idx * BN, panels = (int)min((int64_t)BN, p.N - n0) / 64;
            mbar_expect_tx(res_full, (uint32_t)(panels * kPanelBytes));
            for (int q = 0; q < panels; ++q) tma_load_3d(stage_c + q * kPanelBytes, &tmR, n0 + 64 * q, m0, p.r_bcast ? 0 : b, res_full);
          }
        }
      }
    }
    // no CTA leaves while a peer can still write into its shared memory or arrive on its barriers
    if (csize > 1) cluster_sync();
    return;
  }

  // ---- consumers
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int c = wg - 1;
  const int warp = tid >> 5, lane = tid & 31;
  // hand ring slot `slot` back: to this CTA's producer, or to the producers of every CTA of the cluster (each may have
  // multicast a slice into it), one lane per CTA
  auto release = [&](uint64_t* bar) {
    __syncwarp();
    if (csize == 1) {
      if (lane == 0) mbar_arrive(bar);
    } else if (lane < csize) {
      mbar_arrive_cluster(bar, (uint32_t)lane);
    }
  };
  // staged epilogue: consumer thread 0 issues the tile's TMA stores and tracks their completion
  auto store_thread = [&]() { return STAGED && threadIdx.x == 128; };
  int s = 0, sa = 0;
  uint32_t ph = 0, pha = 0;
  for (int unit = first_unit; unit < num_units; unit += unit_step) {
    const int ctile = unit / p.splits, split = unit % p.splits;
    const int tm_idx = (ctile % cluster_tiles_m) * cm + rm;
    const int tn_idx = (ctile / cluster_tiles_m) * cn + rn;
    const int b = tm_idx / p.m_tiles;
    const int m0 = (tm_idx % p.m_tiles) * (MT * 128);
    const int n0 = tn_idx * BN;
    const int kb_begin = split * p.kb_per_split;
    const int kb_end = min(num_kb, kb_begin + p.kb_per_split);

    float acc[MT][L::kAcc];
    int prev = -1, prev_a = -1;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[s], ph);
      if (split_ring) mbar_wait(&a_full[sa], pha);
      const uint32_t a_addr = smem_u32(smem + sa * a_stride);
      const uint64_t dw = make_wgmma_desc(smem_u32(w_ring + s * w_stride));
      wgmma_fence();
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
        const uint64_t da = make_wgmma_desc(a_addr + (mt * 128 + c * 64) * (kBK * 2));
#pragma unroll
        for (int k = 0; k < kBK / 16; ++k)
          Wgmma<BN>::mma(acc[mt], da + (uint64_t)(2 * k), dw + (uint64_t)(2 * k), (kb > kb_begin || k > 0) ? 1u : 0u);
      }
      wgmma_commit();
      // staged epilogue: with this tile's first MMAs in flight, wait for the previous tile's store to finish reading the staging
      // tile and hand it on (to the producer's residual load, or to this tile's epilogue)
      if (store_thread() && kb == kb_begin && unit != first_unit) {
        bulk_wait_read0();
        mbar_arrive(stage_free);
      }
      // one k-block of MMAs stays in flight; the slots read by the previous one are handed back to the producers
      wgmma_wait<1>();
      if (prev >= 0) {
        release(&empty_bar[prev]);
        if (split_ring) release(&a_empty[prev_a]);
      }
      prev = s;
      prev_a = sa;
      if (++s == stages) { s = 0; ph ^= 1u; }
      if (++sa == a_stages) { sa = 0; pha ^= 1u; }
    }
    wgmma_wait<0>();
    release(&empty_bar[prev]);
    if (split_ring) release(&a_empty[prev_a]);

    // ---- epilogue from registers: this thread holds rows r0 (+8) of each 64-row sub-tile, columns 8j + 2(lane % 4) (+1)
    const int rq = warp * 16 + (lane >> 2);
    const int cq = 2 * (lane & 3);
    if constexpr (STAGED) {
      {
        // ---- staged epilogue (plain epilogue, one split, no row map): the same arithmetic in the same order as below, written
        // into the staging tile and stored by TMA, so the consumers go straight on to the next tile's MMAs.  The tile is
        // 128-byte panels (64 bf16 / 32 fp32 columns x 128 rows, 128B swizzle: 16-byte chunk q of row r sits at chunk q ^ (r % 8)).
        // A warp's bf16 write of one (h, j) covers 8 rows r (r % 8 = lane / 4) x 16 bytes of chunk j % 8: the swizzle puts
        // the 8 rows in 8 different chunks, so the 32 lanes hit 32 different banks.  An fp32 write (8 bytes per lane) covers
        // chunks 2(j % 4) and 2(j % 4) + 1, which rows r and r ^ 1 share: a 2-way conflict, accepted for the rare fp32 output.
        // The residual (bf16 output only) was loaded into the tile by the producer, in the output's layout: each element is
        // read at the position its result is written to.
        const uint32_t tile_par = (uint32_t)((unit - first_unit) / unit_step) & 1u;  // parity of the tile's ordinal in this CTA
        if (p.R) mbar_wait(res_full, tile_par);
        else mbar_wait(stage_free, tile_par ^ 1u);
        __nv_bfloat162 bias_v[BN / 8];
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int64_t n = n0 + 8 * j + cq;
          if (p.bias && n < p.N) bias_v[j] = *reinterpret_cast<const __nv_bfloat162*>(p.bias + n);
        }
        const uint32_t st0 = smem_u32(stage_c);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int r = c * 64 + rq + 8 * h;  // tile row; rows past a_rows are clipped by the TMA store
          const uint32_t row = st0 + (uint32_t)r * 128u, sw = (uint32_t)(r & 7);
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            float v0 = acc[0][4 * j + 2 * h] * p.alpha, v1 = acc[0][4 * j + 2 * h + 1] * p.alpha;
            if (p.bias) {
              const float2 t = __bfloat1622float2(bias_v[j]);
              v0 += t.x;
              v1 += t.y;
            }
            if (p.act == UVX_ACT_GELU) {
              v0 = gelu_fast(v0);
              v1 = gelu_fast(v1);
            }
            if (p.out_f32) {
              const uint32_t chunk = (uint32_t)(2 * (j % 4) + (lane & 3) / 2);
              st_shared_f32x2(row + (j / 4) * kPanelBytes + ((chunk ^ sw) << 4) + (lane & 1) * 8, v0, v1);
            } else {
              const uint32_t addr = row + (j / 8) * kPanelBytes + (((uint32_t)(j % 8) ^ sw) << 4) + (lane & 3) * 4;
              if (p.R) {
                const uint32_t rv = ld_shared_u32(addr);
                const float2 t = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&rv));
                v0 += t.x;
                v1 += t.y;
              }
              const __nv_bfloat162 o = __floats2bfloat162_rn(v0, v1);
              st_shared_u32(addr, *reinterpret_cast<const uint32_t*>(&o));
            }
          }
        }
        // every writer makes its shared-memory writes visible to the async proxy; then one thread stores the panels that lie
        // inside N (TMA clips the M tail and the last panel's columns past N)
        fence_proxy_async();
        named_bar_sync<1, 256>();
        if (store_thread()) {
          const int cols = p.out_f32 ? 32 : 64;
          const int panels = (int)min((int64_t)BN, p.N - n0) / cols;
          for (int q = 0; q < panels; ++q) tma_store_3d(&tmC, stage_c + q * kPanelBytes, n0 + cols * q, m0, b);
          bulk_commit();
        }
        continue;
      }
    }
    if (p.splits > 1) {
      // split-K: park the raw fp32 partial tile in the workspace; splitk_reduce_kernel sums the splits in a fixed order and
      // applies the epilogue (deterministic, and the reduction is spread over every SM)
      float* part = p.ws_partial + (size_t)split * (size_t)(p.a_batch * p.a_rows) * (size_t)p.N;
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t m = (int64_t)m0 + mt * 128 + c * 64 + rq + 8 * h;
          if (m >= p.a_rows) continue;
          float* dst = part + ((size_t)b * p.a_rows + m) * p.N;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int64_t n = n0 + tile_col(8 * j + cq, p.w_perm);
            if (n < p.N) *reinterpret_cast<float2*>(dst + n) = make_float2(acc[mt][4 * j + 2 * h], acc[mt][4 * j + 2 * h + 1]);
          }
        }
      }
      continue;
    }
    if (p.swiglu) {
      const int64_t n_out0 = (int64_t)tn_idx * (BN / 2);
#pragma unroll
      for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int64_t m = (int64_t)m0 + mt * 128 + c * 64 + rq + 8 * h;
          if (m >= p.a_rows) continue;
          const int64_t orow = out_row(p, b, m);
          if (orow < 0) continue;
          bf16* crow = reinterpret_cast<bf16*>(p.C) + orow * p.c_row_stride;
          if (p.swiglu == 16) swiglu_row<BN, 16>(p, acc[mt], h, cq, crow, n_out0);
          else swiglu_row<BN, 8>(p, acc[mt], h, cq, crow, n_out0);
        }
      }
      continue;
    }
    if constexpr (BN == 128) {
      if (p.rope_cos != nullptr && n0 < p.rope_cols) {
        // fused RoPE: the tile is one 128-wide head; output columns d and d + 64 rotate together and sit in this thread's
        // registers (tile columns t and t + 64, or t and t + 16 in the pair-permuted image).  Same rounding as GEMM-then-uvx_rope:
        // the projection is rounded to bf16 first, the rotation runs in fp32 on those values and is rounded once more by the store.
#pragma unroll
        for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const int64_t m = (int64_t)m0 + mt * 128 + c * 64 + rq + 8 * h;
            if (m >= p.a_rows) continue;
            const int64_t orow = out_row(p, b, m);
            if (orow < 0) continue;
            const int64_t pos = p.rope_pos ? (int64_t)p.rope_pos[m] : p.rope_pos_offset + (m % p.rope_rows_per_seq);
            bf16* crow = reinterpret_cast<bf16*>(p.C) + orow * p.c_row_stride + n0;
            const float* a = acc[mt];
            if (!p.w_perm) {
#pragma unroll
              for (int j = 0; j < 8; ++j)
                rope_store(p, a[4 * j + 2 * h], a[4 * j + 2 * h + 1], a[4 * (j + 8) + 2 * h], a[4 * (j + 8) + 2 * h + 1], pos, 8 * j + cq, crow);
            } else {
#pragma unroll
              for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int jj = 0; jj < 2; ++jj) {
                  const int j = 4 * q + jj;
                  rope_store(p, a[4 * j + 2 * h], a[4 * j + 2 * h + 1], a[4 * (j + 2) + 2 * h], a[4 * (j + 2) + 2 * h + 1], pos,
                             16 * q + 8 * jj + cq, crow);
                }
            }
          }
        }
        continue;
      }
    }
    // plain epilogue: alpha, bias, GELU, residual, row remap; bf16 or fp32 out.  The operands are loaded before the first store
    // that could depend on them: the bias columns once per tile, a row's residual before that row's stores.  The compiler cannot
    // move a load above a store to C (C may alias R: the in-place residual stream), so loads interleaved with the stores each
    // waited out a full memory latency.  Hoisting is safe: a thread reads residual elements only at the positions it writes.  Only
    // tiles with MT * BN <= 128 have the registers for it (wider ones spill, and keep the loads next to their use).
    constexpr bool kHoist = MT * BN <= 128;
    __nv_bfloat162 bias_v[BN / 8];
    if constexpr (kHoist) {
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const int64_t n = n0 + tile_col(8 * j + cq, p.w_perm);
        if (p.bias && n < p.N) bias_v[j] = *reinterpret_cast<const __nv_bfloat162*>(p.bias + n);
      }
    }
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t m = (int64_t)m0 + mt * 128 + c * 64 + rq + 8 * h;
        if (m >= p.a_rows) continue;
        const int64_t orow = out_row(p, b, m);
        if (orow < 0) continue;
        const bf16* rrow = p.R ? p.R + (int64_t)b * p.r_batch_stride + m * p.r_row_stride : nullptr;
        __nv_bfloat162 res_v[BN / 8];
        if (kHoist && rrow) {
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const int64_t n = n0 + tile_col(8 * j + cq, p.w_perm);
            if (n < p.N) res_v[j] = *reinterpret_cast<const __nv_bfloat162*>(rrow + n);
          }
        }
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const int64_t n = n0 + tile_col(8 * j + cq, p.w_perm);
          if (n >= p.N) continue;  // ragged last column tile (N % BN != 0); N % 64 == 0 keeps both columns in range
          float v0 = acc[mt][4 * j + 2 * h] * p.alpha, v1 = acc[mt][4 * j + 2 * h + 1] * p.alpha;
          if (p.bias) {
            const float2 t = __bfloat1622float2(kHoist ? bias_v[j] : *reinterpret_cast<const __nv_bfloat162*>(p.bias + n));
            v0 += t.x;
            v1 += t.y;
          }
          if (p.act == UVX_ACT_GELU) {
            v0 = gelu_fast(v0);
            v1 = gelu_fast(v1);
          }
          if (rrow) {
            const float2 t = __bfloat1622float2(kHoist ? res_v[j] : *reinterpret_cast<const __nv_bfloat162*>(rrow + n));
            v0 += t.x;
            v1 += t.y;
          }
          if (p.out_f32)
            *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.C) + orow * p.c_row_stride + n) = make_float2(v0, v1);
          else
            *reinterpret_cast<__nv_bfloat162*>(reinterpret_cast<bf16*>(p.C) + orow * p.c_row_stride + n) = __floats2bfloat162_rn(v0, v1);
        }
      }
    }
  }
  // the stores are complete in global memory before the CTA exits (the next kernel's griddepcontrol.wait must see them)
  if (store_thread()) bulk_wait0();
  if (csize > 1) cluster_sync();
}

// Split-K second pass: sums the fp32 partials in split order and applies the same epilogue as the direct path.
// One thread per 8 consecutive output columns; spread over the whole grid so no single SM has to pull all partials.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const GemmParams p) {
  pdl_trigger();
  pdl_wait();
  const int64_t rows = p.a_batch * p.a_rows;
  const int64_t vec_per_row = p.N / 8;
  const int64_t total = rows * vec_per_row;
  const size_t split_stride = (size_t)rows * (size_t)p.N;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = idx / vec_per_row, n = (idx % vec_per_row) * 8;
    const int64_t b = r / p.a_rows, m = r % p.a_rows;
    const float* src = p.ws_partial + (size_t)r * p.N + n;
    float v[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll 4
    for (int sidx = 0; sidx < p.splits; ++sidx) {
      const float4 t0 = __ldcg(reinterpret_cast<const float4*>(src + sidx * split_stride));
      const float4 t1 = __ldcg(reinterpret_cast<const float4*>(src + sidx * split_stride) + 1);
      v[0] += t0.x; v[1] += t0.y; v[2] += t0.z; v[3] += t0.w;
      v[4] += t1.x; v[5] += t1.y; v[6] += t1.z; v[7] += t1.w;
    }
    const int64_t orow = p.c_row_map ? (int64_t)p.c_row_map[r] : b * p.c_batch_rows + m + p.c_row_offset;
    if (orow < 0) continue;
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] *= p.alpha;
    if (p.bias) {
      float t[8];
      unpack8(*reinterpret_cast<const bf16x8*>(p.bias + n), t);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += t[i];
    }
    if (p.act == UVX_ACT_GELU) {
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = gelu_erf(v[i]);
    }
    if (p.R) {
      float t[8];
      unpack8(*reinterpret_cast<const bf16x8*>(p.R + b * p.r_batch_stride + m * p.r_row_stride + n), t);
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] += t[i];
    }
    if (p.out_f32) {
      float4* dst = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.C) + orow * p.c_row_stride + n);
      dst[0] = make_float4(v[0], v[1], v[2], v[3]);
      dst[1] = make_float4(v[4], v[5], v[6], v[7]);
    } else {
      *reinterpret_cast<bf16x8*>(reinterpret_cast<bf16*>(p.C) + orow * p.c_row_stride + n) = pack8(v);
    }
  }
}

// Split-K second pass fused with the RMSNorm that follows o_proj / down_proj in every Llama layer: one CTA per output row
// sums the partials, applies the epilogue (bias / residual), writes the residual stream C and, from the same registers,
// norm_out = w * bf16(C * rsqrt(mean(C^2) + eps)) (LlamaRMSNorm rounding order on the bf16-rounded C).  bf16 output only.
__global__ void __launch_bounds__(256) splitk_reduce_rmsnorm_kernel(const GemmParams p) {
  pdl_trigger();
  pdl_wait();
  __shared__ float red[32];
  const int64_t r = blockIdx.x;
  const int64_t b = r / p.a_rows, m = r % p.a_rows;
  const int64_t rows = p.a_batch * p.a_rows;
  const size_t split_stride = (size_t)rows * (size_t)p.N;
  const int64_t orow = p.c_row_map ? (int64_t)p.c_row_map[r] : b * p.c_batch_rows + m + p.c_row_offset;
  constexpr int kMaxV = 4;  // up to 256 * 4 * 8 = 8192 columns
  float v[kMaxV][8];
  float sq = 0.f;
  const int nvec = (int)(p.N / 8);
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = threadIdx.x + i * 256;
    if (j < nvec) {
      const int64_t n = (int64_t)j * 8;
      const float* src = p.ws_partial + (size_t)r * p.N + n;
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] = 0.f;
      // loads of four splits are issued together (the kernel is a latency chain: partials -> row sum -> write), sums stay in
      // split order so the result does not depend on the batching
      for (int s0 = 0; s0 < p.splits; s0 += 4) {
        float4 t0[4], t1[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (s0 + u < p.splits) {
            t0[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * split_stride));
            t1[u] = __ldcg(reinterpret_cast<const float4*>(src + (s0 + u) * split_stride) + 1);
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (s0 + u < p.splits) {
            v[i][0] += t0[u].x; v[i][1] += t0[u].y; v[i][2] += t0[u].z; v[i][3] += t0[u].w;
            v[i][4] += t1[u].x; v[i][5] += t1[u].y; v[i][6] += t1[u].z; v[i][7] += t1[u].w;
          }
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) v[i][e] *= p.alpha;
      if (p.bias) {
        float t[8];
        unpack8(*reinterpret_cast<const bf16x8*>(p.bias + n), t);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] += t[e];
      }
      if (p.R) {
        float t[8];
        unpack8(*reinterpret_cast<const bf16x8*>(p.R + b * p.r_batch_stride + m * p.r_row_stride + n), t);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[i][e] += t[e];
      }
      const bf16x8 packed = pack8(v[i]);
      if (orow >= 0) *reinterpret_cast<bf16x8*>(reinterpret_cast<bf16*>(p.C) + orow * p.c_row_stride + n) = packed;
      unpack8(packed, v[i]);  // the norm sees the bf16-rounded residual stream, exactly like a separate kernel would
#pragma unroll
      for (int e = 0; e < 8; ++e) sq += v[i][e] * v[i][e];
    }
  }
  const float rstd = rsqrtf(block_sum(sq, red) / (float)p.N + p.norm_eps);
  if (orow < 0) return;
#pragma unroll
  for (int i = 0; i < kMaxV; ++i) {
    const int j = threadIdx.x + i * 256;
    if (j < nvec) {
      float wv[8], o[8];
      unpack8(*reinterpret_cast<const bf16x8*>(p.norm_w + (int64_t)j * 8), wv);
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] = wv[e] * __bfloat162float(__float2bfloat16_rn(v[i][e] * rstd));
      *reinterpret_cast<bf16x8*>(p.norm_out + orow * p.N + (int64_t)j * 8) = pack8(o);
    }
  }
}


// ---------------------------------------------------------------------------------- decode form (operands swapped)
// Decode batches (a_rows <= 32): 128 weight rows on the wgmma M dimension (64 per consumer warpgroup) and the tokens on N
// (BT = 8 / 16 / 32), so no MMA work is spent on padding rows.  Same ring / producer as gemm_wg_kernel; the weight stream is
// spread over the SMs by deterministic split-K (fp32 partials in [split][row][N], reduced in split order).  A thread holds
// features f and f + 8 of its warp's 16 and tokens 8j + 2(lane % 4) (+1).
template <int BT>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_swap_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const GemmParams p) {
  constexpr int kWBytes = 128 * kBK * 2, kXBytes = BT * kBK * 2, kStage = kWBytes + kXBytes;
  pdl_trigger();
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full_bar = (uint64_t*)(smem + p.stages * kStage);
  uint64_t* empty_bar = full_bar + kMaxStages;
  const int wg = threadIdx.x >> 7, tid = threadIdx.x & 127;
  const int num_kb = (int)((p.K + kBK - 1) / kBK);
  const int num_units = p.n_tiles * p.splits;
  const int stages = p.stages;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], 8);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  if (wg == 0) {
    if (tid == 0) {
      int s = 0;
      uint32_t ph = 0;
      for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
        const int tn_idx = unit / p.splits, split = unit % p.splits;
        const int kb_begin = split * p.kb_per_split, kb_end = min(num_kb, kb_begin + p.kb_per_split);
        const int wt_base = tn_idx * num_kb * 128;
        for (int kb = kb_begin; kb < kb_end; ++kb) {
          mbar_wait(&empty_bar[s], ph ^ 1u);
          uint8_t* sa = smem + s * kStage;
          mbar_expect_tx(&full_bar[s], (uint32_t)kStage);
          tma_load_2d(sa, &tmW, p.w_tiled ? 0 : kb * kBK, p.w_tiled ? wt_base + kb * 128 : tn_idx * 128, &full_bar[s]);
          tma_load_2d(sa + kWBytes, &tmX, kb * kBK, 0, &full_bar[s]);
          if (++s == stages) { s = 0; ph ^= 1u; }
        }
      }
    }
    return;
  }
  const int c = wg - 1, warp = tid >> 5, lane = tid & 31;
  int s = 0;
  uint32_t ph = 0;
  for (int unit = blockIdx.x; unit < num_units; unit += gridDim.x) {
    const int tn_idx = unit / p.splits, split = unit % p.splits;
    const int kb_begin = split * p.kb_per_split, kb_end = min(num_kb, kb_begin + p.kb_per_split);
    float acc[BT / 2];
    int prev = -1;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(&full_bar[s], ph);
      const uint32_t sa = smem_u32(smem + s * kStage);
      const uint64_t dw = make_wgmma_desc(sa + c * 64 * (kBK * 2));
      const uint64_t dx = make_wgmma_desc(sa + kWBytes);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < kBK / 16; ++k) Wgmma<BT>::mma(acc, dw + (uint64_t)(2 * k), dx + (uint64_t)(2 * k), (kb > kb_begin || k > 0) ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();
      if (prev >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
      }
      prev = s;
      if (++s == stages) { s = 0; ph ^= 1u; }
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[prev]);
    const bool partial = p.splits > 1 || p.rope_cos != nullptr;
    float* part = p.ws_partial + (size_t)split * (size_t)p.a_rows * (size_t)p.N;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t n = (int64_t)tn_idx * 128 + tile_col(c * 64 + warp * 16 + (lane >> 2) + 8 * h, p.w_perm);
      if (n >= p.N) continue;
      const float bias = p.bias ? __bfloat162float(p.bias[n]) : 0.f;
#pragma unroll
      for (int j = 0; j < BT / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t m = 8 * j + 2 * (lane & 3) + e;
          if (m >= p.a_rows) continue;
          const float a = acc[4 * j + 2 * h + e];
          if (partial) {
            part[m * p.N + n] = a;
            continue;
          }
          float v = a * p.alpha + bias;
          if (p.act == UVX_ACT_GELU) v = gelu_fast(v);
          if (p.R) v += __bfloat162float(p.R[m * p.r_row_stride + n]);
          reinterpret_cast<bf16*>(p.C)[m * p.c_row_stride + n] = __float2bfloat16_rn(v);
        }
      }
    }
  }
}

// Split-K second pass of the decode form with the fused RoPE: one thread sums 8 columns d .. d+7 of a head and their rotation
// partners d+64 .. d+71 in split order, rounds them to bf16 (what the GEMM would have stored) and rotates heads below rope_cols
// exactly like uvx_rope - the same bits as GEMM + reduce + uvx_rope.
__global__ void __launch_bounds__(256) splitk_reduce_rope_kernel(const GemmParams p) {
  pdl_trigger();
  pdl_wait();
  const int64_t heads = p.N / 128;
  const int64_t total = p.a_rows * heads * 8;
  const size_t split_stride = (size_t)p.a_rows * (size_t)p.N;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int64_t m = idx / (heads * 8), t = (idx / 8) % heads, g = idx % 8;
    const int64_t n1 = t * 128 + g * 8, n2 = n1 + 64;
    float v1[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, v2[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int sidx = 0; sidx < p.splits; ++sidx) {
      const float* src = p.ws_partial + sidx * split_stride + (size_t)m * p.N;
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        v1[e] += __ldcg(src + n1 + e);
        v2[e] += __ldcg(src + n2 + e);
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      v1[e] = __bfloat162float(__float2bfloat16_rn(v1[e] * p.alpha));
      v2[e] = __bfloat162float(__float2bfloat16_rn(v2[e] * p.alpha));
    }
    if (n1 < p.rope_cols) {
      const int64_t pos = p.rope_pos ? (int64_t)p.rope_pos[m] : p.rope_pos_offset + (m % p.rope_rows_per_seq);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        float o1, o2;
        rope_pair(v1[e], v2[e], p.rope_cos[pos * 64 + g * 8 + e], p.rope_sin[pos * 64 + g * 8 + e], o1, o2);
        v1[e] = o1;
        v2[e] = o2;
      }
    }
    bf16* crow = reinterpret_cast<bf16*>(p.C) + m * p.c_row_stride;
    *reinterpret_cast<bf16x8*>(crow + n1) = pack8(v1);
    *reinterpret_cast<bf16x8*>(crow + n2) = pack8(v2);
  }
}

// ---------------------------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static int encode_map(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                      const uint32_t* box, CUtensorMapL2promotion promo,
                      CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_BFLOAT16) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    set_error("cuTensorMapEncodeTiled entry point not available");
    return UVX_ERR_CUDA;
  }
  cuuint64_t gd[3];
  cuuint64_t gs[2];
  cuuint32_t bx[3], es[3];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i < rank - 1; ++i) gs[i] = strides_bytes[i];
  CUresult r = enc(tm, dtype, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, promo, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed with CUresult %d (rank %d dims %llu %llu stride %llu)", (int)r, rank,
              (unsigned long long)dims[0], (unsigned long long)dims[1], (unsigned long long)strides_bytes[0]);
    return UVX_ERR_CUDA;
  }
  return UVX_OK;
}

static int num_sms() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

static int g_gemm_stage_cap = 0;  // tuning only (uvx_debug_gemm_stages): upper bound on the ring depth
static int g_grid_cap = 0;        // tuning only (uvx_debug_gemm_ws grid): upper bound on the persistent grid
static int g_tma_store = -1;      // uvx_debug_gemm_tma_store: 0 = register epilogue everywhere, otherwise staged where it applies
static int g_split_ring = -1;     // uvx_debug_gemm_split_ring: 0 = one ring everywhere, n >= 2 = n activation slots, -1 = default

// after the main kernel: split-K reduce (fused RMSNorm where it applies) or the row norm of a direct epilogue
static int finish_gemm(const uvx_gemm_args* a, const GemmParams& p, cudaStream_t stream) {
  const bool want_norm = a->norm_w && a->norm_out;
  if (p.splits == 1) {
    if (!want_norm) return UVX_OK;
    // direct epilogue (tile-local): the row norm runs as its own kernel on the finished rows
    return uvx_rmsnorm(a->C, a->norm_w, a->norm_out, a->a_batch * a->a_rows, a->N, a->c_row_stride, 0, 0, 0, a->norm_eps, stream);
  }
  if (want_norm && !p.out_f32 && a->N <= 8192 && !a->c_row_map && a->act == UVX_ACT_NONE) {
    launch_k(splitk_reduce_rmsnorm_kernel, dim3((unsigned)(a->a_batch * a->a_rows)), dim3(256), 0, stream, p);
    return check_launch("splitk_reduce_rmsnorm_kernel");
  }
  const int64_t total = a->a_batch * a->a_rows * (a->N / 8);
  int64_t blocks = (total + 255) / 256;
  if (blocks > (int64_t)num_sms() * 8) blocks = (int64_t)num_sms() * 8;
  launch_k(splitk_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, p);
  int rc = check_launch("splitk_reduce_kernel");
  if (rc || !want_norm) return rc;
  return uvx_rmsnorm(a->C, a->norm_w, a->norm_out, a->a_batch * a->a_rows, a->N, a->c_row_stride, 0, 0, 0, a->norm_eps, stream);
}

// cluster shape (cm, cn) actually run for an (MT, BN) tiling: an axis whose tile count it does not divide, or whose operand box
// it cannot cut into whole 8-row swizzle atoms, falls back to 1; at most 8 CTAs (the portable cluster size)
static void legal_cluster(int mt, int bn, int tiles_m_total, int n_tiles, int* cm, int* cn) {
  if (*cm < 1 || *cm > 4 || tiles_m_total % *cm != 0 || bn % (8 * *cm) != 0) *cm = 1;
  if (*cn < 1 || *cn > 4 || n_tiles % *cn != 0 || (mt * 128) % (8 * *cn) != 0) *cn = 1;
  if (*cm * *cn > 8) *cm = *cn = 1;
}

template <int MT, int BN, bool STAGED>
static cudaError_t set_smem_attr() {
  if constexpr (STAGED && !(MT == 1 && BN <= 128)) return cudaErrorInvalidValue;
  else return cudaFuncSetAttribute(gemm_wg_kernel<MT, BN, STAGED>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal);
}

template <int MT, int BN>
static int launch_gemm(const uvx_gemm_args* a, int splits, int cm, int cn, cudaStream_t stream) {
  using L = WgLayout<MT, BN>;
  const int m_tiles = (int)((a->a_rows + MT * 128 - 1) / (MT * 128));
  const int n_tiles = (int)((a->N + BN - 1) / BN);
  legal_cluster(MT, BN, m_tiles * (int)a->a_batch, n_tiles, &cm, &cn);
  // Split ring (weight-streaming prefill: one m-tile covers every row of the single batch, and no cluster cuts the A box): the
  // A box holds only the rows that exist (rounded to a swizzle atom), and A and W get rings of their own.  The weight ring takes
  // what the activation ring leaves (<2, 128> at M = 201: 5 x 26 KB + 5 x 16 KB, against 4 stages of 32 + 16 KB in one ring).
  // The A box comes from L2, but its latency still needs a lead of 3 k-blocks (H100 80GB HBM3 at 700 W, gate|up at M = 201:
  // 123.9 / 116.9 us with 3 / 4 stages of one ring, 102.4 / 101.8 / 103.7 us with 4 / 5 / 6 A slots).  It runs where the W ring
  // gets deeper than the one ring: at 256 rows the box cannot shrink, 5 A slots leave 4 W slots, and gate|up takes 106.8 us
  // against 102.1 us in one ring.  Where two m-tiles share the W box through a cluster (q|k|v at 129..256 rows) one ring is
  // faster too (31.2 us, against 32.4 with 6 A slots).  scripts/prefill_gemm_ab.py measures these; DESIGN §3.
  const int box_rows = (int)((a->a_rows + 7) / 8 * 8);
  int split_a = g_split_ring > 0 ? (g_split_ring < kMaxAStages ? g_split_ring : kMaxAStages) : 5;
  if (split_a < 2) split_a = 2;
  int split_w = (L::kRingMax - split_a * box_rows * kBK * 2) / L::kWBytes;
  if (split_w > kMaxWStages) split_w = kMaxWStages;
  const bool split_ring = BN <= 128 && g_split_ring != 0 && a->a_batch == 1 && m_tiles == 1 && cn == 1 &&
                          (g_split_ring > 0 || split_w > L::kStages);
  const int a_box_rows = split_ring ? box_rows : MT * 128;
  CUtensorMap tmA, tmW;
  {
    uint64_t dims[3] = {(uint64_t)a->K, (uint64_t)a->a_rows, (uint64_t)a->a_batch};
    uint64_t st[2] = {(uint64_t)a->a_row_stride * 2, (uint64_t)(a->a_batch > 1 ? a->a_batch_stride : a->a_row_stride) * 2};
    uint32_t box[3] = {kBK, (uint32_t)(a_box_rows / cn), 1};  // a CTA loads its 1/cn share of the A box
    int rc = encode_map(&tmA, a->A, 3, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc) return rc;
  }
  const bool tiled = a->w_tiled != 0;
  if (tiled) {
    // pre-tiled image [n_tiles][K/64][BN][64] (built once by the host, ops.TiledWeight): a 2-D map over [rows, 64] whose BN-row
    // boxes are contiguous BN*128-byte runs of DRAM
    UVX_REQUIRE(a->w_tiled == BN && a->K % kBK == 0, "uvx_gemm_bf16: tiled weights need BN == tile rows and K %% 64 == 0");
    const uint64_t n_tiles_w = (uint64_t)((a->N + BN - 1) / BN);
    uint64_t dims[2] = {(uint64_t)kBK, n_tiles_w * (uint64_t)(a->K / kBK) * (uint64_t)BN};
    uint64_t st[1] = {(uint64_t)kBK * 2};
    uint32_t box[2] = {kBK, (uint32_t)(BN / cm)};  // and its 1/cm share of the W box
    int rc = encode_map(&tmW, a->W, 2, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
    uint64_t st[1] = {(uint64_t)a->w_row_stride * 2};
    uint32_t box[2] = {kBK, (uint32_t)(BN / cm)};
    int rc = encode_map(&tmW, a->W, 2, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.w_tiled = tiled ? 1 : 0;
  p.w_perm = a->w_perm == 1 ? 1 : 0;
  p.swiglu = a->act == UVX_ACT_SWIGLU ? (a->w_tiled == 128 ? 16 : 8) : 0;
  p.rope_cos = a->rope_cos;
  p.rope_sin = a->rope_sin;
  p.rope_pos = a->rope_positions;
  p.rope_rows_per_seq = a->rope_rows_per_seq > 0 ? a->rope_rows_per_seq : 1;
  p.rope_pos_offset = a->rope_pos_offset;
  p.rope_cols = a->rope_cos ? (int)a->rope_cols : 0;
  if (p.swiglu || p.rope_cos || p.w_perm) splits = 1;  // fused epilogues are tile-local: no split-K
  p.a_rows = a->a_rows;
  p.a_batch = a->a_batch;
  p.K = a->K;
  p.N = a->N;
  p.C = a->C;
  p.c_row_stride = a->c_row_stride;
  p.c_batch_rows = a->c_batch_rows;
  p.c_row_offset = a->c_row_offset;
  p.c_row_map = a->c_row_map;
  p.bias = (const bf16*)a->bias;
  p.R = (const bf16*)a->R;
  p.r_row_stride = a->r_row_stride;
  p.r_batch_stride = a->r_batch_stride;
  p.alpha = a->alpha;
  p.act = a->act;
  p.out_f32 = a->out_dtype == UVX_DT_F32;
  p.norm_w = (const bf16*)a->norm_w;
  p.norm_out = (bf16*)a->norm_out;
  p.norm_eps = a->norm_eps;
  p.m_tiles = m_tiles;
  p.n_tiles = n_tiles;
  p.num_tiles = p.m_tiles * (int)a->a_batch * p.n_tiles;
  p.cm = cm;
  p.cn = cn;
  p.a_box_rows = a_box_rows;
  const int num_kb = (int)((a->K + kBK - 1) / kBK);
  if (a->N % BN != 0) splits = 1;  // ragged column tiles exist only in the direct epilogue
  // split-K needs the caller's workspace: [splits][rows][N] fp32 partial sums
  const size_t per_split = (size_t)a->a_batch * (size_t)a->a_rows * (size_t)a->N * 4;
  while (splits > 1 && (!a->workspace || per_split * (size_t)splits > (size_t)a->workspace_bytes)) --splits;
  if (splits > num_kb) splits = num_kb;
  if (splits < 1) splits = 1;
  p.kb_per_split = (num_kb + splits - 1) / splits;
  p.splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;  // no empty split
  p.ws_partial = (float*)a->workspace;
  // Staged epilogue (output tile through shared memory, TMA store; the residual loaded by TMA ahead of the epilogue): the
  // tensor-bound calls (more than 256 rows, or a batch) with the plain epilogue on 128 x 64 / 128 x 128 tiles.  Same bits as
  // the register epilogue.  The tile's shared memory comes out of the ring (128 x 128 bf16: 7 -> 6 stages, fp32: 5).
  CUtensorMap tmC, tmR;
  memset(&tmC, 0, sizeof(tmC));
  memset(&tmR, 0, sizeof(tmR));
  const bool staged = MT == 1 && BN <= 128 && g_tma_store != 0 && (a->a_rows > 256 || a->a_batch > 1) && p.splits == 1 &&
                      cm * cn == 1 && !a->c_row_map && !p.swiglu && !p.rope_cos && !p.w_perm && !(a->norm_w && a->norm_out) &&
                      (!a->R || (!p.out_f32 && a->r_row_stride > 0 && (uintptr_t)a->R % 16 == 0));
  if (staged) {
    const uint64_t es = p.out_f32 ? 4 : 2;
    const uint64_t row_bytes = (uint64_t)a->c_row_stride * es;
    uint64_t dims[3] = {(uint64_t)a->N, (uint64_t)a->a_rows, (uint64_t)a->a_batch};
    uint64_t st[2] = {row_bytes, a->a_batch > 1 ? (uint64_t)a->c_batch_rows * row_bytes : row_bytes};
    uint32_t box[3] = {(uint32_t)(128 / es), 128, 1};
    int rc = encode_map(&tmC, (const char*)a->C + a->c_row_offset * (int64_t)row_bytes, 3, dims, st, box,
                        CU_TENSOR_MAP_L2_PROMOTION_NONE, p.out_f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16);
    if (rc) return rc;
    if (a->R) {
      // a residual shared by every batch (the conv stem's positional embedding) gets a map without the batch dimension
      p.r_bcast = a->a_batch == 1 || a->r_batch_stride == 0;
      uint64_t rdims[3] = {(uint64_t)a->N, (uint64_t)a->a_rows, p.r_bcast ? 1 : (uint64_t)a->a_batch};
      uint64_t rst[2] = {(uint64_t)a->r_row_stride * 2, (uint64_t)(p.r_bcast ? a->r_row_stride : a->r_batch_stride) * 2};
      uint32_t rbox[3] = {64, 128, 1};
      rc = encode_map(&tmR, a->R, 3, rdims, rst, rbox, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
      if (rc) return rc;
    }
    p.staged_bytes = BN / 64 * (p.out_f32 ? 2 : 1) * kPanelBytes;
  }
  int ring_bytes;
  if (split_ring) {
    // the MMAs' reads past the last activation slot (rows a_box_rows .. MT * 128 - 1) land in the weight ring
    const int a_bytes = a_box_rows * kBK * 2;
    p.a_stages = split_a;
    p.stages = split_w;
    if (g_gemm_stage_cap >= 2 && p.stages > g_gemm_stage_cap) p.stages = g_gemm_stage_cap;
    UVX_REQUIRE(p.stages >= 2 && (MT * 128 - a_box_rows) * kBK * 2 <= p.stages * L::kWBytes, "uvx_gemm_bf16: split ring does not fit");
    p.w_early = (a->flags & UVX_GEMM_W_STATIC) ? 1 : 0;
    ring_bytes = p.a_stages * a_bytes + p.stages * L::kWBytes;
  } else {
    p.stages = (L::kRingMax - p.staged_bytes) / L::kStageBytes;
    if (p.stages > L::kStages) p.stages = L::kStages;
    if (g_gemm_stage_cap >= 2 && p.stages > g_gemm_stage_cap) p.stages = g_gemm_stage_cap;
    ring_bytes = p.stages * L::kStageBytes;
  }
  const int smem = ring_bytes + p.staged_bytes + 1024 + kBarBytes;
  static bool attr_set[2] = {false, false};
  if (!attr_set[staged]) {
    cudaError_t e = staged ? set_smem_attr<MT, BN, true>() : set_smem_attr<MT, BN, false>();
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(gemm_wg_kernel<%d,%d,%d>, smem %d): %s", MT, BN, (int)staged, kSmemTotal, cudaGetErrorString(e));
      return UVX_ERR_CUDA;
    }
    attr_set[staged] = true;
  }
  // persistent grid: a whole number of clusters, no more than fit on the GPU at once (clusters stay inside one GPC, so with
  // 4-CTA clusters a few SMs stay idle)
  const int csize = cm * cn;
  const int units = p.num_tiles / csize * p.splits;
  int max_units = num_sms();
  if (csize > 1) {
    static int max_clusters[9] = {0};
    if (!max_clusters[csize]) {
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3((unsigned)csize);
      cfg.blockDim = dim3(kGemmThreads);
      cfg.dynamicSmemBytes = (size_t)smem;
      cudaLaunchAttribute attr;
      attr.id = cudaLaunchAttributeClusterDimension;
      attr.val.clusterDim.x = (unsigned)csize;
      attr.val.clusterDim.y = 1;
      attr.val.clusterDim.z = 1;
      cfg.attrs = &attr;
      cfg.numAttrs = 1;
      cudaError_t e = cudaOccupancyMaxActiveClusters(&max_clusters[csize], gemm_wg_kernel<MT, BN, false>, &cfg);
      if (e != cudaSuccess || max_clusters[csize] < 1) {
        set_error("cudaOccupancyMaxActiveClusters(gemm_wg_kernel<%d,%d>, %d CTAs): %s", MT, BN, csize,
                  e != cudaSuccess ? cudaGetErrorString(e) : "no cluster fits");
        max_clusters[csize] = 0;
        return UVX_ERR_CUDA;
      }
    }
    max_units = max_clusters[csize];
  }
  int clusters = units < max_units ? units : max_units;
  if (g_grid_cap > 0 && clusters * csize > g_grid_cap) clusters = g_grid_cap / csize > 1 ? g_grid_cap / csize : 1;
  const dim3 grid((unsigned)(clusters * csize));
  if (csize > 1)
    launch_k_cluster(gemm_wg_kernel<MT, BN, false>, grid, dim3(kGemmThreads), (size_t)smem, stream, (unsigned)csize, tmA, tmW, tmC, tmR, p);
  else if (staged)
    launch_k(gemm_wg_kernel<MT, BN, (MT == 1 && BN <= 128)>, grid, dim3(kGemmThreads), (size_t)smem, stream, tmA, tmW, tmC, tmR, p);
  else
    launch_k(gemm_wg_kernel<MT, BN, false>, grid, dim3(kGemmThreads), (size_t)smem, stream, tmA, tmW, tmC, tmR, p);
  int rc = check_launch("gemm_wg_kernel");
  if (rc) return rc;
  return finish_gemm(a, p, stream);
}

// Weight-streaming forms, for calls with a_batch == 1, a plain bf16 output and few rows (uvx_debug_gemm_ws / UVX_GEMM_WS):
//   a_rows <= 32   the decode form (gemm_swap_kernel): tokens on the wgmma N dimension, split-K over the weight stream;
//   a_rows <= 256  (mode 1 only) the single-pass form of gemm_wg_kernel: 128-wide tiles, one K pass per tile, no split-K.
static int g_ws_enable = -1;  // -1: UVX_GEMM_WS env or 2.  0 = never, 1 = both forms, 2 = the decode form only

static int gemm_ws_enabled() {
  if (g_ws_enable < 0) {
    const char* e = getenv("UVX_GEMM_WS");
    g_ws_enable = e ? atoi(e) : 2;
  }
  return g_ws_enable;
}

static bool gemm_ws_common(const uvx_gemm_args* a) {
  if (!gemm_ws_enabled() || (a->flags & 2)) return false;
  if (a->a_batch != 1 || a->out_dtype != UVX_DT_BF16 || a->c_row_map || a->c_row_offset != 0) return false;
  return a->w_tiled == 0 || a->w_tiled == 128;
}

static bool gemm_swap_eligible(const uvx_gemm_args* a) {
  if (!gemm_ws_common(a) || a->a_rows > 32 || a->act == UVX_ACT_SWIGLU) return false;
  return a->workspace && (size_t)a->workspace_bytes >= (size_t)a->a_rows * (size_t)a->N * 4;
}

static bool gemm_ws_eligible(const uvx_gemm_args* a) {
  return gemm_ws_common(a) && gemm_ws_enabled() == 1 && a->a_rows <= 256 && a->N % 128 == 0;
}

template <int BT>
static int launch_gemm_swap(const uvx_gemm_args* a, cudaStream_t stream) {
  constexpr int kStage = 128 * kBK * 2 + BT * kBK * 2;
  CUtensorMap tmX, tmW;
  {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->a_rows};
    uint64_t st[1] = {(uint64_t)a->a_row_stride * 2};
    uint32_t box[2] = {kBK, (uint32_t)BT};
    int rc = encode_map(&tmX, a->A, 2, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_128B);
    if (rc) return rc;
  }
  const int num_kb = (int)((a->K + kBK - 1) / kBK);
  const int n_tiles = (int)((a->N + 127) / 128);
  if (a->w_tiled) {
    UVX_REQUIRE(a->K % kBK == 0, "uvx_gemm_bf16: tiled weights need K %% 64 == 0");
    uint64_t dims[2] = {(uint64_t)kBK, (uint64_t)n_tiles * (uint64_t)num_kb * 128};
    uint64_t st[1] = {(uint64_t)kBK * 2};
    uint32_t box[2] = {kBK, 128};
    int rc = encode_map(&tmW, a->W, 2, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  } else {
    uint64_t dims[2] = {(uint64_t)a->K, (uint64_t)a->N};
    uint64_t st[1] = {(uint64_t)a->w_row_stride * 2};
    uint32_t box[2] = {kBK, 128};
    int rc = encode_map(&tmW, a->W, 2, dims, st, box, CU_TENSOR_MAP_L2_PROMOTION_L2_256B);
    if (rc) return rc;
  }
  GemmParams p;
  memset(&p, 0, sizeof(p));
  p.a_rows = a->a_rows;
  p.a_batch = 1;
  p.K = a->K;
  p.N = a->N;
  p.C = a->C;
  p.c_row_stride = a->c_row_stride;
  p.c_batch_rows = a->a_rows;
  p.bias = (const bf16*)a->bias;
  p.R = (const bf16*)a->R;
  p.r_row_stride = a->r_row_stride;
  p.r_batch_stride = a->r_batch_stride;
  p.alpha = a->alpha;
  p.act = a->act;
  p.norm_w = (const bf16*)a->norm_w;
  p.norm_out = (bf16*)a->norm_out;
  p.norm_eps = a->norm_eps;
  p.w_tiled = a->w_tiled ? 1 : 0;
  p.w_perm = a->w_perm == 1 ? 1 : 0;
  p.rope_cos = a->rope_cos;
  p.rope_sin = a->rope_sin;
  p.rope_pos = a->rope_positions;
  p.rope_rows_per_seq = a->rope_rows_per_seq > 0 ? a->rope_rows_per_seq : 1;
  p.rope_pos_offset = a->rope_pos_offset;
  p.rope_cols = a->rope_cos ? (int)a->rope_cols : 0;
  p.n_tiles = n_tiles;
  p.num_tiles = n_tiles;
  const int sms = num_sms();
  int splits = 1;
  if (n_tiles * 2 <= sms && num_kb >= 16) {   // spread the weight stream over the SMs (>= 8 k-blocks per split)
    splits = sms / n_tiles;
    if (splits > num_kb / 8) splits = num_kb / 8;
    if (splits > 16) splits = 16;
    if (splits < 1) splits = 1;
  }
  if (a->N % 8 != 0) splits = 1;
  const size_t per_split = (size_t)a->a_rows * (size_t)a->N * 4;
  while (splits > 1 && per_split * (size_t)splits > (size_t)a->workspace_bytes) --splits;
  p.kb_per_split = (num_kb + splits - 1) / splits;
  p.splits = (num_kb + p.kb_per_split - 1) / p.kb_per_split;
  p.ws_partial = (float*)a->workspace;
  p.stages = (kSmemTotal - 1024 - 256) / kStage;
  if (p.stages > kMaxStages) p.stages = kMaxStages;
  if (g_gemm_stage_cap >= 2 && p.stages > g_gemm_stage_cap) p.stages = g_gemm_stage_cap;
  const int smem = p.stages * kStage + 1024 + 2 * kMaxStages * 8;
  static bool attr_set = false;
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(gemm_swap_kernel<BT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemTotal);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(gemm_swap_kernel<%d>): %s", BT, cudaGetErrorString(e));
      return UVX_ERR_CUDA;
    }
    attr_set = true;
  }
  const int units = n_tiles * p.splits;
  int grid = units < sms ? units : sms;
  if (g_grid_cap > 0 && grid > g_grid_cap) grid = g_grid_cap;
  launch_k(gemm_swap_kernel<BT>, dim3((unsigned)grid), dim3(kGemmThreads), (size_t)smem, stream, tmX, tmW, p);
  int rc = check_launch("gemm_swap_kernel");
  if (rc) return rc;
  if (p.rope_cos) {   // the partial sums always go through the RoPE reduce pass
    const int64_t total = a->a_rows * (a->N / 128) * 8;
    const int64_t blocks = (total + 255) / 256;
    launch_k(splitk_reduce_rope_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, p);
    return check_launch("splitk_reduce_rope_kernel");
  }
  return finish_gemm(a, p, stream);
}

}  // namespace uvx

static int forced = -1, forced_splits = -1;

// tuning hook (scripts/gemm_sweep.py): force a tile config (MT*1000+BN, 0 = heuristic) and a split count (0 = heuristic)
extern "C" int uvx_debug_gemm_override(int cfg, int splits) {
  forced = cfg;
  forced_splits = splits;
  return UVX_OK;
}

// tuning hook: cap the shared-memory ring depth (0 = as deep as fits)
extern "C" int uvx_debug_gemm_stages(int n) {
  uvx::g_gemm_stage_cap = n;
  return UVX_OK;
}

// tuning hook of the weight-streaming forms: enable (0 = never, 1 = decode form for rows <= 32 and single-pass form up to 256 rows,
// 2 = decode form only; -1 = UVX_GEMM_WS env, default 2) and an upper bound on the persistent grid (0 = one CTA per SM); `mode` is
// accepted and ignored
extern "C" int uvx_debug_gemm_ws(int enable, int mode, int grid) {
  (void)mode;
  uvx::g_ws_enable = enable;
  uvx::g_grid_cap = grid > 0 ? grid : 0;
  return UVX_OK;
}

static int forced_cm = 0, forced_cn = 0;
static int g_cluster_enable = -1;  // -1: UVX_GEMM_CLUSTER env (0 = no clusters), default on

// tuning hook: thread-block cluster shape of gemm_wg_kernel, cm tiles along M x cn along N ((0, 0) = heuristic, (1, 1) = none);
// an axis that does not divide the tile grid falls back to 1
extern "C" int uvx_debug_gemm_cluster(int cm, int cn) {
  forced_cm = cm;
  forced_cn = cn;
  return UVX_OK;
}

// tuning hook: the staged (shared memory + TMA store) epilogue of the tensor-bound calls: 0 = register epilogue everywhere,
// -1 (default) or > 0 = staged wherever it applies.  Never changes the result bits.
extern "C" int uvx_debug_gemm_tma_store(int on) {
  uvx::g_tma_store = on;
  return UVX_OK;
}

// tuning hook: the split weight / activation ring of calls one m-tile covers: 0 = the one ring of A + W stages, n >= 2 = split
// with n activation slots (at most 8) wherever the shape allows, -1 (default) = split with 5 where the W ring gets deeper than
// the one ring (launch_gemm).  Never changes the result bits.
extern "C" int uvx_debug_gemm_split_ring(int a_stages) {
  uvx::g_split_ring = a_stages;
  return UVX_OK;
}

// Hooks of tuning knobs this kernel does not have (L2 prefetch distance, phase timestamps, pipeline isolation): accepted for ABI
// compatibility, no effect.
extern "C" int uvx_debug_gemm_mode(int mode) { (void)mode; return UVX_OK; }
extern "C" int uvx_debug_gemm_times(void* dev_buf) { (void)dev_buf; return UVX_OK; }
extern "C" int uvx_debug_gemm_pf(int pf) { (void)pf; return UVX_OK; }
extern "C" int uvx_debug_gemm_ws_times(void* dev_buf) { (void)dev_buf; return UVX_OK; }

static void read_forced() {
  if (forced < 0) {
    const char* e = getenv("UVX_GEMM_CFG");
    forced = e ? atoi(e) : 0;
    const char* s = getenv("UVX_GEMM_SPLITS");
    forced_splits = s ? atoi(s) : 0;
  }
}

// Tile / split selection for 132 SMs.  Row sub-tiles: MT = 2 when one CTA tile covers 129..256 rows of a single batch (every weight
// byte read once); the accumulators of an MT x BN tile must fit the consumers' registers, so MT = 2 pairs with BN <= 128.
static void pick_cfg(int64_t rows, int64_t batch, int64_t N, int64_t K, int sms, int* mt_out, int* bn_out, int* splits) {
  const int num_kb = (int)((K + 63) / 64);
  int mt, bn;
  if (rows <= 256 && batch == 1) {
    mt = rows > 128 ? 2 : 1;
    bn = N % 128 == 0 ? 128 : 64;
    // enough 128 x 128 tiles to fill most SMs without split-K: no reduce pass, and the same tiling as the fused-RoPE q|k|v GEMM;
    // unless 256 x 128 tiles alone fill every SM (gate|up): then one W read per tile instead of two is faster (same bits)
    if (bn == 128 && 2 * (N / 128) >= (sms * 3) / 5 && N / 128 < sms && num_kb <= 80) mt = 1;
  } else {
    // tensor-bound regime (encoder, training): 128-row tiles; 256 wide when that still fills one wave of SMs and K is long (the
    // Llama GEMMs of adapter training: the cfg3 step is ~3 % slower with them 128 wide).  With the 20 k-blocks of the Whisper
    // encoder (K = 1280) 128-wide tiles win (H100 at 400 W, T = 1500: q|k|v 1500 x 3840 63.6 -> 47.6 us, fc1 1500 x 5120
    // 80.5 -> 69.1 us)
    mt = 1;
    const int64_t m_tiles = (rows + 127) / 128 * batch;
    if (N % 256 == 0 && m_tiles * (N / 256) >= sms && num_kb >= 32) bn = 256;
    else bn = (N % 128 == 0 && m_tiles * (N / 128) >= sms / 2) ? 128 : 64;
  }
  const int64_t tiles = ((rows + mt * 128 - 1) / (mt * 128)) * batch * ((N + bn - 1) / bn);
  int sp = 1;
  if (tiles * 2 <= sms && num_kb >= 16) {  // too few tiles to occupy the SMs: split K (>= 8 k-blocks per split)
    sp = (int)(sms / tiles);
    if (sp > num_kb / 8) sp = num_kb / 8;
    if (sp > 16) sp = 16;
    if (sp < 1) sp = 1;
  }
  *mt_out = mt;
  *bn_out = bn;
  *splits = sp;
}

// Cluster shape for the final (MT, BN).  Prefill rows (<= 256, one batch) against a large weight: every CTA pulled its own copy of
// the A box for each k-block (2-3 bytes of L2 -> SM traffic per weight byte); multicast along N cuts the A share to 1/cn and
// along M lets 128-row tiles share one W read.  Chosen per tiling by scripts/gemm_cluster_sweep.py (DESIGN §3).  The
// tensor-bound regime (encoder, training) runs without clusters.
static void pick_cluster(int64_t rows, int64_t batch, int mt, int* cm, int* cn) {
  *cm = *cn = 1;
  if (g_cluster_enable < 0) {
    const char* e = getenv("UVX_GEMM_CLUSTER");
    g_cluster_enable = e ? atoi(e) : 1;
  }
  if (forced_cm > 0 || forced_cn > 0) {
    *cm = forced_cm > 0 ? forced_cm : 1;
    *cn = forced_cn > 0 ? forced_cn : 1;
    return;
  }
  if (!g_cluster_enable || rows > 256 || batch != 1) return;
  // H100 80GB HBM3 at 400 W, M = 201, us per call (scripts/gemm_cluster_sweep.py; (cm, cn) = (1, 1) first):
  //   q|k|v  6144 x 4096  MT 1: 42.2 | (2,1) 36.5 | (2,2) 33.9 | (1,2) 41.5 | (1,4) 34.9
  //   gate|up 28672 x 4096 MT 2: 135.9 | (1,2) 148.6 | (1,4) 137.4   (MT 1: 169.6 | (2,2) 141.9)
  //   o 4096 x 4096 MT 2 split 4: 34.5 | (1,2) 35.2 | (1,4) 48.0;  down 4096 x 14336 MT 2 split 4: 81.1 | (1,2) 76.8 | (1,4) 126.8
  // so two 128-row tiles share both boxes; 256-row tiles (W already read once per tile) run without a cluster
  if (mt == 1 && rows > 128) {
    *cm = 2;
    *cn = 2;
  }
}

extern "C" int uvx_gemm_bf16(const uvx_gemm_args* a, uvx_stream_t stream_) {
  using namespace uvx;
  cudaStream_t stream = (cudaStream_t)stream_;
  UVX_REQUIRE(a && a->A && a->W && a->C, "uvx_gemm_bf16: null pointer");
  UVX_REQUIRE(a->a_batch >= 1 && a->a_rows >= 1 && a->K >= 8 && a->N >= 64, "uvx_gemm_bf16: empty problem");
  UVX_REQUIRE(a->K % 8 == 0 && a->N % 64 == 0, "uvx_gemm_bf16: K %% 8 and N %% 64 required (K=%lld N=%lld)",
              (long long)a->K, (long long)a->N);
  UVX_REQUIRE(a->a_row_stride % 8 == 0 && a->w_row_stride % 8 == 0 && (a->a_batch == 1 || a->a_batch_stride % 8 == 0),
              "uvx_gemm_bf16: strides must be multiples of 8 elements");
  UVX_REQUIRE(((uintptr_t)a->A % 16 == 0) && ((uintptr_t)a->W % 16 == 0) && ((uintptr_t)a->C % 16 == 0),
              "uvx_gemm_bf16: 16-byte aligned bases required");
  UVX_REQUIRE(a->c_row_stride % 8 == 0 && (!a->R || (a->r_row_stride % 8 == 0 && a->r_batch_stride % 8 == 0)),
              "uvx_gemm_bf16: output / residual strides must be multiples of 8");
  UVX_REQUIRE(a->a_rows < (1ll << 31) && a->K < (1ll << 31) && a->N < (1ll << 31), "uvx_gemm_bf16: dimension too large");
  UVX_REQUIRE(!a->workspace || (uintptr_t)a->workspace % 256 == 0, "uvx_gemm_bf16: workspace must be 256-byte aligned");
  UVX_REQUIRE(!(a->norm_w && a->norm_out) || (a->out_dtype == UVX_DT_BF16 && !a->c_row_map && a->c_row_offset == 0 &&
                                              (a->a_batch == 1 || a->c_batch_rows == a->a_rows)),
              "uvx_gemm_bf16: fused RMSNorm needs a plain bf16 output");
  UVX_REQUIRE(a->w_tiled == 0 || a->w_tiled == 64 || a->w_tiled == 128 || a->w_tiled == 208 || a->w_tiled == 256,
              "uvx_gemm_bf16: w_tiled must be 64 / 128 / 208 / 256");
  UVX_REQUIRE(a->w_perm == 0 || (a->w_perm == 1 && a->w_tiled == 128 && a->N % 128 == 0 && a->act != UVX_ACT_SWIGLU),
              "uvx_gemm_bf16: the pair-permuted image (w_perm = 1) is a 128-row image of whole heads");
  UVX_REQUIRE(a->act != UVX_ACT_SWIGLU || (a->w_tiled != 0 && !a->bias && !a->R && !a->norm_w && a->out_dtype == UVX_DT_BF16 &&
                                           a->N % (a->w_tiled == 128 ? 32 : 16) == 0),
              "uvx_gemm_bf16: UVX_ACT_SWIGLU needs the interleaved gate|up image, bf16 output, no bias / residual / norm");
  UVX_REQUIRE(!a->rope_cos || (a->rope_sin && a->a_batch == 1 && a->alpha == 1.0f && !a->bias && !a->R && a->act == UVX_ACT_NONE &&
                               a->rope_cols % 128 == 0 && (a->w_tiled == 0 || a->w_tiled == 128) && a->N % 128 == 0),
              "uvx_gemm_bf16: fused RoPE needs head_dim 128 tiles, a_batch 1, no bias / residual / activation");
  read_forced();
  const int sms = num_sms();
  int mt, bn, splits;
  pick_cfg(a->a_rows, a->a_batch, a->N, a->K, sms, &mt, &bn, &splits);
  if (forced <= 0 && forced_splits <= 0 && gemm_swap_eligible(a)) {
    if (a->a_rows <= 8) return launch_gemm_swap<8>(a, stream);
    if (a->a_rows <= 16) return launch_gemm_swap<16>(a, stream);
    return launch_gemm_swap<32>(a, stream);
  }
  const bool ws = forced <= 0 && forced_splits <= 0 && gemm_ws_eligible(a);
  if (ws) {
    mt = 1;
    bn = 128;
    splits = 1;
  } else if (forced > 0) {
    // forced MT*1000 + BN; tile widths that do not divide N fall back to the heuristic's
    const int fb = forced % 1000, fm = forced / 1000;
    if (fb == 64 || fb == 128 || fb == 208 || fb == 256) {
      if (a->N % fb == 0 || fb == 208) bn = fb;
      mt = fm == 2 ? 2 : 1;
    }
  }
  if (forced_splits > 0 && !ws) splits = forced_splits;
  if (a->w_tiled) bn = (int)a->w_tiled;  // the image was cut for one tile width: that width is the configuration
  if (a->rope_cos) {                     // one 128-wide head per tile, both rotation halves in the same accumulator row
    mt = 1;
    bn = 128;
  }
  if (bn > 128) mt = 1;                  // register budget of the consumers
  int cm, cn;
  pick_cluster(a->a_rows, a->a_batch, mt, &cm, &cn);
  switch (mt * 1000 + bn) {
    case 1064: return launch_gemm<1, 64>(a, splits, cm, cn, stream);
    case 1128: return launch_gemm<1, 128>(a, splits, cm, cn, stream);
    case 1208: return launch_gemm<1, 208>(a, splits, cm, cn, stream);
    case 1256: return launch_gemm<1, 256>(a, splits, cm, cn, stream);
    case 2064: return launch_gemm<2, 64>(a, splits, cm, cn, stream);
    case 2128: return launch_gemm<2, 128>(a, splits, cm, cn, stream);
    default: return launch_gemm<1, 64>(a, splits, cm, cn, stream);
  }
}
