// uvx_attention: fused softmax(Q K^T * scale + mask) V, flash style (online softmax, fp32 statistics).
//
// Round-1 implementation: 64-query x 64-key tiles, 4 warps, K/V double-buffered in shared memory with
// cp.async, bf16 mma.sync.m16n8k16 with fp32 accumulators, ldmatrix operand fetch.  Masks are computed from
// indices (key length per clip, causal offset, block-causal streaming) - no dense mask tensor is read, and
// key tiles that are fully masked are skipped.  Serves the Whisper encoder (head_dim 64, uvx_attention_enc_tc),
// the Llama prefill / training attention (head_dim 128) and the single-token decode steps.
#include <stdlib.h>

#include <type_traits>

#include "uvx_common.cuh"

namespace uvx {

static constexpr int kAM = 64;  // queries per CTA
static constexpr int kAN = 64;  // keys per tile
static constexpr int kAThreads = 128;

struct AttnParams {
  const bf16 *q, *k, *v;
  bf16* o;
  int64_t q_rs, q_bs, k_rs, k_bs, v_rs, v_bs, o_rs, o_bs;
  const int32_t* kv_len;
  const int32_t* kv_start;  // optional [B]: keys before it are masked (left-padded batches)
  float* lse;  // optional [B, Hq, Sq]: natural-log sum-exp of the scaled scores (for the backward)
  int Sq, Skv, group, Hq;  // group = Hq / Hkv
  int causal, block;
  float scale_log2;  // scale * log2(e)
};

// Paged form: k / v address a pool layer [n_pages, 64, Hkv, D]; key tile t of batch row b is page table[b * table_stride + t]
// (k_bs / v_bs are the page strides, k_rs / v_rs the row strides inside a page).
struct PagedAttnParams : AttnParams {
  const int32_t* table;
  int64_t table_stride;
};

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(dst);
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(d), "l"(src), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void ldsm_x4(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];" : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(a));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3, const void* p) {
  const uint32_t a = (uint32_t)__cvta_generic_to_shared(p);
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3)
               : "r"(a));
}
__device__ __forceinline__ void mma_bf16(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

template <int D, bool kPaged = false>
__global__ void __launch_bounds__(kAThreads) attn_fwd_kernel(const std::conditional_t<kPaged, PagedAttnParams, AttnParams> p) {
  pdl_trigger();
  pdl_wait();
  constexpr int LD = D + 8;  // padded row (bf16 elements): 16-byte aligned, conflict-free ldmatrix
  extern __shared__ __align__(16) uint8_t attn_smem[];
  bf16* sQ = reinterpret_cast<bf16*>(attn_smem);
  bf16* sK = sQ + kAM * LD;       // 2 stages
  bf16* sV = sK + 2 * kAN * LD;   // 2 stages

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int g = lane >> 2, t4 = lane & 3;
  const int m0 = blockIdx.x * kAM;
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / p.group;
  const bf16* qb = p.q + (int64_t)b * p.q_bs + (int64_t)h * D;
  const bf16* kb = p.k + (kPaged ? 0 : (int64_t)b * p.k_bs) + (int64_t)hk * D;
  const bf16* vb = p.v + (kPaged ? 0 : (int64_t)b * p.v_bs) + (int64_t)hk * D;

  int kv_end = p.Skv;
  if (p.kv_len) kv_end = min(kv_end, max(p.kv_len[b], 0));
  const int shift = p.Skv - p.Sq;
  const int last_q = min(m0 + kAM, p.Sq) - 1;
  if (p.causal) kv_end = min(kv_end, last_q + shift + 1);
  if (p.block > 0) kv_end = min(kv_end, (last_q / p.block + 1) * p.block);
  const int kv_begin = p.kv_start ? min(max(p.kv_start[b], 0), kv_end) : 0;
  const int tile0 = kv_begin / kAN;  // tiles entirely in the left padding are skipped
  const int n_tiles = (kv_end + kAN - 1) / kAN;

  constexpr int CH = D / 8;  // 16-byte chunks per row
  auto load_q = [&]() {
    for (int i = tid; i < kAM * CH; i += kAThreads) {
      const int r = i / CH, c = i % CH;
      const bool ok = (m0 + r) < p.Sq;
      cp_async16(sQ + r * LD + c * 8, qb + (int64_t)(ok ? m0 + r : 0) * p.q_rs + c * 8, ok);
    }
  };
  auto load_kv = [&](int tile, int stage) {
    const int n0 = tile * kAN;
    bf16* dk = sK + stage * kAN * LD;
    bf16* dv = sV + stage * kAN * LD;
    if constexpr (kPaged) {
      // the tile is one page: row r of the tile is row r of the page (only tiles below kv_end are ever looked up)
      const int64_t pg = p.table[(int64_t)b * p.table_stride + tile];
      const bf16* kp = kb + pg * p.k_bs;
      const bf16* vp = vb + pg * p.v_bs;
      for (int i = tid; i < kAN * CH; i += kAThreads) {
        const int r = i / CH, c = i % CH;
        const bool ok = (n0 + r) < kv_end;
        const int64_t row = ok ? r : 0;
        cp_async16(dk + r * LD + c * 8, kp + row * p.k_rs + c * 8, ok);
        cp_async16(dv + r * LD + c * 8, vp + row * p.v_rs + c * 8, ok);
      }
    } else {
      for (int i = tid; i < kAN * CH; i += kAThreads) {
        const int r = i / CH, c = i % CH;
        // rows outside [kv_begin, kv_end) are zero-filled, never read: the cache tail past a sequence's length may hold
        // anything (torch.empty), and a masked probability of 0 times a NaN/Inf V row would still poison P.V
        const bool ok = (n0 + r) < kv_end && (n0 + r) >= kv_begin;
        const int64_t row = ok ? n0 + r : 0;
        cp_async16(dk + r * LD + c * 8, kb + row * p.k_rs + c * 8, ok);
        cp_async16(dv + r * LD + c * 8, vb + row * p.v_rs + c * 8, ok);
      }
    }
  };

  load_q();
  if (n_tiles > tile0) load_kv(tile0, 0);
  cp_async_commit();

  float o_acc[D / 8][4];
#pragma unroll
  for (int i = 0; i < D / 8; ++i) o_acc[i][0] = o_acc[i][1] = o_acc[i][2] = o_acc[i][3] = 0.f;
  float row_m[2] = {-INFINITY, -INFINITY}, row_l[2] = {0.f, 0.f};
  uint32_t qf[D / 16][4];
  const int qrow0 = m0 + warp * 16 + g;  // this thread's rows: qrow0 and qrow0 + 8

  for (int tile = tile0; tile < n_tiles; ++tile) {
    const int stage = (tile - tile0) & 1;
    if (tile + 1 < n_tiles) load_kv(tile + 1, stage ^ 1);
    cp_async_commit();
    cp_async_wait<1>();
    __syncthreads();
    if (tile == tile0) {
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk)
        ldsm_x4(qf[kk][0], qf[kk][1], qf[kk][2], qf[kk][3], sQ + (warp * 16 + (lane & 15)) * LD + kk * 16 + (lane >> 4) * 8);
    }
    const bf16* tk = sK + stage * kAN * LD;
    const bf16* tv = sV + stage * kAN * LD;

    float s[kAN / 8][4];
#pragma unroll
    for (int i = 0; i < kAN / 8; ++i) s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f;
#pragma unroll
    for (int kk = 0; kk < D / 16; ++kk) {
#pragma unroll
      for (int nb = 0; nb < kAN / 16; ++nb) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4(b0, b1, b2, b3, tk + (nb * 16 + (lane >> 4) * 8 + (lane & 7)) * LD + kk * 16 + ((lane >> 3) & 1) * 8);
        mma_bf16(s[2 * nb], qf[kk], b0, b1);
        mma_bf16(s[2 * nb + 1], qf[kk], b2, b3);
      }
    }

    // ---- mask + online softmax (scores kept unscaled; scale folded into the exp2 argument)
    const int n0 = tile * kAN;
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nb = 0; nb < kAN / 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = n0 + nb * 8 + t4 * 2 + (e & 1);
        const int qr = qrow0 + (e >> 1) * 8;
        bool ok = key < kv_end && key >= kv_begin;
        if (p.causal) ok = ok && (key <= qr + shift);
        if (p.block > 0) ok = ok && (key / p.block <= qr / p.block);
        if (!ok) s[nb][e] = -INFINITY;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], s[nb][e]);
      }
    }
    float corr[2], mref[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 1));
      tmax[r] = fmaxf(tmax[r], __shfl_xor_sync(0xffffffffu, tmax[r], 2));
      const float m_new = fmaxf(row_m[r], tmax[r]);
      mref[r] = (m_new == -INFINITY) ? 0.f : m_new;
      corr[r] = exp2f((row_m[r] - mref[r]) * p.scale_log2);  // row_m = -inf -> 0
      row_m[r] = m_new;
      row_l[r] *= corr[r];
    }
    float psum[2] = {0.f, 0.f};
#pragma unroll
    for (int nb = 0; nb < kAN / 8; ++nb) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float pv = exp2f((s[nb][e] - mref[e >> 1]) * p.scale_log2);
        s[nb][e] = pv;
        psum[e >> 1] += pv;
      }
    }
    row_l[0] += psum[0];
    row_l[1] += psum[1];
#pragma unroll
    for (int i = 0; i < D / 8; ++i) {
      o_acc[i][0] *= corr[0];
      o_acc[i][1] *= corr[0];
      o_acc[i][2] *= corr[1];
      o_acc[i][3] *= corr[1];
    }

    // ---- O += P V
#pragma unroll
    for (int ks = 0; ks < kAN / 16; ++ks) {
      uint32_t pa[4];
      pa[0] = pack_bf16(s[2 * ks][0], s[2 * ks][1]);
      pa[1] = pack_bf16(s[2 * ks][2], s[2 * ks][3]);
      pa[2] = pack_bf16(s[2 * ks + 1][0], s[2 * ks + 1][1]);
      pa[3] = pack_bf16(s[2 * ks + 1][2], s[2 * ks + 1][3]);
#pragma unroll
      for (int db = 0; db < D / 16; ++db) {
        uint32_t b0, b1, b2, b3;
        ldsm_x4_t(b0, b1, b2, b3, tv + (ks * 16 + ((lane >> 3) & 1) * 8 + (lane & 7)) * LD + db * 16 + (lane >> 4) * 8);
        mma_bf16(o_acc[2 * db], pa, b0, b1);
        mma_bf16(o_acc[2 * db + 1], pa, b2, b3);
      }
    }
    __syncthreads();  // everyone done with this stage before it is refilled
  }
  cp_async_wait<0>();

  // ---- finalize: divide by the row sum (quad-reduced) and store
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    row_l[r] += __shfl_xor_sync(0xffffffffu, row_l[r], 1);
    row_l[r] += __shfl_xor_sync(0xffffffffu, row_l[r], 2);
  }
  if (p.lse && t4 == 0) {
    float* lp = p.lse + ((int64_t)b * p.Hq + h) * p.Sq;
    const float ln2 = 0.6931471805599453f;
    if (qrow0 < p.Sq) lp[qrow0] = row_m[0] * p.scale_log2 * ln2 + logf(row_l[0]);
    if (qrow0 + 8 < p.Sq) lp[qrow0 + 8] = row_m[1] * p.scale_log2 * ln2 + logf(row_l[1]);
  }
  const float inv0 = row_l[0] > 0.f ? 1.f / row_l[0] : 0.f;
  const float inv1 = row_l[1] > 0.f ? 1.f / row_l[1] : 0.f;
  bf16* ob = p.o + (int64_t)b * p.o_bs + (int64_t)h * D;
#pragma unroll
  for (int i = 0; i < D / 8; ++i) {
    const int col = i * 8 + t4 * 2;
    if (qrow0 < p.Sq)
      *reinterpret_cast<uint32_t*>(ob + (int64_t)qrow0 * p.o_rs + col) = pack_bf16(o_acc[i][0] * inv0, o_acc[i][1] * inv0);
    if (qrow0 + 8 < p.Sq)
      *reinterpret_cast<uint32_t*>(ob + (int64_t)(qrow0 + 8) * p.o_rs + col) = pack_bf16(o_acc[i][2] * inv1, o_acc[i][3] * inv1);
  }
}

template <int D, bool kPaged = false>
static int launch_attn(const uvx_attn_args* a, cudaStream_t st, const int32_t* table = nullptr, int64_t table_stride = 0) {
  constexpr int LD = D + 8;
  const size_t smem = (size_t)(kAM + 4 * kAN) * LD * 2;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_fwd_kernel<D, kPaged>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attn_fwd_kernel<%d>): %s", D, cudaGetErrorString(e));
      return UVX_ERR_CUDA;
    }
    attr = true;
  }
  std::conditional_t<kPaged, PagedAttnParams, AttnParams> p;
  if constexpr (kPaged) {
    p.table = table;
    p.table_stride = table_stride;
  }
  p.q = (const bf16*)a->q;
  p.k = (const bf16*)a->k;
  p.v = (const bf16*)a->v;
  p.o = (bf16*)a->o;
  p.q_rs = a->q_rs; p.q_bs = a->q_bs; p.k_rs = a->k_rs; p.k_bs = a->k_bs;
  p.v_rs = a->v_rs; p.v_bs = a->v_bs; p.o_rs = a->o_rs; p.o_bs = a->o_bs;
  p.kv_len = a->kv_len;
  p.kv_start = a->kv_start;
  p.lse = a->lse;
  p.Hq = (int)a->Hq;
  p.Sq = (int)a->Sq;
  p.Skv = (int)a->Skv;
  p.group = (int)(a->Hq / a->Hkv);
  p.causal = a->causal;
  p.block = a->block;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  dim3 grid((unsigned)((a->Sq + kAM - 1) / kAM), (unsigned)a->Hq, (unsigned)a->B);
  launch_k(attn_fwd_kernel<D, kPaged>, dim3(grid), dim3(kAThreads), smem, st, p);
  return check_launch("attn_fwd_kernel");
}

int launch_attn_wg(const uvx_attn_args* a, cudaStream_t st);  // attention_wg.cu (TMA + wgmma, a tile of queries per head)
bool attn_wg_eligible(const uvx_attn_args* a);
static int g_attn_wg = -1;  // UVX_ATTN_TC=0 keeps every shape on the mma.sync kernel (A/B runs, tests)

}  // namespace uvx

// tuning hook: 1 = wgmma kernel for every shape with a tile of queries per head (default), 0 = mma.sync kernel everywhere,
// -1 = UVX_ATTN_TC / default
extern "C" int uvx_debug_attn_tc(int on) {
  uvx::g_attn_wg = on;
  return UVX_OK;
}

extern "C" int uvx_attention(const uvx_attn_args* a, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(a && a->q && a->k && a->v && a->o, "uvx_attention: null pointer");
  UVX_REQUIRE(a->D == 64 || a->D == 128, "uvx_attention: head_dim must be 64 or 128 (got %lld)", (long long)a->D);
  UVX_REQUIRE(a->B >= 1 && a->Hq >= 1 && a->Hkv >= 1 && a->Hq % a->Hkv == 0 && a->Sq >= 1 && a->Skv >= 1,
              "uvx_attention: bad shape");
  UVX_REQUIRE(a->B < 65536 && a->Hq < 65536, "uvx_attention: grid too large");
  UVX_REQUIRE(a->q_rs % 8 == 0 && a->k_rs % 8 == 0 && a->v_rs % 8 == 0 && a->o_rs % 2 == 0 && a->q_bs % 8 == 0 &&
                  a->k_bs % 8 == 0 && a->v_bs % 8 == 0,
              "uvx_attention: strides must keep 16-byte alignment");
  UVX_REQUIRE(((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) % 16 == 0 && (uintptr_t)a->o % 4 == 0,
              "uvx_attention: base pointers must be 16-byte aligned");
  if (g_attn_wg < 0) {
    const char* e = getenv("UVX_ATTN_TC");
    g_attn_wg = e ? atoi(e) : 1;
  }
  // prefill / training / encoder shapes (a tile of queries per head): TMA + wgmma kernel; single-token decode steps stay on the
  // mma.sync kernel below
  if (g_attn_wg && attn_wg_eligible(a)) return launch_attn_wg(a, (cudaStream_t)stream);
  return a->D == 64 ? launch_attn<64>(a, (cudaStream_t)stream) : launch_attn<128>(a, (cudaStream_t)stream);
}

extern "C" int uvx_attention_paged(const uvx_attn_args* a, const int32_t* table, int64_t table_stride, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(a && a->q && a->k && a->v && a->o && a->kv_len && table, "uvx_attention_paged: null pointer");
  UVX_REQUIRE(a->D == 64 || a->D == 128, "uvx_attention_paged: head_dim must be 64 or 128 (got %lld)", (long long)a->D);
  UVX_REQUIRE(a->B >= 1 && a->B < 65536 && a->Hq >= 1 && a->Hq < 65536 && a->Hkv >= 1 && a->Hq % a->Hkv == 0 && a->Sq >= 1 &&
                  a->Skv >= 1,
              "uvx_attention_paged: bad shape");
  UVX_REQUIRE(table_stride >= (a->Skv + kAN - 1) / kAN, "uvx_attention_paged: a table row of %lld pages cannot cover Skv = %lld",
              (long long)table_stride, (long long)a->Skv);
  UVX_REQUIRE(!a->kv_start && !a->lse && a->block == 0 && (!a->causal || a->Sq == 1),
              "uvx_attention_paged: no kv_start, no lse, no block mask, causal only with Sq == 1");
  UVX_REQUIRE(a->k_bs == (int64_t)kAN * a->k_rs && a->v_bs == (int64_t)kAN * a->v_rs,
              "uvx_attention_paged: k_bs / v_bs must be one page of 64 rows");
  UVX_REQUIRE(a->q_rs % 8 == 0 && a->k_rs % 8 == 0 && a->v_rs % 8 == 0 && a->o_rs % 2 == 0 && a->q_bs % 8 == 0,
              "uvx_attention_paged: strides must keep 16-byte alignment");
  UVX_REQUIRE(((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) % 16 == 0 && (uintptr_t)a->o % 4 == 0,
              "uvx_attention_paged: base pointers must be 16-byte aligned");
  return a->D == 64 ? launch_attn<64, true>(a, (cudaStream_t)stream, table, table_stride)
                    : launch_attn<128, true>(a, (cudaStream_t)stream, table, table_stride);
}

// Whisper-encoder entry over the fused projection: qkv [B*S, row_stride] with head h's q / k / v at columns q_col + 64h,
// k_col + 64h, v_col + 64h; output o[b*S + i, 64h .. 64h+63].  Same dispatch and masks as uvx_attention (non-causal, key length
// per clip, optional block-causal streaming mask), addressed through strides - no copy of q / k / v.
extern "C" int uvx_attention_enc_tc(const void* qkv, int64_t row_stride, int64_t B, int64_t S, int64_t H, int64_t q_col,
                                    int64_t k_col, int64_t v_col, void* o, int64_t o_rs, const int32_t* kv_len, int32_t block,
                                    float scale, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(qkv && o, "uvx_attention_enc_tc: null pointer");
  UVX_REQUIRE(B >= 1 && B < 65536 && H >= 1 && H < 65536 && S >= 1, "uvx_attention_enc_tc: bad shape");
  UVX_REQUIRE(row_stride % 8 == 0 && o_rs % 8 == 0 && q_col % 8 == 0 && k_col % 8 == 0 && v_col % 8 == 0 &&
                  (uintptr_t)qkv % 16 == 0 && (uintptr_t)o % 16 == 0,
              "uvx_attention_enc_tc: alignment");
  const bf16* base = (const bf16*)qkv;
  uvx_attn_args a;
  memset(&a, 0, sizeof(a));
  a.q = base + q_col;
  a.k = base + k_col;
  a.v = base + v_col;
  a.o = o;
  a.B = B;
  a.Hq = a.Hkv = H;
  a.Sq = a.Skv = S;
  a.D = 64;
  a.q_rs = a.k_rs = a.v_rs = row_stride;
  a.q_bs = a.k_bs = a.v_bs = S * row_stride;
  a.o_rs = o_rs;
  a.o_bs = S * o_rs;
  a.kv_len = kv_len;
  a.block = block;
  a.scale = scale;
  return uvx_attention(&a, stream);
}
