// Flash attention on the Hopper tensor cores (TMA + mbarrier + wgmma), head_dim 64 or 128: the Whisper encoder (non-causal, key
// length / block-causal masks) and the Llama prefill / training forward (causal GQA, optional LSE, left padding).
//
// One warpgroup per CTA owns 64 queries of one head.  Thread 0 loads the Q tile once and double-buffers 64-key K / V tiles with
// 4-D TMA boxes {64 d, 1 head, 64 rows, 1 batch} (128B swizzle, one box per 64-wide d panel) on mbarriers.  S = Q K^T is
// wgmma m64n64k16 with both operands K-major in shared memory; the online softmax (fp32, scores unscaled, scale folded into the
// exp2 argument) runs on the accumulator registers; O += P V is wgmma m64nDk16 with P straight from registers (the accumulator
// fragment re-packed to bf16 is the A fragment) and V read MN-major from the same TMA layout.  Masks come from indices; key tiles
// outside [kv_start, kv_len) / above the causal diagonal are never loaded, and V rows of a partly valid tile that lie outside
// that range are zeroed in shared memory (a cache tail may hold anything, and 0 * NaN would still poison P V).
#include <type_traits>

#include "uvx_common.cuh"
#include "tc_ptx.cuh"

namespace uvx {

struct AttnWgParams {
  bf16* o;
  int64_t o_rs, o_bs;
  const int32_t* kv_len;
  const int32_t* kv_start;
  float* lse;
  int Sq, Skv, group, Hq;
  int causal, block;
  float scale_log2;
  const int32_t* kv_row;  // device-indexed form: K / V batch coordinate of query batch b
  const int32_t* past;    // device-indexed form: causal shift (keys already in the cache) of query batch b
};

// Paged device-indexed form: kv_row[b] is a row of the page table, and key tile t lives in page table[kv_row[b] * table_stride + t]
// of the pool layer the K / V tensor maps cover as {D, Hkv, 64, n_pages}.
struct AttnWgPagedParams : AttnWgParams {
  const int32_t* table;
  int64_t table_stride;
};

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  __nv_bfloat162 t = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&t);
}

static constexpr int kWQ = 64;          // queries per CTA
static constexpr int kWK = 64;          // keys per tile
static constexpr int kPanel = 64 * 128;  // one 64-row x 64-d panel, 128B swizzled

template <int D>
struct AttnWgSmem {
  static constexpr int kP = D / 64;                   // d panels
  static constexpr int kQ = 0;
  static constexpr int kK = kQ + kP * kPanel;         // 2 stages
  static constexpr int kV = kK + 2 * kP * kPanel;     // 2 stages
  static constexpr int kBar = kV + 2 * kP * kPanel;
  static constexpr int kBytes = kBar + 64 + 1024;     // + barriers + alignment slack
};

// kIndexed: the K / V batch coordinate and the causal shift come from device memory (p.kv_row[b], p.past[b]) instead of b and
// Skv - Sq, so one captured launch serves whichever cache row and prompt offset the host writes between replays.
template <int D, bool kIndexed = false, bool kPaged = false>
__global__ void __launch_bounds__(128, 1)
attn_wg_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
               const std::conditional_t<kPaged, AttnWgPagedParams, AttnWgParams> p) {
  static_assert(!kPaged || kIndexed, "the paged form is device-indexed");
  using L = AttnWgSmem<D>;
  constexpr int P = L::kP;
  pdl_trigger();
  extern __shared__ uint8_t attn_wg_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)attn_wg_raw + 1023) & ~(uintptr_t)1023);
  uint64_t* full = (uint64_t*)(smem + L::kBar);   // [0], [1]: K/V stages; [2]: Q
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int m0 = blockIdx.x * kWQ;
  const int h = blockIdx.y, b = blockIdx.z;
  const int hk = h / p.group;
  const int kb = kIndexed ? p.kv_row[b] : b;

  int kv_end = p.Skv;
  if (p.kv_len) kv_end = min(kv_end, max(p.kv_len[b], 0));
  const int shift = kIndexed ? p.past[b] : p.Skv - p.Sq;
  const int last_q = min(m0 + kWQ, p.Sq) - 1;
  if (p.causal) kv_end = min(kv_end, last_q + shift + 1);
  if (p.block > 0) kv_end = min(kv_end, (last_q / p.block + 1) * p.block);
  const int kv_begin = p.kv_start ? min(max(p.kv_start[b], 0), kv_end) : 0;
  const int tile0 = kv_begin / kWK;
  const int n_tiles = (kv_end + kWK - 1) / kWK;

  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_init(&full[2], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  pdl_wait();
  auto load_kv = [&](int tile, int stage) {
    mbar_expect_tx(&full[stage], (uint32_t)(2 * P * kPanel));
    if constexpr (kPaged) {
      // the tile is one whole page (only tiles below kv_end are ever looked up)
      const int pg = p.table[(int64_t)kb * p.table_stride + tile];
#pragma unroll
      for (int pn = 0; pn < P; ++pn) {
        tma_load_4d(smem + L::kK + (stage * P + pn) * kPanel, &tmK, pn * 64, hk, 0, pg, &full[stage]);
        tma_load_4d(smem + L::kV + (stage * P + pn) * kPanel, &tmV, pn * 64, hk, 0, pg, &full[stage]);
      }
    } else {
#pragma unroll
      for (int pn = 0; pn < P; ++pn) {
        tma_load_4d(smem + L::kK + (stage * P + pn) * kPanel, &tmK, pn * 64, hk, tile * kWK, kb, &full[stage]);
        tma_load_4d(smem + L::kV + (stage * P + pn) * kPanel, &tmV, pn * 64, hk, tile * kWK, kb, &full[stage]);
      }
    }
  };
  if (tid == 0 && n_tiles > tile0) {
    mbar_expect_tx(&full[2], (uint32_t)(P * kPanel));
#pragma unroll
    for (int pn = 0; pn < P; ++pn) tma_load_4d(smem + L::kQ + pn * kPanel, &tmQ, pn * 64, h, m0, b, &full[2]);
    if (n_tiles > tile0) load_kv(tile0, 0);
  }

  float o[D / 2];
#pragma unroll
  for (int i = 0; i < D / 2; ++i) o[i] = 0.f;
  float row_m[2] = {-INFINITY, -INFINITY}, row_l[2] = {0.f, 0.f};
  const int t4 = lane & 3;
  const int qrow0 = m0 + warp * 16 + (lane >> 2);  // this thread's rows: qrow0 and qrow0 + 8
  const uint32_t sQ = smem_u32(smem + L::kQ);
  if (n_tiles > tile0) mbar_wait(&full[2], 0);

  for (int tile = tile0; tile < n_tiles; ++tile) {
    const int it = tile - tile0, stage = it & 1;
    if (tid == 0 && tile + 1 < n_tiles) load_kv(tile + 1, stage ^ 1);  // that stage was released at the end of the last iteration
    mbar_wait(&full[stage], (uint32_t)((it >> 1) & 1));
    const int n0 = tile * kWK;
    uint8_t* vst = smem + L::kV + stage * P * kPanel;
    if (n0 < kv_begin || n0 + kWK > kv_end) {
      // partly valid tile: zero the V rows outside [kv_begin, kv_end) (whole 128-byte rows: the swizzle permutes within a row)
      for (int i = tid; i < P * kWK * 8; i += 128) {
        const int pn = i / (kWK * 8), r = (i / 8) % kWK, c = i % 8;
        const int key = n0 + r;
        if (key < kv_begin || key >= kv_end) reinterpret_cast<uint4*>(vst + pn * kPanel + r * 128)[c] = make_uint4(0u, 0u, 0u, 0u);
      }
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
    }

    // ---- S = Q K^T
    float s[kWK / 2];
    const uint32_t sK = smem_u32(smem + L::kK + stage * P * kPanel);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < D / 16; ++k) {
      const uint64_t da = make_wgmma_desc(sQ + (k >> 2) * kPanel) + (uint64_t)(2 * (k & 3));
      const uint64_t db = make_wgmma_desc(sK + (k >> 2) * kPanel) + (uint64_t)(2 * (k & 3));
      Wgmma<kWK>::mma(s, da, db, k > 0 ? 1u : 0u);
    }
    wgmma_commit();
    wgmma_wait<0>();

    // ---- mask + online softmax
    float tmax[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < kWK / 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = n0 + j * 8 + t4 * 2 + (e & 1);
        const int qr = qrow0 + (e >> 1) * 8;
        bool ok = key < kv_end && key >= kv_begin;
        if (p.causal) ok = ok && (key <= qr + shift);
        if (p.block > 0) ok = ok && (key / p.block <= qr / p.block);
        if (!ok) s[4 * j + e] = -INFINITY;
        tmax[e >> 1] = fmaxf(tmax[e >> 1], s[4 * j + e]);
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
    for (int i = 0; i < kWK / 2; ++i) {
      const float pv = exp2f((s[i] - mref[(i >> 1) & 1]) * p.scale_log2);
      s[i] = pv;
      psum[(i >> 1) & 1] += pv;
    }
    row_l[0] += psum[0];
    row_l[1] += psum[1];
#pragma unroll
    for (int i = 0; i < D / 2; ++i) o[i] *= corr[(i >> 1) & 1];

    // ---- O += P V (P from registers)
    const uint64_t dv = make_wgmma_desc_mn(smem_u32(vst), kPanel);
    wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < kWK / 16; ++ks) {
      uint32_t pa[4];
      pa[0] = pack_bf16x2(s[8 * ks + 0], s[8 * ks + 1]);
      pa[1] = pack_bf16x2(s[8 * ks + 2], s[8 * ks + 3]);
      pa[2] = pack_bf16x2(s[8 * ks + 4], s[8 * ks + 5]);
      pa[3] = pack_bf16x2(s[8 * ks + 6], s[8 * ks + 7]);
      // 16 keys = 16 rows of 128 B per panel
      WgmmaRS<D>::mma(o, pa, dv + (uint64_t)(ks * (16 * 128 >> 4)), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    __syncthreads();  // every thread is done with this stage before it is refilled
  }

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
  for (int j = 0; j < D / 8; ++j) {
    const int col = j * 8 + t4 * 2;
    if (qrow0 < p.Sq)
      *reinterpret_cast<uint32_t*>(ob + (int64_t)qrow0 * p.o_rs + col) = pack_bf16x2(o[4 * j] * inv0, o[4 * j + 1] * inv0);
    if (qrow0 + 8 < p.Sq)
      *reinterpret_cast<uint32_t*>(ob + (int64_t)(qrow0 + 8) * p.o_rs + col) = pack_bf16x2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1);
  }
}

typedef CUresult (*AwEncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                               const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

// [B, S, H, D] view of q / k / v (row stride rs, batch stride bs, heads D elements apart), boxes {64 d, 1 head, 64 rows, 1 batch}
static int aw_encode(CUtensorMap* tm, const void* base, int64_t D, int64_t H, int64_t S, int64_t B, int64_t rs, int64_t bs) {
  static AwEncodeFn enc = nullptr;
  if (!enc) {
    void* fp = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fp, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess) {
      set_error("cuTensorMapEncodeTiled entry point not available");
      return UVX_ERR_CUDA;
    }
    enc = (AwEncodeFn)fp;
  }
  cuuint64_t dims[4] = {(cuuint64_t)D, (cuuint64_t)H, (cuuint64_t)S, (cuuint64_t)B};
  cuuint64_t strides[3] = {(cuuint64_t)D * 2, (cuuint64_t)rs * 2, (cuuint64_t)(B > 1 ? bs : rs * S) * 2};
  cuuint32_t box[4] = {64, 1, 64, 1}, es[4] = {1, 1, 1, 1};
  CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("uvx_attention (wgmma): cuTensorMapEncodeTiled failed (%d)", (int)r);
    return UVX_ERR_CUDA;
  }
  return UVX_OK;
}

// shapes the wgmma kernel takes: a tile of queries per head, strides TMA can describe
bool attn_wg_eligible(const uvx_attn_args* a) {
  if (a->Sq < 16) return false;  // decode steps: latency-bound, mma.sync kernel
  if (a->q_bs <= 0 && a->B > 1) return false;
  if (a->k_bs <= 0 && a->B > 1) return false;
  if (a->v_bs <= 0 && a->B > 1) return false;
  if (a->o_rs % 2 != 0 || (uintptr_t)a->o % 4 != 0) return false;
  return true;
}

// kPaged: kv_batch is the pool's page count and the K / V maps cover it as {D, Hkv, 64, n_pages}
template <int D, bool kIndexed, bool kPaged = false>
static int launch_wg(const uvx_attn_args* a, int64_t kv_batch, const int32_t* kv_row, const int32_t* past, cudaStream_t st,
                     const int32_t* table = nullptr, int64_t table_stride = 0) {
  using L = AttnWgSmem<D>;
  CUtensorMap tq, tk, tv;
  const int64_t kv_rows = kPaged ? kWK : a->Skv;
  int rc = aw_encode(&tq, a->q, D, a->Hq, a->Sq, a->B, a->q_rs, a->q_bs);
  if (!rc) rc = aw_encode(&tk, a->k, D, a->Hkv, kv_rows, kv_batch, a->k_rs, a->k_bs);
  if (!rc) rc = aw_encode(&tv, a->v, D, a->Hkv, kv_rows, kv_batch, a->v_rs, a->v_bs);
  if (rc) return rc;
  static bool attr = false;
  if (!attr) {
    cudaError_t e = cudaFuncSetAttribute(attn_wg_kernel<D, kIndexed, kPaged>, cudaFuncAttributeMaxDynamicSharedMemorySize, L::kBytes);
    if (e != cudaSuccess) {
      set_error("cudaFuncSetAttribute(attn_wg_kernel<%d>): %s", D, cudaGetErrorString(e));
      return UVX_ERR_CUDA;
    }
    attr = true;
  }
  std::conditional_t<kPaged, AttnWgPagedParams, AttnWgParams> p;
  if constexpr (kPaged) {
    p.table = table;
    p.table_stride = table_stride;
  }
  p.o = (bf16*)a->o;
  p.o_rs = a->o_rs;
  p.o_bs = a->o_bs;
  p.kv_len = a->kv_len;
  p.kv_start = a->kv_start;
  p.lse = a->lse;
  p.Sq = (int)a->Sq;
  p.Skv = (int)a->Skv;
  p.group = (int)(a->Hq / a->Hkv);
  p.Hq = (int)a->Hq;
  p.causal = a->causal;
  p.block = a->block;
  p.scale_log2 = a->scale * 1.4426950408889634f;
  p.kv_row = kv_row;
  p.past = past;
  dim3 grid((unsigned)((a->Sq + kWQ - 1) / kWQ), (unsigned)a->Hq, (unsigned)a->B);
  launch_k(attn_wg_kernel<D, kIndexed, kPaged>, grid, dim3(128), (size_t)L::kBytes, st, tq, tk, tv, p);
  return check_launch("attn_wg_kernel");
}

int launch_attn_wg(const uvx_attn_args* a, cudaStream_t st) {
  return a->D == 64 ? launch_wg<64, false>(a, a->B, nullptr, nullptr, st) : launch_wg<128, false>(a, a->B, nullptr, nullptr, st);
}

}  // namespace uvx

extern "C" int uvx_attention_indexed(const uvx_attn_args* a, int64_t kv_batch, const int32_t* kv_row, const int32_t* past,
                                     uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(a && a->q && a->k && a->v && a->o && kv_row && past && a->kv_len, "uvx_attention_indexed: null pointer");
  UVX_REQUIRE(a->D == 64 || a->D == 128, "uvx_attention_indexed: head_dim must be 64 or 128 (got %lld)", (long long)a->D);
  UVX_REQUIRE(a->B >= 1 && a->B < 65536 && a->Hq >= 1 && a->Hq < 65536 && a->Hkv >= 1 && a->Hq % a->Hkv == 0 && a->Sq >= 1 &&
                  a->Skv >= 1 && kv_batch >= 1,
              "uvx_attention_indexed: bad shape");
  UVX_REQUIRE(a->causal == 1 && a->block == 0 && !a->kv_start && !a->lse,
              "uvx_attention_indexed: causal, no block mask, no kv_start, no lse");
  UVX_REQUIRE(a->q_rs % 8 == 0 && a->k_rs % 8 == 0 && a->v_rs % 8 == 0 && a->q_bs % 8 == 0 && a->k_bs % 8 == 0 &&
                  a->v_bs % 8 == 0 && a->o_rs % 2 == 0,
              "uvx_attention_indexed: strides must keep 16-byte alignment");
  UVX_REQUIRE(((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) % 16 == 0 && (uintptr_t)a->o % 4 == 0,
              "uvx_attention_indexed: base pointers must be 16-byte aligned");
  return a->D == 64 ? launch_wg<64, true>(a, kv_batch, kv_row, past, (cudaStream_t)stream)
                    : launch_wg<128, true>(a, kv_batch, kv_row, past, (cudaStream_t)stream);
}

extern "C" int uvx_attention_indexed_paged(const uvx_attn_args* a, int64_t n_pages, const int32_t* table, int64_t table_stride,
                                           const int32_t* kv_row, const int32_t* past, uvx_stream_t stream) {
  using namespace uvx;
  UVX_REQUIRE(a && a->q && a->k && a->v && a->o && kv_row && past && a->kv_len && table, "uvx_attention_indexed_paged: null pointer");
  UVX_REQUIRE(a->D == 64 || a->D == 128, "uvx_attention_indexed_paged: head_dim must be 64 or 128 (got %lld)", (long long)a->D);
  UVX_REQUIRE(a->B >= 1 && a->B < 65536 && a->Hq >= 1 && a->Hq < 65536 && a->Hkv >= 1 && a->Hq % a->Hkv == 0 && a->Sq >= 1 &&
                  a->Skv >= 1 && n_pages >= 1,
              "uvx_attention_indexed_paged: bad shape");
  UVX_REQUIRE(table_stride >= (a->Skv + kWK - 1) / kWK, "uvx_attention_indexed_paged: a table row of %lld pages cannot cover Skv = %lld",
              (long long)table_stride, (long long)a->Skv);
  UVX_REQUIRE(a->causal == 1 && a->block == 0 && !a->kv_start && !a->lse,
              "uvx_attention_indexed_paged: causal, no block mask, no kv_start, no lse");
  UVX_REQUIRE(a->k_bs == (int64_t)kWK * a->k_rs && a->v_bs == (int64_t)kWK * a->v_rs,
              "uvx_attention_indexed_paged: k_bs / v_bs must be one page of 64 rows");
  UVX_REQUIRE(a->q_rs % 8 == 0 && a->k_rs % 8 == 0 && a->v_rs % 8 == 0 && a->q_bs % 8 == 0 && a->o_rs % 2 == 0,
              "uvx_attention_indexed_paged: strides must keep 16-byte alignment");
  UVX_REQUIRE(((uintptr_t)a->q | (uintptr_t)a->k | (uintptr_t)a->v) % 16 == 0 && (uintptr_t)a->o % 4 == 0,
              "uvx_attention_indexed_paged: base pointers must be 16-byte aligned");
  return a->D == 64 ? launch_wg<64, true, true>(a, n_pages, kv_row, past, (cudaStream_t)stream, table, table_stride)
                    : launch_wg<128, true, true>(a, n_pages, kv_row, past, (cudaStream_t)stream, table, table_stride);
}
