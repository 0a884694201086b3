// Expression cost matrix on the Hopper tensor cores (wgmma + TMA + mbarrier), fp32-accurate through a 3xTF32 split:
//   x = hi + lo  (hi = tf32(x), lo = x - hi),  A.B ~= Ahi.Bhi + Ahi.Blo + Alo.Bhi  accumulated in fp32 registers.
// GT[j][i] (op)= prob(metric(A_i, B_j)); the operands come from the row pre-passes of gene_cost.cu, split by spb_split_tf32.
//
// Per CTA (persistent, one per SM): tile = 128 fixed cells (wgmma M, two warpgroups of 64) x 256 moving cells (wgmma N).
//   warp 8      TMA producer: 2-stage ring, per k-block (32 features = one 128-byte swizzle row) four 2-D tensor-map loads
//               (Bfix hi/lo 128x32, Amov hi/lo 256x32) into the canonical K-major SWIZZLE_128B layout
//   warps 0-7   two consumer warpgroups, fixed cells 64 w .. 64 w + 63: 4 k-steps x 3 products of
//               wgmma.m64n256k8.tf32 per k-block (128 fp32 accumulators per thread), then the epilogue
//               (cost -> probability, store to GT) straight from the registers. The producer runs ahead into the next
//               tile while the epilogue runs; the epilogue is a few per cent of a tile's MMA time at G ~ 2000.
#include "wgmma.cuh"

namespace {

constexpr int TM = 128;   // fixed cells per tile (2 x wgmma M)
constexpr int TN = 256;   // moving cells per tile (wgmma N)
constexpr int TK = 32;    // features per k-block (128 bytes)
constexpr int kTcStages = 2;
constexpr int kTcConsumers = 256;               // two warpgroups
constexpr int kTcThreads = kTcConsumers + 32;   // + the producer warp

struct __align__(1024) TcSmem {
  float bfix_hi[kTcStages][TM * TK];  // 16 KB each, SWIZZLE_128B K-major (8-row groups of 1024 B)
  float bfix_lo[kTcStages][TM * TK];
  float amov_hi[kTcStages][TN * TK];  // 32 KB each
  float amov_lo[kTcStages][TN * TK];
  uint64_t full[kTcStages];
  uint64_t empty[kTcStages];  // one arrive per consumer warpgroup
};

__device__ __forceinline__ float tc_cost_to_prob(float dot, float ta, float tb, int metric, int prob_type, float neg_inv2b) {
  float e;
  if (metric == SPB_METRIC_KL) e = (ta - tb) - dot;  // tb = centring term c_j of the fixed cell
  else if (metric == SPB_METRIC_SYMKL) e = 0.5f * ((ta + tb) - dot);             // utils.py:922-932
  else if (metric == SPB_METRIC_COS) e = fmaf(-0.5f, dot, 0.5f);
  else {
    e = fmaxf(ta + tb - 2.0f * dot, 0.0f);
    if (metric == SPB_METRIC_SQRT_EUC) e = sqrtf(e);
  }
  if (prob_type == SPB_PROB_GAUSS) return __expf(e * neg_inv2b);
  if (prob_type == SPB_PROB_COS) return 1.0f - e;
  return e;
}

// Tile order: bands of kBand fixed-cell tiles, moving-cell tiles fastest inside a band, so the tiles in flight (one
// per SM) touch ~kBand B-side and ~SMs/kBand A-side operand panels (tens of MB, L2 resident) instead of one A panel each.
constexpr int kBand = 16;
__device__ __forceinline__ void tile_coords(int tile, int tiles_i, int tiles_j, int& ti, int& tj) {
  const int per_band = kBand * tiles_i;
  const int band = tile / per_band, r = tile % per_band;
  const int bh = min(kBand, tiles_j - band * kBand);
  ti = r / bh;
  tj = band * kBand + r % bh;
}

__global__ void __launch_bounds__(kTcThreads, 1)
gene_cost_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
                    const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
                    const float* __restrict__ rtA, const float* __restrict__ rtB, int64_t NA, int64_t NB, int nkb,
                    int tiles_i, int tiles_j, int metric, int prob_type, float neg_inv2b, int accumulate,
                    float* __restrict__ GT, int64_t ldx) {
  extern __shared__ uint8_t tc_smem_raw[];
  // SWIZZLE_128B operands need 1024-byte aligned tiles: align the dynamic shared-memory window by hand
  TcSmem& sm = *reinterpret_cast<TcSmem*>(tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int ntiles = tiles_i * tiles_j;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kTcStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kTcConsumers / 32) {
    // ===== TMA producer =====
    if (lane == 0) {
      int it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        int ti, tj;
        tile_coords(tile, tiles_i, tiles_j, ti, tj);
        for (int kb = 0; kb < nkb; ++kb, ++it) {
          const int s = it % kTcStages;
          if (it >= kTcStages) mbar_wait(&sm.empty[s], ((it / kTcStages) - 1) & 1);
          mbar_expect_tx(&sm.full[s], (uint32_t)((2 * TM + 2 * TN) * TK * 4));
          tma_load_2d(sm.bfix_hi[s], &map_b_hi, kb * TK, tj * TM, &sm.full[s]);
          tma_load_2d(sm.bfix_lo[s], &map_b_lo, kb * TK, tj * TM, &sm.full[s]);
          tma_load_2d(sm.amov_hi[s], &map_a_hi, kb * TK, ti * TN, &sm.full[s]);
          tma_load_2d(sm.amov_lo[s], &map_a_lo, kb * TK, ti * TN, &sm.full[s]);
        }
      }
    }
    return;
  }

  // ===== consumer warpgroups: wgmma "A" (M side) = fixed cells, "B" (N side) = moving cells =====
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int row0 = wg * 64 + (t >> 5) * 16 + (lane >> 2);  // this thread's rows row0, row0 + 8 of the tile
  const int col0 = 2 * (lane & 3);                           // and columns 8 n + col0 + {0, 1}
  const uint32_t a_off = (uint32_t)(wg * 64 * TK * 4);       // this warpgroup's 64 fixed-cell rows (8 KB, 1024-aligned)
  float acc[TN / 2];
  int it = 0;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    int ti, tj;
    tile_coords(tile, tiles_i, tiles_j, ti, tj);
#pragma unroll
    for (int c = 0; c < TN / 2; ++c) acc[c] = 0.f;
    for (int kb = 0; kb < nkb; ++kb, ++it) {
      const int s = it % kTcStages;
      mbar_wait(&sm.full[s], (it / kTcStages) & 1);
      const uint64_t d_bhi = wgmma_desc_k_sw128((const uint8_t*)sm.bfix_hi[s] + a_off);
      const uint64_t d_blo = wgmma_desc_k_sw128((const uint8_t*)sm.bfix_lo[s] + a_off);
      const uint64_t d_ahi = wgmma_desc_k_sw128(sm.amov_hi[s]), d_alo = wgmma_desc_k_sw128(sm.amov_lo[s]);
      wgmma_fence_operand(acc);
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < TK / 8; ++k) {
        const uint64_t adv = (uint64_t)((k * 8 * 4) >> 4);  // 32 bytes per K = 8 step inside the 128-byte swizzle row
        wgmma_tf32_m64n256k8(acc, d_blo + adv, d_ahi + adv, 1);  // small cross terms first
        wgmma_tf32_m64n256k8(acc, d_bhi + adv, d_alo + adv, 1);
        wgmma_tf32_m64n256k8(acc, d_bhi + adv, d_ahi + adv, 1);
      }
      wgmma_commit();
      // the previous k-block's MMAs are done reading their stage: hand it back to the producer
      wgmma_wait<1>();
      wgmma_fence_operand(acc);
      if (kb > 0 && t == 0) mbar_arrive(&sm.empty[(it - 1) % kTcStages]);
    }
    wgmma_wait<0>();
    wgmma_fence_operand(acc);
    if (t == 0) mbar_arrive(&sm.empty[(it - 1) % kTcStages]);

    const int64_t i0 = (int64_t)ti * TN;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t j = (int64_t)tj * TM + row0 + 8 * h;
      if (j >= NB) continue;
      const float tb = rtB != nullptr ? rtB[j] : 0.f;
      float* dst = GT + j * ldx + i0 + col0;
#pragma unroll
      for (int n = 0; n < TN / 8; ++n) {  // fully unrolled: acc must stay in registers
        const int64_t i = i0 + 8 * n + col0;
        if (i >= ldx) continue;  // ldx % 4 == 0 and i even: i + 1 < ldx as well
        float o[2];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float ta = (rtA != nullptr && i + u < NA) ? rtA[i + u] : 0.f;
          o[u] = i + u < NA ? tc_cost_to_prob(acc[4 * n + 2 * h + u], ta, tb, metric, prob_type, neg_inv2b) : 0.f;
        }
        float2* d2 = reinterpret_cast<float2*>(dst + 8 * n);
        if (accumulate) {
          const float2 old = *d2;
          o[0] *= old.x;
          o[1] *= old.y;
        }
        *d2 = make_float2(o[0], o[1]);
      }
    }
  }
}

// x -> (hi, lo): hi keeps the 10 explicit mantissa bits a tf32 operand keeps, lo = x - hi (exact in fp32)
__global__ void split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = x[i];
    const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    hi[i] = h;
    lo[i] = v - h;
  }
}

// dst[r][.] = src[idx[r]][.]: one thread per (row, 16-byte vector) with kVec, per (row, word) otherwise
template <bool kVec>
__global__ void __launch_bounds__(256)
gather_rows_kernel(const uint32_t* __restrict__ src, int64_t ld_src, int64_t width, const int32_t* __restrict__ idx, int64_t n,
                   uint32_t* __restrict__ dst, int64_t ld_dst) {
  const int64_t per = kVec ? width / 4 : width;
  const int64_t total = n * per;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = t / per, c = t - r * per;
    const int64_t s = (int64_t)__ldg(idx + r);
    if constexpr (kVec) {
      reinterpret_cast<uint4*>(dst + r * ld_dst)[c] = __ldg(reinterpret_cast<const uint4*>(src + s * ld_src) + c);
    } else {
      dst[r * ld_dst + c] = __ldg(src + s * ld_src + c);
    }
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

int make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t Gp, int64_t pitch, int box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return SPB_EUNSUPPORTED;
  const cuuint64_t dims[2] = {(cuuint64_t)Gp, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)pitch * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)TK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 700 + (int)r;
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" int spb_split_tf32(const float* x, float* hi, float* lo, int64_t n, void* stream) {
  if (n <= 0) return 0;
  split_tf32_kernel<<<1184, 256, 0, ST>>>(x, hi, lo, n);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_gene_cost_tc(const float* A_hi, const float* A_lo, int64_t lda, const float* rowtermA, const float* B_hi,
                                const float* B_lo, int64_t ldb, const float* rowtermB, int64_t NA, int64_t NB, int64_t G,
                                int32_t metric, int32_t prob_type, float prob_param, int32_t accumulate, float* GT,
                                int64_t ldx, void* stream) {
  if (lda % 4 != 0 || ldb % 4 != 0 || ldx % 4 != 0) return SPB_EINVAL;
  const int64_t Gp = ((G + TK - 1) / TK) * TK;
  if (lda < Gp || ldb < Gp) return SPB_EINVAL;  // operands must be zero-padded to a multiple of 32 features
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  int rc;
  if ((rc = make_map(&ma_hi, A_hi, NA, Gp, lda, TN))) return rc;
  if ((rc = make_map(&ma_lo, A_lo, NA, Gp, lda, TN))) return rc;
  if ((rc = make_map(&mb_hi, B_hi, NB, Gp, ldb, TM))) return rc;
  if ((rc = make_map(&mb_lo, B_lo, NB, Gp, ldb, TM))) return rc;
  const int tiles_i = (int)((ldx + TN - 1) / TN), tiles_j = (int)((NB + TM - 1) / TM);
  const float neg_inv2b = prob_type == SPB_PROB_GAUSS ? -1.0f / (2.0f * prob_param) : 0.f;
  static int n_sm_dev[SPB_MAX_DEVICES] = {};  // SM count + shared-memory opt-in, per device
  const int dev_ = spb_current_device();
  if (n_sm_dev[dev_] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev_);
    cudaError_t e = cudaFuncSetAttribute(gene_cost_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TcSmem) + 1024);
    if (e != cudaSuccess) return (int)e;
    n_sm_dev[dev_] = n;
  }
  const int n_sm = n_sm_dev[dev_];
  const int grid = min(n_sm, tiles_i * tiles_j);
  gene_cost_tc_kernel<<<grid, kTcThreads, sizeof(TcSmem) + 1024, ST>>>(ma_hi, ma_lo, mb_hi, mb_lo, rowtermA, rowtermB, NA, NB,
                                                                        (int)(Gp / TK), tiles_i, tiles_j, metric, prob_type,
                                                                        neg_inv2b, accumulate, GT, ldx);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_gather_rows(const void* src, int64_t ld_src, int64_t width, const int32_t* idx, int64_t n, void* dst,
                               int64_t ld_dst, void* stream) {
  if (n < 0 || width < 0 || ld_src < width || ld_dst < width) return SPB_EINVAL;
  if (n == 0 || width == 0) return 0;
  const bool vec = width % 4 == 0 && ld_src % 4 == 0 && ld_dst % 4 == 0 && ((uintptr_t)src & 15) == 0 &&
                   ((uintptr_t)dst & 15) == 0;
  const int64_t work = n * (vec ? width / 4 : width);
  const int blocks = (int)std::min<int64_t>((work + 255) / 256, (int64_t)spb_num_sms() * 16);
  const uint32_t* s = static_cast<const uint32_t*>(src);
  uint32_t* d = static_cast<uint32_t*>(dst);
  if (vec) gather_rows_kernel<true><<<blocks, 256, 0, ST>>>(s, ld_src, width, idx, n, d, ld_dst);
  else gather_rows_kernel<false><<<blocks, 256, 0, ST>>>(s, ld_src, width, idx, n, d, ld_dst);
  SPB_CHECK_LAUNCH();
  return 0;
}
