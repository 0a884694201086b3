// K^T P K contraction on the Hopper tensor cores (wgmma + TMA + mbarrier):
//     UtWU[k][l] = sum_n U[n][k] w[n] U[n][l]          (morpho_class.py:1266-1268  U^T diag(K_NA) U;  SparseVFC U^T P U)
//     UtX[k][e]  = sum_n U[n][k] X[n][e]               (morpho_class.py:1279       U^T PXB_term;      SparseVFC U^T P Y)
// as ONE K-major GEMM  C = A B^T, fp32-accurate through the 3xTF32 split  x = hi + lo,
// a b ~= a_hi b_hi + a_hi b_lo + a_lo b_hi  accumulated in fp32 registers.
//
// The tensor core's fp32 accumulation TRUNCATES, which biases a sum of all-positive terms (U > 0, w >= 0) by ~4e-6
// relative; so the contraction runs on the CENTRED kernel  D = U - 1 m^T  (m_k = mean_n U[n][k]):
//     A = D^T  [K][N]                       (constant over the EM: gram_center_kernel, once)
//     B = [ w o D^T ; X^T ; w^T ]  [K + E + 1][N]   (rebuilt every iteration by gram_prepare_kernel)
//     UtWU = D^T W D + m v^T + v m^T + (sum w) m m^T,   v = D^T w  (the extra B row),   UtX = D^T X + m (sum_n X)^T
// whose terms change sign, so the truncation errors cancel instead of adding up (same idea as the centred KL contraction
// of gene_cost_tc.cu). The rank-one corrections are applied in fp64 by gram_reduce_kernel.
//
// Work unit = (output tile 128 x <=256, slice of the reduction dimension n). Every unit flushes its fp32 accumulators
// to a scratch slab; gram_reduce_kernel folds the slices in fp64 in a fixed order (deterministic), symmetrises the K x K
// block and writes the fp64 outputs the solve kernels consume. Slices are short (<= kMaxSliceKb k-blocks) so the fp32
// accumulation inside the tensor core never runs over more than a few thousand terms.
//
//   warp 8     TMA producer: 2-stage ring; per k-block (32 reduction elements = one 128-byte swizzle row) the A tile
//              (128 rows, hi and lo) and the B tile (128 or 256 rows, hi and lo) as 2-D tensor-map boxes of 128 rows
//   warps 0-7  two consumer warpgroups (A rows 64 w .. 64 w + 63): 4 k-steps x 3 products of wgmma.m64nNk8.tf32 per
//              k-block, N = 128 or 256 (the tile's columns rounded up), then the accumulators -> scratch slab
#include "wgmma.cuh"

namespace {

constexpr int GM = 128;  // output rows per tile (2 x wgmma M)
constexpr int GN = 256;  // output columns per tile (largest wgmma N)
constexpr int GK = 32;   // reduction elements per k-block (128 bytes)
constexpr int kGStages = 2;
constexpr int kGConsumers = 256;             // two warpgroups
constexpr int kGThreads = kGConsumers + 32;  // + the producer warp
constexpr int kMaxTiles = 16;     // (K + E) <= 515 -> at most 5 x 3 tiles, upper block triangle + right-hand sides
constexpr int kMaxSliceKb = 128;  // k-blocks per unit: fp32 accumulation over at most 4096 reduction elements

struct __align__(1024) GramSmem {
  float a_hi[kGStages][GM * GK];  // 16 KB each, SWIZZLE_128B K-major
  float a_lo[kGStages][GM * GK];
  float b_hi[kGStages][GN * GK];  // 32 KB each (two stacked 128-row boxes)
  float b_lo[kGStages][GN * GK];
  uint64_t full[kGStages];
  uint64_t empty[kGStages];  // one arrive per consumer warpgroup
};

struct GramPlan {
  int ntiles;           // tiles computed
  int nslices;          // slices of the reduction dimension
  int kb_per_slice;     // k-blocks per slice
  int nkb;              // k-blocks in total
  int K, E;
  int8_t mt[kMaxTiles], nt[kMaxTiles];
  int16_t ncols[kMaxTiles];     // columns of the tile (multiple of 16)
  int8_t index[8][4];           // (mt, nt) -> tile slot or -1
};

template <int N>
__device__ __forceinline__ void gram_wgmma(float (&acc)[N / 2], uint64_t a, uint64_t b) {
  if constexpr (N == 256) wgmma_tf32_m64n256k8(acc, a, b, 1);
  else wgmma_tf32_m64n128k8(acc, a, b, 1);
}

// Consumer warpgroup of one unit with an N-column accumulator: MMAs over the unit's k-blocks, then the scratch slab.
template <int N>
__device__ __forceinline__ void gram_consume(GramSmem& sm, int kb0, int kb1, float* __restrict__ scratch) {
  const int wg = threadIdx.x >> 7, t = threadIdx.x & 127, lane = threadIdx.x & 31;
  const uint32_t a_off = (uint32_t)(wg * 64 * GK * 4);  // this warpgroup's 64 A rows (8 KB, 1024-aligned)
  float acc[N / 2];
#pragma unroll
  for (int c = 0; c < N / 2; ++c) acc[c] = 0.f;
  for (int kb = kb0, it = 0; kb < kb1; ++kb, ++it) {
    const int s = it % kGStages;
    mbar_wait(&sm.full[s], (it / kGStages) & 1);
    const uint64_t d_ahi = wgmma_desc_k_sw128((const uint8_t*)sm.a_hi[s] + a_off);
    const uint64_t d_alo = wgmma_desc_k_sw128((const uint8_t*)sm.a_lo[s] + a_off);
    const uint64_t d_bhi = wgmma_desc_k_sw128(sm.b_hi[s]), d_blo = wgmma_desc_k_sw128(sm.b_lo[s]);
    wgmma_fence_operand(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < GK / 8; ++k) {
      const uint64_t adv = (uint64_t)((k * 8 * 4) >> 4);
      gram_wgmma<N>(acc, d_alo + adv, d_bhi + adv);  // small cross terms first
      gram_wgmma<N>(acc, d_ahi + adv, d_blo + adv);
      gram_wgmma<N>(acc, d_ahi + adv, d_bhi + adv);
    }
    wgmma_commit();
    wgmma_wait<1>();  // the previous k-block's stage is no longer read: hand it back to the producer
    wgmma_fence_operand(acc);
    if (it > 0 && t == 0) mbar_arrive(&sm.empty[(it - 1) % kGStages]);
  }
  wgmma_wait<0>();
  wgmma_fence_operand(acc);
  const int row = wg * 64 + (t >> 5) * 16 + (lane >> 2), col = 2 * (lane & 3);
  float* dst = scratch + ((int64_t)blockIdx.x * GM + row) * GN + col;
#pragma unroll
  for (int n = 0; n < N / 8; ++n) {
    *reinterpret_cast<float2*>(dst + 8 * n) = make_float2(acc[4 * n], acc[4 * n + 1]);
    *reinterpret_cast<float2*>(dst + 8 * GN + 8 * n) = make_float2(acc[4 * n + 2], acc[4 * n + 3]);
  }
}

// One CTA = one work unit (tile, slice).
__global__ void __launch_bounds__(kGThreads, 1)
gram_tc_kernel(const __grid_constant__ CUtensorMap map_a_hi, const __grid_constant__ CUtensorMap map_a_lo,
               const __grid_constant__ CUtensorMap map_b_hi, const __grid_constant__ CUtensorMap map_b_lo,
               const GramPlan plan, float* __restrict__ scratch) {
  extern __shared__ uint8_t g_smem_raw[];
  GramSmem& sm = *reinterpret_cast<GramSmem*>(g_smem_raw + ((1024u - (smem_u32(g_smem_raw) & 1023u)) & 1023u));
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tile = blockIdx.x % plan.ntiles, slice = blockIdx.x / plan.ntiles;
  const int mt = plan.mt[tile], nt = plan.nt[tile], ncols = plan.ncols[tile];
  const int kb0 = slice * plan.kb_per_slice, kb1 = min(plan.nkb, kb0 + plan.kb_per_slice);
  // 128-row boxes of the B operand = wgmma N / 128. A tile narrower than 128 columns (e.g. the right-hand sides alone, E + 1
  // columns) still runs N = 128 on zero-filled rows: its MMAs are a small share of the contraction, and gram_reduce_kernel
  // reads only the tile's ncols columns.
  const int nb_boxes = ncols > 128 ? 2 : 1;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kGStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], 2);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kGConsumers / 32) {
    if (lane == 0) {
      for (int kb = kb0, it = 0; kb < kb1; ++kb, ++it) {
        const int s = it % kGStages;
        if (it >= kGStages) mbar_wait(&sm.empty[s], ((it / kGStages) - 1) & 1);
        mbar_expect_tx(&sm.full[s], (uint32_t)((2 * GM + 2 * 128 * nb_boxes) * GK * 4));
        tma_load_2d(sm.a_hi[s], &map_a_hi, kb * GK, mt * GM, &sm.full[s]);
        tma_load_2d(sm.a_lo[s], &map_a_lo, kb * GK, mt * GM, &sm.full[s]);
        for (int b = 0; b < nb_boxes; ++b) {
          tma_load_2d(sm.b_hi[s] + b * 128 * GK, &map_b_hi, kb * GK, nt * GN + b * 128, &sm.full[s]);
          tma_load_2d(sm.b_lo[s] + b * 128 * GK, &map_b_lo, kb * GK, nt * GN + b * 128, &sm.full[s]);
        }
      }
    }
    return;
  }
  if (nb_boxes == 2) gram_consume<256>(sm, kb0, kb1, scratch);
  else gram_consume<128>(sm, kb0, kb1, scratch);
}

// fp64 fold of the slice partials in slice order; K x K block symmetrised over the tiles that were computed.
__device__ __forceinline__ bool gram_entry(const GramPlan& plan, const float* __restrict__ scratch, int k, int l, double& out) {
  const int slot = plan.index[k / GM][l / GN];
  if (slot < 0) return false;
  const float* p = scratch + ((int64_t)slot * GM + (k % GM)) * GN + (l % GN);
  const int64_t stride = (int64_t)plan.ntiles * GM * GN;
  double s = 0.0;
  for (int sl = 0; sl < plan.nslices; ++sl) s += (double)p[sl * stride];
  out = s;
  return true;
}
__global__ void gram_reduce_kernel(const GramPlan plan, const float* __restrict__ scratch, const float* __restrict__ mean,
                                   const double* __restrict__ sums, double* __restrict__ UtWU, double* __restrict__ UtX,
                                   int ldx_out) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x, k = blockIdx.y;
  const int K = plan.K, E = plan.E - 1;  // plan.E counts the extra w row
  if (k >= K || l >= K + E) return;
  const double mk = (double)mean[k];
  double a = 0.0, b = 0.0;
  if (l >= K) {  // U^T X = D^T X + m_k sum_n X_e
    gram_entry(plan, scratch, k, l, a);
    UtX[k * ldx_out + (l - K)] = a + mk * sums[1 + (l - K)];
    return;
  }
  const bool ha = gram_entry(plan, scratch, k, l, a), hb = gram_entry(plan, scratch, l, k, b);
  const double g = (ha && hb) ? 0.5 * (k <= l ? __dadd_rn(a, b) : __dadd_rn(b, a)) : (ha ? a : b);
  double vk = 0.0, vl = 0.0;  // v = D^T w
  gram_entry(plan, scratch, k, K + E, vk);
  gram_entry(plan, scratch, l, K + E, vl);
  const double ml = (double)mean[l];
  // the two cross terms are added in an order that does not depend on which of (k, l), (l, k) this thread owns
  // (explicit rounding of every operation: an fma contraction chosen differently on the two sides would break symmetry)
  const double c1 = __dmul_rn(ml, vk), c2 = __dmul_rn(mk, vl);
  const double cross = k <= l ? __dadd_rn(c1, c2) : __dadd_rn(c2, c1);
  UtWU[(int64_t)k * K + l] = __dadd_rn(__dadd_rn(g, cross), __dmul_rn(__dmul_rn(mk, ml), sums[0]));
}

// Row means of U^T and the centred, tf32-split A operand (once per alignment; U is constant over the EM).
__global__ void __launch_bounds__(256)
gram_center_kernel(const float* __restrict__ UT, int64_t ldn, int64_t N, float* __restrict__ mean, float* __restrict__ Ahi,
                   float* __restrict__ Alo) {
  __shared__ double red[8];
  __shared__ float s_mean;
  const int row = blockIdx.x;
  const float* src = UT + (int64_t)row * ldn;
  double acc = 0.0;
  for (int64_t n = threadIdx.x; n < N; n += 256) acc += (double)src[n];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int q = 0; q < 8; ++q) t += red[q];
    s_mean = (float)(t / (double)N);
    mean[row] = s_mean;
  }
  __syncthreads();
  const float m = s_mean;
  for (int64_t n = threadIdx.x; n < ldn; n += 256) {
    const float v = n < N ? src[n] - m : 0.f;
    const float h = __uint_as_float(__float_as_uint(v) & 0xFFFFE000u);
    Ahi[(int64_t)row * ldn + n] = h;
    Alo[(int64_t)row * ldn + n] = v - h;
  }
}

// B operand of the iteration: rows k < K = w o (U^T - m_k), rows K..K+E-1 = X^T, row K+E = w; written already split into
// tf32 hi / lo parts. The X and w rows also accumulate sum_n X_e (sums[1 + e]) and sum_n w (sums[0]) in fp64.
__global__ void __launch_bounds__(256)
gram_prepare_kernel(const float* __restrict__ UT, int64_t ldn, int64_t N, int K, int E, const float* __restrict__ mean,
                    const float* __restrict__ w, const float* __restrict__ X, int64_t ldxx, float* __restrict__ Bhi,
                    float* __restrict__ Blo, double* __restrict__ sums) {
  const int row = blockIdx.y;
  const float* src = row < K ? UT + (int64_t)row * ldn : (row < K + E ? X + (int64_t)(row - K) * ldxx : w);
  const float m = row < K ? mean[row] : 0.f;
  float* hi = Bhi + (int64_t)row * ldn;
  float* lo = Blo + (int64_t)row * ldn;
  double tot = 0.0;
  for (int64_t n = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; n < N; n += (int64_t)gridDim.x * blockDim.x * 4) {
    float4 v = *reinterpret_cast<const float4*>(src + n);
    if (n + 3 >= N) {  // ragged tail: the padding of the inputs is not trusted
      if (n + 1 >= N) v.y = 0.f;
      if (n + 2 >= N) v.z = 0.f;
      v.w = 0.f;
      if (n + 3 < N) v.w = src[n + 3];
    }
    if (row < K) {
      const float4 ww = *reinterpret_cast<const float4*>(w + n);
      v.x = (v.x - m) * ww.x; v.y = (v.y - m) * ww.y; v.z = (v.z - m) * ww.z; v.w = (v.w - m) * ww.w;
      if (n + 3 >= N) {
        if (n + 1 >= N) v.y = 0.f;
        if (n + 2 >= N) v.z = 0.f;
        if (n + 3 >= N) v.w = 0.f;
      }
    } else {
      tot += 0.0;
    }
    float4 h;
    h.x = __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
    h.y = __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
    h.z = __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
    h.w = __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
    *reinterpret_cast<float4*>(hi + n) = h;
    *reinterpret_cast<float4*>(lo + n) = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
  }
  (void)tot;
  (void)sums;
}

// sum_n w (sums[0]) and sum_n X_e (sums[1 + e]): one block per row, fixed summation order (reproducible)
__global__ void __launch_bounds__(1024)
gram_sums_kernel(int64_t N, int E, const float* __restrict__ w, const float* __restrict__ X, int64_t ldxx,
                 double* __restrict__ sums) {
  __shared__ double red[32];
  const int row = blockIdx.x;  // 0 = w, 1 + e = X_e
  const float* src = row == 0 ? w : X + (int64_t)(row - 1) * ldxx;
  double t = 0.0;
  for (int64_t n = threadIdx.x; n < N; n += 1024) t += (double)src[n];
  t = warp_sum(t);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
  __syncthreads();
  if (threadIdx.x < 32) {
    double x = red[threadIdx.x];
    x = warp_sum(x);
    if (threadIdx.x == 0) sums[row] = x;
  }
  if (row == 0 && threadIdx.x == 0)
    for (int e = E; e < 3; ++e) sums[1 + e] = 0.0;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn g_encode_fn() {
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
// [rows][N] fp32, row pitch ldn; boxes of 128 rows x 32 reduction elements; out-of-range rows / columns read as zero
int g_make_map(CUtensorMap* map, const float* base, int64_t rows, int64_t N, int64_t ldn) {
  EncodeTiledFn fn = g_encode_fn();
  if (fn == nullptr) return SPB_EUNSUPPORTED;
  const cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ldn * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)GK, 128u};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : 700 + (int)r;
}

// Tiles: the block upper triangle of the K x K part plus every tile that holds right-hand-side columns; slices sized so
// that the grid fills the GPU about twice and no unit accumulates more than kMaxSliceKb k-blocks in fp32.
int make_plan(int K, int E, int64_t N, GramPlan* plan) {
  if (K < 1 || E < 1 || K + E > 4 * GN || K > 8 * GM) return SPB_EUNSUPPORTED;  // E counts X rows + the w row
  GramPlan& p = *plan;
  p.K = K;
  p.E = E;
  p.ntiles = 0;
  const int n_mt = (K + GM - 1) / GM, n_nt = (K + E + GN - 1) / GN;
  for (int a = 0; a < 8; ++a)
    for (int b = 0; b < 4; ++b) p.index[a][b] = -1;
  for (int nt = 0; nt < n_nt; ++nt)
    for (int mt = 0; mt < n_mt; ++mt) {
      const int col_end = (nt + 1) * GN;                  // exclusive
      const bool upper = col_end > mt * GM;               // tile touches the upper triangle (l >= k for some entry)
      const bool rhs = E > 0 && col_end > K && nt * GN < K + E;
      if (!upper && !rhs) continue;
      if (p.ntiles >= kMaxTiles) return SPB_EUNSUPPORTED;
      int nc = K + E - nt * GN;
      nc = nc > GN ? GN : nc;
      nc = ((nc + 15) / 16) * 16;
      p.mt[p.ntiles] = (int8_t)mt;
      p.nt[p.ntiles] = (int8_t)nt;
      p.ncols[p.ntiles] = (int16_t)nc;
      p.index[mt][nt] = (int8_t)p.ntiles;
      ++p.ntiles;
    }
  p.nkb = (int)((N + GK - 1) / GK);
  int want = (2 * spb_num_sms() + p.ntiles - 1) / p.ntiles;  // slices for ~2 units per SM
  int per = (p.nkb + want - 1) / want;
  if (per < 8) per = 8;
  if (per > kMaxSliceKb) per = kMaxSliceKb;
  p.kb_per_slice = per;
  p.nslices = (p.nkb + per - 1) / per;
  return 0;
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" int spb_gram_tc_scratch_floats(int32_t K, int32_t E, int64_t N, int64_t* floats) {
  GramPlan plan;
  const int rc = make_plan(K, E + 1, N, &plan);
  if (rc) return rc;
  *floats = (int64_t)plan.ntiles * plan.nslices * GM * GN;
  return 0;
}

extern "C" int spb_gram_center(const float* UT, int64_t ldn, int64_t N, int32_t K, float* mean, float* A_hi, float* A_lo,
                               void* stream) {
  if (K < 1 || N < 1 || ldn < N) return SPB_EINVAL;
  gram_center_kernel<<<K, 256, 0, ST>>>(UT, ldn, N, mean, A_hi, A_lo);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_gram_prepare(const float* UT, int64_t ldn, int64_t N, int32_t K, const float* mean, const float* w,
                                const float* X, int64_t ldxx, int32_t E, float* B_hi, float* B_lo, double* sums4,
                                void* stream) {
  if (ldn % 4 != 0 || (E > 0 && ldxx % 4 != 0) || K < 1 || E < 0 || E > 3) return SPB_EINVAL;
  gram_sums_kernel<<<1 + E, 1024, 0, ST>>>(N, E, w, X, ldxx, sums4);
  SPB_CHECK_LAUNCH();
  int gx = (int)((N / 4 + 255) / 256);
  if (gx > 592) gx = 592;
  if (gx < 1) gx = 1;
  const int n_sm = spb_num_sms();
  if ((int64_t)gx * (K + E + 1) > n_sm * 64) gx = (n_sm * 64) / (K + E + 1) + 1;  // enough CTAs, short rows need no more
  gram_prepare_kernel<<<dim3(gx, K + E + 1), 256, 0, ST>>>(UT, ldn, N, K, E, mean, w, X, ldxx, B_hi, B_lo, sums4);
  SPB_CHECK_LAUNCH();
  return 0;
}

// per-device shared-memory opt-in of the contraction kernel (idempotent; also called by spb_nonrigid_warm)
int spb_gram_tc_warm() {
  static bool attr_set[SPB_MAX_DEVICES] = {};
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(gram_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(GramSmem) + 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  return 0;
}

extern "C" int spb_gram_tc(const float* A_hi, const float* A_lo, const float* B_hi, const float* B_lo, int64_t ldn, int64_t N,
                           int32_t K, int32_t E, const float* mean, const double* sums4, float* scratch,
                           int64_t scratch_floats, double* UtWU, double* UtX, void* stream) {
  if (ldn % 4 != 0 || N < 1) return SPB_EINVAL;
  GramPlan plan;
  int rc = make_plan(K, E + 1, N, &plan);
  if (rc) return rc;
  if (scratch_floats < (int64_t)plan.ntiles * plan.nslices * GM * GN) return SPB_EINVAL;
  CUtensorMap ma_hi, ma_lo, mb_hi, mb_lo;
  if ((rc = g_make_map(&ma_hi, A_hi, K, N, ldn))) return rc;
  if ((rc = g_make_map(&ma_lo, A_lo, K, N, ldn))) return rc;
  if ((rc = g_make_map(&mb_hi, B_hi, K + E + 1, N, ldn))) return rc;
  if ((rc = g_make_map(&mb_lo, B_lo, K + E + 1, N, ldn))) return rc;
  if ((rc = spb_gram_tc_warm())) return rc;
  gram_tc_kernel<<<plan.ntiles * plan.nslices, kGThreads, sizeof(GramSmem) + 1024, ST>>>(ma_hi, ma_lo, mb_hi, mb_lo, plan, scratch);
  SPB_CHECK_LAUNCH();
  gram_reduce_kernel<<<dim3((K + E + 127) / 128, K), 128, 0, ST>>>(plan, scratch, mean, sums4, UtWU, UtX, 3);
  SPB_CHECK_LAUNCH();
  return 0;
}
