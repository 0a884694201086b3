// Expression cost / probability matrix (replaces calc_distance + calc_probability for the representation layers:
// spateo/alignment/methods/utils.py:647-788, 866-985). One-off per pair, outside the EM loop.
//
// GT[j][i] = prob(metric(A_i, B_j)), written in the layout the E-step sweeps stream (one contiguous row per fixed cell).
// v1 contraction: FP32-FMA register-tiled GEMM (128x128x16 tiles, 8x8 micro-tiles) — fp32-accurate dot products are
// required because the KL cost is a small difference of O(7) terms that is then divided by 2*beta^2 ~ 0.02.
#include "common.cuh"

namespace {

constexpr int kPadG = 16;  // feature pitch granularity produced by the prep kernels

// Xn = (X + .01) / rowsum, rowterm = sum Xn log(Xn + 1e-8)  (moving side), or out = log(Xn + 1e-8) (fixed side)
// (utils.py:683-695). Both log terms are shifted by +log(G): KL = sum Xn (logX + c) - sum Xn (logY + c) for any c, and
// with c = log G the summands are O(Xn) instead of O(7 Xn), which cuts the fp32 rounding of the rank-G contraction.
// Fixed side with `center_w` (a probability profile, e.g. the mean moving row): the row is additionally centred by
// c_j = sum_g w_g (log Y_jg + c), returned as its row term, so that sum_g Xn_ig * out_jg = dot_ij - c_j stays near zero for
// every partial sum — this removes the truncation bias of the tensor-core fp32 accumulators (measured -3e-5 on e without
// it) and shrinks the fp32 rounding of the SIMT path as well. The epilogue adds c_j back: e = rowA_i - dot - c_j.
// One CTA per row; output pitch ldout >= G rounded up to 16, tail zero-filled.
__global__ void kl_prepare_rows_kernel(const float* __restrict__ X, int64_t G, int64_t ldin, float* __restrict__ out,
                                       int64_t ldout, float* __restrict__ rowterm, int is_fixed,
                                       const float* __restrict__ center_w) {
  const int64_t r = blockIdx.x;
  const float* x = X + r * ldin;
  float s = 0.f;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) s += x[g] + 0.01f;
  __shared__ float red[32];
  __shared__ double redd[32];
  __shared__ float total;
  __shared__ float centre;
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) total = t;
  }
  __syncthreads();
  const float inv = 1.0f / total;
  const float shift = logf((float)G);
  // moving side: xl = sum Xn (log Xn + log G);  fixed side with a centring profile w: xl = sum_g w_g (log Yn_g + log G)
  double xl = 0.0;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
    const float xn = (x[g] + 0.01f) * inv;
    const float lg = logf(xn + 1e-8f) + shift;
    if (!is_fixed) xl += (double)xn * (double)lg;
    else if (center_w != nullptr) xl += (double)center_w[g] * (double)lg;
  }
  xl = warp_sum(xl);
  if ((threadIdx.x & 31) == 0) redd[threadIdx.x >> 5] = xl;
  __syncthreads();
  if (threadIdx.x < 32) {
    double t = threadIdx.x < (blockDim.x >> 5) ? redd[threadIdx.x] : 0.0;
    t = warp_sum(t);
    if (threadIdx.x == 0) {
      centre = (is_fixed && center_w != nullptr) ? (float)t : 0.f;
      if (rowterm != nullptr) rowterm[r] = (float)t;
    }
  }
  __syncthreads();
  const float cj = centre;
  for (int64_t g = threadIdx.x; g < ldout; g += blockDim.x) {
    float o = 0.f;
    if (g < G) {
      const float xn = (x[g] + 0.01f) * inv;
      o = is_fixed ? (logf(xn + 1e-8f) + shift) - cj : xn;
    }
    out[r * ldout + g] = o;
  }
}

__global__ void rows_sqnorm_kernel(const float* __restrict__ X, int64_t G, int64_t ldin, float* __restrict__ rowterm) {
  const int64_t r = blockIdx.x;
  float s = 0.f;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
    const float v = X[r * ldin + g];
    s = fmaf(v, v, s);
  }
  __shared__ float red[32];
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) rowterm[r] = t;
  }
}

// out = X / max(|X|, 1e-8) (utils.py:736-739), zero-padded to ldout
__global__ void rows_normalize_kernel(const float* __restrict__ X, int64_t G, int64_t ldin, float* __restrict__ out,
                                      int64_t ldout) {
  const int64_t r = blockIdx.x;
  float s = 0.f;
  for (int64_t g = threadIdx.x; g < G; g += blockDim.x) {
    const float v = X[r * ldin + g];
    s = fmaf(v, v, s);
  }
  __shared__ float red[32];
  __shared__ float total;
  s = warp_sum(s);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x < 32) {
    float t = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    t = warp_sum(t);
    if (threadIdx.x == 0) total = t;
  }
  __syncthreads();
  const float inv = 1.0f / fmaxf(sqrtf(total), 1e-8f);
  for (int64_t g = threadIdx.x; g < ldout; g += blockDim.x) out[r * ldout + g] = g < G ? X[r * ldin + g] * inv : 0.f;
}

__device__ __forceinline__ float cost_to_prob(float dot, float ta, float tb, int metric, int prob_type, float neg_inv2b) {
  float e;
  if (metric == SPB_METRIC_KL) e = (ta - tb) - dot;                            // utils.py:697 (tb = centring term c_j)
  else if (metric == SPB_METRIC_SYMKL) e = 0.5f * ((ta + tb) - dot);             // utils.py:922-932
  else if (metric == SPB_METRIC_COS) e = fmaf(-0.5f, dot, 0.5f);               // utils.py:742
  else {
    e = fmaxf(ta + tb - 2.0f * dot, 0.0f);                                     // utils.py:780-783
    if (metric == SPB_METRIC_SQRT_EUC) e = sqrtf(e);                           // utils.py:786 ("square_euc" quirk)
  }
  if (prob_type == SPB_PROB_GAUSS) return __expf(e * neg_inv2b);               // utils.py:977
  if (prob_type == SPB_PROB_COS) return 1.0f - e;                              // utils.py:979
  return e;                                                                    // utils.py:981
}

constexpr int BM = 128, BN = 128, BK = 16, LDS_PAD = 4;

typedef unsigned long long u64;
__device__ __forceinline__ u64 pk2(float a, float b) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void upk2(u64 v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
// Hopper has no packed fp32x2 instructions: each pair operation is two scalar round-to-nearest operations (same bits)
__device__ __forceinline__ u64 add2p(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  return pk2(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
constexpr int kFlush = 16;  // k-blocks (of 16 features) between folds of the register partial sums
__device__ __forceinline__ u64 fma2p(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  upk2(a, a0, a1);
  upk2(b, b0, b1);
  upk2(c, c0, c1);
  return pk2(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}

__global__ void __launch_bounds__(256, 2)
gene_cost_kernel(const float* __restrict__ A, int64_t lda, const float* __restrict__ rtA, const float* __restrict__ B,
                 int64_t ldb, const float* __restrict__ rtB, int64_t NA, int64_t NB, int64_t Gp, int metric,
                 int prob_type, float neg_inv2b, int accumulate, float* __restrict__ GT, int64_t ldx) {
  __shared__ __align__(16) float As[2][BK][BM + LDS_PAD];  // moving cells i
  __shared__ __align__(16) float Bs[2][BK][BN + LDS_PAD];  // fixed cells j
  const int t = threadIdx.x;
  const int tx = t & 15, ty = t >> 4;
  const int64_t i0 = (int64_t)blockIdx.x * BM, j0 = (int64_t)blockIdx.y * BN;
  const int lrow = t >> 2, lq = t & 3;  // loader: rows lrow, lrow + 64; float4 quad lq
  // 8 (fixed cells j) x 8 (moving cells i) micro-tile held as 8 x 4 fp32-pair accumulators; the inner product is an FFMA
  // pair with a scalar-broadcast j operand
  u64 acc2[8][4];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc2[a][b] = 0ull;

  float4 ra[2], rb[2];
  auto gload = [&](int64_t k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t ia = i0 + lrow + 64 * h, jb = j0 + lrow + 64 * h;
      ra[h] = ia < NA ? *reinterpret_cast<const float4*>(A + ia * lda + k0 + lq * 4) : make_float4(0, 0, 0, 0);
      rb[h] = jb < NB ? *reinterpret_cast<const float4*>(B + jb * ldb + k0 + lq * 4) : make_float4(0, 0, 0, 0);
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = lrow + 64 * h;
      As[buf][lq * 4 + 0][row] = ra[h].x; As[buf][lq * 4 + 1][row] = ra[h].y;
      As[buf][lq * 4 + 2][row] = ra[h].z; As[buf][lq * 4 + 3][row] = ra[h].w;
      Bs[buf][lq * 4 + 0][row] = rb[h].x; Bs[buf][lq * 4 + 1][row] = rb[h].y;
      Bs[buf][lq * 4 + 2][row] = rb[h].z; Bs[buf][lq * 4 + 3][row] = rb[h].w;
    }
  };
  const int nk = (int)(Gp / BK);
  // Two-level accumulation: every kFlush k-blocks (256 features) the register partial sums are folded into per-thread
  // fp32 totals kept in shared memory, so a partial sum never grows beyond 1/8 of the final magnitude. This cuts the
  // rounding of the rank-G contraction ~20x (rms 8e-6 -> 4e-7 on e at G = 2000) for 2 % more issue slots.
  extern __shared__ u64 tot2[];  // [32][256] packed pairs, thread-contiguous
  const bool two_level = nk > kFlush;
  gload(0);
  sstore(0);
  __syncthreads();
  for (int kb = 0; kb < nk; ++kb) {
    const int buf = kb & 1;
    if (kb + 1 < nk) gload((int64_t)(kb + 1) * BK);
#pragma unroll
    for (int kk = 0; kk < BK; ++kk) {
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][kk][ty * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][kk][64 + ty * 4]);
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][kk][tx * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][kk][64 + tx * 4]);
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
      const u64 av2[4] = {pk2(a0.x, a0.y), pk2(a0.z, a0.w), pk2(a1.x, a1.y), pk2(a1.z, a1.w)};
#pragma unroll
      for (int a = 0; a < 8; ++a) {
        const u64 bb = pk2(bv[a], bv[a]);
#pragma unroll
        for (int b = 0; b < 4; ++b) acc2[a][b] = fma2p(bb, av2[b], acc2[a][b]);
      }
    }
    if (two_level && ((kb % kFlush) == kFlush - 1) && kb + 1 < nk) {
      const bool first = kb == kFlush - 1;
#pragma unroll
      for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) {
          const int q = (a * 4 + b) * 256 + t;
          tot2[q] = first ? acc2[a][b] : add2p(tot2[q], acc2[a][b]);
          acc2[a][b] = 0ull;
        }
    }
    if (kb + 1 < nk) {
      sstore(buf ^ 1);
      __syncthreads();
    }
  }
  if (two_level) {
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
      for (int b = 0; b < 4; ++b) acc2[a][b] = add2p(tot2[(a * 4 + b) * 256 + t], acc2[a][b]);
  }
  float acc[8][8];
#pragma unroll
  for (int a = 0; a < 8; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) upk2(acc2[a][b], acc[a][2 * b], acc[a][2 * b + 1]);
  // epilogue: acc[a][b] -> j = j0 + (a<4 ? ty*4+a : 64+ty*4+a-4), i = i0 + (b<4 ? tx*4+b : 64+tx*4+b-4)
  float ta[8];
#pragma unroll
  for (int b = 0; b < 8; ++b) {
    const int64_t i = i0 + (b < 4 ? tx * 4 + b : 64 + tx * 4 + b - 4);
    ta[b] = (rtA != nullptr && i < NA) ? rtA[i] : 0.f;
  }
#pragma unroll
  for (int a = 0; a < 8; ++a) {
    const int64_t j = j0 + (a < 4 ? ty * 4 + a : 64 + ty * 4 + a - 4);
    if (j >= NB) continue;
    const float tb = rtB != nullptr ? rtB[j] : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t ib = i0 + h * 64 + tx * 4;
      float o[4];
#pragma unroll
      for (int b = 0; b < 4; ++b) {
        const int64_t i = ib + b;
        o[b] = i < NA ? cost_to_prob(acc[a][h * 4 + b], ta[h * 4 + b], tb, metric, prob_type, neg_inv2b) : 0.f;
      }
      float4* dst = reinterpret_cast<float4*>(GT + j * ldx + ib);
      if (accumulate) {
        const float4 old = *dst;
        o[0] *= old.x; o[1] *= old.y; o[2] *= old.z; o[3] *= old.w;
      }
      *dst = make_float4(o[0], o[1], o[2], o[3]);
    }
  }
}

__global__ void label_cost_kernel(const int32_t* __restrict__ labA, const int32_t* __restrict__ labB,
                                  const float* __restrict__ LT, int nB_labels, int64_t NA, int64_t NB, int accumulate,
                                  float* __restrict__ GT, int64_t ldx) {
  const int64_t j = blockIdx.y;
  const int lb = labB[j];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ldx; i += (int64_t)gridDim.x * blockDim.x) {
    float v = i < NA ? LT[(int64_t)labA[i] * nB_labels + lb] : 0.f;
    if (accumulate) v *= GT[j * ldx + i];
    GT[j * ldx + i] = v;
  }
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" int spb_kl_prepare_rows(const float* X, int64_t n, int64_t G, int64_t ldin, float* out, int64_t ldout,
                                   float* rowterm, int32_t is_fixed, const float* center_w, void* stream) {
  if (n <= 0) return 0;
  if (ldout % kPadG != 0 || ldout < G) return SPB_EINVAL;
  kl_prepare_rows_kernel<<<(unsigned)n, 256, 0, ST>>>(X, G, ldin, out, ldout, rowterm, is_fixed, center_w);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_rows_sqnorm(const float* X, int64_t n, int64_t G, int64_t ldin, float* rowterm, void* stream) {
  if (n <= 0) return 0;
  rows_sqnorm_kernel<<<(unsigned)n, 256, 0, ST>>>(X, G, ldin, rowterm);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_rows_normalize(const float* X, int64_t n, int64_t G, int64_t ldin, float* out, int64_t ldout,
                                  void* stream) {
  if (n <= 0) return 0;
  if (ldout % kPadG != 0 || ldout < G) return SPB_EINVAL;
  rows_normalize_kernel<<<(unsigned)n, 256, 0, ST>>>(X, G, ldin, out, ldout);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_gene_cost(const float* A, int64_t lda, const float* rowtermA, const float* B, int64_t ldb,
                             const float* rowtermB, int64_t NA, int64_t NB, int64_t G, int32_t metric, int32_t prob_type,
                             float prob_param, int32_t accumulate, float* GT, int64_t ldx, void* stream) {
  if (lda % 4 != 0 || ldb % 4 != 0 || ldx % BM != 0) return SPB_EINVAL;
  const int64_t Gp = ((G + BK - 1) / BK) * BK;
  if (lda < Gp || ldb < Gp) return SPB_EINVAL;  // operands must be zero-padded to a multiple of 16 features
  const float neg_inv2b = prob_type == SPB_PROB_GAUSS ? -1.0f / (2.0f * prob_param) : 0.f;
  dim3 grid((unsigned)(ldx / BM), (unsigned)((NB + BN - 1) / BN));
  const size_t dyn = 32 * 256 * sizeof(unsigned long long);  // second-level accumulators
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(gene_cost_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  gene_cost_kernel<<<grid, 256, dyn, ST>>>(A, lda, rowtermA, B, ldb, rowtermB, NA, NB, Gp, metric, prob_type, neg_inv2b,
                                         accumulate, GT, ldx);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_label_cost(const int32_t* labA, const int32_t* labB, const float* LT, int32_t nB_labels, int64_t NA,
                              int64_t NB, int32_t accumulate, float* GT, int64_t ldx, void* stream) {
  dim3 grid((unsigned)((ldx + 1023) / 1024), (unsigned)NB);
  label_cost_kernel<<<grid, 256, 0, ST>>>(labA, labB, LT, nB_labels, NA, NB, accumulate, GT, ldx);
  SPB_CHECK_LAUNCH();
  return 0;
}
