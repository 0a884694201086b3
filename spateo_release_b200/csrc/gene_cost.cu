// Expression cost / probability matrix (replaces calc_distance + calc_probability for the representation layers:
// spateo/alignment/methods/utils.py:647-788, 866-985). One-off per pair, outside the EM loop.
//
// GT[j][i] = prob(metric(A_i, B_j)), written in the layout the E-step sweeps stream (one contiguous row per fixed cell).
// This file holds the row pre-passes that turn expression rows into contraction operands, and the label layer. The
// contraction is gene_cost_tc.cu (wgmma, 3xTF32 split): fp32-accurate dot products are required because the KL cost is a
// small difference of O(7) terms that is then divided by 2*beta^2 ~ 0.02.
#include "common.cuh"

namespace {

constexpr int kPadG = 16;  // feature pitch granularity produced by the prep kernels

// Xn = (X + .01) / rowsum, rowterm = sum Xn log(Xn + 1e-8)  (moving side), or out = log(Xn + 1e-8) (fixed side)
// (utils.py:683-695). Both log terms are shifted by +log(G): KL = sum Xn (logX + c) - sum Xn (logY + c) for any c, and
// with c = log G the summands are O(Xn) instead of O(7 Xn), which cuts the fp32 rounding of the rank-G contraction.
// Fixed side with `center_w` (a probability profile, e.g. the mean moving row): the row is additionally centred by
// c_j = sum_g w_g (log Y_jg + c), returned as its row term, so that sum_g Xn_ig * out_jg = dot_ij - c_j stays near zero for
// every partial sum — this reduces the rounding bias of the tensor-core fp32 accumulators. At G = 2,000 (benchmark data,
// H100) the max error on e is 2.3e-5 with it and 5.4e-5 without; the fp32 reference is 3.3e-5 off float64. The log G
// shift moves that error by < 1e-6 at this G. The epilogue adds c_j back: e = rowA_i - dot - c_j.
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

// GT[j][i] (op)= LT[labA[i]][labB[j]]. Fixed cells stride over grid.y, which is capped at 65,535 blocks.
constexpr int64_t kMaxGridY = 65535;

__global__ void label_cost_kernel(const int32_t* __restrict__ labA, const int32_t* __restrict__ labB,
                                  const float* __restrict__ LT, int nB_labels, int64_t NA, int64_t NB, int accumulate,
                                  float* __restrict__ GT, int64_t ldx) {
  for (int64_t j = blockIdx.y; j < NB; j += gridDim.y) {
    const int lb = labB[j];
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < ldx; i += (int64_t)gridDim.x * blockDim.x) {
      float v = i < NA ? LT[(int64_t)labA[i] * nB_labels + lb] : 0.f;
      if (accumulate) v *= GT[j * ldx + i];
      GT[j * ldx + i] = v;
    }
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

extern "C" int spb_label_cost(const int32_t* labA, const int32_t* labB, const float* LT, int32_t nB_labels, int64_t NA,
                              int64_t NB, int32_t accumulate, float* GT, int64_t ldx, void* stream) {
  if (NB <= 0 || ldx <= 0) return 0;
  dim3 grid((unsigned)((ldx + 1023) / 1024), (unsigned)std::min<int64_t>(NB, kMaxGridY));
  label_cost_kernel<<<grid, 256, 0, ST>>>(labA, labB, LT, nB_labels, NA, NB, accumulate, GT, ldx);
  SPB_CHECK_LAUNCH();
  return 0;
}
