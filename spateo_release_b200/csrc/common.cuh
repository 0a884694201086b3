// Shared device helpers for the sm_90a kernels: bulk-async (TMA 1-D) copies, mbarriers, warp reductions,
// digamma, small dense linear algebra in fp64.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/spateo_b200.h"

#define SPB_STAGES 3

extern "C" int64_t spb_launch_count(void);
int spb_gram_tc_warm();  // gram_tc.cu
void spb_count_launch(int n = 1);

// kernel attributes (dynamic shared-memory opt-in) are per device: index the "already set" flags by the current device
#define SPB_MAX_DEVICES 64
static inline int spb_current_device() {
  int d = 0;
  cudaGetDevice(&d);
  return (d >= 0 && d < SPB_MAX_DEVICES) ? d : 0;
}

// SM count of the current device, for grid sizing (cached per device)
static inline int spb_num_sms() {
  static int n_dev[SPB_MAX_DEVICES] = {};
  const int d = spb_current_device();
  if (n_dev[d] == 0) {
    int n = 0;
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, d);
    n_dev[d] = n > 0 ? n : 1;
  }
  return n_dev[d];
}

#define SPB_CHECK_LAUNCH()                      \
  do {                                          \
    cudaError_t e__ = cudaGetLastError();       \
    if (e__ != cudaSuccess) return (int)e__;    \
    spb_count_launch();                         \
  } while (0)

// ---------------------------------------------------------------------------------------------------------------------
// mbarrier + cp.async.bulk (global -> shared, completes on an mbarrier). SASS: UBLKCP / SYNCS.
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ uint32_t mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n"
      "selp.u32 %0, 1, 0, p;\n"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk copy: dst/src 16-byte aligned, bytes % 16 == 0
__device__ __forceinline__ void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

__device__ __forceinline__ float ex2f(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ---------------------------------------------------------------------------------------------------------------------
// reductions
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-reduce NV doubles (blockDim.x multiple of 32, <= 1024) and atomically add them to dst[0..NV).
template <int NV>
__device__ __forceinline__ void block_reduce_atomic(double (&v)[NV], double* dst) {
  __shared__ double red_[32][NV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = warp_sum(v[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) red_[warp][q] = v[q];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double x = lane < nw ? red_[lane][q] : 0.0;
      x = warp_sum(x);
      if (lane == 0) atomicAdd(dst + q, x);
    }
  }
  __syncthreads();
}

// Deterministic grid-wide sum of NV doubles per block: every block stores its block-reduced partials, the LAST block to
// arrive (atomic ticket) adds the gridDim.x partials of each value in a fixed order and writes (or adds to) dst. Unlike
// block_reduce_atomic the result does not depend on block scheduling, so replicas of the EM on several GPUs stay bit-identical
// (column-sharded pair) and runs are reproducible. partials: [gridDim.x][NV]; counter: zero before the first use (it is
// reset by the last block). blockDim.x multiple of 32, <= 1024.
template <int NV>
__device__ __forceinline__ void grid_reduce_ordered(double (&v)[NV], double* __restrict__ partials, unsigned int* counter,
                                                    double* dst, bool accumulate) {
  __shared__ double red_[32][NV];
  __shared__ bool is_last_;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
  for (int q = 0; q < NV; ++q) v[q] = warp_sum(v[q]);
  if (lane == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) red_[warp][q] = v[q];
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int q = 0; q < NV; ++q) {
      double x = lane < nw ? red_[lane][q] : 0.0;
      x = warp_sum(x);
      if (lane == 0) partials[(size_t)blockIdx.x * NV + q] = x;
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last_ = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last_) return;
  __threadfence();
  for (int q = warp; q < NV; q += nw) {
    double x = 0.0;
    for (unsigned b = lane; b < gridDim.x; b += 32) x += partials[(size_t)b * NV + q];
    x = warp_sum(x);
    if (lane == 0) dst[q] = accumulate ? dst[q] + x : x;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

// ---------------------------------------------------------------------------------------------------------------------
// digamma for x > 0 (scipy.special.psi on the reference path, utils.py:1434)
// ---------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double digamma_pos(double x) {
  double r = 0.0;
  while (x < 10.0) {
    r -= 1.0 / x;
    x += 1.0;
  }
  const double f = 1.0 / (x * x);
  // asymptotic series: ln x - 1/2x - sum B_2n / (2n x^2n)
  const double t = f * (-1.0 / 12.0 + f * (1.0 / 120.0 + f * (-1.0 / 252.0 + f * (1.0 / 240.0 + f * (-1.0 / 132.0 + f * (691.0 / 32760.0 + f * (-1.0 / 12.0)))))));
  return r + log(x) - 0.5 / x + t;
}

// ---------------------------------------------------------------------------------------------------------------------
// DxD (D<=3) SVD by two-sided Jacobi on A^T A, singular values sorted descending (LAPACK order, needed for the
// reflection fix C[-1,-1] = det(U Vh), morpho_class.py:1370-1374). A = U diag(s) Vh. Row-major 3x3 storage.
// ---------------------------------------------------------------------------------------------------------------------
__device__ inline void svd_small(const double* A, int D, double* U, double* S, double* Vh) {
  double W[9], V[9];
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < D; ++j) {
      W[i * 3 + j] = A[i * 3 + j];
      V[i * 3 + j] = (i == j) ? 1.0 : 0.0;
    }
  // one-sided (Hestenes) Jacobi: rotate column pairs of W until they are mutually orthogonal; A V = W
  for (int sweep = 0; sweep < 60; ++sweep) {
    bool rotated = false;
    for (int p = 0; p < D; ++p)
      for (int q = p + 1; q < D; ++q) {
        double al = 0, be = 0, ga = 0;
        for (int k = 0; k < D; ++k) {
          al += W[k * 3 + p] * W[k * 3 + p];
          be += W[k * 3 + q] * W[k * 3 + q];
          ga += W[k * 3 + p] * W[k * 3 + q];
        }
        if (ga == 0.0 || fabs(ga) <= 1e-17 * sqrt(al * be)) continue;
        rotated = true;
        const double zeta = (be - al) / (2.0 * ga);
        const double tt = (zeta >= 0 ? 1.0 : -1.0) / (fabs(zeta) + sqrt(1.0 + zeta * zeta));
        const double c = 1.0 / sqrt(1.0 + tt * tt), sn = c * tt;
        for (int k = 0; k < D; ++k) {
          const double wp = W[k * 3 + p], wq = W[k * 3 + q];
          W[k * 3 + p] = c * wp - sn * wq;
          W[k * 3 + q] = sn * wp + c * wq;
          const double vp = V[k * 3 + p], vq = V[k * 3 + q];
          V[k * 3 + p] = c * vp - sn * vq;
          V[k * 3 + q] = sn * vp + c * vq;
        }
      }
    if (!rotated) break;
  }
  double nrm[3] = {0, 0, 0};
  for (int c = 0; c < D; ++c) {
    double s2 = 0;
    for (int k = 0; k < D; ++k) s2 += W[k * 3 + c] * W[k * 3 + c];
    nrm[c] = sqrt(s2);
  }
  int ord[3] = {0, 1, 2};
  for (int a = 0; a < D; ++a)
    for (int b = a + 1; b < D; ++b)
      if (nrm[ord[b]] > nrm[ord[a]]) {
        int t = ord[a];
        ord[a] = ord[b];
        ord[b] = t;
      }
  const double smax = nrm[ord[0]] > 0 ? nrm[ord[0]] : 1.0;
  for (int c = 0; c < D; ++c) {
    const int oc = ord[c];
    S[c] = nrm[oc];
    for (int k = 0; k < D; ++k) Vh[c * 3 + k] = V[k * 3 + oc];
    if (nrm[oc] > 1e-300 && nrm[oc] > 1e-15 * smax) {
      for (int r = 0; r < D; ++r) U[r * 3 + c] = W[r * 3 + oc] / nrm[oc];
    } else {
      // null direction: any unit vector orthogonal to the columns already chosen
      for (int e = 0; e < D; ++e) {
        double w[3] = {0, 0, 0};
        w[e] = 1.0;
        for (int pc = 0; pc < c; ++pc) {
          double dp = 0;
          for (int r = 0; r < D; ++r) dp += w[r] * U[r * 3 + pc];
          for (int r = 0; r < D; ++r) w[r] -= dp * U[r * 3 + pc];
        }
        double n2 = 0;
        for (int r = 0; r < D; ++r) n2 += w[r] * w[r];
        if (n2 > 1e-6) {
          n2 = sqrt(n2);
          for (int r = 0; r < D; ++r) U[r * 3 + c] = w[r] / n2;
          break;
        }
      }
    }
  }
}

__device__ inline double det_small(const double* M, int D) {
  if (D == 2) return M[0] * M[4] - M[1] * M[3];
  return M[0] * (M[4] * M[8] - M[5] * M[7]) - M[1] * (M[3] * M[8] - M[5] * M[6]) + M[2] * (M[3] * M[7] - M[4] * M[6]);
}

// R = U diag(1,..,det(U Vh)) Vh  — the proper rotation closest to A (Kabsch)
__device__ inline void rotation_from(const double* A, int D, double* R) {
  double U[9], S[3], Vh[9], UV[9];
  svd_small(A, D, U, S, Vh);
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < D; ++j) {
      double s = 0;
      for (int k = 0; k < D; ++k) s += U[i * 3 + k] * Vh[k * 3 + j];
      UV[i * 3 + j] = s;
    }
  const double dt = det_small(UV, D);
  for (int i = 0; i < D; ++i)
    for (int j = 0; j < D; ++j) {
      double s = 0;
      for (int k = 0; k < D; ++k) s += U[i * 3 + k] * (k == D - 1 ? dt : 1.0) * Vh[k * 3 + j];
      R[i * 3 + j] = s;
    }
}
