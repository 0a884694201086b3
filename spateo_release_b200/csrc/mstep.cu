// M-step of the morpho-align EM on the device (spateo/alignment/methods/morpho_class.py:1202-1469): gamma / alpha
// (digamma), the non-rigid inducing-point solve (U^T diag(K_NA) U contraction, symmetric eigen pseudo-inverse, field
// application), the rigid Procrustes update from weighted moments, sigma2, and the per-row state refresh.
// All scalar state lives in `spb_scalars` on the device: no host synchronisation inside an iteration.
#include "common.cuh"

namespace {

constexpr double kLog2e = 1.4426950408889634;
constexpr double kTwoPi = 6.283185307179586;

// ---------------------------------------------------------------------------------------------------------------------
__global__ void iter_begin_kernel(spb_em_params p, int iter) {
  spb_scalars* sc = p.sc;
  const int K = p.K;
  if (iter < 0) iter = sc->iter + 1;  // graph replay: the iteration counter lives on the device
  for (int q = threadIdx.x; q < K * K; q += blockDim.x) p.UtWU[q] = 0.0;
  for (int q = threadIdx.x; q < K * 3; q += blockDim.x) p.UtPXB[q] = 0.0;
  for (int q = threadIdx.x; q < 32; q += blockDim.x) p.moments[q] = 0.0;
  if (threadIdx.x == 0) {
    sc->iter = iter;
    sc->step = p.svi ? fmin(1.0, 10.0 / (iter + 1.0)) : 1.0;  // morpho_class.py:894
    for (int q = 0; q < 8; ++q) sc->sums[q] = 0.0;
    sc->dotKS = 0.0;
    sc->visited = 0.0;
    const double s2 = sc->sigma2, g = sc->gamma;
    const double outlier_s = p.samples_s * (double)p.NA;                                   // utils.py:1051
    sc->omega = pow(kTwoPi * s2, 0.5 * p.D) * (1.0 - g) / (g * outlier_s);                 // utils.py:1053
    const double cq = -kLog2e / (2.0 * s2);
    sc->c_q = (float)cq;
    sc->c_s = (float)(cq * sc->sigma2_variance);                                           // utils.py:1049
  }
}

// Sp running averages, sigma2_related, gamma (morpho_class.py:1178-1200, 1214-1224)
__global__ void scalar_update_kernel(spb_em_params p) {
  spb_scalars* sc = p.sc;
  const double step = sc->step;
  const double nsp = sc->sums[0], ns2 = sc->sums[1], nS = sc->sums[2], S2 = sc->sums[3];
  if (p.svi) {
    sc->Sp_spatial = step * nsp + (1.0 - step) * sc->Sp_spatial;
    sc->Sp = step * nS + (1.0 - step) * sc->Sp;
    sc->Sp_sigma2 = step * ns2 + (1.0 - step) * sc->Sp_sigma2;
  } else {
    sc->Sp_spatial = nsp;
    sc->Sp = nS;
    sc->Sp_sigma2 = ns2;
  }
  sc->SpK = nS;
  sc->sigma2_related = S2 / ((double)p.D * sc->Sp_sigma2);
  double g = exp(digamma_pos(p.gamma_a + sc->Sp_spatial) - digamma_pos(p.gamma_a + p.gamma_b + (double)(p.NB_total > 0 ? p.NB_total : p.NBb)));
  sc->gamma = fmax(fmin(g, 0.99), 0.01);
}

// alpha_i (morpho_class.py:1238-1252)
__global__ void alpha_update_kernel(spb_em_params p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.NA) return;
  const spb_scalars* sc = p.sc;
  const double kap = (double)p.kappa[i];
  const double a = exp(digamma_pos(kap + (double)p.K_NA_spatial[i]) - digamma_pos(kap * (double)p.NA + sc->Sp_spatial));
  if (p.svi) {
    const double step = sc->step;
    p.alpha[i] = (float)(step * a + (1.0 - step) * (double)p.alpha[i]);
  } else {
    p.alpha[i] = (float)a;
  }
}

// PXB_term = P@XB - RnA * K_NA (SVI: running average) (morpho_class.py:1270-1276)
__global__ void pxb_term_kernel(spb_em_params p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.NA) return;
  const double step = p.sc->step;
  const float k = p.K_NA[i];
  for (int d = 0; d < 3; ++d) {
    const int64_t o = (int64_t)d * p.ldx + i;
    const float nw = p.PXB[o] - p.RnA[o] * k;
    p.PXB_term[o] = p.svi ? (float)(step * (double)nw + (1.0 - step) * (double)p.PXB_term[o]) : nw;
  }
}

// U^T diag(w) U  and  U^T X3 with fp64 products (spb_weighted_gram: the reference-accurate path of SparseVFC above 32 inducing
// points): 64 x 64 output tiles of the block upper triangle, 256 threads x (4 x 4) register tiles, operands converted to
// double ONCE while they are staged through shared memory (32 rows of n per chunk), atomics into the K x K accumulator.
// grid.x = row chunks, grid.y = (kt, lt) tile pairs with kt <= lt.
constexpr int kGT = 64;        // tile edge
constexpr int kGC = 32;        // rows of n per shared-memory chunk
constexpr int kAccRows = 128;  // granularity of the row chunks
inline int gram_rows_per_block(int64_t N, int npairs) {
  const int64_t want_chunks = (2 * spb_num_sms() + npairs - 1) / npairs;  // ~2 CTAs per SM
  int64_t rows = (N + want_chunks - 1) / want_chunks;
  rows = ((rows + kAccRows - 1) / kAccRows) * kAccRows;
  if (rows < 2 * kAccRows) rows = 2 * kAccRows;
  if (rows > 16384) rows = 16384;
  return (int)rows;
}
__global__ void __launch_bounds__(256)
weighted_gram_kernel(const float* __restrict__ UT, int64_t ldx, int N, int K, const float* __restrict__ w,
                     const float* __restrict__ X3, double* __restrict__ UtWU, double* __restrict__ UtX,
                     int rows_per_block, int ntile) {
  __shared__ double As[kGC][kGT + 1];
  __shared__ double Bs[kGC][kGT + 1];
  __shared__ double Xs[kGC][3];
  int kt = 0, lt = 0;
  {
    int q = blockIdx.y;
    for (kt = 0; kt < ntile; ++kt) {
      const int cnt = ntile - kt;
      if (q < cnt) {
        lt = kt + q;
        break;
      }
      q -= cnt;
    }
  }
  const int ty = threadIdx.x >> 4, tx = threadIdx.x & 15;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  double accx = 0.0;  // U^T X entry (threads < 192 of diagonal tiles: row kk = tid / 3, column d = tid % 3)
  const int r_begin = blockIdx.x * rows_per_block;
  const int r_end = min(N, r_begin + rows_per_block);
  for (int r0 = r_begin; r0 < r_end; r0 += kGC) {
    const int nr = min(kGC, r_end - r0);
    __syncthreads();
    for (int q = threadIdx.x; q < kGT * kGC; q += 256) {
      const int kk = q / kGC, rr = q % kGC;  // a warp reads 32 consecutive n of one row: coalesced
      const int k = kt * kGT + kk, l = lt * kGT + kk;
      const bool ok = rr < nr;
      const float wv = ok ? w[r0 + rr] : 0.f;
      As[rr][kk] = (ok && k < K) ? (double)UT[(int64_t)k * ldx + r0 + rr] : 0.0;
      // w * u is rounded to fp32 first, like the reference's fp32 product (and the small-K kernel)
      Bs[rr][kk] = (ok && l < K) ? (double)(UT[(int64_t)l * ldx + r0 + rr] * wv) : 0.0;
    }
    if (kt == lt && threadIdx.x < kGC * 3) {
      const int rr = threadIdx.x / 3, d = threadIdx.x % 3;
      Xs[rr][d] = rr < nr ? (double)X3[(int64_t)d * ldx + r0 + rr] : 0.0;
    }
    __syncthreads();
#pragma unroll 8
    for (int rr = 0; rr < kGC; ++rr) {
      double a[4], b[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        a[q] = As[rr][ty * 4 + q];
        b[q] = Bs[rr][tx * 4 + q];
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] += a[i] * b[j];
    }
    if (kt == lt && threadIdx.x < kGT * 3) {
      const int kk = threadIdx.x / 3, d = threadIdx.x % 3;
      for (int rr = 0; rr < kGC; ++rr) accx += As[rr][kk] * Xs[rr][d];
    }
  }
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) {
      const int k = kt * kGT + ty * 4 + a, l = lt * kGT + tx * 4 + b;
      if (k < K && l < K) {
        atomicAdd(&UtWU[(int64_t)k * K + l], acc[a][b]);
        if (kt != lt) atomicAdd(&UtWU[(int64_t)l * K + k], acc[a][b]);
      }
    }
  if (kt == lt && threadIdx.x < kGT * 3) {
    const int k = kt * kGT + threadIdx.x / 3, d = threadIdx.x % 3;
    if (k < K) atomicAdd(&UtX[k * 3 + d], accx);
  }
}

// Small inducing sets (K <= 32): every thread owns a few of the K x (K + 3) entries, rows are staged through shared memory
// in chunks of 128, fp64 products and accumulation as in weighted_gram_kernel (same numerics, ~10x less time at K = 15).
constexpr int kSmallK = 32;
__global__ void __launch_bounds__(256)
gram_small_kernel(const float* __restrict__ UT, int64_t ldx, int N, int K, const float* __restrict__ w,
                  const float* __restrict__ X3, double* __restrict__ UtWU, double* __restrict__ UtX, int rows_per_block,
                  double* __restrict__ partials, unsigned int* counter) {
  constexpr int kChunk = 128, kPitch = kChunk + 1;
  __shared__ float As[kSmallK][kPitch];
  __shared__ float Bs[kSmallK + 3][kPitch];
  __shared__ bool is_last;
  const int KB = K + 3, nent = K * KB;
  constexpr int kPer = (kSmallK * (kSmallK + 3) + 255) / 256;  // 5 entries per thread at most
  double acc[kPer];
  int ek[kPer], el[kPer];
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    const int e = threadIdx.x + q * 256;
    acc[q] = 0.0;
    ek[q] = e < nent ? e / KB : -1;
    el[q] = e < nent ? e % KB : 0;
  }
  const int r_begin = blockIdx.x * rows_per_block, r_end = min(N, r_begin + rows_per_block);
  for (int r0 = r_begin; r0 < r_end; r0 += kChunk) {
    const int nr = min(kChunk, r_end - r0);
    __syncthreads();
    for (int q = threadIdx.x; q < KB * kChunk; q += 256) {
      const int row = q / kChunk, rr = q % kChunk;
      const bool ok = rr < nr;
      float a = 0.f, b = 0.f;
      if (ok) {
        if (row < K) {
          a = UT[(int64_t)row * ldx + r0 + rr];
          b = a * w[r0 + rr];
        } else {
          b = X3[(int64_t)(row - K) * ldx + r0 + rr];
        }
      }
      if (row < K) As[row][rr] = a;
      Bs[row][rr] = b;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < kPer; ++q) {
      if (ek[q] < 0) continue;
      const float* ar = As[ek[q]];
      const float* br = Bs[el[q]];
      double s = 0.0;
      for (int rr = 0; rr < kChunk; ++rr) s += (double)ar[rr] * (double)br[rr];
      acc[q] += s;
    }
  }
  // deterministic fold over the CTAs: partials[block][entry], the last CTA to arrive adds them in block order
#pragma unroll
  for (int q = 0; q < kPer; ++q)
    if (ek[q] >= 0) partials[(size_t)blockIdx.x * nent + threadIdx.x + q * 256] = acc[q];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(counter, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
#pragma unroll
  for (int q = 0; q < kPer; ++q) {
    if (ek[q] < 0) continue;
    const int e = threadIdx.x + q * 256;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    unsigned b = 0;
    for (; b + 4 <= gridDim.x; b += 4) {
      s0 += partials[(size_t)(b + 0) * nent + e];
      s1 += partials[(size_t)(b + 1) * nent + e];
      s2 += partials[(size_t)(b + 2) * nent + e];
      s3 += partials[(size_t)(b + 3) * nent + e];
    }
    for (; b < gridDim.x; ++b) s0 += partials[(size_t)b * nent + e];
    const double t = (s0 + s1) + (s2 + s3);
    if (el[q] < K) UtWU[(int64_t)ek[q] * K + el[q]] = t;
    else UtX[ek[q] * 3 + (el[q] - K)] = t;
  }
  if (threadIdx.x == 0) *counter = 0u;
}

// SparseVFC E-step (dynamo scVectorField.SparseVFC get_P + bookkeeping; SURVEY.md Appendix E — parity unpinned):
//   V_i = U_i C, r_i = |Y_i - V_i|^2, P_i = t1 / (t1 + t2), t1 = exp(-r / 2 sigma2), then the clamp to minP.
// sums: [0] sum P_pre r  [1] sum P_pre  [2] sum P r  [3] sum P  [4] #{P > theta}
__global__ void __launch_bounds__(128)
vfc_estep_kernel(const float* __restrict__ UT, int64_t ldn, int N, int M, int D, const double* __restrict__ Cf,
                 const double* __restrict__ Y, double sigma2, double t2, double minP, double theta,
                 double* __restrict__ P, double* __restrict__ V, float* __restrict__ Pf, float* __restrict__ PY3,
                 double* __restrict__ sums) {
  double v[5] = {0, 0, 0, 0, 0};
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < N) {
    double acc[3] = {0, 0, 0};
    for (int m = 0; m < M; ++m) {
      const double u = (double)UT[(int64_t)m * ldn + i];
      acc[0] += u * Cf[m * 3 + 0];
      acc[1] += u * Cf[m * 3 + 1];
      acc[2] += u * Cf[m * 3 + 2];
    }
    double r = 0.0, y[3] = {0, 0, 0};
    for (int d = 0; d < D; ++d) {
      y[d] = Y[(int64_t)i * D + d];
      const double df = y[d] - acc[d];
      r += df * df;
      V[(int64_t)i * D + d] = acc[d];
    }
    const double t1 = exp(-r / (2.0 * sigma2));
    const double ppre = t1 / (t1 + t2);
    const double p = fmax(ppre, minP);
    P[i] = p;
    Pf[i] = (float)p;
    for (int d = 0; d < 3; ++d) PY3[(int64_t)d * ldn + i] = d < D ? (float)(p * y[d]) : 0.f;
    v[0] = ppre * r; v[1] = ppre; v[2] = p * r; v[3] = p; v[4] = ppre > theta ? 1.0 : 0.0;
  }
  block_reduce_atomic<5>(v, sums);
}

// SigmaInv = sigma2 lambda Gamma + U^T W U (SVI running average) (morpho_class.py:1266-1277)
__global__ void nonrigid_blend_kernel(spb_em_params p) {
  const int K = p.K;
  const spb_scalars* sc = p.sc;
  const double step = sc->step, s2l = sc->sigma2 * p.lambdaVF;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < K * K; q += gridDim.x * blockDim.x) {
    const double nw = s2l * (double)p.Gamma[q] + p.UtWU[q];
    double a = p.svi ? step * nw + (1.0 - step) * p.SigmaInv[q] : nw;
    if (p.g_on && p.g_nonrigid) a += (sc->sigma2 * p.g_weight * sc->Sp / (double)p.g_NI) * p.g_G1[q];  // :1282-1285
    p.SigmaInv[q] = a;
  }
}

// Symmetric eigen-decomposition by parallel cyclic Jacobi in shared memory (K <= 64), pseudo-inverse with scipy's
// cutoff rtol = K * eps(float32) (scipy.linalg.pinv on the reference's fp32 matrix, utils.py:1435), Coff = Sigma UPXB.
__global__ void __launch_bounds__(256) nonrigid_solve_kernel(spb_em_params p) {
  extern __shared__ double sh[];
  const int K = p.K;
  const int Kp = (K + 1) & ~1;
  double* A = sh;                  // [Kp][Kp]
  double* V = A + Kp * Kp;         // [Kp][Kp]
  double* cs = V + Kp * Kp;        // [Kp] (c, s) per pair
  int* top = reinterpret_cast<int*>(cs + Kp);
  int* bot = top + Kp / 2;
  __shared__ double s_off, s_diag;
  const spb_scalars* sc = p.sc;
  const double step = sc->step, s2l = sc->sigma2 * p.lambdaVF;
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int q = tid; q < Kp * Kp; q += nt) {
    const int r = q / Kp, c = q % Kp;
    double a = 0.0;
    if (r < K && c < K) {
      const double nw = s2l * (double)p.Gamma[r * K + c] + p.UtWU[r * K + c];
      a = p.svi ? step * nw + (1.0 - step) * p.SigmaInv[r * K + c] : nw;
      // guidance term; it is added to the stored (running-average) matrix like the reference does (:1282-1285)
      if (p.g_on && p.g_nonrigid) a += (sc->sigma2 * p.g_weight * sc->Sp / (double)p.g_NI) * p.g_G1[r * K + c];
      p.SigmaInv[r * K + c] = a;
    }
    A[q] = a;
    V[q] = (r == c) ? 1.0 : 0.0;
  }
  if (tid < Kp / 2) {
    top[tid] = 2 * tid;
    bot[tid] = 2 * tid + 1;
  }
  __syncthreads();
  // symmetrise (atomics order may differ between the two triangles by rounding)
  for (int q = tid; q < Kp * Kp; q += nt) {
    const int r = q / Kp, c = q % Kp;
    if (r < c) {
      const double m = 0.5 * (A[r * Kp + c] + A[c * Kp + r]);
      A[r * Kp + c] = m;
      A[c * Kp + r] = m;
    }
  }
  __syncthreads();
  // Warm start: SigmaInv changes little from one EM iteration to the next, so in the eigenbasis V0 of the previous
  // iteration it is already nearly diagonal. Rotate A <- V0^T A V0 (two K^3 products in shared memory) and continue the
  // Jacobi sweeps from V = V0: 2-4 sweeps instead of 8-10 from the identity.
  double* ws = p.jacobi_ws;
  const bool warm = ws != nullptr && ws[0] == (double)K;
  if (warm) {
    double* T = cs + Kp + Kp;  // [Kp][Kp] scratch behind the index arrays
    const double* V0 = ws + 1;
    for (int q = tid; q < Kp * Kp; q += nt) {
      const int r = q / Kp, c = q % Kp;
      V[q] = (r < K && c < K) ? V0[r * K + c] : (r == c ? 1.0 : 0.0);
    }
    __syncthreads();
    for (int q = tid; q < Kp * Kp; q += nt) {  // T = A V
      const int r = q / Kp, c = q % Kp;
      double t = 0.0;
      for (int e = 0; e < Kp; ++e) t += A[r * Kp + e] * V[e * Kp + c];
      T[q] = t;
    }
    __syncthreads();
    for (int q = tid; q < Kp * Kp; q += nt) {  // A = V^T T (upper triangle, mirrored: exactly symmetric)
      const int r = q / Kp, c = q % Kp;
      if (r <= c) {
        double t = 0.0;
        for (int e = 0; e < Kp; ++e) t += V[e * Kp + r] * T[e * Kp + c];
        A[r * Kp + c] = t;
        A[c * Kp + r] = t;
      }
    }
    __syncthreads();
  }
  const int npair = Kp / 2;
  for (int sweep = 0; sweep < 30; ++sweep) {
    // convergence: off-diagonal mass below 1e-30 of the diagonal mass (eigenvalues then carry ~1e-15 relative error)
    {
      double off = 0, dg = 0;
      for (int q = tid; q < Kp * Kp; q += nt) {
        const double a = A[q];
        if (q / Kp == q % Kp) dg += a * a; else off += a * a;
      }
      off = warp_sum(off);
      dg = warp_sum(dg);
      __shared__ double r_off[8], r_dg[8];
      if ((tid & 31) == 0) {
        r_off[tid >> 5] = off;
        r_dg[tid >> 5] = dg;
      }
      __syncthreads();
      if (tid == 0) {
        double o = 0, d = 0;
        for (int w = 0; w < (nt >> 5); ++w) {
          o += r_off[w];
          d += r_dg[w];
        }
        s_off = o;
        s_diag = d;
      }
      __syncthreads();
    }
    if (s_off <= 1e-30 * s_diag || s_off == 0.0) break;
    // One sweep = Kp - 1 rounds of Kp / 2 disjoint pairs (round-robin tournament: index Kp - 1 stays, the others rotate; the
    // pairs of a round follow from the round number alone). A round is TWO barrier-separated phases: the rotations from the
    // current matrix, then A <- J^T A J in one pass over 2 x 2 blocks (block (a, b) = rows of pair a x columns of pair b only
    // touches its own four entries, so rows and columns need no barrier in between) together with V <- V J.
    const int m = Kp - 1;
    for (int stp = 0; stp < m; ++stp) {
      auto pair_of = [&](int i, int& pp, int& qq) {
        const int x = i == 0 ? stp % m : (stp + i) % m;
        const int y = i == 0 ? m : (stp - i + m) % m;
        pp = min(x, y);
        qq = max(x, y);
      };
      if (tid < npair) {
        int pp, qq;
        pair_of(tid, pp, qq);
        const double apq = A[pp * Kp + qq];
        double c = 1.0, sn = 0.0;
        if (fabs(apq) > 1e-300) {
          const double theta = (A[qq * Kp + qq] - A[pp * Kp + pp]) / (2.0 * apq);
          const double t = (theta >= 0 ? 1.0 : -1.0) / (fabs(theta) + sqrt(theta * theta + 1.0));
          c = 1.0 / sqrt(t * t + 1.0);
          sn = t * c;
        }
        cs[2 * tid] = c;
        cs[2 * tid + 1] = sn;
        top[tid] = pp;  // the round's pairs, for the update phase
        bot[tid] = qq;
      }
      __syncthreads();
      for (int q = tid; q < npair * npair; q += nt) {
        const int pa = q / npair, pb = q % npair;
        const int p0 = top[pa], q0 = bot[pa], r0 = top[pb], t0 = bot[pb];
        const double ca = cs[2 * pa], sa = cs[2 * pa + 1], cb = cs[2 * pb], sb = cs[2 * pb + 1];
        const double apr = A[p0 * Kp + r0], apt = A[p0 * Kp + t0], aqr = A[q0 * Kp + r0], aqt = A[q0 * Kp + t0];
        const double xpr = ca * apr - sa * aqr, xpt = ca * apt - sa * aqt;  // rows: J_a^T A
        const double xqr = sa * apr + ca * aqr, xqt = sa * apt + ca * aqt;
        A[p0 * Kp + r0] = cb * xpr - sb * xpt;                              // columns: (.) J_b
        A[p0 * Kp + t0] = sb * xpr + cb * xpt;
        A[q0 * Kp + r0] = cb * xqr - sb * xqt;
        A[q0 * Kp + t0] = sb * xqr + cb * xqt;
      }
      for (int q = tid; q < npair * Kp; q += nt) {
        const int pr = q / Kp, k = q % Kp;
        const int pp = top[pr], qq = bot[pr];
        const double c = cs[2 * pr], sn = cs[2 * pr + 1];
        const double vp = V[k * Kp + pp], vq = V[k * Kp + qq];
        V[k * Kp + pp] = c * vp - sn * vq;
        V[k * Kp + qq] = sn * vp + c * vq;
      }
      __syncthreads();
    }
  }
  __syncthreads();
  // eigenvalues on the diagonal of A; invert above the cutoff
  if (tid == 0) {
    double mx = 0;
    for (int r = 0; r < K; ++r) mx = fmax(mx, fabs(A[r * Kp + r]));
    s_diag = mx * (double)K * p.pinv_eps;
  }
  __syncthreads();
  const double cutoff = s_diag;
  for (int r = tid; r < Kp; r += nt) {
    const double ev = (r < K) ? A[r * Kp + r] : 0.0;
    cs[r] = (r < K && fabs(ev) > cutoff) ? 1.0 / ev : 0.0;
  }
  __syncthreads();
  for (int q = tid; q < K * K; q += nt) {
    const int r = q / K, c = q % K;
    if (r <= c) {  // upper triangle, mirrored: Sigma is exactly symmetric like SigmaInv
      double s = 0;
      for (int e = 0; e < Kp; ++e) s += V[r * Kp + e] * cs[e] * V[c * Kp + e];
      p.Sigma[q] = s;
      p.Sigma[c * K + r] = s;
    }
    if (ws != nullptr) ws[1 + q] = V[r * Kp + c];  // eigenbasis for the next iteration's warm start
  }
  if (ws != nullptr && tid == 0) ws[0] = (double)K;
  if (p.g_on && p.g_nonrigid) {  // U^T PXB_term += c_g U_I^T (X_BI - R_AI)   (:1286-1288)
    const double cg = sc->sigma2 * p.g_weight * sc->Sp / (double)p.g_NI;
    for (int q = tid; q < K * 3; q += nt) {
      const int k = q / 3, d = q % 3;
      double s = 0;
      for (int n = 0; n < p.g_NI; ++n) s += p.g_UI[(int64_t)n * K + k] * (p.g_XB[n * 3 + d] - p.g_RA[n * 3 + d]);
      p.UtPXB[q] += cg * s;
    }
  }
  __syncthreads();
  __threadfence_block();
  for (int q = tid; q < K * 3; q += nt) {
    const int r = q / 3, d = q % 3;
    double s = 0;
    for (int c = 0; c < K; ++c) s += p.Sigma[r * K + c] * p.UtPXB[c * 3 + d];
    p.Coff[q] = s;
  }
  if (p.g_on && p.g_nonrigid) {  // V_AI = U_I Coff (:1294-1295)
    __syncthreads();
    for (int q = tid; q < p.g_NI * 3; q += nt) {
      const int n = q / 3, d = q % 3;
      double s = 0;
      for (int k = 0; k < K; ++k) s += p.g_UI[(int64_t)n * K + k] * p.Coff[k * 3 + d];
      p.g_VA[q] = s;
    }
  }
}

// VnA = U Coff, SigmaDiag = sigma2 * diag(U Sigma U^T) (morpho_class.py:1293-1298)
__global__ void __launch_bounds__(128) field_apply_kernel(spb_em_params p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.NA) return;
  const int K = p.K;
  const double s2 = p.sc->sigma2;
  double v0 = 0, v1 = 0, v2 = 0, quad = 0;
  for (int k = 0; k < K; ++k) {
    const double uk = (double)p.UT[(int64_t)k * p.ldx + i];
    v0 += uk * p.Coff[k * 3 + 0];
    v1 += uk * p.Coff[k * 3 + 1];
    v2 += uk * p.Coff[k * 3 + 2];
    double tk = 0;
    for (int l = 0; l < K; ++l) tk += p.Sigma[(int64_t)k * K + l] * (double)p.UT[(int64_t)l * p.ldx + i];
    quad += uk * tk;
  }
  p.VnA[i] = (float)v0;
  p.VnA[p.ldx + i] = (float)v1;
  p.VnA[2 * p.ldx + i] = (float)v2;
  p.SigmaDiag[i] = (float)(s2 * quad);
}

// Same outputs from a FACTOR of Sigma: Sigma = G G^T with G = V_kept diag(1 / sqrt(ev_kept)) [K][ldg], only the first *rank
// columns non-zero (eigenvalues above the pseudo-inverse cutoff, sorted first). diag(U Sigma U^T)_n = |G^T u_n|^2 costs
// K * rank instead of K^2 per moving cell; the spectrum of SigmaInv decays fast, so rank << K for large inducing sets.
__global__ void __launch_bounds__(128) field_apply_lowrank_kernel(spb_em_params p, const double* __restrict__ G, int ldg,
                                                                  const int32_t* __restrict__ rank_ptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.NA) return;
  const int K = p.K, r = min(*rank_ptr, K);
  const double s2 = p.sc->sigma2;
  double v0 = 0, v1 = 0, v2 = 0;
  for (int k = 0; k < K; ++k) {
    const double uk = (double)p.UT[(int64_t)k * p.ldx + i];
    v0 += uk * p.Coff[k * 3 + 0];
    v1 += uk * p.Coff[k * 3 + 1];
    v2 += uk * p.Coff[k * 3 + 2];
  }
  double quad = 0.0;
  for (int j0 = 0; j0 < r; j0 += 8) {
    double t[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int k = 0; k < K; ++k) {
      const double uk = (double)p.UT[(int64_t)k * p.ldx + i];
      const double* g = G + (int64_t)k * ldg + j0;  // columns beyond the rank are zero: the last chunk may overrun it
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) t[jj] += uk * ((j0 + jj < ldg) ? g[jj] : 0.0);
    }
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) quad += t[jj] * t[jj];
  }
  p.VnA[i] = (float)v0;
  p.VnA[p.ldx + i] = (float)v1;
  p.VnA[2 * p.ldx + i] = (float)v2;
  p.SigmaDiag[i] = (float)(s2 * quad);
}

// weighted moments for the rigid update and sigma2 (morpho_class.py:1312-1318, 1356-1357, 1427)
//  [0..2] sum K x   [3..5] sum K v   [6..8] sum (P@XB)_i   [9..17] sum K x v^T   [18..26] sum x (P@XB)_i^T
//  [27] sum K_NA_sigma2 * SigmaDiag   [28] sum K
__global__ void __launch_bounds__(256) rigid_moments_kernel(spb_em_params p) {
  double m[29];
#pragma unroll
  for (int q = 0; q < 29; ++q) m[q] = 0.0;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < p.NA; i += gridDim.x * blockDim.x) {
    const double k = p.K_NA[i];
    double x[3], v[3], px[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      x[d] = p.xa[(int64_t)d * p.ldx + i];
      v[d] = p.VnA[(int64_t)d * p.ldx + i];
      px[d] = p.PXB[(int64_t)d * p.ldx + i];
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      m[d] += k * x[d];
      m[3 + d] += k * v[d];
      m[6 + d] += px[d];
#pragma unroll
      for (int e = 0; e < 3; ++e) {
        m[9 + d * 3 + e] += k * x[d] * v[e];
        m[18 + d * 3 + e] += x[d] * px[e];
      }
    }
    m[27] += (double)p.K_NA_sigma2[i] * (double)p.SigmaDiag[i];
    m[28] += k;
  }
  grid_reduce_ordered<29>(m, p.red_scratch, p.red_counter + 1, p.moments, false);
}

// rotation / translation / sigma2 (morpho_class.py:1320-1402, 1426-1435) — one thread, fp64
__global__ void rigid_solve_kernel(spb_em_params p, int iter) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  spb_scalars* sc = p.sc;
  if (iter < 0) iter = sc->iter;
  const int D = p.D;
  const double* m = p.moments;
  const double Sp = sc->Sp, SpK = m[28];
  double PXA[3], PVA[3], PXB[3];
  for (int d = 0; d < 3; ++d) {
    PXA[d] = m[d];
    PVA[d] = m[3 + d];
    PXB[d] = m[6 + d];
  }
  double c = 0.0;
  double PXAa[3], PXBa[3], PVAa[3];  // the "augmented" arrays of the reference's aliasing quirk (SURVEY Appendix B-5)
  double deno = Sp, denoV = Sp;
  for (int d = 0; d < 3; ++d) {
    PXAa[d] = PXA[d];
    PXBa[d] = PXB[d];
    PVAa[d] = PVA[d];
  }
  const bool g_rigid = p.g_on && p.g_rigid;
  double cg = 0.0;
  if (g_rigid) {  // morpho_class.py:1322-1327 — scalar means added to every axis, in place
    cg = sc->sigma2 * p.g_weight * Sp / (double)p.g_NI;
    double sv = 0.0;
    for (int n = 0; n < p.g_NI; ++n)
      for (int d = 0; d < D; ++d) sv += p.g_VA[n * 3 + d];
    const double meanVA = sv / ((double)p.g_NI * D);
    for (int d = 0; d < D; ++d) {
      PXBa[d] += cg * p.g_meanXB;
      PXAa[d] += cg * p.g_meanXA;
      PVAa[d] += cg * meanVA;
    }
    deno += cg * (double)p.g_NI;
    denoV += cg * (double)p.g_NI;
  }
  if (p.nn_init) {
    c = sc->sigma2 * p.nn_init_weight * Sp / p.inl_SP;
    for (int d = 0; d < 3; ++d) {
      PXBa[d] += c * p.inl_Sb[d];
      PXAa[d] += c * p.inl_Sa[d];
    }
    deno += c * p.inl_SP;
  }
  double muB[3], muA[3], muV[3];
  for (int d = 0; d < 3; ++d) {
    muB[d] = PXBa[d] / deno;
    muA[d] = PXAa[d] / deno;
    muV[d] = PVAa[d] / denoV;
  }
  double A[9];
  for (int q = 0; q < 9; ++q) A[q] = 0.0;
  for (int d1 = 0; d1 < D; ++d1)
    for (int d2 = 0; d2 < D; ++d2) {
      const double T1 = m[9 + d1 * 3 + d2] - muA[d1] * PVA[d2] - PXA[d1] * muV[d2] + SpK * muA[d1] * muV[d2];
      const double T2 = m[18 + d1 * 3 + d2] - muA[d1] * PXB[d2] - PXA[d1] * muB[d2] + SpK * muA[d1] * muB[d2];
      double a = T2 - T1;  // -(T1 - T2), transposed below
      if (p.nn_init) {
        const double E = -(p.inl_Mab[d1 * 3 + d2] - muA[d1] * p.inl_Sb[d2] - p.inl_Sa[d1] * muB[d2] +
                           p.inl_SP * muA[d1] * muB[d2]);
        a -= c * E;
      }
      A[d2 * 3 + d1] = a;
    }
  if (g_rigid) {  // A -= c_g (X_AI_hat^T (V_AI_hat - X_BI_hat))^T   (:1347-1350, 1360-1363)
    for (int n = 0; n < p.g_NI; ++n)
      for (int d1 = 0; d1 < D; ++d1) {
        const double ah = p.g_XA[n * 3 + d1] - muA[d1];
        for (int d2 = 0; d2 < D; ++d2) {
          const double w = (p.g_VA[n * 3 + d2] - muV[d2]) - (p.g_XB[n * 3 + d2] - muB[d2]);
          A[d2 * 3 + d1] -= cg * ah * w;
        }
      }
  }
  double Rn[9];
  rotation_from(A, D, Rn);
  const double step = sc->step;
  const bool blend = p.svi && step < 1.0;
  if (p.update_R) {
    for (int d1 = 0; d1 < D; ++d1)
      for (int d2 = 0; d2 < D; ++d2) {
        const int q = d1 * 3 + d2;
        sc->R[q] = blend ? step * Rn[q] + (1.0 - step) * sc->R[q] : Rn[q];
      }
  }
  double tn[3];
  double tden = Sp;
  for (int d = 0; d < D; ++d) {
    double s = PXBa[d] - PVAa[d];
    for (int e = 0; e < D; ++e) s -= PXAa[e] * sc->R[d * 3 + e];
    if (g_rigid) {  // :1384-1388
      double gsum = 0.0;
      for (int n = 0; n < p.g_NI; ++n) {
        double r = p.g_XB[n * 3 + d] - p.g_VA[n * 3 + d];
        for (int e = 0; e < D; ++e) r -= p.g_XA[n * 3 + e] * sc->R[d * 3 + e];
        gsum += r;
      }
      s += cg * gsum;
    }
    if (p.nn_init) {
      double r = p.inl_Sb[d];
      for (int e = 0; e < D; ++e) r -= p.inl_Sa[e] * sc->R[d * 3 + e];
      s += c * r;
    }
    tn[d] = s;
  }
  if (g_rigid) tden += cg * (double)p.g_NI;
  if (p.nn_init) tden += c * p.inl_SP;
  for (int d = 0; d < D; ++d) {
    const double t = tn[d] / tden;
    sc->t[d] = blend ? step * t + (1.0 - step) * sc->t[d] : t;
  }
  if (p.g_on) {  // R_AI <- R_AI R^T + t (morpho_class.py:1407-1408: iterates R_AI itself, starting from zeros)
    for (int n = 0; n < p.g_NI; ++n) {
      double r[3] = {p.g_RA[n * 3], p.g_RA[n * 3 + 1], p.g_RA[n * 3 + 2]}, o[3] = {0, 0, 0};
      for (int d = 0; d < D; ++d) {
        double s = sc->t[d];
        for (int e = 0; e < D; ++e) s += r[e] * sc->R[d * 3 + e];
        o[d] = s;
      }
      for (int d = 0; d < 3; ++d) p.g_RA[n * 3 + d] = o[d];
    }
  }
  // sigma2 (morpho_class.py:1426-1435)
  sc->dotKS = m[27];
  double s2 = fmax(sc->sigma2_related + m[27] / sc->Sp_sigma2, 1e-3);
  sc->sigma2_variance = fmin(sc->sigma2_variance * p.sigma2_variance_decress, p.sigma2_variance_end);
  if (iter < 100) s2 = fmax(s2, 1e-2);
  sc->sigma2 = s2;
  if (p.trace && p.trace_buf) {
    double* tr = p.trace_buf + (int64_t)iter * SPB_TRACE_STRIDE;
    tr[0] = sc->sigma2; tr[1] = sc->gamma; tr[2] = sc->Sp; tr[3] = sc->Sp_spatial;
    tr[4] = sc->Sp_sigma2; tr[5] = sc->sigma2_variance; tr[6] = sc->sigma2_related; tr[7] = sc->visited;
  }
}

// RnA = XA R^T + t, XAHat = VnA + RnA, and next E-step's model multiplier (morpho_class.py:1404, 293, 1087)
__global__ void row_update_kernel(spb_em_params p) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= p.NA) return;
  const spb_scalars* sc = p.sc;
  float x[3];
  for (int d = 0; d < 3; ++d) x[d] = p.xa[(int64_t)d * p.ldx + i];
  for (int d = 0; d < 3; ++d) {
    float r = 0.f;
    if (d < p.D) {
      double s = sc->t[d];
      for (int e = 0; e < p.D; ++e) s += (double)x[e] * sc->R[d * 3 + e];
      r = (float)s;
    }
    const int64_t o = (int64_t)d * p.ldx + i;
    p.RnA[o] = r;
    p.XAHat[o] = p.VnA[o] + r;
  }
  const double a = (double)p.alpha[i], sd = (double)p.SigmaDiag[i], s2 = sc->sigma2;
  p.mm[i] = (float)(a * exp(-sd / s2));
  p.lm[i] = (float)(log2(a) - sd * kLog2e / s2);
}

// closing similarity (morpho_class.py:1451-1468) from the last E-step's moments
__global__ void optimal_rigid_kernel(spb_em_params p, double* out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const spb_scalars* sc = p.sc;
  const int D = p.D;
  const double* m = p.moments;
  const double Sp = sc->Sp, SpK = m[28];
  double muA[3], muB[3];
  for (int d = 0; d < 3; ++d) {
    muA[d] = m[d] / Sp;
    muB[d] = m[6 + d] / Sp;
  }
  double A[9];
  for (int q = 0; q < 9; ++q) A[q] = 0.0;
  for (int d1 = 0; d1 < D; ++d1)
    for (int d2 = 0; d2 < D; ++d2)
      A[d1 * 3 + d2] = m[18 + d2 * 3 + d1] - m[6 + d1] * muA[d2] - muB[d1] * m[d2] + SpK * muB[d1] * muA[d2];
  double R[9];
  for (int q = 0; q < 9; ++q) R[q] = 0.0;
  rotation_from(A, D, R);
  for (int q = 0; q < 9; ++q) out[q] = R[q];
  for (int d = 0; d < 3; ++d) {
    double s = 0.0;
    if (d < D) {
      s = muB[d];
      for (int e = 0; e < D; ++e) s -= muA[e] * R[d * 3 + e];
    }
    out[9 + d] = s;
  }
}

}  // namespace

#define ST ((cudaStream_t)stream)

extern "C" int spb_iter_begin(const spb_em_params* p, int32_t iter, void* stream) {
  iter_begin_kernel<<<1, 256, 0, ST>>>(*p, iter);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_update_gamma_alpha(const spb_em_params* p, void* stream) {
  scalar_update_kernel<<<1, 1, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  alpha_update_kernel<<<(p->NA + 255) / 256, 256, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_nonrigid_accumulate(const spb_em_params* p, void* stream) {
  pxb_term_kernel<<<(p->NA + 255) / 256, 256, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  if (p->UT_hi != nullptr) {  // tensor-core contraction (wgmma, 3xTF32): every K the caller prepared operands for
    int rc = spb_gram_prepare(p->UT, p->ldx, p->NA, p->K, p->UT_mean, p->K_NA, p->PXB_term, p->ldx, 3, p->GB_hi, p->GB_lo,
                              p->gram_sums, stream);
    if (rc) return rc;
    return spb_gram_tc(p->UT_hi, p->UT_lo, p->GB_hi, p->GB_lo, p->ldx, p->NA, p->K, 3, p->UT_mean, p->gram_sums,
                       p->gram_scratch, p->gram_scratch_floats, p->UtWU, p->UtPXB, stream);
  }
  if (p->K > kSmallK) return SPB_EINVAL;  // above 32 inducing points the caller prepares the tensor-core operands
  int rows = (p->NA + 295) / 296;
  rows = ((rows + 127) / 128) * 128;
  const int nblk = (p->NA + rows - 1) / rows;
  if ((int64_t)nblk * p->K * (p->K + 3) > p->red_scratch_doubles) return SPB_EINVAL;
  gram_small_kernel<<<nblk, 256, 0, ST>>>(p->UT, p->ldx, p->NA, p->K, p->K_NA, p->PXB_term, p->UtWU, p->UtPXB, rows,
                                          p->red_scratch, p->red_counter + 2);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_weighted_gram(const float* UT, int64_t ldx, int64_t N, int32_t K, const float* w, const float* X3,
                                 double* UtWU, double* UtX, void* stream) {
  cudaError_t e = cudaMemsetAsync(UtWU, 0, sizeof(double) * (size_t)K * K, ST);
  if (e != cudaSuccess) return (int)e;
  e = cudaMemsetAsync(UtX, 0, sizeof(double) * (size_t)K * 3, ST);
  if (e != cudaSuccess) return (int)e;
  if (K <= kSmallK) {
    int rows = (int)((N + 295) / 296);
    rows = ((rows + 127) / 128) * 128;
    // stand-alone call (no spb_em_params): the block partials live in a small per-device buffer owned by the library
    static double* scratch[SPB_MAX_DEVICES] = {};
    static unsigned int* ticket[SPB_MAX_DEVICES] = {};
    const int dev_ = spb_current_device();
    const int nblk = (int)((N + rows - 1) / rows);
    if (scratch[dev_] == nullptr) {
      if (cudaMalloc(&scratch[dev_], sizeof(double) * 320 * kSmallK * (kSmallK + 3)) != cudaSuccess) return SPB_EUNSUPPORTED;
      if (cudaMalloc(&ticket[dev_], sizeof(unsigned int)) != cudaSuccess) return SPB_EUNSUPPORTED;
      cudaMemset(ticket[dev_], 0, sizeof(unsigned int));
    }
    if (nblk > 320) return SPB_EUNSUPPORTED;
    gram_small_kernel<<<nblk, 256, 0, ST>>>(UT, ldx, (int)N, K, w, X3, UtWU, UtX, rows, scratch[dev_], ticket[dev_]);
    SPB_CHECK_LAUNCH();
    return 0;
  }
  const int ntile = (K + kGT - 1) / kGT;
  const int npairs = ntile * (ntile + 1) / 2;
  const int rows_per_block = gram_rows_per_block(N, npairs);
  dim3 grid((unsigned)((N + rows_per_block - 1) / rows_per_block), npairs);
  weighted_gram_kernel<<<grid, 256, 0, ST>>>(UT, ldx, (int)N, K, w, X3, UtWU, UtX, rows_per_block, ntile);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_vfc_estep(const float* UT, int64_t ldn, int64_t N, int32_t M, int32_t D, const double* C,
                             const double* Y, double sigma2, double gamma, double a, double minP, double theta,
                             double* P, double* V, float* Pf, float* PY3, double* sums5, void* stream) {
  if (D < 1 || D > 3) return SPB_EINVAL;
  cudaError_t e = cudaMemsetAsync(sums5, 0, sizeof(double) * 5, ST);
  if (e != cudaSuccess) return (int)e;
  const double t2 = pow(kTwoPi * sigma2, 0.5 * D) * (1.0 - gamma) / (gamma * a);
  vfc_estep_kernel<<<(unsigned)((N + 127) / 128), 128, 0, ST>>>(UT, ldn, (int)N, M, D, C, Y, sigma2, t2, minP, theta, P, V,
                                                                 Pf, PY3, sums5);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_nonrigid_blend(const spb_em_params* p, void* stream) {
  nonrigid_blend_kernel<<<(p->K * p->K + 255) / 256, 256, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

static int ensure_nonrigid_solve_attr() {
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(nonrigid_solve_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 112 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  return 0;
}

// One-time per-device kernel attributes of the non-rigid phase, so that the phase can be captured in a CUDA graph before
// any of its kernels has been launched eagerly.
extern "C" int spb_nonrigid_warm(void) {
  const int rc = ensure_nonrigid_solve_attr();
  return rc ? rc : spb_gram_tc_warm();
}

extern "C" int spb_nonrigid_solve(const spb_em_params* p, void* stream) {
  if (p->K > SPB_MAX_K_FUSED) return SPB_EUNSUPPORTED;
  const int Kp = (p->K + 1) & ~1;
  const size_t smem = sizeof(double) * (3 * Kp * Kp + 2 * Kp) + sizeof(int) * Kp;  // A, V, warm-start scratch, rotations, pairing
  int rc = ensure_nonrigid_solve_attr();
  if (rc) return rc;
  // small matrices are latency-bound on the block barriers of the rotation rounds: fewer threads, cheaper barriers
  const int threads = Kp <= 16 ? 32 : (Kp <= 32 ? 64 : 256);
  nonrigid_solve_kernel<<<1, threads, smem, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_field_apply(const spb_em_params* p, void* stream) {
  field_apply_kernel<<<(p->NA + 127) / 128, 128, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_field_apply_lowrank(const spb_em_params* p, const double* G, int32_t ldg, const int32_t* rank, void* stream) {
  if (G == nullptr || rank == nullptr || ldg < 1) return SPB_EINVAL;
  field_apply_lowrank_kernel<<<(p->NA + 127) / 128, 128, 0, ST>>>(*p, G, ldg, rank);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_rigid_moments(const spb_em_params* p, void* stream) {
  int blocks = (p->NA + 255) / 256;
  if (blocks > 592) blocks = 592;
  if ((int64_t)blocks * 29 > p->red_scratch_doubles) return SPB_EINVAL;
  rigid_moments_kernel<<<blocks, 256, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_rigid_solve(const spb_em_params* p, int32_t iter, void* stream) {
  rigid_solve_kernel<<<1, 32, 0, ST>>>(*p, iter);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_row_update(const spb_em_params* p, void* stream) {
  row_update_kernel<<<(p->NA + 255) / 256, 256, 0, ST>>>(*p);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_optimal_rigid(const spb_em_params* p, double* out12, void* stream) {
  optimal_rigid_kernel<<<1, 32, 0, ST>>>(*p, out12);
  SPB_CHECK_LAUNCH();
  return 0;
}

#define SPB_TRY(x)          \
  do {                      \
    int rc__ = (x);         \
    if (rc__ != 0) return rc__; \
  } while (0)

// One EM iteration (morpho_class.py:280-294) as a fixed launch sequence. ``iter`` < 0: the iteration index is taken from
// the device scalars (previous + 1), which makes the sequence capturable ONCE in a CUDA graph and replayable for every
// iteration of a phase (``nonrigid`` = 0 before nonrigid_start_iter, 1 after).
extern "C" int spb_em_iteration_ex(const spb_em_params* p, int32_t iter, int32_t nonrigid, void* stream) {
  if (nonrigid && p->K > SPB_MAX_K_FUSED) return SPB_EUNSUPPORTED;
  SPB_TRY(spb_iter_begin(p, iter, stream));
  SPB_TRY(spb_gather_cols(p, iter, stream));
  SPB_TRY(spb_estep_col_lists(p, stream));
  SPB_TRY(spb_estep_sweep1(p, iter, stream));
  SPB_TRY(spb_col_finalize(p, stream));
  if (p->sparse_k > 0) SPB_TRY(spb_estep_col_select(p, iter, stream));
  SPB_TRY(spb_estep_sweep2(p, iter, stream));
  SPB_TRY(spb_row_finalize(p, stream));
  SPB_TRY(spb_update_gamma_alpha(p, stream));
  if (nonrigid) {
    SPB_TRY(spb_nonrigid_accumulate(p, stream));
    SPB_TRY(spb_nonrigid_solve(p, stream));
    SPB_TRY(spb_field_apply(p, stream));
  }
  SPB_TRY(spb_rigid_moments(p, stream));
  SPB_TRY(spb_rigid_solve(p, iter, stream));
  SPB_TRY(spb_row_update(p, stream));
  return 0;
}

extern "C" int spb_em_iteration(const spb_em_params* p, int32_t iter, void* stream) {
  if (iter < 0) return SPB_EINVAL;
  // latched flag == monotone in iter (morpho_class.py:289-291)
  return spb_em_iteration_ex(p, iter, iter > p->nonrigid_start_iter ? 1 : 0, stream);
}
