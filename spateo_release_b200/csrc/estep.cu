// Fused E-step of the morpho-align EM (replaces calc_distance("euc") + get_P_core + every reduction that consumes P:
// spateo/alignment/methods/utils.py:993-1096, morpho_class.py:1147-1200). P is never materialised in the loop.
//
//   sweep 1  streams GT (one contiguous row per fixed cell j) through a 3-stage bulk-async (TMA 1-D) shared-memory
//            ring and produces the four column sums  C1=sum_i s, C2=sum_i s m, C3=sum_i q m, C4=sum_i q m g.
//   col_finalize   turns them into the per-column constants a_j, b_j, c_j (and K_NB_j).
//   sweep 2  streams GT again and accumulates, per moving cell i (thread-owned registers), K_NA_spatial, K_NA_sigma2,
//            sum_j Psigma d, K_NA and the D components of P @ XB.
//   Pair arithmetic is written on fp32 pairs (two moving cells per value, explicitly rounded scalar operations).
//   row_finalize   reduces the per-segment partials in fp64 and forms the global sums.
//
// Algorithmic HBM traffic: 4 bytes per cell pair per sweep (the fp32 g_ij), 8 B/pair/iteration in total.
// Thread mapping: a CTA covers SPB_ROW_TILE = 512 moving cells: 128 consumer threads own 4 consecutive rows each (one
// float4 of a GT row), one extra warp is the bulk-copy producer (160 threads, 96 registers, ~50 KB of shared memory:
// 4 CTAs per SM). Column constants are broadcast from shared memory. 512-row tiles rather than 1024: finer exact culling
// and shorter tails.
#include "common.cuh"

namespace {

constexpr int kRowTile = SPB_ROW_TILE;    // rows per CTA
constexpr int kConsumers = kRowTile / 4;  // consumer threads, 4 consecutive rows each
constexpr int kThreads = kConsumers + 32;
constexpr int kCtas = 2048 / kRowTile;    // resident CTAs per SM the sweeps are built for (96 registers, ~100 KB of shared memory per 1024 rows)
constexpr int kColF4 = SPB_COLCONST_FLOATS / 4;  // float4 per column constant record (sweep 1 uses the first two)
constexpr int kColStage = SPB_COL_STAGE;  // columns per pipeline stage (the host sizes column segments in whole stages)
constexpr int kStages = 3;                // stages of the shared-memory ring
constexpr int kQuarter = 32 * 4;          // rows of one consumer warp: the granularity of the culling within a row block
static_assert(kColStage == 8, "one 64-bit word holds the quarter masks of a stage");

struct __align__(16) SmemLayout {
  float tile[kStages][kColStage][kRowTile];  // kColStage x 4 KB per stage
  float4 cols[kStages][kColStage][kColF4];   // per-column constants, pre-duplicated for packed math (80 B / column)
  float red[2][kConsumers / 32][32];         // sweep-1 cross-warp staging
  uint64_t quarters[kStages];                // byte jj of the stage's column jj: colquarters | colspatial << 4
  uint64_t full[kStages];
  uint64_t empty[kStages];
};

// Column work lists. Every row block owns a compacted list of the columns of this iteration that can interact with it
// (build_col_lists_kernel): with culling on, a column whose squared distance to the block's bounding box makes
// exp(-d / 2 sigma2) flush to zero in fp32 contributes EXACTLY nothing to any sum and is dropped — bit-identical results,
// less HBM traffic. A CTA (rb, seg) takes a contiguous slice of its block's list.
struct ColRange {
  int begin, end;
};
// SVI: the column batch of the CURRENT iteration (morpho_class.py:894-896). The iteration index is read from the device
// scalars (spb_iter_begin writes it), so a captured CUDA graph of one iteration can be replayed for every iteration.
__device__ __forceinline__ const int32_t* batch_cols(const int32_t* __restrict__ batch_base, const spb_scalars* __restrict__ sc,
                                                     int NBb) {
  return batch_base ? batch_base + (int64_t)sc->iter * NBb : nullptr;
}
__device__ __forceinline__ ColRange col_range(const int32_t* __restrict__ colcount, int rb, int seg, int nseg) {
  const int count = colcount[rb];
  int cps = (count + nseg - 1) / nseg;
  cps = ((cps + kColStage - 1) / kColStage) * kColStage;
  ColRange r;
  r.begin = min(count, seg * cps);
  r.end = min(count, r.begin + cps);
  return r;
}

// One stage = the live quarters (512 B each) of kColStage GT rows + the columns' constants. A column's live quarters
// (colquarters: the quarters whose weights q can be non-zero) are copied as one bulk copy per run of adjacent quarters (a
// 4-bit mask has at most two runs); the other quarters of the slot keep stale data that the owning consumer warp never
// reads. Slots past the end of the slice have no live quarter and take the all-zero constant entry at index NBb (the
// constant arrays are zero-padded). The stage's masks, with the spatially live quarters (colspatial) in the high nibble
// of each byte, go to sm.quarters before the arrive on the full barrier, which publishes them with the copies.
// kFeat > 0 (posterior transfer): a column with a live quarter also brings its kFeat-float feature panel row
// fsrc[frow * ldf ..] (frow = fcol_index[j], or j) to fdst[stage][slot][0 .. kFeat).
template <int kFeat = 0>
__device__ __forceinline__ void producer_loop(SmemLayout& sm, const float* __restrict__ GT, int64_t ldx,
                                              const int32_t* __restrict__ col_index, const int32_t* __restrict__ list,
                                              const uint8_t* __restrict__ quarters, const uint8_t* __restrict__ spatial,
                                              const float* __restrict__ colsrc, int col_floats, int i0, ColRange cr, int NBb,
                                              int lane, const float* __restrict__ fsrc = nullptr, int64_t ldf = 0,
                                              const int32_t* __restrict__ fcol_index = nullptr, float* fdst = nullptr) {
  const int nst = (cr.end - cr.begin + kColStage - 1) / kColStage;
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    if (st >= kStages) mbar_wait(&sm.empty[s], ((st / kStages) - 1) & 1);
    const int pb = cr.begin + st * kColStage;
    const bool slot = lane < kColStage, live = slot && pb + lane < cr.end;
    const uint32_t qm = live ? quarters[pb + lane] : 0u;
    const uint32_t wm = live ? qm | (uint32_t)spatial[pb + lane] << 4 : 0u;
    const uint32_t bytes = slot ? __popc(qm) * kQuarter * 4 + col_floats * 4 + (qm != 0u ? kFeat * 4 : 0) : 0u;
    const uint32_t total = __reduce_add_sync(0xffffffffu, bytes);
    const uint32_t lo = __reduce_or_sync(0xffffffffu, lane < 4 ? wm << (8 * lane) : 0u);
    const uint32_t hi = __reduce_or_sync(0xffffffffu, (lane >= 4 && slot) ? wm << (8 * (lane - 4)) : 0u);
    if (lane == 0) {
      sm.quarters[s] = ((uint64_t)hi << 32) | lo;
      mbar_expect_tx(&sm.full[s], total);
    }
    __syncwarp();
    if (slot) {
      const int j = live ? list[pb + lane] : NBb;  // NBb = zero-constant pad entry
      if (qm != 0u) {
        const int64_t row = col_index ? (int64_t)col_index[j] : (int64_t)j;
        const float* src = GT + row * ldx + i0;
        for (uint32_t m = qm; m != 0u;) {
          const int q0 = __ffs(m) - 1;
          const int len = __ffs(~(m >> q0)) - 1;  // length of the run of set bits starting at q0
          bulk_g2s(&sm.tile[s][lane][q0 * kQuarter], src + q0 * kQuarter, len * kQuarter * 4, &sm.full[s]);
          m &= ~(((1u << len) - 1u) << q0);
        }
        if constexpr (kFeat > 0) {
          const int64_t frow = fcol_index ? (int64_t)fcol_index[j] : (int64_t)j;
          bulk_g2s(fdst + (s * kColStage + lane) * kFeat, fsrc + frow * ldf, kFeat * 4, &sm.full[s]);
        }
      }
      bulk_g2s(&sm.cols[s][lane][0], colsrc + (int64_t)j * col_floats, col_floats * 4, &sm.full[s]);
    }
  }
}

// A consumer warp reads the cost matrix and forms the weights q only for a column whose q bit (low nibble) is set, and forms
// the spatial weights s only where its s bit (high nibble) is set. A clear bit means every pair of the warp's 128 rows with
// that column has an fp32 ex2 argument below -126 (build_col_lists_kernel): ex2(c_q d + lm) = +0 or ex2(c_s d) = +0. Sweep 1
// would have reduced exact zeros and sweep 2 would have added exact zeros (an accumulator that starts at +0 is never -0, so
// x + 0 = x). Skipping is therefore bit-identical.
__device__ __forceinline__ bool quarter_q(uint64_t wq, int jj) { return (wq >> (8 * jj)) & 1u; }
__device__ __forceinline__ bool quarter_s(uint64_t wq, int jj) { return (wq >> (8 * jj + 4)) & 1u; }

// ---- fp32 pairs: two moving cells per value. Hopper has no packed fp32x2 instructions, so every pair operation is two
// scalar operations with explicit round-to-nearest (no contraction: the same bits as a packed add / mul / fma) ----------
typedef unsigned long long u64;
__device__ __forceinline__ u64 pk(float a, float b) {
  u64 r;
  asm("mov.b64 %0, {%1, %2};" : "=l"(r) : "f"(a), "f"(b));
  return r;
}
__device__ __forceinline__ void upk(u64 v, float& a, float& b) { asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v)); }
__device__ __forceinline__ u64 add2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1);
  upk(b, b0, b1);
  return pk(__fadd_rn(a0, b0), __fadd_rn(a1, b1));
}
__device__ __forceinline__ u64 sub2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1);
  upk(b, b0, b1);
  return pk(__fsub_rn(a0, b0), __fsub_rn(a1, b1));
}
__device__ __forceinline__ u64 mul2(u64 a, u64 b) {
  float a0, a1, b0, b1;
  upk(a, a0, a1);
  upk(b, b0, b1);
  return pk(__fmul_rn(a0, b0), __fmul_rn(a1, b1));
}
__device__ __forceinline__ u64 fma2(u64 a, u64 b, u64 c) {
  float a0, a1, b0, b1, c0, c1;
  upk(a, a0, a1);
  upk(b, b0, b1);
  upk(c, c0, c1);
  return pk(__fmaf_rn(a0, b0, c0), __fmaf_rn(a1, b1, c1));
}
__device__ __forceinline__ u64 ex2_2(u64 v) {
  float a, b;
  upk(v, a, b);
  return pk(ex2f(a), ex2f(b));
}
__device__ __forceinline__ float hsum(u64 v) {
  float a, b;
  upk(v, a, b);
  return a + b;
}
// squared distance of two moving cells (packed) to one fixed cell whose coordinates are pre-duplicated (y,y)
// kDim = 2: slices without a third coordinate skip its term (fma(0, 0, r) = r exactly, so the result is bit-identical to the
// 3-term form on zero-padded coordinates — col_select_kernel's scalar pair_weight relies on that)
template <int kDim = 3>
__device__ __forceinline__ u64 sqdist2(u64 x0, u64 x1, u64 x2, u64 y0, u64 y1, u64 y2) {
  const u64 d0 = sub2(x0, y0), d1 = sub2(x1, y1);
  u64 r = fma2(d1, d1, mul2(d0, d0));
  if constexpr (kDim == 3) {
    const u64 d2 = sub2(x2, y2);
    r = fma2(d2, d2, r);
  }
  return r;
}

// Butterfly transpose-reduce: NV (= 32 or 16) per-lane values are summed across the 32 lanes of a warp in
// (NV - 1) + log2(32 / NV) shuffles; afterwards acc[0] of lane l holds the warp total of value (l * NV / 32).
template <int N, int OFF, int NV>
__device__ __forceinline__ void bfly_step(float (&acc)[NV], int lane) {
  if constexpr (N >= 1) {
    const bool up = (lane & OFF) != 0;
#pragma unroll
    for (int q = 0; q < N; ++q) {
      const float mine = up ? acc[q + N] : acc[q];
      const float theirs = up ? acc[q] : acc[q + N];
      acc[q] = mine + __shfl_xor_sync(0xffffffffu, theirs, OFF);
    }
  } else {
    acc[0] += __shfl_xor_sync(0xffffffffu, acc[0], OFF);
  }
}
template <int NV>
__device__ __forceinline__ void butterfly_reduce(float (&acc)[NV], int lane) {
  bfly_step<NV / 2, 16, NV>(acc, lane);
  bfly_step<NV / 4, 8, NV>(acc, lane);
  bfly_step<NV / 8, 4, NV>(acc, lane);
  bfly_step<NV / 16, 2, NV>(acc, lane);
  bfly_step<NV / 32, 1, NV>(acc, lane);
}

// ---- per-thread state and per-stage math of the two sweeps --------------
struct RowRegs {  // 4 consecutive moving cells as two packed pairs (a = rows r, r+1; b = rows r+2, r+3)
  u64 xa0, xb0, xa1, xb1, xa2, xb2, lma, lmb, mma, mmb;
};
__device__ __forceinline__ RowRegs load_rows(const float* __restrict__ XA, int64_t ldx, const float* __restrict__ lm,
                                             const float* __restrict__ mm, int r) {
  const float4 X0 = *reinterpret_cast<const float4*>(XA + r);
  const float4 X1 = *reinterpret_cast<const float4*>(XA + ldx + r);
  const float4 X2 = *reinterpret_cast<const float4*>(XA + 2 * ldx + r);
  const float4 LM = *reinterpret_cast<const float4*>(lm + r);
  RowRegs R;
  R.xa0 = pk(X0.x, X0.y), R.xb0 = pk(X0.z, X0.w), R.xa1 = pk(X1.x, X1.y), R.xb1 = pk(X1.z, X1.w);
  R.xa2 = pk(X2.x, X2.y), R.xb2 = pk(X2.z, X2.w);
  R.lma = pk(LM.x, LM.y), R.lmb = pk(LM.z, LM.w);
  if (mm) {
    const float4 MM = *reinterpret_cast<const float4*>(mm + r);
    R.mma = pk(MM.x, MM.y), R.mmb = pk(MM.z, MM.w);
  } else {
    R.mma = R.mmb = 0ull;
  }
  return R;
}

// sweep 1, one pipeline stage: per column the four partial sums of this thread's 4 rows (index v * kColStage + jj)
// sweep 1, a stage whose columns are "spatially dead" for this row block (exp2(c_s d) flushes to 0 for every pair: the narrow
// spatial posterior has no mass here): only the two sums of the sigma2 / full posteriors are formed — half the MUFU work.
template <int kDim = 3>
__device__ __forceinline__ void sweep1_stage_q(const SmemLayout& sm, int s, int tid, const RowRegs& R,
                                               u64 CQ, uint64_t wq, float (&acc)[2 * kColStage]) {
#pragma unroll
  for (int jj = 0; jj < kColStage; ++jj) {
    if (!quarter_q(wq, jj)) {
      acc[0 * kColStage + jj] = acc[1 * kColStage + jj] = 0.f;
      continue;
    }
    const ulonglong2 ya = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][0]);
    const ulonglong2 yb = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][1]);
    const ulonglong2 g = *reinterpret_cast<const ulonglong2*>(&sm.tile[s][jj][tid * 4]);
    const u64 da = sqdist2<kDim>(R.xa0, R.xa1, R.xa2, ya.x, ya.y, yb.x);
    const u64 db = sqdist2<kDim>(R.xb0, R.xb1, R.xb2, ya.x, ya.y, yb.x);
    const u64 qa = ex2_2(fma2(CQ, da, R.lma)), qb = ex2_2(fma2(CQ, db, R.lmb));
    acc[0 * kColStage + jj] = hsum(add2(qa, qb));
    acc[1 * kColStage + jj] = hsum(fma2(qa, g.x, mul2(qb, g.y)));
  }
}

template <int kDim = 3>
__device__ __forceinline__ void sweep1_stage(const SmemLayout& sm, int s, int tid, const RowRegs& R,
                                             u64 CQ, u64 CS, uint64_t wq, float (&acc)[4 * kColStage]) {
#pragma unroll
  for (int jj = 0; jj < kColStage; ++jj) {
    acc[0 * kColStage + jj] = acc[1 * kColStage + jj] = acc[2 * kColStage + jj] = acc[3 * kColStage + jj] = 0.f;
    const bool ql = quarter_q(wq, jj), sl = quarter_s(wq, jj);
    if (!ql && !sl) continue;
    const ulonglong2 ya = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][0]);  // (y0,y0) (y1,y1)
    const ulonglong2 yb = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][1]);  // (y2,y2) (0,0)
    const u64 da = sqdist2<kDim>(R.xa0, R.xa1, R.xa2, ya.x, ya.y, yb.x);
    const u64 db = sqdist2<kDim>(R.xb0, R.xb1, R.xb2, ya.x, ya.y, yb.x);
    if (sl) {
      const u64 sa = ex2_2(mul2(CS, da)), sb = ex2_2(mul2(CS, db));
      acc[0 * kColStage + jj] = hsum(add2(sa, sb));
      acc[1 * kColStage + jj] = hsum(fma2(sa, R.mma, mul2(sb, R.mmb)));
    }
    if (ql) {
      const ulonglong2 g = *reinterpret_cast<const ulonglong2*>(&sm.tile[s][jj][tid * 4]);
      const u64 qa = ex2_2(fma2(CQ, da, R.lma)), qb = ex2_2(fma2(CQ, db, R.lmb));
      acc[2 * kColStage + jj] = hsum(add2(qa, qb));
      acc[3 * kColStage + jj] = hsum(fma2(qa, g.x, mul2(qb, g.y)));
    }
  }
}

// sweep 2 accumulators: [row pair a | b] x {K_NA_spatial/m, K_NA_sigma2, sum Psigma d, K_NA, (P@XB)_x, _y, _z}
struct S2Acc {
  u64 spa, spb, s2a, s2b, sda, sdb, ka, kb, pxa, pxb, pya, pyb, pza, pzb;
  __device__ __forceinline__ void clear() {
    const u64 Z = pk(0.f, 0.f);
    spa = spb = s2a = s2b = sda = sdb = ka = kb = pxa = pxb = pya = pyb = pza = pzb = Z;
  }
  __device__ __forceinline__ void store(float* __restrict__ out, int64_t ldx) const {
    auto st4 = [&](int q, u64 a, u64 b) {
      float4 v;
      upk(a, v.x, v.y);
      upk(b, v.z, v.w);
      *reinterpret_cast<float4*>(out + (int64_t)q * ldx) = v;
    };
    st4(0, spa, spb);
    st4(1, s2a, s2b);
    st4(2, sda, sdb);
    st4(3, ka, kb);
    st4(4, pxa, pxb);
    st4(5, pya, pyb);
    st4(6, pza, pzb);
  }
};

// kSparse (sparse_calculation_mode, utils.py:1085-1094): only pairs whose weight q g reaches the column's top-k threshold
// tau_j (col_select_kernel) enter K_NA and P @ XB; the spatial and sigma2 posteriors stay dense as in the reference.
__device__ __forceinline__ u64 keep_ge(u64 w, float tau) {
  float a, b;
  upk(w, a, b);
  return pk(a >= tau ? a : 0.f, b >= tau ? b : 0.f);
}

// kSpatial = false: stage of spatially dead columns (see sweep1_stage_q) — K_NA_spatial receives exact zeros from them
template <bool kSparse, int kDim = 3, bool kSpatial = true>
__device__ __forceinline__ void sweep2_stage(const SmemLayout& sm, int s, int tid, const RowRegs& R,
                                             u64 CQ, u64 CS, uint64_t wq, S2Acc& A) {
#pragma unroll
  for (int jj = 0; jj < kColStage; ++jj) {
    const bool ql = quarter_q(wq, jj), sl = kSpatial && quarter_s(wq, jj);
    if (!ql && !sl) continue;
    const ulonglong2 c0 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][0]);  // (y0,y0) (y1,y1)
    const ulonglong2 c1 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][1]);  // (y2,y2) (a,a)
    const u64 da = sqdist2<kDim>(R.xa0, R.xa1, R.xa2, c0.x, c0.y, c1.x);
    const u64 db = sqdist2<kDim>(R.xb0, R.xb1, R.xb2, c0.x, c0.y, c1.x);
    if (sl) {
      const u64 sa = ex2_2(mul2(CS, da)), sb = ex2_2(mul2(CS, db));
      A.spa = fma2(sa, c1.y, A.spa);
      A.spb = fma2(sb, c1.y, A.spb);
    }
    if (!ql) continue;
    const ulonglong2 c2 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][2]);  // (b,b)  (c,c)
    const ulonglong2 c3 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][3]);  // (c y0, c y0) (c y1, c y1)
    const ulonglong2 g = *reinterpret_cast<const ulonglong2*>(&sm.tile[s][jj][tid * 4]);
    const u64 qa = ex2_2(fma2(CQ, da, R.lma)), qb = ex2_2(fma2(CQ, db, R.lmb));
    const u64 ta = mul2(qa, c2.x), tb = mul2(qb, c2.x);
    A.s2a = add2(A.s2a, ta);
    A.s2b = add2(A.s2b, tb);
    A.sda = fma2(ta, da, A.sda);
    A.sdb = fma2(tb, db, A.sdb);
    u64 wa = mul2(qa, g.x), wb = mul2(qb, g.y);
    if constexpr (kSparse) {
      const float tau = sm.cols[s][jj][4].z;
      wa = keep_ge(wa, tau);
      wb = keep_ge(wb, tau);
    }
    // P = w c and P y = w (c y): the column factor rides in the pre-multiplied constants (one packed op less per pair)
    A.ka = fma2(wa, c2.y, A.ka);
    A.kb = fma2(wb, c2.y, A.kb);
    A.pxa = fma2(wa, c3.x, A.pxa);
    A.pxb = fma2(wb, c3.x, A.pxb);
    A.pya = fma2(wa, c3.y, A.pya);
    A.pyb = fma2(wb, c3.y, A.pyb);
    if constexpr (kDim == 3) {
      const u64 cy2 = *reinterpret_cast<const u64*>(&sm.cols[s][jj][4]);  // (c y2, c y2)
      A.pza = fma2(wa, cy2, A.pza);
      A.pzb = fma2(wb, cy2, A.pzb);
    }
  }
}

__device__ __forceinline__ float sqdist(float x0, float x1, float x2, const float4& y) {
  const float d0 = x0 - y.x, d1 = x1 - y.y, d2 = x2 - y.z;
  return fmaf(d2, d2, fmaf(d1, d1, d0 * d0));
}

// ---------------------------------------------------------------------------------------------------------------------
// sweep 1: column sums
// ---------------------------------------------------------------------------------------------------------------------
template <int kDim = 3>
__global__ void __launch_bounds__(kThreads, kCtas)
estep_sweep1_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                    const float* __restrict__ colgeom, const float* __restrict__ XA, const float* __restrict__ lm,
                    const float* __restrict__ mm, const spb_scalars* __restrict__ sc, float* __restrict__ colpart,
                    int NBb, int nbb_pad, const int32_t* __restrict__ collist, const uint8_t* __restrict__ colquarters,
                    const uint8_t* __restrict__ colspatial, const int32_t* __restrict__ colcount,
                    const int32_t* __restrict__ colsplit) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  SmemLayout& sm = *reinterpret_cast<SmemLayout*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rb = blockIdx.x, seg = blockIdx.y;
  const int i0 = rb * kRowTile;
  const ColRange cr = col_range(colcount, rb, seg, gridDim.y);
  const int32_t* list = collist + (int64_t)rb * nbb_pad;
  const uint8_t* quarters = colquarters + (int64_t)rb * nbb_pad;
  const uint8_t* spatial = colspatial + (int64_t)rb * nbb_pad;
  const int32_t* col_index = batch_cols(batch_base, sc, NBb);
  const int split = colsplit[rb];  // list positions >= split: spatially dead columns
  // partials are stored by list position: a stage's kColStage values of one sum are one aligned 32-byte sector
  // (segments begin at multiples of kColStage, nbb_pad is a multiple of 8)
  float* part = colpart + (int64_t)rb * 4 * nbb_pad;
  if (cr.begin >= cr.end) return;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp == kConsumers / 32) {
    producer_loop(sm, GT, ldx, col_index, list, quarters, spatial, colgeom, 8, i0, cr, NBb, lane);
    return;
  }
  // ---- consumers: 4 rows per thread = 2 packed row pairs ----
  const u64 CQ = pk(sc->c_q, sc->c_q), CS = pk(sc->c_s, sc->c_s);
  const RowRegs R = load_rows(XA, ldx, lm, mm, i0 + tid * 4);
  const int nst = (cr.end - cr.begin + kColStage - 1) / kColStage;
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    mbar_wait(&sm.full[s], (st / kStages) & 1);
    const int pb = cr.begin + st * kColStage;
    constexpr int NV = 4 * kColStage;  // partial sums per thread per stage, index v * kColStage + jj
    const int buf = st & 1;
    const uint64_t wq = sm.quarters[s] >> warp;  // bits 8 jj, 8 jj + 4: this warp's q and s bits of column jj
    if (pb >= split) {
      // all columns of the stage are spatially dead: sums 0 and 1 are exact zeros (not stored: col_finalize knows them from
      // the list position), only 2 and 3 are computed and reduced
      constexpr int NQ = 2 * kColStage;
      float acc[NQ];
      sweep1_stage_q<kDim>(sm, s, tid, R, CQ, wq, acc);
      __syncwarp();
      if (lane == 0) mbar_arrive(&sm.empty[s]);
      butterfly_reduce<NQ>(acc, lane);
      constexpr int kShiftQ = (NQ == 32) ? 0 : (NQ == 16 ? 1 : 2);
      if ((lane & ((1 << kShiftQ) - 1)) == 0) sm.red[buf][warp][lane >> kShiftQ] = acc[0];
      named_bar_sync(1, kConsumers);
      if (warp == 0 && lane < NQ) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < kConsumers / 32; ++w) t += sm.red[buf][w][lane];
        const int v = 2 + lane / kColStage, jj = lane % kColStage;
        if (pb + jj < cr.end) part[(int64_t)v * nbb_pad + pb + jj] = t;
      }
      continue;
    }
    float acc[NV];
    sweep1_stage<kDim>(sm, s, tid, R, CQ, CS, wq, acc);
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);  // stage buffer is free again
    butterfly_reduce<NV>(acc, lane);
    constexpr int kShift = (NV == 32) ? 0 : (NV == 16 ? 1 : 2);  // lane -> value index
    if ((lane & ((1 << kShift) - 1)) == 0) sm.red[buf][warp][lane >> kShift] = acc[0];
    named_bar_sync(1, kConsumers);
    if (warp == 0 && lane < NV) {
      float t = 0.f;
#pragma unroll
      for (int w = 0; w < kConsumers / 32; ++w) t += sm.red[buf][w][lane];
      const int v = lane / kColStage, jj = lane % kColStage;
      if (pb + jj < cr.end) part[(int64_t)v * nbb_pad + pb + jj] = t;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// column constants
// ---------------------------------------------------------------------------------------------------------------------
// One warp owns 32 consecutive columns; the kFinWarps warps of a CTA split the row blocks between them (the fold over ~100
// row-block partials per column is a chain of dependent loads otherwise) and combine through shared memory in fp64.
constexpr int kFinWarps = 8;
__global__ void __launch_bounds__(32 * kFinWarps)
col_finalize_kernel(const float* __restrict__ colpart, const uint32_t* __restrict__ keepmask,
                    const uint32_t* __restrict__ livemask, const int2* __restrict__ keepoff, int kstride, int nrb, int nbb_pad,
                    int NBb, const float* __restrict__ colgeom,
                    const spb_scalars* __restrict__ sc, float* __restrict__ colconst, float* __restrict__ K_NB) {
  __shared__ double part[kFinWarps][4][32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int j = blockIdx.x * 32 + lane;
  const uint32_t below = (1u << lane) - 1u;
  double C[4] = {0, 0, 0, 0};
  // a (row block, column) partial exists only if the column is on the row block's list; the others are never written or read
  // (this warp's row blocks: warp, warp + kFinWarps, ...; lane t fetches the mask words and list offsets of the t-th one, they
  // are then broadcast, and four row blocks' loads are in flight before the first add: the fold stays in row-block order).
  // Sweep 1 stored the partials by list position: the column's position is the offset of its group (spatially live / dead)
  // in this 32-column word plus the listed columns of the group below it (build_col_lists_kernel's compaction). A spatially
  // dead column's sums 0 and 1 are exact zeros and were not stored.
  const int nmine = (nrb - warp + kFinWarps - 1) / kFinWarps;
  for (int base = 0; base < nmine; base += 32) {
    const int t = base + lane;
    const int64_t w = (int64_t)(warp + t * kFinWarps) * kstride + blockIdx.x;
    const uint32_t mymask = t < nmine ? keepmask[w] : 0u;
    const uint32_t mylive = t < nmine ? livemask[w] : 0u;
    const int2 myoff = t < nmine ? keepoff[w] : make_int2(0, 0);
    const int cnt = min(32, nmine - base);
    for (int u0 = 0; u0 < cnt; u0 += 4) {
      float tmp[4][4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int src = (u0 + u) & 31;
        const uint32_t bits = __shfl_sync(0xffffffffu, mymask, src);
        const uint32_t lbits = __shfl_sync(0xffffffffu, mylive, src);
        const int off_live = __shfl_sync(0xffffffffu, myoff.x, src), off_dead = __shfl_sync(0xffffffffu, myoff.y, src);
        const bool on = (u0 + u < cnt) && ((bits >> lane) & 1u);
        const bool live = (lbits >> lane) & 1u;
        const int pos = live ? off_live + __popc(lbits & below) : off_dead + __popc(bits & ~lbits & below);
        const int rb = warp + (base + u0 + u) * kFinWarps;
        const float* p = colpart + (int64_t)rb * 4 * nbb_pad + pos;
#pragma unroll
        for (int v = 0; v < 4; ++v) tmp[u][v] = (on && (live || v >= 2)) ? p[(int64_t)v * nbb_pad] : 0.f;
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
#pragma unroll
        for (int v = 0; v < 4; ++v) C[v] += (double)tmp[u][v];
      }
    }
  }
#pragma unroll
  for (int v = 0; v < 4; ++v) part[warp][v][lane] = C[v];
  __syncthreads();
  if (warp != 0 || j >= NBb) return;
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    double t = 0.0;
    for (int w = 0; w < kFinWarps; ++w) t += part[w][v][lane];  // fixed order: deterministic
    C[v] = t;
  }
  const double omega = sc->omega;
  const double inl = 1.0 - omega / (omega + C[0]);          // utils.py:1055
  const double a = 1.0 / (omega + C[1]);                     // utils.py:1059
  const double b = inl / (C[2] + 1e-8);                      // utils.py:1073
  const double c = inl / (C[3] + 1e-8);                      // utils.py:1083
  const float* yg = colgeom + (int64_t)j * 8;  // (y0,y0,y1,y1,y2,y2,0,0)
  const float y0 = yg[0], y1 = yg[2], y2 = yg[4];
  const float af = (float)a, bf = (float)b, cf = (float)c;
  float4* out = reinterpret_cast<float4*>(colconst + (int64_t)j * SPB_COLCONST_FLOATS);
  const float cy0 = cf * y0, cy1 = cf * y1, cy2 = cf * y2;
  out[0] = make_float4(y0, y0, y1, y1);
  out[1] = make_float4(y2, y2, af, af);
  out[2] = make_float4(bf, bf, cf, cf);
  out[3] = make_float4(cy0, cy0, cy1, cy1);
  out[4] = make_float4(cy2, cy2, 0.f, 0.f);  // [18..19] = tau (sparse mode top-k threshold), 0 = keep everything
  K_NB[j] = (float)(c * C[3]);                                // column sum of P (morpho_class.py:1176)
}

// ---------------------------------------------------------------------------------------------------------------------
// sweep 2: row statistics
// ---------------------------------------------------------------------------------------------------------------------
template <bool kSparse, int kDim = 3>
__global__ void __launch_bounds__(kThreads, kCtas)
estep_sweep2_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                    const float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                    const spb_scalars* __restrict__ sc, float* __restrict__ rowpart, int NBb, int nbb_pad,
                    const int32_t* __restrict__ collist, const uint8_t* __restrict__ colquarters,
                    const uint8_t* __restrict__ colspatial, const int32_t* __restrict__ colcount,
                    const int32_t* __restrict__ colsplit) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  SmemLayout& sm = *reinterpret_cast<SmemLayout*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rb = blockIdx.x, seg = blockIdx.y;
  const int i0 = rb * kRowTile;
  const int split = colsplit[rb];  // list positions >= split: spatially dead columns (no spatial-posterior work)
  const ColRange cr = col_range(colcount, rb, seg, gridDim.y);
  const int32_t* list = collist + (int64_t)rb * nbb_pad;
  const uint8_t* quarters = colquarters + (int64_t)rb * nbb_pad;
  const uint8_t* spatial = colspatial + (int64_t)rb * nbb_pad;
  const int32_t* col_index = batch_cols(batch_base, sc, NBb);
  const int j_begin = cr.begin, j_end = cr.end;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int nst = j_begin < j_end ? (j_end - j_begin + kColStage - 1) / kColStage : 0;
  if (warp == kConsumers / 32) {
    if (j_begin < j_end)
      producer_loop(sm, GT, ldx, col_index, list, quarters, spatial, colconst, SPB_COLCONST_FLOATS, i0, cr, NBb, lane);
    return;
  }
  const u64 CQ = pk(sc->c_q, sc->c_q), CS = pk(sc->c_s, sc->c_s);
  const int r = i0 + tid * 4;
  const RowRegs R = load_rows(XA, ldx, lm, nullptr, r);
  S2Acc A;
  A.clear();
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    mbar_wait(&sm.full[s], (st / kStages) & 1);
    const uint64_t wq = sm.quarters[s] >> warp;
    if (j_begin + st * kColStage >= split) sweep2_stage<kSparse, kDim, false>(sm, s, tid, R, CQ, CS, wq, A);
    else sweep2_stage<kSparse, kDim, true>(sm, s, tid, R, CQ, CS, wq, A);
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);
  }
  A.store(rowpart + ((int64_t)seg * 8) * ldx + r, ldx);
}

// per row: fold the segment partials (fp64), write the fp32 statistics, accumulate the global sums (ordered: reproducible)
__device__ __forceinline__ void row_stats_store(const double (&a)[7], int i, int ldx, const float* __restrict__ mm,
                                                float* __restrict__ K_NA_spatial, float* __restrict__ K_NA_sigma2,
                                                float* __restrict__ K_NA, float* __restrict__ PXB, double (&v)[4]) {
  const double ksp = a[0] * (double)mm[i];
  K_NA_spatial[i] = (float)ksp;
  K_NA_sigma2[i] = (float)a[1];
  K_NA[i] = (float)a[3];
  PXB[i] = (float)a[4];
  PXB[ldx + i] = (float)a[5];
  PXB[2 * ldx + i] = (float)a[6];
  v[0] = ksp; v[1] = a[1]; v[2] = a[3]; v[3] = a[2];
}

__global__ void __launch_bounds__(256)
row_finalize_kernel(const float* __restrict__ rowpart, int nseg, int ldx, int NA, const float* __restrict__ mm,
                    float* __restrict__ K_NA_spatial, float* __restrict__ K_NA_sigma2, float* __restrict__ K_NA,
                    float* __restrict__ PXB, spb_scalars* sc, double* __restrict__ red_scratch, unsigned int* red_counter) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0, 0, 0, 0};  // Sp_spatial, Sp_sigma2, Sp, S2
  if (i < NA) {
    double a[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int s = 0; s < nseg; ++s) {
#pragma unroll
      for (int q = 0; q < 7; ++q) a[q] += (double)rowpart[((int64_t)s * 8 + q) * ldx + i];
    }
    row_stats_store(a, i, ldx, mm, K_NA_spatial, K_NA_sigma2, K_NA, PXB, v);
  }
  grid_reduce_ordered<4>(v, red_scratch, red_counter, sc->sums, false);
}

// ---- column-sharded pair ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
row_fold_kernel(const float* __restrict__ rowpart, int nseg, int ldx, int NA, int add, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NA) return;
  double a[7] = {0, 0, 0, 0, 0, 0, 0};
  for (int s = 0; s < nseg; ++s) {
#pragma unroll
    for (int q = 0; q < 7; ++q) a[q] += (double)rowpart[((int64_t)s * 8 + q) * ldx + i];
  }
#pragma unroll
  for (int q = 0; q < 7; ++q) out[(int64_t)q * ldx + i] = add ? out[(int64_t)q * ldx + i] + a[q] : a[q];
}

__global__ void __launch_bounds__(256)
row_stats_finalize_kernel(const double* __restrict__ stat, int ldx, int NA, const float* __restrict__ mm,
                          float* __restrict__ K_NA_spatial, float* __restrict__ K_NA_sigma2, float* __restrict__ K_NA,
                          float* __restrict__ PXB, spb_scalars* sc, double* __restrict__ red_scratch,
                          unsigned int* red_counter) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0, 0, 0, 0};
  if (i < NA) {
    double a[7];
#pragma unroll
    for (int q = 0; q < 7; ++q) a[q] = stat[(int64_t)q * ldx + i];
    row_stats_store(a, i, ldx, mm, K_NA_spatial, K_NA_sigma2, K_NA, PXB, v);
  }
  grid_reduce_ordered<4>(v, red_scratch, red_counter, sc->sums, false);
}

__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// Row statistics of the whole pair from every rank's partial sums, read straight from the peers' memory over NVLink:
// block 0 announces "my partials of this epoch are complete" in every peer's flag array (system-scope release; the fold
// kernel that produced them has finished), every block waits until all peers have announced the epoch, then each row sums
// the W partial vectors IN RANK ORDER (so all ranks obtain the same bits) and finishes as row_finalize does.
__global__ void __launch_bounds__(256)
row_stats_p2p_kernel(const uint64_t* __restrict__ peer_stat, int parity, int rank, int world, uint64_t* flags,
                     const uint64_t* __restrict__ peer_flags, uint64_t epoch, int ldx, int NA, const float* __restrict__ mm,
                     float* __restrict__ K_NA_spatial, float* __restrict__ K_NA_sigma2, float* __restrict__ K_NA,
                     float* __restrict__ PXB, spb_scalars* sc, double* __restrict__ red_scratch, unsigned int* red_counter) {
  if (blockIdx.x == 0 && threadIdx.x < world) {
    __threadfence_system();
    st_release_sys(reinterpret_cast<uint64_t*>(peer_flags[threadIdx.x]) + rank, epoch);
  }
  if (threadIdx.x < world) {
    while (ld_acquire_sys(flags + threadIdx.x) < epoch) {
    }
  }
  __syncthreads();
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  double v[4] = {0, 0, 0, 0};
  if (i < NA) {
    double a[7] = {0, 0, 0, 0, 0, 0, 0};
    for (int r = 0; r < world; ++r) {
      const double* src = reinterpret_cast<const double*>(peer_stat[r]) + (int64_t)parity * 8 * ldx;
#pragma unroll
      for (int q = 0; q < 7; ++q) a[q] += src[(int64_t)q * ldx + i];
    }
    row_stats_store(a, i, ldx, mm, K_NA_spatial, K_NA_sigma2, K_NA, PXB, v);
  }
  grid_reduce_ordered<4>(v, red_scratch, red_counter, sc->sums, false);
}

// bounding box of the current positions of each 128-row quarter of each row block and the largest row term lm of the
// quarter (valid rows only): warp w reduces the rows of consumer warp w of the sweeps
__global__ void __launch_bounds__(kConsumers) block_bounds_kernel(const float* __restrict__ XA, const float* __restrict__ lm,
                                                                  int ldx, int NA, float* __restrict__ bbox) {
  const int rb = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  float lo[3] = {3e38f, 3e38f, 3e38f}, hi[3] = {-3e38f, -3e38f, -3e38f}, lmax = -INFINITY;
  for (int q = 0; q < 4; ++q) {
    const int i = rb * kRowTile + threadIdx.x * 4 + q;
    if (i < NA) {
#pragma unroll
      for (int d = 0; d < 3; ++d) {
        const float x = XA[(int64_t)d * ldx + i];
        lo[d] = fminf(lo[d], x);
        hi[d] = fmaxf(hi[d], x);
      }
      lmax = fmaxf(lmax, lm[i]);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if (lane == 0) bbox[(rb * 4 + warp) * 8 + 6] = lmax;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xffffffffu, lo[d], o));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xffffffffu, hi[d], o));
    }
    if (lane == 0) {
      bbox[(rb * 4 + warp) * 8 + d] = lo[d];
      bbox[(rb * 4 + warp) * 8 + 3 + d] = hi[d];
    }
  }
}

__device__ __forceinline__ float box_dist2(const float (&lo)[3], const float (&hi)[3], const float (&y)[3]) {
  float d2 = 0.f;
#pragma unroll
  for (int d = 0; d < 3; ++d) {
    const float g = fmaxf(fmaxf(lo[d] - y[d], y[d] - hi[d]), 0.f);
    d2 = fmaf(g, g, d2);
  }
  return d2;
}

// Per row block: order-preserving compaction of the columns that are not provably zero for every row of the block.
// With dmin the distance from y_j to a bounding box and lmax the largest row term lm = log2(alpha e^(-SigmaDiag/sigma2))
// of its rows, every pair (i, j) of the box's rows has an fp32 ex2 argument below -126 in the sweeps
//   for the weight q = ex2(c_q d + lm)   when  c_q dmin^2 + lmax < -127,
//   for the spatial weight s = ex2(c_s d) when  c_s dmin^2 < -127
// (log2 domain; the 1e-5 relative margin on c_q and c_s and the one unit between -127 and -126 cover the rounding of d and
// of the fma), so that weight flushes to +0. The cost matrix enters only through q g, so it is read only where q can be
// non-zero. Per 128-row quarter the two tests give the listed column's quarter masks: colquarters (q: the quarter's cost
// rows are read) and colspatial (s is formed). A column is listed when either test passes against the block's box; it is
// spatially live (before colsplit) when the s test passes. Dropped pairs would have added exact zeros.
// One CTA per row block, 32 warps, each warp owns a contiguous range of columns: pass 1 evaluates the block test once (the
// keep bits go to shared memory), one block barrier turns the per-warp counts into offsets, pass 2 scatters the listed
// columns with their quarter masks. The keep bits, the spatially live bits and each word's two list offsets are also
// published (keepmask, livemask, keepoff): col_finalize folds only the partial column sums that sweep 1 wrote, so the dropped
// (row block, column) combinations are neither zeroed (a 157-313 MB write per iteration) nor read, and finds each partial
// at its list position (sweep 1 stores them there, one full 32-byte sector per stage and sum instead of 4-byte scatters).
constexpr int kListThreads = 1024;
// geom: one record per column, `gstride` floats apart, coordinate d at float offset d * gstep (the 16-byte xb4 records when the
// columns are all fixed cells: half the L2 traffic of the duplicated colgeom layout, which every row block re-reads in full)
__device__ __forceinline__ void load_col(const float* __restrict__ geom, int gstride, int gstep, int j, bool in, int cull,
                                         float (&y)[3]) {
  const float* p = geom + (int64_t)(in ? j : 0) * gstride;
  if (gstride == 4) {  // one 16-byte load per column
    const float4 v = cull ? *reinterpret_cast<const float4*>(p) : make_float4(0.f, 0.f, 0.f, 0.f);
    y[0] = v.x, y[1] = v.y, y[2] = v.z;
  } else {
#pragma unroll
    for (int d = 0; d < 3; ++d) y[d] = cull ? p[d * gstep] : 0.f;
  }
}

__global__ void __launch_bounds__(kListThreads) build_col_lists_kernel(const float* __restrict__ bbox, const float* __restrict__ geom,
                                                                       int gstride, int gstep,
                                                                       int NBb, spb_scalars* __restrict__ sc, int cull,
                                                                       int32_t* __restrict__ collist, uint8_t* __restrict__ colquarters,
                                                                       uint8_t* __restrict__ colspatial, int32_t* __restrict__ colcount, int32_t* __restrict__ colsplit,
                                                                       int nbb_pad, uint32_t* __restrict__ colmask,
                                                                       uint32_t* __restrict__ keepmask, uint32_t* __restrict__ livemask,
                                                                       int2* __restrict__ keepoff, int kstride) {
  extern __shared__ uint32_t keep_bits[];  // [2][nwords]: one word per 32 columns — kept at all | spatially live
  __shared__ int warp_cnt[2][32];
  __shared__ int live_quarters;
  const int rb = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float cq = sc->c_q * (1.0f - 1e-5f);
  const float cs = sc->c_s * (1.0f - 1e-5f);  // c_s = c_q * sigma2_variance
  float qlo[4][3], qhi[4][3], lo[3], hi[3];   // quarter boxes and the block's box (their union)
  float qlm[4], blm = -INFINITY;              // largest row term of each quarter and of the block
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    qlm[q] = bbox[(rb * 4 + q) * 8 + 6];
    blm = fmaxf(blm, qlm[q]);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
      qlo[q][d] = bbox[(rb * 4 + q) * 8 + d];
      qhi[q][d] = bbox[(rb * 4 + q) * 8 + 3 + d];
      lo[d] = q ? fminf(lo[d], qlo[q][d]) : qlo[q][d];
      hi[d] = q ? fmaxf(hi[d], qhi[q][d]) : qhi[q][d];
    }
  }
  if (threadIdx.x == 0) live_quarters = 0;
  const int nwords = (NBb + 31) / 32;
  uint32_t* live_bits = keep_bits + nwords;
  const int wpw = (nwords + 31) / 32;  // words per warp
  const int w0 = warp * wpw, w1 = min(nwords, w0 + wpw);
  int cnt = 0, cnt_live = 0;
  constexpr int kU = 4;  // words per trip: the 12 coordinate loads of a trip are independent (the loop is latency-bound)
  for (int wb = w0; wb < w1; wb += kU) {
    float yy[kU][3];
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int j = (wb + u) * 32 + lane;
      load_col(geom, gstride, gstep, j, (wb + u < w1) && j < NBb, cull, yy[u]);
    }
#pragma unroll
    for (int u = 0; u < kU; ++u) {
      const int wd = wb + u;
      if (wd >= w1) break;  // warp-uniform
      const int j = wd * 32 + lane;
      bool keep = false, live = false;
      if (j < NBb) {
        keep = live = true;
        if (cull) {
          const float d2 = box_dist2(lo, hi, yy[u]);
          live = cs * d2 >= -127.0f;
          keep = live || cq * d2 + blm >= -127.0f;
        }
      }
      const uint32_t bits = __ballot_sync(0xffffffffu, keep), lbits = __ballot_sync(0xffffffffu, live);
      if (lane == 0) {
        keep_bits[wd] = bits;
        live_bits[wd] = lbits;
      }
      cnt += __popc(bits & ~lbits);  // kept but spatially dead
      cnt_live += __popc(lbits);
    }
  }
  if (lane == 0) {
    warp_cnt[0][warp] = cnt_live;
    warp_cnt[1][warp] = cnt;
  }
  __syncthreads();
  int off_live = 0, off_dead = 0, total_live = 0, total_dead = 0;
#pragma unroll
  for (int grp = 0; grp < 2; ++grp) {
    const int c = warp_cnt[grp][lane];
    int inc = c;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    const int mine = __shfl_sync(0xffffffffu, inc - c, warp);  // exclusive prefix of this warp
    const int tot = __shfl_sync(0xffffffffu, inc, 31);
    if (grp == 0) off_live = mine, total_live = tot;
    else off_dead = mine, total_dead = tot;
  }
  off_dead += total_live;  // the spatially dead columns follow the live ones in the list
  int32_t* list = collist + (int64_t)rb * nbb_pad;
  uint8_t* qlist = colquarters + (int64_t)rb * nbb_pad;
  uint8_t* slist = colspatial + (int64_t)rb * nbb_pad;
  int nq = 0;  // quarters of this lane's listed columns whose cost rows are read
  float ynext[3];
  if (w0 < w1) load_col(geom, gstride, gstep, w0 * 32 + lane, w0 * 32 + lane < NBb, cull, ynext);
  for (int wd = w0; wd < w1; ++wd) {
    const uint32_t bits = keep_bits[wd], lbits = live_bits[wd], dbits = bits & ~lbits;
    const int j = wd * 32 + lane;
    const float y[3] = {ynext[0], ynext[1], ynext[2]};
    if (wd + 1 < w1) load_col(geom, gstride, gstep, j + 32, j + 32 < NBb, cull, ynext);  // next word's column, in flight
    const uint32_t below = (1u << lane) - 1u;
    int pos = -1;
    if ((lbits >> lane) & 1u) pos = off_live + __popc(lbits & below);
    else if ((dbits >> lane) & 1u) pos = off_dead + __popc(dbits & below);
    if (pos >= 0) {
      uint32_t qm = 0xFu, sm = 0xFu;  // without culling every quarter of every column is read and computed
      if (cull) {
        qm = sm = 0u;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float d2 = box_dist2(qlo[q], qhi[q], y);
          qm |= (cq * d2 + qlm[q] >= -127.0f) ? 1u << q : 0u;
          sm |= (cs * d2 >= -127.0f) ? 1u << q : 0u;
        }
      }
      list[pos] = j;
      qlist[pos] = (uint8_t)qm;
      slist[pos] = (uint8_t)sm;
      nq += __popc(qm);
    }
    if (lane == 0) {  // col_finalize folds only the listed (row block, column) partials and finds them by list position
      keepmask[(int64_t)rb * kstride + wd] = bits;
      livemask[(int64_t)rb * kstride + wd] = lbits;
      keepoff[(int64_t)rb * kstride + wd] = make_int2(off_live, off_dead);
    }
    if (((bits >> lane) & 1u) && colmask != nullptr && rb < 32 * SPB_COLMASK_WORDS)
      atomicOr(colmask + (int64_t)j * SPB_COLMASK_WORDS + (rb >> 5), 1u << (rb & 31));
    off_live += __popc(lbits);
    off_dead += __popc(dbits);
  }
  nq = __reduce_add_sync(0xffffffffu, nq);
  if (lane == 0) atomicAdd(&live_quarters, nq);
  __syncthreads();
  if (threadIdx.x == 0) {
    colcount[rb] = total_live + total_dead;
    colsplit[rb] = total_live;
    atomicAdd(&sc->visited, 0.25 * (double)live_quarters);  // in whole (row block, column) tiles
  }
}

// gather this iteration's fixed-slice coordinates (SVI batch or all columns) (morpho_class.py:1149)
__global__ void gather_cols_kernel(const float* __restrict__ xb4, const int32_t* __restrict__ batch_base,
                                   const spb_scalars* __restrict__ sc, int NBb, float* __restrict__ colgeom) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= NBb) return;
  const int32_t* idx = batch_cols(batch_base, sc, NBb);
  const int64_t src = idx ? idx[j] : j;
  const float4 y = reinterpret_cast<const float4*>(xb4)[src];
  float4* out = reinterpret_cast<float4*>(colgeom + (int64_t)j * 8);
  out[0] = make_float4(y.x, y.x, y.y, y.y);
  out[1] = make_float4(y.z, y.z, 0.f, 0.f);
}

// dense P for the caller (utils.py:1083): P[i][j] = qm_ij g_ij c_j, transposed through shared memory
__global__ void materialize_P_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                                     const float* __restrict__ colconst, const float* __restrict__ XA,
                                     const float* __restrict__ lm, const spb_scalars* __restrict__ sc, int NA, int NBb,
                                     float* __restrict__ P, int64_t ldp) {
  __shared__ float tile[32][33];
  const int32_t* col_index = batch_cols(batch_base, sc, NBb);
  const float c_q = sc->c_q;
  const int jb = blockIdx.y * 32, ib = blockIdx.x * 32;
  for (int jj = threadIdx.y; jj < 32; jj += blockDim.y) {
    const int j = jb + jj, i = ib + threadIdx.x;
    float p = 0.f;
    if (j < NBb && i < NA) {
      const int64_t row = col_index ? col_index[j] : j;
      const float* cc = colconst + (int64_t)j * SPB_COLCONST_FLOATS;
      const float4 ya = make_float4(cc[0], cc[2], cc[4], 0.f);
      const float cj = cc[10];
      const float d = sqdist(XA[i], XA[ldx + i], XA[2 * ldx + i], ya);
      p = ex2f(fmaf(c_q, d, lm[i])) * GT[row * ldx + i] * cj;
    }
    tile[jj][threadIdx.x] = p;
  }
  __syncthreads();
  for (int ii = threadIdx.y; ii < 32; ii += blockDim.y) {
    const int i = ib + ii, j = jb + threadIdx.x;
    if (i < NA && j < NBb) P[(int64_t)i * ldp + j] = tile[threadIdx.x][ii];
  }
}


// ---------------------------------------------------------------------------------------------------------------------
// sparse_calculation_mode: per-column top-k of the full posterior (utils.py:1085-1094 -> _dense_to_sparse :1369-1404)
// ---------------------------------------------------------------------------------------------------------------------
// Within a column P_ij = w_ij c_j with w = q g, so the k largest P are the k largest w. One CTA owns one column (its GT
// row is contiguous) and finds the k-th largest w EXACTLY by a 3-level radix select on the float bits (12 + 12 + 7 bits;
// w >= 0 so the bit pattern is monotone). After the first level the surviving candidates are gathered into shared
// memory, so the column is normally read twice; that second read also sums the mass above the selected bin:
//   tau_j   -> colconst[j][18..19]  (sweep 2 keeps pairs with w >= tau_j; exact ties at tau_j are all kept)
//   K_NB_j  = c_j * sum_{w >= tau_j} w
// The weight is evaluated with the same instruction sequence as the packed sweep (sub, mul, fma, fma, fma, ex2, mul), so
// both kernels see bit-identical w.
constexpr int kSelThreads = 512;
constexpr int kSelBins = 4096;
constexpr int kSelCap = 8192;

__device__ __forceinline__ float pair_weight(float x0, float x1, float x2, float y0, float y1, float y2, float cq,
                                             float lmi, float g) {
  const float d0 = __fsub_rn(x0, y0), d1 = __fsub_rn(x1, y1), d2 = __fsub_rn(x2, y2);
  const float d = __fmaf_rn(d2, d2, __fmaf_rn(d1, d1, __fmul_rn(d0, d0)));
  return __fmul_rn(ex2f(__fmaf_rn(cq, d, lmi)), g);
}

struct SelShared {
  uint32_t wcnt[kSelThreads / 32];
  float wsum[kSelThreads / 32];
  uint32_t bsel, above_cnt, sel_cnt, total;
  float above_sum, sel_sum, total_sum;
  int ncand;
};

// histogram of (key >> shift) & (nb - 1) over the values whose key matches (prefix, pmask); zero weights are skipped
// mask (optional): bit rb set <=> row block rb (SPB_ROW_TILE rows) can hold a non-zero weight for this column; the other blocks
// are provably all-zero (build_col_lists_kernel) and are skipped — a warp never straddles two row blocks
template <typename F>
__device__ __forceinline__ void sel_for_each(const float* __restrict__ g, const float* __restrict__ XA, int64_t ldx,
                                             const float* __restrict__ lm, int NA, float y0, float y1, float y2, float cq,
                                             F&& f, const uint32_t* __restrict__ mask = nullptr) {
  for (int i = threadIdx.x * 4; i < NA; i += kSelThreads * 4) {
    if (mask != nullptr) {
      const int rb = i / kRowTile;
      if (((mask[rb >> 5] >> (rb & 31)) & 1u) == 0u) continue;
    }
    const float4 G = *reinterpret_cast<const float4*>(g + i);
    const float4 X0 = *reinterpret_cast<const float4*>(XA + i);
    const float4 X1 = *reinterpret_cast<const float4*>(XA + ldx + i);
    const float4 X2 = *reinterpret_cast<const float4*>(XA + 2 * ldx + i);
    const float4 L = *reinterpret_cast<const float4*>(lm + i);
    f(i, pair_weight(X0.x, X1.x, X2.x, y0, y1, y2, cq, L.x, G.x));
    if (i + 1 < NA) f(i + 1, pair_weight(X0.y, X1.y, X2.y, y0, y1, y2, cq, L.y, G.y));
    if (i + 2 < NA) f(i + 2, pair_weight(X0.z, X1.z, X2.z, y0, y1, y2, cq, L.z, G.z));
    if (i + 3 < NA) f(i + 3, pair_weight(X0.w, X1.w, X2.w, y0, y1, y2, cq, L.w, G.w));
  }
}

// block-wide sum in a fixed order (warp butterfly, then warps in sequence); ends with a barrier so `red` can be reused
__device__ __forceinline__ float sel_block_sum(float v, float* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float t = 0.f;
  for (int w = 0; w < kSelThreads / 32; ++w) t += red[w];
  __syncthreads();
  return t;
}

__global__ void __launch_bounds__(kSelThreads)
col_select_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                  float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                  const spb_scalars* __restrict__ sc, int NA, int topk, float* __restrict__ K_NB,
                  const uint32_t* __restrict__ colmask) {
  extern __shared__ __align__(16) uint8_t sel_raw[];
  uint32_t* hist = reinterpret_cast<uint32_t*>(sel_raw);
  float* sums = reinterpret_cast<float*>(hist + kSelBins);
  float* cand = sums + kSelBins;
  __shared__ SelShared sh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int jb = blockIdx.x;
  float* cc = colconst + (int64_t)jb * SPB_COLCONST_FLOATS;
  const float y0 = cc[0], y1 = cc[2], y2 = cc[4], cj = cc[10];
  const int32_t* col_index = batch_cols(batch_base, sc, (int)gridDim.x);
  const int64_t row = col_index ? (int64_t)col_index[jb] : (int64_t)jb;
  const float* g = GT + row * ldx;
  const float cq = sc->c_q;
  __shared__ uint32_t s_mask[SPB_COLMASK_WORDS];
  if (colmask != nullptr && tid < SPB_COLMASK_WORDS) s_mask[tid] = colmask[(int64_t)jb * SPB_COLMASK_WORDS + tid];
  __syncthreads();
  const uint32_t* mask = colmask != nullptr ? s_mask : nullptr;
  uint32_t prefix = 0, pmask = 0, remaining = (uint32_t)min(topk, NA);
  float kept = 0.f;
  bool use_cand = false;
  int ncand = 0;
  float tau = 0.f;
  for (int pass = 0; pass < 3; ++pass) {
    const int shift = pass == 0 ? 19 : (pass == 1 ? 7 : 0);
    const int nb = pass == 2 ? 128 : kSelBins;
    for (int t = tid; t < nb; t += kSelThreads) {
      hist[t] = 0u;
      sums[t] = 0.f;
    }
    __syncthreads();
    // level 0 only counts (one shared-memory atomic per non-zero weight); the mass above the selected bin is summed in
    // registers by the pass that gathers the survivors
    const bool with_sums = pass > 0;
    auto add = [&](int, float w) {
      const uint32_t key = __float_as_uint(w);
      if (key != 0u && (key & pmask) == prefix) {
        const uint32_t b = (key >> shift) & (uint32_t)(nb - 1);
        atomicAdd(&hist[b], 1u);
        if (with_sums) atomicAdd(&sums[b], w);
      }
    };
    if (!use_cand) {
      sel_for_each(g, XA, ldx, lm, NA, y0, y1, y2, cq, add, mask);
    } else {
      for (int t = tid; t < ncand; t += kSelThreads) add(t, cand[t]);
    }
    __syncthreads();
    // suffix scan over bins (high bins first): thread t owns bins [t * per, (t + 1) * per)
    const int per = nb >= kSelThreads ? nb / kSelThreads : 1;
    const bool owner = tid * per < nb;
    uint32_t mycnt = 0;
    float mysum = 0.f;
    if (owner)
      for (int q = 0; q < per; ++q) {
        mycnt += hist[tid * per + q];
        mysum += sums[tid * per + q];
      }
    uint32_t c = mycnt;
    float sm_ = mysum;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const uint32_t c2 = __shfl_down_sync(0xffffffffu, c, off);
      const float s2 = __shfl_down_sync(0xffffffffu, sm_, off);
      if (lane + off < 32) {
        c += c2;
        sm_ += s2;
      }
    }
    if (lane == 0) {
      sh.wcnt[warp] = c;
      sh.wsum[warp] = sm_;
    }
    __syncthreads();
    uint32_t hi_c = 0;
    float hi_s = 0.f;
    for (int w = warp + 1; w < kSelThreads / 32; ++w) {
      hi_c += sh.wcnt[w];
      hi_s += sh.wsum[w];
    }
    const uint32_t above_c = c - mycnt + hi_c;  // count in bins owned by higher threads
    const float above_s = sm_ - mysum + hi_s;
    if (tid == 0) {
      sh.total = c + hi_c;
      sh.total_sum = sm_ + hi_s;
    }
    if (owner && above_c < remaining && remaining <= above_c + mycnt) {
      uint32_t run_c = above_c;
      float run_s = above_s;
      for (int q = per - 1; q >= 0; --q) {
        const uint32_t h = hist[tid * per + q];
        if (run_c + h >= remaining) {
          sh.bsel = (uint32_t)(tid * per + q);
          sh.above_cnt = run_c;
          sh.above_sum = run_s;
          sh.sel_cnt = h;
          sh.sel_sum = sums[tid * per + q];
          break;
        }
        run_c += h;
        run_s += sums[tid * per + q];
      }
    }
    __syncthreads();
    if (sh.total < remaining) {  // fewer non-zero weights than k (only possible at the first level): keep everything
      float acc = 0.f;
      sel_for_each(g, XA, ldx, lm, NA, y0, y1, y2, cq, [&](int, float w) { acc += w; }, mask);
      kept += sel_block_sum(acc, sh.wsum);
      tau = 0.f;
      break;
    }
    const uint32_t bsel = sh.bsel;
    prefix |= bsel << shift;
    pmask |= (uint32_t)(nb - 1) << shift;
    if (pass == 2) {
      kept += sh.above_sum + sh.sel_sum;  // every copy of the threshold value is kept
      tau = __uint_as_float(prefix);
      break;
    }
    if (pass > 0) kept += sh.above_sum;
    remaining -= sh.above_cnt;
    const uint32_t sel_cnt = sh.sel_cnt;
    __syncthreads();
    if (pass == 0) {
      // second read of the column: mass of the bins above the selected one (registers, fixed reduction order) and, when
      // they fit, the survivors of the selected bin into shared memory so the remaining levels never touch global memory
      const bool fits = sel_cnt <= (uint32_t)kSelCap;
      if (tid == 0) sh.ncand = 0;
      __syncthreads();
      float acc = 0.f;
      sel_for_each(g, XA, ldx, lm, NA, y0, y1, y2, cq, [&](int, float w) {
        const uint32_t kb = __float_as_uint(w) >> 19;
        if (kb > bsel) acc += w;
        else if (fits && kb == bsel && w != 0.f) cand[atomicAdd(&sh.ncand, 1)] = w;
      }, mask);
      kept += sel_block_sum(acc, sh.wsum);
      ncand = sh.ncand;
      use_cand = fits;
    }
  }
  if (tid == 0) {
    cc[18] = tau;
    cc[19] = tau;
    K_NB[jb] = cj * kept;
  }
}

// COO entries of the sparse posterior: per column the (up to) k pairs with w >= tau_j, explicit zeros filling columns
// with fewer than k non-zero weights (the reference's sort keeps exactly k entries per column). Unordered within the
// column; the host sorts the k values.
__global__ void __launch_bounds__(kSelThreads)
col_emit_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                const float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                const spb_scalars* __restrict__ sc, int NA, int topk, int32_t* __restrict__ rows,
                float* __restrict__ vals) {
  __shared__ int cnt;
  const int jb = blockIdx.x, tid = threadIdx.x;
  const float* cc = colconst + (int64_t)jb * SPB_COLCONST_FLOATS;
  const float y0 = cc[0], y1 = cc[2], y2 = cc[4], cj = cc[10], tau = cc[18];
  const int32_t* col_index = batch_cols(batch_base, sc, (int)gridDim.x);
  const int64_t row = col_index ? (int64_t)col_index[jb] : (int64_t)jb;
  const float* g = GT + row * ldx;
  const float cq = sc->c_q;
  const int k = min(topk, NA);
  int32_t* r = rows + (int64_t)jb * topk;
  float* v = vals + (int64_t)jb * topk;
  if (tid == 0) cnt = 0;
  __syncthreads();
  sel_for_each(g, XA, ldx, lm, NA, y0, y1, y2, cq, [&](int i, float w) {
    if (w > tau) {
      const int s = atomicAdd(&cnt, 1);
      if (s < k) {
        r[s] = i;
        v[s] = w * cj;
      }
    }
  });
  __syncthreads();
  // ties at the threshold (and, when tau == 0, the zero fill) until k entries exist
  for (int i0 = 0; i0 < NA; i0 += kSelThreads * 4) {
    if (__syncthreads_or(cnt >= k)) break;  // block-uniform: every atomic of the previous round precedes the barrier
    const int i = i0 + tid * 4;
    if (i < NA) {
      const float4 G = *reinterpret_cast<const float4*>(g + i);
      const float4 X0 = *reinterpret_cast<const float4*>(XA + i);
      const float4 X1 = *reinterpret_cast<const float4*>(XA + ldx + i);
      const float4 X2 = *reinterpret_cast<const float4*>(XA + 2 * ldx + i);
      const float4 L = *reinterpret_cast<const float4*>(lm + i);
      const float w4[4] = {pair_weight(X0.x, X1.x, X2.x, y0, y1, y2, cq, L.x, G.x),
                           pair_weight(X0.y, X1.y, X2.y, y0, y1, y2, cq, L.y, G.y),
                           pair_weight(X0.z, X1.z, X2.z, y0, y1, y2, cq, L.z, G.z),
                           pair_weight(X0.w, X1.w, X2.w, y0, y1, y2, cq, L.w, G.w)};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        if (i + q < NA && w4[q] == tau) {
          const int s = atomicAdd(&cnt, 1);
          if (s < k) {
            r[s] = i + q;
            v[s] = w4[q] * cj;
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// argmax of the posterior along both axes without materialising it (get_optimal_mapping_relationship,
// spateo/alignment/utils.py:157-191: X_max_index = row maxima of pi, Y_max_index = column maxima)
// ---------------------------------------------------------------------------------------------------------------------
// key = (float bits of p) << 32 | (0xffffffff - index): unsigned max picks the largest value, lowest index on ties
__device__ __forceinline__ unsigned long long argmax_key(float p, int idx) {
  return ((unsigned long long)__float_as_uint(p) << 32) | (unsigned long long)(0xffffffffu - (uint32_t)idx);
}

__global__ void __launch_bounds__(kSelThreads)
col_argmax_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                  const float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                  const spb_scalars* __restrict__ sc, int NA, unsigned long long* __restrict__ colbest) {
  __shared__ unsigned long long red[kSelThreads / 32];
  const int jb = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* cc = colconst + (int64_t)jb * SPB_COLCONST_FLOATS;
  const float y0 = cc[0], y1 = cc[2], y2 = cc[4], cj = cc[10];
  const int32_t* col_index = batch_cols(batch_base, sc, (int)gridDim.x);
  const int64_t row = col_index ? (int64_t)col_index[jb] : (int64_t)jb;
  unsigned long long best = 0ull;
  sel_for_each(GT + row * ldx, XA, ldx, lm, NA, y0, y1, y2, sc->c_q, [&](int i, float w) {
    const unsigned long long key = argmax_key(w * cj, i);
    best = key > best ? key : best;
  });
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other > best ? other : best;
  }
  if (lane == 0) red[warp] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < kSelThreads / 32; ++w) best = red[w] > best ? red[w] : best;
    colbest[jb] = best;
  }
}

// one thread per moving cell, blockIdx.y = column segment; partial results are merged with a 64-bit atomicMax.
// colmap (optional): output column index of every launch position, -1 = no column (skipped); without it the key carries j.
// A column-sharded pair passes its block's global column indices, so the ranks' keys merge with a plain maximum.
__global__ void __launch_bounds__(256)
row_argmax_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                  const float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                  const spb_scalars* __restrict__ sc, int NA, int NBb, const int32_t* __restrict__ colmap,
                  unsigned long long* __restrict__ rowbest) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NA) return;
  const int per = (NBb + gridDim.y - 1) / gridDim.y;
  const int j0 = blockIdx.y * per, j1 = min(NBb, j0 + per);
  const float x0 = XA[i], x1 = XA[ldx + i], x2 = XA[2 * ldx + i], li = lm[i], cq = sc->c_q;
  const int32_t* col_index = batch_cols(batch_base, sc, NBb);
  unsigned long long best = 0ull;
  for (int j = j0; j < j1; ++j) {
    const int jo = colmap ? colmap[j] : j;
    if (jo < 0) continue;
    const float4 c0 = *reinterpret_cast<const float4*>(colconst + (int64_t)j * SPB_COLCONST_FLOATS);
    const float4 c1 = *reinterpret_cast<const float4*>(colconst + (int64_t)j * SPB_COLCONST_FLOATS + 4);
    const float cj = colconst[(int64_t)j * SPB_COLCONST_FLOATS + 10];
    const int64_t row = col_index ? (int64_t)col_index[j] : (int64_t)j;
    float w = pair_weight(x0, x1, x2, c0.x, c0.z, c1.x, cq, li, GT[row * ldx + i]);
    w = w >= colconst[(int64_t)j * SPB_COLCONST_FLOATS + 18] ? w : 0.f;  // sparse mode: entries below the column's top-k are absent
    const unsigned long long key = argmax_key(w * cj, jo);
    best = key > best ? key : best;
  }
  if (j0 < j1) atomicMax(rowbest + i, best);
}

// ---------------------------------------------------------------------------------------------------------------------
// posterior transfer: P @ F_B and P^T @ F_A of the last E-step without forming P
// ---------------------------------------------------------------------------------------------------------------------
// Both kernels visit the (row block, column) tiles and 128-row quarters of the E-step's work lists with the grid and
// pipeline of the sweeps, and form P_ij = (q_ij g_ij) c_j with sweep 2's instruction sequence (sparse mode: w < tau_j
// is absent). Features are processed in panels of kXferPanel; a panel reads the listed cost tiles once. Skipped pairs
// are exact zeros, so culling changes no bit. No float atomics: every fold has a fixed order.
constexpr int kXferPanel = SPB_TRANSFER_PANEL;
constexpr int kXferCtas = 3;  // 4 x 16 fp32 accumulators (or feature registers) per thread: 3 CTAs of 160 threads per SM
static_assert(kXferPanel == 16, "one butterfly of 16 values per column, two 32-byte sectors per feature and stage");

struct __align__(16) XferSmem {
  SmemLayout base;
  float fpan[kStages][kColStage][kXferPanel];           // rows kernel: F_B panel rows of the staged columns
  float red[2][kColStage][kConsumers / 32][kXferPanel];  // cols kernel: warp totals of the staged columns
};

// P of this thread's 4 rows with staged column jj (a column whose q bit is set for the warp)
template <bool kSparse, int kDim>
__device__ __forceinline__ void xfer_weights(const SmemLayout& sm, int s, int jj, int tid, const RowRegs& R, u64 CQ,
                                             float (&p)[4]) {
  const ulonglong2 c0 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][0]);  // (y0,y0) (y1,y1)
  const ulonglong2 c1 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][1]);  // (y2,y2) (a,a)
  const ulonglong2 c2 = *reinterpret_cast<const ulonglong2*>(&sm.cols[s][jj][2]);  // (b,b)  (c,c)
  const ulonglong2 g = *reinterpret_cast<const ulonglong2*>(&sm.tile[s][jj][tid * 4]);
  const u64 da = sqdist2<kDim>(R.xa0, R.xa1, R.xa2, c0.x, c0.y, c1.x);
  const u64 db = sqdist2<kDim>(R.xb0, R.xb1, R.xb2, c0.x, c0.y, c1.x);
  const u64 qa = ex2_2(fma2(CQ, da, R.lma)), qb = ex2_2(fma2(CQ, db, R.lmb));
  u64 wa = mul2(qa, g.x), wb = mul2(qb, g.y);
  if constexpr (kSparse) {
    const float tau = sm.cols[s][jj][4].z;
    wa = keep_ge(wa, tau);
    wb = keep_ge(wb, tau);
  }
  upk(mul2(wa, c2.y), p[0], p[1]);
  upk(mul2(wb, c2.y), p[2], p[3]);
}

// P @ F_B, one feature panel: grid and pipeline of sweep 2; per-segment fp32 partials part[seg][kXferPanel][ldx]
template <bool kSparse, int kDim = 3>
__global__ void __launch_bounds__(kThreads, kXferCtas)
transfer_rows_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                     const int32_t* __restrict__ fbatch_base, const float* __restrict__ colconst,
                     const float* __restrict__ XA, const float* __restrict__ lm, const spb_scalars* __restrict__ sc,
                     const float* __restrict__ FB, int64_t ldf, float* __restrict__ part, int NBb, int nbb_pad,
                     const int32_t* __restrict__ collist, const uint8_t* __restrict__ colquarters,
                     const uint8_t* __restrict__ colspatial, const int32_t* __restrict__ colcount) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  XferSmem& xs = *reinterpret_cast<XferSmem*>(smem_raw);
  SmemLayout& sm = xs.base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rb = blockIdx.x, seg = blockIdx.y;
  const int i0 = rb * kRowTile;
  const ColRange cr = col_range(colcount, rb, seg, gridDim.y);
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  const int nst = cr.begin < cr.end ? (cr.end - cr.begin + kColStage - 1) / kColStage : 0;
  if (warp == kConsumers / 32) {
    if (nst > 0)
      producer_loop<kXferPanel>(sm, GT, ldx, batch_cols(batch_base, sc, NBb), collist + (int64_t)rb * nbb_pad,
                                colquarters + (int64_t)rb * nbb_pad, colspatial + (int64_t)rb * nbb_pad, colconst,
                                SPB_COLCONST_FLOATS, i0, cr, NBb, lane, FB, ldf, batch_cols(fbatch_base, sc, NBb),
                                &xs.fpan[0][0][0]);
    return;
  }
  const u64 CQ = pk(sc->c_q, sc->c_q);
  const int r = i0 + tid * 4;
  const RowRegs R = load_rows(XA, ldx, lm, nullptr, r);
  float acc[4][kXferPanel];
#pragma unroll
  for (int q = 0; q < 4; ++q)
#pragma unroll
    for (int f = 0; f < kXferPanel; ++f) acc[q][f] = 0.f;
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    mbar_wait(&sm.full[s], (st / kStages) & 1);
    const uint64_t wq = sm.quarters[s] >> warp;
#pragma unroll
    for (int jj = 0; jj < kColStage; ++jj) {
      if (!quarter_q(wq, jj)) continue;
      float p[4];
      xfer_weights<kSparse, kDim>(sm, s, jj, tid, R, CQ, p);
      const float4* fr = reinterpret_cast<const float4*>(&xs.fpan[s][jj][0]);
#pragma unroll
      for (int v = 0; v < kXferPanel / 4; ++v) {
        const float4 f = fr[v];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          acc[q][4 * v + 0] = fmaf(p[q], f.x, acc[q][4 * v + 0]);
          acc[q][4 * v + 1] = fmaf(p[q], f.y, acc[q][4 * v + 1]);
          acc[q][4 * v + 2] = fmaf(p[q], f.z, acc[q][4 * v + 2]);
          acc[q][4 * v + 3] = fmaf(p[q], f.w, acc[q][4 * v + 3]);
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);
  }
  float* out = part + (int64_t)seg * kXferPanel * ldx + r;
#pragma unroll
  for (int f = 0; f < kXferPanel; ++f)
    *reinterpret_cast<float4*>(out + (int64_t)f * ldx) = make_float4(acc[0][f], acc[1][f], acc[2][f], acc[3][f]);
}

// per moving cell: the segment partials of one panel folded in fp64 in segment order (row_finalize), written to or (add:
// the next column chunk of a streamed E-step) added into out[kXferPanel][ldx]
__global__ void __launch_bounds__(256)
transfer_row_fold_kernel(const float* __restrict__ part, int nseg, int ldx, int NA, int add, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NA) return;
#pragma unroll 4
  for (int f = 0; f < kXferPanel; ++f) {
    double a = 0.0;
    for (int s = 0; s < nseg; ++s) a += (double)part[((int64_t)s * kXferPanel + f) * ldx + i];
    double* o = out + (int64_t)f * ldx + i;
    *o = add ? *o + a : a;
  }
}

// P^T @ F_A, one feature panel: grid and pipeline of sweep 1. Each consumer thread holds its 4 rows of the panel; per
// staged column a warp reduces its quarter with the butterfly, warp 0 adds the four warps in order (sweep 1) and stores
// the row block's partials by list position, part[rb][kXferPanel][nbb_pad]: one 32-byte sector per feature and stage.
template <bool kSparse, int kDim = 3>
__global__ void __launch_bounds__(kThreads, kXferCtas)
transfer_cols_kernel(const float* __restrict__ GT, int64_t ldx, const int32_t* __restrict__ batch_base,
                     const float* __restrict__ colconst, const float* __restrict__ XA, const float* __restrict__ lm,
                     const spb_scalars* __restrict__ sc, const float* __restrict__ FA, float* __restrict__ part, int NBb,
                     int nbb_pad, const int32_t* __restrict__ collist, const uint8_t* __restrict__ colquarters,
                     const uint8_t* __restrict__ colspatial, const int32_t* __restrict__ colcount) {
  extern __shared__ __align__(128) uint8_t smem_raw[];
  XferSmem& xs = *reinterpret_cast<XferSmem*>(smem_raw);
  SmemLayout& sm = xs.base;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int rb = blockIdx.x, seg = blockIdx.y;
  const int i0 = rb * kRowTile;
  const ColRange cr = col_range(colcount, rb, seg, gridDim.y);
  if (cr.begin >= cr.end) return;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&sm.full[s], 1);
      mbar_init(&sm.empty[s], kConsumers / 32);
    }
    fence_mbar_init();
  }
  __syncthreads();
  if (warp == kConsumers / 32) {
    producer_loop(sm, GT, ldx, batch_cols(batch_base, sc, NBb), collist + (int64_t)rb * nbb_pad,
                  colquarters + (int64_t)rb * nbb_pad, colspatial + (int64_t)rb * nbb_pad, colconst, SPB_COLCONST_FLOATS,
                  i0, cr, NBb, lane);
    return;
  }
  const u64 CQ = pk(sc->c_q, sc->c_q);
  const int r = i0 + tid * 4;
  const RowRegs R = load_rows(XA, ldx, lm, nullptr, r);
  float fa[kXferPanel][4];
#pragma unroll
  for (int f = 0; f < kXferPanel; ++f) {
    const float4 v = *reinterpret_cast<const float4*>(FA + (int64_t)f * ldx + r);
    fa[f][0] = v.x, fa[f][1] = v.y, fa[f][2] = v.z, fa[f][3] = v.w;
  }
  float* out = part + (int64_t)rb * kXferPanel * nbb_pad;
  const int nst = (cr.end - cr.begin + kColStage - 1) / kColStage;
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    mbar_wait(&sm.full[s], (st / kStages) & 1);
    const int pb = cr.begin + st * kColStage;
    const int buf = st & 1;
    const uint64_t wq = sm.quarters[s] >> warp;
#pragma unroll
    for (int jj = 0; jj < kColStage; ++jj) {
      float v[kXferPanel];
      if (quarter_q(wq, jj)) {
        float p[4];
        xfer_weights<kSparse, kDim>(sm, s, jj, tid, R, CQ, p);
#pragma unroll
        for (int f = 0; f < kXferPanel; ++f)
          v[f] = fmaf(p[3], fa[f][3], fmaf(p[2], fa[f][2], fmaf(p[1], fa[f][1], p[0] * fa[f][0])));
      } else {
#pragma unroll
        for (int f = 0; f < kXferPanel; ++f) v[f] = 0.f;
      }
      butterfly_reduce<kXferPanel>(v, lane);  // lanes 2f and 2f + 1: the warp total of feature f
      if ((lane & 1) == 0) xs.red[buf][jj][warp][lane >> 1] = v[0];
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);
    named_bar_sync(1, kConsumers);
    if (warp == 0) {
      const int f = lane >> 1, j0 = (lane & 1) * 4;
      float t[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        t[k] = 0.f;
#pragma unroll
        for (int w = 0; w < kConsumers / 32; ++w) t[k] += xs.red[buf][j0 + k][w][f];
      }
      // segments begin at multiples of kColStage and only the last one of a list ends inside a stage: the positions past
      // the list's end hold zeros that no fold reads
      *reinterpret_cast<float4*>(out + (int64_t)f * nbb_pad + pb + j0) = make_float4(t[0], t[1], t[2], t[3]);
    }
  }
}

// per column: the row blocks' partials of one panel summed in fp64 in row-block order, found by list position with the
// keepmask / livemask / keepoff lookup of col_finalize; out[j][0 .. nf) of the [NBb][ldo] result
__global__ void __launch_bounds__(128)
transfer_col_fold_kernel(const float* __restrict__ part, const uint32_t* __restrict__ keepmask,
                         const uint32_t* __restrict__ livemask, const int2* __restrict__ keepoff, int kstride, int nrb,
                         int nbb_pad, int NBb, int nf, float* __restrict__ out, int64_t ldo) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= NBb) return;
  const int wd = j >> 5, bit = j & 31;
  const uint32_t below = (1u << bit) - 1u;
  double C[kXferPanel];
#pragma unroll
  for (int f = 0; f < kXferPanel; ++f) C[f] = 0.0;
  for (int rb = 0; rb < nrb; ++rb) {
    const int64_t w = (int64_t)rb * kstride + wd;
    const uint32_t bits = keepmask[w];
    if (((bits >> bit) & 1u) == 0u) continue;
    const uint32_t lbits = livemask[w];
    const int2 off = keepoff[w];
    const int pos = ((lbits >> bit) & 1u) ? off.x + __popc(lbits & below) : off.y + __popc(bits & ~lbits & below);
    const float* q = part + (int64_t)rb * kXferPanel * nbb_pad + pos;
#pragma unroll
    for (int f = 0; f < kXferPanel; ++f) C[f] += (double)q[(int64_t)f * nbb_pad];
  }
#pragma unroll
  for (int f = 0; f < kXferPanel; ++f)
    if (f < nf) out[(int64_t)j * ldo + f] = (float)C[f];
}

template <typename K>
int xfer_smem_opt_in(K kernel, bool (&attr_set)[SPB_MAX_DEVICES]) {
  const int dev_ = spb_current_device();
  if (attr_set[dev_]) return 0;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(XferSmem));
  if (e != cudaSuccess) return (int)e;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
  if (e != cudaSuccess) return (int)e;
  attr_set[dev_] = true;
  return 0;
}

template <bool SP, int DIM>
int launch_transfer_rows(const spb_em_params* p, const int32_t* gtb, const int32_t* fb, const float* FB, int64_t ldf,
                         float* part, cudaStream_t st) {
  static bool attr_set[SPB_MAX_DEVICES] = {};
  if (int rc = xfer_smem_opt_in(transfer_rows_kernel<SP, DIM>, attr_set)) return rc;
  transfer_rows_kernel<SP, DIM><<<dim3(p->ldx / kRowTile, p->seg2), kThreads, sizeof(XferSmem), st>>>(
      p->GT, p->ldx, gtb, fb, p->colconst, p->XAHat, p->lm, p->sc, FB, ldf, part, p->NBb, p->nbb_pad, p->collist,
      p->colquarters, p->colspatial, p->colcount);
  return 0;
}

template <bool SP, int DIM>
int launch_transfer_cols(const spb_em_params* p, const int32_t* gtb, const float* FA, float* part, cudaStream_t st) {
  static bool attr_set[SPB_MAX_DEVICES] = {};
  if (int rc = xfer_smem_opt_in(transfer_cols_kernel<SP, DIM>, attr_set)) return rc;
  transfer_cols_kernel<SP, DIM><<<dim3(p->ldx / kRowTile, p->seg1), kThreads, sizeof(XferSmem), st>>>(
      p->GT, p->ldx, gtb, p->colconst, p->XAHat, p->lm, p->sc, FA, part, p->NBb, p->nbb_pad, p->collist, p->colquarters,
      p->colspatial, p->colcount);
  return 0;
}

template <int DIM = 3>
int launch_sweep1(const spb_em_params* p, const int32_t* bidx, cudaStream_t st) {
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(estep_sweep1_kernel<DIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmemLayout));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(estep_sweep1_kernel<DIM>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  dim3 grid(p->ldx / kRowTile, p->seg1);
  estep_sweep1_kernel<DIM><<<grid, kThreads, sizeof(SmemLayout), st>>>(p->GT, p->ldx, bidx, p->colgeom, p->XAHat, p->lm, p->mm, p->sc,
                                                                      p->colpart, p->NBb, p->nbb_pad, p->collist, p->colquarters, p->colspatial, p->colcount,
                                                                      p->colsplit);
  return 0;
}

template <bool SP, int DIM = 3>
int launch_sweep2(const spb_em_params* p, const int32_t* bidx, cudaStream_t st) {
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(estep_sweep2_kernel<SP, DIM>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SmemLayout));
    if (e != cudaSuccess) return (int)e;
    e = cudaFuncSetAttribute(estep_sweep2_kernel<SP, DIM>, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  dim3 grid(p->ldx / kRowTile, p->seg2);
  estep_sweep2_kernel<SP, DIM><<<grid, kThreads, sizeof(SmemLayout), st>>>(p->GT, p->ldx, bidx, p->colconst, p->XAHat, p->lm, p->sc,
                                                                          p->rowpart, p->NBb, p->nbb_pad, p->collist, p->colquarters, p->colspatial, p->colcount,
                                                                          p->colsplit);
  return 0;
}

}  // namespace

// base of the SVI batch schedule [max_iter][NBb]; the kernels pick the row of the current iteration (sc->iter)
static inline const int32_t* batch_ptr(const spb_em_params* p, int /*iter*/) {
  return (p->svi && p->batch_idx) ? p->batch_idx : nullptr;
}
// schedule the GT readers index their rows by: none when GT holds this call's columns in list order (p->gt_by_position)
static inline const int32_t* gt_batch_ptr(const spb_em_params* p, int iter) {
  return p->gt_by_position ? nullptr : batch_ptr(p, iter);
}

extern "C" int spb_gather_cols(const spb_em_params* p, int32_t iter, void* stream) {
  gather_cols_kernel<<<(p->NBb + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p->xb4, batch_ptr(p, iter), p->sc, p->NBb, p->colgeom);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_estep_col_lists(const spb_em_params* p, void* stream) {
  const int nrb = p->ldx / kRowTile;
  block_bounds_kernel<<<nrb, kConsumers, 0, (cudaStream_t)stream>>>(p->XAHat, p->lm, p->ldx, p->NA, p->bbox);
  SPB_CHECK_LAUNCH();
  // sparse mode also records, per column, which row blocks can hold a non-zero weight (col_select skips the others)
  uint32_t* colmask = (p->sparse_k > 0 && nrb <= 32 * SPB_COLMASK_WORDS) ? p->colmask : nullptr;
  if (colmask) {
    cudaError_t e = cudaMemsetAsync(colmask, 0, sizeof(uint32_t) * SPB_COLMASK_WORDS * (size_t)p->nbb_pad, (cudaStream_t)stream);
    if (e != cudaSuccess) return (int)e;
  }
  const size_t smem = 2 * sizeof(uint32_t) * (size_t)((p->NBb + 31) / 32);
  if (smem > 200 * 1024) return SPB_EUNSUPPORTED;  // 800 k columns per iteration
  static bool attr_set[SPB_MAX_DEVICES] = {};
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(build_col_lists_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  const bool all_cols = !(p->svi && p->batch_idx);  // the iteration's columns are the fixed cells themselves, in order
  build_col_lists_kernel<<<nrb, kListThreads, smem, (cudaStream_t)stream>>>(
      p->bbox, all_cols ? p->xb4 : p->colgeom, all_cols ? 4 : 8, all_cols ? 1 : 2, p->NBb, p->sc, p->cull, p->collist,
      p->colquarters, p->colspatial, p->colcount, p->colsplit, p->nbb_pad, colmask, p->keepmask, p->livemask,
      reinterpret_cast<int2*>(p->keepoff), (p->nbb_pad + 31) / 32);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_estep_sweep1(const spb_em_params* p, int32_t iter, void* stream) {
  int rc;
  // writes the partial column sums of every (row block, listed column) combination by list position; col_finalize reads
  // exactly those (keepmask, livemask, keepoff)
  if (p->D == 2) rc = launch_sweep1<2>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  else rc = launch_sweep1<>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  if (rc) return rc;
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_col_finalize(const spb_em_params* p, void* stream) {
  col_finalize_kernel<<<(p->NBb + 31) / 32, 32 * kFinWarps, 0, (cudaStream_t)stream>>>(
      p->colpart, p->keepmask, p->livemask, reinterpret_cast<const int2*>(p->keepoff), (p->nbb_pad + 31) / 32, p->ldx / kRowTile, p->nbb_pad, p->NBb, p->colgeom, p->sc, p->colconst, p->K_NB);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_estep_sweep2(const spb_em_params* p, int32_t iter, void* stream) {
  int rc;
  if (p->sparse_k > 0 && p->D == 2) rc = launch_sweep2<true, 2>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  else if (p->sparse_k > 0) rc = launch_sweep2<true>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  else if (p->D == 2) rc = launch_sweep2<false, 2>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  else rc = launch_sweep2<false>(p, gt_batch_ptr(p, iter), (cudaStream_t)stream);
  if (rc) return rc;
  SPB_CHECK_LAUNCH();
  return 0;
}


extern "C" int spb_estep_col_select(const spb_em_params* p, int32_t iter, void* stream) {
  if (p->sparse_k <= 0) return SPB_EINVAL;
  const size_t smem = sizeof(uint32_t) * kSelBins + sizeof(float) * kSelBins + sizeof(float) * kSelCap;
  static bool attr_set[SPB_MAX_DEVICES] = {};  // the opt-in is per device (one process may drive several GPUs)
  const int dev_ = spb_current_device();
  if (!attr_set[dev_]) {
    cudaError_t e = cudaFuncSetAttribute(col_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return (int)e;
    attr_set[dev_] = true;
  }
  col_select_kernel<<<p->NBb, kSelThreads, smem, (cudaStream_t)stream>>>(p->GT, p->ldx, gt_batch_ptr(p, iter), p->colconst,
                                                                      p->XAHat, p->lm, p->sc, p->NA, p->sparse_k, p->K_NB,
                                                                      (p->cull && p->ldx / kRowTile <= 32 * SPB_COLMASK_WORDS) ? p->colmask : nullptr);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_sparse_P_emit(const spb_em_params* p, int32_t iter, int32_t* rows, float* vals, void* stream) {
  if (p->sparse_k <= 0) return SPB_EINVAL;
  col_emit_kernel<<<p->NBb, kSelThreads, 0, (cudaStream_t)stream>>>(p->GT, p->ldx, gt_batch_ptr(p, iter), p->colconst, p->XAHat,
                                                                    p->lm, p->sc, p->NA, p->sparse_k, rows, vals);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_posterior_argmax_mapped(const spb_em_params* p, int32_t iter, const int32_t* colmap, uint64_t* rowbest,
                                           uint64_t* colbest, void* stream) {
  cudaStream_t st = (cudaStream_t)stream;
  if (colbest) {
    col_argmax_kernel<<<p->NBb, kSelThreads, 0, st>>>(p->GT, p->ldx, gt_batch_ptr(p, iter), p->colconst, p->XAHat, p->lm,
                                                      p->sc, p->NA, (unsigned long long*)colbest);
    SPB_CHECK_LAUNCH();
  }
  if (rowbest) {
    cudaError_t e = cudaMemsetAsync(rowbest, 0, sizeof(uint64_t) * (size_t)p->NA, st);
    if (e != cudaSuccess) return (int)e;
    const int nrow = (p->NA + 255) / 256;
    int nseg = (spb_num_sms() * 8 + nrow - 1) / nrow;  // ~8 CTAs per SM
    nseg = nseg < 1 ? 1 : (nseg > p->NBb ? p->NBb : nseg);
    row_argmax_kernel<<<dim3(nrow, nseg), 256, 0, st>>>(p->GT, p->ldx, gt_batch_ptr(p, iter), p->colconst, p->XAHat, p->lm,
                                                        p->sc, p->NA, p->NBb, colmap, (unsigned long long*)rowbest);
    SPB_CHECK_LAUNCH();
  }
  return 0;
}


extern "C" int spb_row_finalize(const spb_em_params* p, void* stream) {
  if ((int64_t)((p->NA + 255) / 256) * 4 > p->red_scratch_doubles) return SPB_EINVAL;
  row_finalize_kernel<<<(p->NA + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      p->rowpart, p->seg2, p->ldx, p->NA, p->mm, p->K_NA_spatial, p->K_NA_sigma2, p->K_NA, p->PXB, p->sc, p->red_scratch,
      p->red_counter);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_row_fold(const spb_em_params* p, int32_t parity, void* stream) {
  if (p->rowstat == nullptr) return SPB_EINVAL;
  row_fold_kernel<<<(p->NA + 255) / 256, 256, 0, (cudaStream_t)stream>>>(p->rowpart, p->seg2, p->ldx, p->NA, p->fold_add,
                                                                          p->rowstat + (int64_t)(parity & 1) * 8 * p->ldx);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_row_stats_finalize(const spb_em_params* p, int32_t parity, void* stream) {
  if (p->rowstat == nullptr || (int64_t)((p->NA + 255) / 256) * 4 > p->red_scratch_doubles) return SPB_EINVAL;
  row_stats_finalize_kernel<<<(p->NA + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      p->rowstat + (int64_t)(parity & 1) * 8 * p->ldx, p->ldx, p->NA, p->mm, p->K_NA_spatial, p->K_NA_sigma2, p->K_NA, p->PXB,
      p->sc, p->red_scratch, p->red_counter);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_row_stats_p2p(const spb_em_params* p, int32_t parity, uint64_t epoch, void* stream) {
  if (p->peer_rowstat == nullptr || p->peer_flags == nullptr || p->shard_flags == nullptr || p->shard_world < 1 ||
      p->shard_world > 32 || (int64_t)((p->NA + 255) / 256) * 4 > p->red_scratch_doubles)
    return SPB_EINVAL;
  row_stats_p2p_kernel<<<(p->NA + 255) / 256, 256, 0, (cudaStream_t)stream>>>(
      p->peer_rowstat, parity & 1, p->shard_rank, p->shard_world, p->shard_flags, p->peer_flags, epoch, p->ldx, p->NA, p->mm,
      p->K_NA_spatial, p->K_NA_sigma2, p->K_NA, p->PXB, p->sc, p->red_scratch, p->red_counter);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_materialize_P(const spb_em_params* p, int32_t iter, float* P, int64_t ldp, void* stream) {
  dim3 grid((p->NA + 31) / 32, (p->NBb + 31) / 32), block(32, 8);
  materialize_P_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(p->GT, p->ldx, gt_batch_ptr(p, iter), p->colconst, p->XAHat,
                                                                p->lm, p->sc, p->NA, p->NBb, P, ldp);
  SPB_CHECK_LAUNCH();
  return 0;
}

extern "C" int spb_posterior_transfer_rows(const spb_em_params* p, int32_t iter, const float* FB, int64_t ldf, int32_t F,
                                           float* part, double* out, void* stream) {
  if (F < 1 || ldf < F || ldf % kXferPanel != 0 || FB == nullptr || part == nullptr || out == nullptr) return SPB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t* gtb = gt_batch_ptr(p, iter);
  const int32_t* fb = batch_ptr(p, iter);  // F_B rows are fixed cells (the rows of xb4), whatever the cost matrix's layout
  for (int f0 = 0; f0 < F; f0 += kXferPanel) {
    int rc;
    const float* panel = FB + f0;
    if (p->sparse_k > 0 && p->D == 2) rc = launch_transfer_rows<true, 2>(p, gtb, fb, panel, ldf, part, st);
    else if (p->sparse_k > 0) rc = launch_transfer_rows<true, 3>(p, gtb, fb, panel, ldf, part, st);
    else if (p->D == 2) rc = launch_transfer_rows<false, 2>(p, gtb, fb, panel, ldf, part, st);
    else rc = launch_transfer_rows<false, 3>(p, gtb, fb, panel, ldf, part, st);
    if (rc) return rc;
    SPB_CHECK_LAUNCH();
    transfer_row_fold_kernel<<<(p->NA + 255) / 256, 256, 0, st>>>(part, p->seg2, p->ldx, p->NA, p->fold_add,
                                                                   out + (int64_t)f0 * p->ldx);
    SPB_CHECK_LAUNCH();
  }
  return 0;
}

extern "C" int spb_posterior_transfer_cols(const spb_em_params* p, int32_t iter, const float* FA, int32_t F, float* part,
                                           float* out, int64_t ldo, void* stream) {
  if (F < 1 || ldo < F || FA == nullptr || part == nullptr || out == nullptr) return SPB_EINVAL;
  cudaStream_t st = (cudaStream_t)stream;
  const int32_t* gtb = gt_batch_ptr(p, iter);
  for (int f0 = 0; f0 < F; f0 += kXferPanel) {
    int rc;
    const float* panel = FA + (int64_t)f0 * p->ldx;
    if (p->sparse_k > 0 && p->D == 2) rc = launch_transfer_cols<true, 2>(p, gtb, panel, part, st);
    else if (p->sparse_k > 0) rc = launch_transfer_cols<true, 3>(p, gtb, panel, part, st);
    else if (p->D == 2) rc = launch_transfer_cols<false, 2>(p, gtb, panel, part, st);
    else rc = launch_transfer_cols<false, 3>(p, gtb, panel, part, st);
    if (rc) return rc;
    SPB_CHECK_LAUNCH();
    transfer_col_fold_kernel<<<(p->NBb + 127) / 128, 128, 0, st>>>(
        part, p->keepmask, p->livemask, reinterpret_cast<const int2*>(p->keepoff), (p->nbb_pad + 31) / 32,
        p->ldx / kRowTile, p->nbb_pad, p->NBb, F - f0 < kXferPanel ? F - f0 : kXferPanel, out + f0, ldo);
    SPB_CHECK_LAUNCH();
  }
  return 0;
}
