"""Read ceiling of the E-step sweeps: how fast can the sweeps' bulk-copy producer stream the cost matrix, by layout and column
order, with the real work lists of the benchmark pair?

Usage (one H100): python profiles/sweep_stream.py [--out DIR] [--reps N]
Builds a standalone CUDA source with nvcc in DIR (a temporary directory by default) and loads it with ctypes; nothing is
added to the library. Prints one JSON document (card, power limit, every figure below) and writes it to
DIR/sweep_stream.json.

The pair is ``bench.py``'s flagship workload (100k x 100k x 2000 genes, 3-D, full EM, K = 15). Its work lists (collist,
colquarters, colcount, colsplit) are taken from the real EM at iterations 0, 60 and 150. For each of them, read-only
producers are timed with CUDA events. They use the sweeps' grid, column segments, 3-stage ring of bulk copies (the live
512-byte quarters of 8 columns and each column's 32-byte record per stage) and consumer warps that do no math:
  (a) today's layout GT[N_B][ldx] and today's column order, no partial stores;
  (b) (a) plus sweep 1's former column-indexed partial stores: 32 scattered 4-byte stores per stage into [nrb][4][nbb_pad];
  (c) k-d ordered columns (``kd_order`` of the fixed cells, the lists re-sorted within their live / dead groups as the list
      builder would order them) and GT in row-block panels [nrb][N_B][512] (same bytes): one bulk copy per run of list
      entries that are adjacent columns with all four quarters live, otherwise one per run of live quarters as today;
  (d) a plain sequential read of the same number of bytes as (a).
Go / no-go for the panel layout: the summed time of (c) over the three iterations must be at least 8 % below that of (a).
"""

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CU = r"""
#include <cstdint>
constexpr int kRowTile = 512, kStage = 8, kStages = 3, kQuarter = 128, kConsumers = 128, kThreads = kConsumers + 32;
struct __align__(16) Smem {
  float tile[kStages][kStage][kRowTile];
  float cols[kStages][kStage][8];
  uint64_t full[kStages], empty[kStages];
};
__device__ __forceinline__ uint32_t su32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(su32(b)), "r"(c)); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* b, uint32_t n) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(su32(b)), "r"(n) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(su32(b)) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint64_t* b, uint32_t par) {
  uint32_t ok = 0;
  while (!ok)
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}\n"
                 : "=r"(ok) : "r"(su32(b)), "r"(par) : "memory");
}
__device__ __forceinline__ void bulk(void* d, const void* s, uint32_t n, uint64_t* b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(su32(d)), "l"(s), "r"(n), "r"(su32(b)) : "memory");
}

// panel = 0: GT[j][ldx] (row block i0 at column offset i0); panel = 1: GT[rb][ncols][512]
// store = 0: none; 1: sweep 1's former scattered partial stores colpart[(rb * 4 + v) * nbb_pad + list[pos]]
extern "C" __global__ void __launch_bounds__(kThreads, 4)
stream_kernel(const float* __restrict__ GT, long long ldx, int panel, int ncols, const int* __restrict__ collist,
              const unsigned char* __restrict__ colq, const int* __restrict__ colcount, int nbb_pad,
              const float* __restrict__ colgeom, int store, float* __restrict__ colpart, float* __restrict__ sink) {
  extern __shared__ __align__(128) unsigned char raw[];
  Smem& sm = *reinterpret_cast<Smem*>(raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, rb = blockIdx.x, seg = blockIdx.y;
  const int count = colcount[rb];
  int cps = (count + gridDim.y - 1) / gridDim.y;
  cps = ((cps + kStage - 1) / kStage) * kStage;
  const int begin = min(count, seg * cps), end = min(count, begin + cps);
  if (begin >= end) return;
  const int* list = collist + (long long)rb * nbb_pad;
  const unsigned char* qs = colq + (long long)rb * nbb_pad;
  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) { mbar_init(&sm.full[s], 1); mbar_init(&sm.empty[s], kConsumers / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const int nst = (end - begin + kStage - 1) / kStage;
  if (warp == kConsumers / 32) {  // producer
    for (int st = 0; st < nst; ++st) {
      const int s = st % kStages;
      if (st >= kStages) mbar_wait(&sm.empty[s], ((st / kStages) - 1) & 1);
      const int pb = begin + st * kStage;
      const bool slot = lane < kStage, live = slot && pb + lane < end;
      const uint32_t qm = live ? qs[pb + lane] : 0u;
      const int j = live ? list[pb + lane] : 0;
      const uint32_t total = __reduce_add_sync(0xffffffffu, slot ? __popc(qm) * kQuarter * 4 + 32 : 0u);
      // panel runs: slot l continues a run when it and slot l - 1 are full columns and adjacent
      const int jprev = __shfl_up_sync(0xffffffffu, j, 1);
      const uint32_t qprev = __shfl_up_sync(0xffffffffu, qm, 1);
      const bool full = panel && qm == 0xFu;
      const bool cont = full && lane > 0 && qprev == 0xFu && jprev + 1 == j;
      const uint32_t contb = __ballot_sync(0xffffffffu, cont);
      if (lane == 0) mbar_expect_tx(&sm.full[s], total);
      __syncwarp();
      if (slot) {
        if (full) {
          if (!cont) {
            int len = 1;
            while (lane + len < kStage && ((contb >> (lane + len)) & 1u)) ++len;
            const float* src = GT + ((long long)rb * ncols + j) * kRowTile;
            bulk(&sm.tile[s][lane][0], src, len * kRowTile * 4, &sm.full[s]);
          }
        } else if (qm != 0u) {
          const float* src = panel ? GT + ((long long)rb * ncols + j) * kRowTile : GT + (long long)j * ldx + (long long)rb * kRowTile;
          for (uint32_t m = qm; m != 0u;) {
            const int q0 = __ffs(m) - 1;
            const int len = __ffs(~(m >> q0)) - 1;
            bulk(&sm.tile[s][lane][q0 * kQuarter], src + q0 * kQuarter, len * kQuarter * 4, &sm.full[s]);
            m &= ~(((1u << len) - 1u) << q0);
          }
        }
        bulk(&sm.cols[s][lane][0], colgeom + (long long)j * 8, 32, &sm.full[s]);
      }
    }
    return;
  }
  float acc = 0.f;
  for (int st = 0; st < nst; ++st) {
    const int s = st % kStages;
    mbar_wait(&sm.full[s], (st / kStages) & 1);
    const int pb = begin + st * kStage;
    const float x = sm.tile[s][lane & 7][tid * 4];
    acc += x;
    __syncwarp();
    if (lane == 0) mbar_arrive(&sm.empty[s]);
    if (store == 1 && warp == 0) {
      const int v = lane / kStage, jj = lane % kStage;
      if (pb + jj < end) colpart[((long long)rb * 4 + v) * nbb_pad + list[pb + jj]] = x;
    }
  }
  if (acc == -1.f) sink[0] = acc;  // never true: keeps the shared-memory reads
}

extern "C" __global__ void read_kernel(const float4* __restrict__ p, long long n4, float* __restrict__ sink) {
  float acc = 0.f;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    const float4 v = p[i];
    acc += v.x + v.y + v.z + v.w;
  }
  if (acc == -1.f) sink[0] = acc;
}

extern "C" int launch_stream(const float* GT, long long ldx, int panel, int ncols, const int* collist, const unsigned char* colq,
                             const int* colcount, int nbb_pad, const float* colgeom, int store, float* colpart, float* sink,
                             int nrb, int seg, void* stream) {
  const int smem = (int)sizeof(Smem);
  static bool attr = false;
  if (!attr) {
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    cudaFuncSetAttribute(stream_kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
    attr = true;
  }
  stream_kernel<<<dim3(nrb, seg), kThreads, smem, (cudaStream_t)stream>>>(GT, ldx, panel, ncols, collist, colq, colcount, nbb_pad,
                                                                         colgeom, store, colpart, sink);
  return (int)cudaGetLastError();
}
extern "C" int launch_read(const float* p, long long bytes, float* sink, int blocks, void* stream) {
  read_kernel<<<blocks, 512, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(p), bytes / 16, sink);
  return (int)cudaGetLastError();
}
"""


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def build(out):
    src = os.path.join(out, "sweep_stream.cu")
    lib = os.path.join(out, "sweep_stream.so")
    with open(src, "w") as f:
        f.write(CU)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    subprocess.run([nvcc, "-shared", "-Xcompiler", "-fPIC", "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17",
                    "-o", lib, src], check=True)
    L = C.CDLL(lib)
    P, I, LL = C.c_void_p, C.c_int, C.c_longlong
    L.launch_stream.argtypes = [P, LL, I, I, P, P, P, I, P, I, P, P, I, I, P]
    L.launch_read.argtypes = [P, LL, P, I, P]
    return L


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--iters", default="0,60,150")
    args = ap.parse_args()
    out = args.out or tempfile.mkdtemp(prefix="sweep_stream_")
    os.makedirs(out, exist_ok=True)
    L = build(out)

    import torch

    import bench
    import spateo_release_b200 as st
    from spateo_release_b200 import _capi
    from spateo_release_b200.alignment.morpho_class import kd_order

    dev = torch.device("cuda:0")
    torch.cuda.set_device(dev)
    A, B = bench.make_pair_on_device(args.cells, args.genes, 3, seed=0, device=dev)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(sampleA=B, sampleB=A, SVI_mode=False, max_iter=200, K=15, nn_init=True, verbose=False,
                                 device="0", materialize_P=False, vecfld_key_added="vf")
    m.prepare()
    m.reset_state()
    stp = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    s, NB, ldx = m._state, m.NB, m.ldx
    nrb = ldx // _capi.ROW_TILE
    nbb_pad = int(m._params.nbb_pad)
    seg = int(m._params.seg1)
    assert m._GT.shape[0] == NB and not m._streamed
    # k-d order of the fixed cells: rank[j] = new index of column j
    perm = kd_order(np.asarray(m.coordsB))
    rank = torch.empty((NB,), dtype=torch.int64, device=dev)
    rank[torch.from_numpy(perm).to(dev)] = torch.arange(NB, device=dev)
    colgeom = torch.zeros((nbb_pad, 8), dtype=torch.float32, device=dev)
    colpart = torch.zeros((nrb, 4, nbb_pad), dtype=torch.float32, device=dev)
    sink = torch.zeros((4,), dtype=torch.float32, device=dev)
    GT = m._GT  # [N_B][ldx]; read as [nrb][N_B][512] for the panel layout (same bytes, contents do not matter here)

    def time_it(fn):
        fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ms.append(e0.elapsed_time(e1))
        return float(np.median(ms))

    results = []
    prev = 0
    for it in [int(x) for x in args.iters.split(",")]:
        if it > prev:
            m.run_em(n_iter=it - prev, start=prev)
        m._estep_only(it, stp)
        torch.cuda.synchronize()
        prev = it
        collist = s["collist"].clone()
        colq = s["colquarters"].clone()
        count = s["colcount"].clone()
        split = s["colsplit"].clone()
        pos = torch.arange(nbb_pad, device=dev)[None, :]
        listed = pos < count[:, None]
        # the list builder's order under k-d ordered columns: live group, then dead group, each by new column index
        key = torch.where(listed, (pos >= split[:, None]).long() * NB + rank[collist.long().clamp(0, NB - 1)],
                          torch.full_like(collist, 2 * NB + 1, dtype=torch.int64))
        order = torch.argsort(key, dim=1, stable=True)
        kd_list = torch.where(listed, rank[torch.gather(collist, 1, order).long().clamp(0, NB - 1)],
                              torch.zeros_like(collist, dtype=torch.int64)).int().contiguous()
        kd_q = torch.gather(colq, 1, order).contiguous()
        quarters = int(sum(bin(v).count("1") * c for v, c in enumerate(torch.bincount(
            torch.where(listed, colq.long(), 0).flatten(), minlength=16).tolist())))
        gt_bytes = quarters * 512

        def stream(lst, q, panel, store):
            return lambda: L.launch_stream(GT.data_ptr(), ldx, panel, NB, lst.data_ptr(), q.data_ptr(), count.data_ptr(), nbb_pad,
                                           colgeom.data_ptr(), store, colpart.data_ptr(), sink.data_ptr(), nrb, seg, stp)

        t = {
            "a_today": time_it(stream(collist, colq, 0, 0)),
            "b_today_scattered_stores": time_it(stream(collist, colq, 0, 1)),
            "c_kd_panels": time_it(stream(kd_list, kd_q, 1, 0)),
            "d_sequential": time_it(lambda: L.launch_read(GT.data_ptr(), gt_bytes, sink.data_ptr(), 132 * 8, stp)),
        }
        results.append(dict(iteration=it, visited_pair_fraction=quarters / (4.0 * nrb * NB), gt_bytes=gt_bytes,
                            ms=t, GBs={k: gt_bytes / (v * 1e-3) / 1e9 for k, v in t.items()}))
        print(json.dumps(results[-1]), file=sys.stderr, flush=True)

    ta = sum(r["ms"]["a_today"] for r in results)
    tc = sum(r["ms"]["c_kd_panels"] for r in results)
    doc = dict(card=card(), workload=f"bench pair {args.cells} x {args.cells} x {args.genes} genes, 3-D, full EM, K = 15",
               seg=seg, reps=args.reps, iterations=results,
               c_time_reduction_vs_a=1.0 - tc / ta, go_panel_layout=bool(tc <= 0.92 * ta))
    text = json.dumps(doc)
    print(text)
    with open(os.path.join(out, "sweep_stream.json"), "w") as f:
        f.write(text + "\n")


if __name__ == "__main__":
    main()
