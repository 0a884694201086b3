#!/usr/bin/env python
"""bench.py — cell-pairs/sec through the morpho_align EM loop (BASELINE.json metric) on an H100.

Workload (default, = BASELINE configs[1]): one synthetic 3-D slice pair per GPU, 100,000 x 100,000 cells, 2,000 genes,
KL dissimilarity, full EM (SVI_mode=False), K=15 inducing points, nn_init=True, max_iter=200. A *step* is one complete
200-iteration EM over one slice pair.

  value        = (N_A * N_B * max_iter * n_gpus) / (max-over-ranks device time of one step), cost matrix resident in HBM
                 (SURVEY.md 8(d): EM loop only), product defaults (exact zero-tile culling on).
  value_dense  = the same loop with culling off: every sweep launch reads all N_A x N_B pairs (the plain 8 B/pair figure).
  e2e          = the same pairs divided by the wall time of the PUBLIC call ``st.align.morpho_align([A, B], ...)`` on
                 plain (unpinned) host arrays: slice copies, constructor, coarse rigid + variational initialisation,
                 H2D of expression and coordinates, expression-cost precompute, the EM loop, closing similarity, D2H of
                 every result. ``e2e.device_only`` keeps the narrower figure (H2D + cost matrix + EM + D2H on a
                 pre-constructed solver with pinned inputs).
  roofline     = E-step sweep kernels: 4 B per cell pair per sweep (algorithmic) / CUDA-event time of each launch, against
                 MEASURED_PEAKS.json hbm_gbs; ``roofline_dense`` = the culling-off launches.
  cpu_baseline = the numpy oracle (port of the reference CPU path) on a bounded sample, host cores stated.

``--impl reference`` times the reference's CPU algorithm (oracle port of the pure-Python reference) on a bounded sample: ONE EM iteration of a 20,000 x 20,000 pair per step
(BASELINE.md section 4), W + K steps really executed; its ``config`` describes that sample.
Other workloads: ``--workload vfc`` (BASELINE configs[4]), ``--workload chain`` (configs[2], multi-GPU slice chain).
Multi-GPU (torchrun): one independent slice pair per rank (weak scaling) + ONE all-gather of the per-pair rigid
transforms per step for the chain composition.

``--dump-outputs DIR`` (pair workload): after the timed steps, the results of the last timed EM step as a caller of
``Morpho_pairwise`` receives them (aligned coordinates, rigid transforms, scalars, column / row sums), one
``DIR/<name>.npy`` each (float32 / float64, a few MB at the default size). The inputs are seeded, so two builds run with
the same arguments can be compared output for output.
"""

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--dim", type=int, default=3)
    ap.add_argument("--max-iter", type=int, default=200)
    ap.add_argument("--K", type=int, default=15)
    ap.add_argument("--svi", action="store_true", help="default SVI mode (batch = N_B/10) instead of the full EM")
    ap.add_argument("--e2e-steps", type=int, default=5)
    ap.add_argument("--cpu-cells", type=int, default=20000, help="cells per slice of the bounded CPU sample")
    ap.add_argument("--cpu-iters", type=int, default=1, help="EM iterations per step of the CPU sample")
    ap.add_argument("--cpu-baseline-steps", type=int, default=2, help="steps of the cpu_baseline leg of the b200 arm")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-secondary", action="store_true",
                    help="skip the secondary EM-loop timings (default SVI mode; K=200 inducing points) of SURVEY.md 8(d) config 2")
    ap.add_argument("--workload", default="pair", choices=["pair", "vfc", "chain", "shard"],
                    help="pair = BASELINE configs[1] (headline); vfc = configs[4] SparseVFC; chain = configs[2] (16-slice chain "
                         "sharded over the GPUs, torchrun); shard = ONE pair column-sharded over the GPUs (strong scaling)")
    ap.add_argument("--chain-slices", type=int, default=16)
    ap.add_argument("--chain-cells", type=int, default=50000)
    ap.add_argument("--vfc-cells", type=int, default=1000000)
    ap.add_argument("--vfc-M", type=int, default=500)
    ap.add_argument("--vfc-iters", type=int, default=50)
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the outputs of the last timed step as DIR/<name>.npy (pair workload)")
    args = ap.parse_args()
    if args.dump_outputs is not None and (args.impl != "b200" or args.workload != "pair"):
        ap.error("--dump-outputs is implemented for the default pair workload")
    return args


# results of Morpho_pairwise a caller reads after run(), in the caller's row order (P is not materialised in the timed path)
DUMP_KEYS = ("XAHat", "RnA", "VnA", "optimal_RnA", "R", "t", "optimal_R", "optimal_t", "sigma2", "gamma", "sigma2_variance",
             "K_NA", "K_NB")


def dump_outputs(m, out_dir):
    """Closes the solver's last EM run (D2H of the results, as ``run()`` does) and writes each result as <name>.npy."""
    m._finish()
    os.makedirs(out_dir, exist_ok=True)
    for key in DUMP_KEYS:
        a = np.asarray(getattr(m, key))
        a = a.astype(np.float64 if a.dtype == np.float64 else np.float32)
        np.save(os.path.join(out_dir, f"{key}.npy"), a)


# ---------------------------------------------------------------------------------------------------------------------
# synthetic data (SURVEY.md §8(d)) generated on the device, returned as plain host arrays
# ---------------------------------------------------------------------------------------------------------------------
def make_pair_on_device(n, G, dim, seed, device):
    import torch

    from spateo_release_b200.anndata_lite import AnnDataLite

    g = torch.Generator(device=device)
    g.manual_seed(1234 + seed)
    coords = torch.rand((n, dim), generator=g, device=device, dtype=torch.float64) * 100
    if dim == 3:
        coords[:, 2] *= 0.2  # a 20-unit thick 3-D slab
    W = torch.randn((dim, G), generator=g, device=device, dtype=torch.float64)
    phi = torch.rand((G,), generator=g, device=device, dtype=torch.float64) * 2 * np.pi

    def counts(c):
        lam = torch.exp(torch.sin(c @ W / 30.0 + phi)).float()
        return torch.poisson(lam, generator=g)

    expA = counts(coords)
    perm = torch.randperm(n, generator=g, device=device)
    base = coords[perm]
    expB = counts(base)
    th = 0.5
    R = torch.eye(dim, dtype=torch.float64, device=device)
    R[0, 0], R[0, 1], R[1, 0], R[1, 1] = np.cos(th), -np.sin(th), np.sin(th), np.cos(th)
    coordsB = base @ R.T + 5.0 + torch.randn((n, dim), generator=g, device=device, dtype=torch.float64) * 0.3

    import pandas as pd

    var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
    # plain (pageable) host arrays, as a user's AnnData holds them
    A = AnnDataLite(expA.cpu().numpy(), var=var.copy(), obsm={"spatial": coords.cpu().numpy()})
    B = AnnDataLite(expB.cpu().numpy(), var=var.copy(), obsm={"spatial": coordsB.cpu().numpy()})
    torch.cuda.synchronize()
    return A, B


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,"
             "clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,"
             "clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(
                ["nvidia-smi", f"--id={self.index}", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "200"],
                stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.thread = threading.Thread(target=self._read, daemon=True)
            self.thread.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=5)
        except Exception:
            pass
        sm, mx, pw, reasons = [], [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            f = [x.strip() for x in r.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0])); mx.append(float(f[1])); pw.append(float(f[2]))
            except ValueError:
                continue
            for nme, v in zip(names, f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(nme)
        if not sm:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["no samples"]}
        return {"sm_mhz": float(np.median(sm)), "sm_max_mhz": float(max(mx)), "power_w_max": float(max(pw)),
                "samples": len(sm), "reasons": sorted(reasons)}


# ---------------------------------------------------------------------------------------------------------------------
# CPU baseline: the oracle port of the reference's numpy path on a bounded sample
# ---------------------------------------------------------------------------------------------------------------------
def cpu_em_sample(n_cells, G, dim, iters, warm=0, steps=1):
    """Returns (pairs_per_sec, seconds_per_step, description, steps_executed). EM loop only, cost matrix precomputed (like
    `value`); every step runs ``iters`` further iterations of the same EM."""
    from oracle.morpho_oracle import MorphoPairOracle
    from spateo_release_b200.synthetic import make_slice_pair

    try:  # torchrun exports OMP_NUM_THREADS=1; the CPU arm is meant to use every host core
        from threadpoolctl import threadpool_limits

        threadpool_limits(limits=os.cpu_count())
    except Exception:
        pass

    (cA, eA), (cB, eB) = make_slice_pair(n_cells, n_cells, G, dim=dim, seed=0, as_anndata=False,
                                         z_thickness=20.0 if dim == 3 else None)
    np.random.seed(0)
    o = MorphoPairOracle(cB, cA, [eB], [eA], dtype="float32", SVI_mode=False, max_iter=iters * (warm + steps), K=15,
                         nn_init=False)
    o.prepare()
    times = []
    it = 0
    for s in range(warm + steps):
        t0 = time.perf_counter()
        for _ in range(iters):
            o.em_iteration(it)
            it += 1
        times.append(time.perf_counter() - t0)
    sec = float(np.mean(times[warm:]))
    pairs = float(n_cells) * n_cells * iters
    desc = (f"oracle port of Morpho_pairwise EM (float32 numpy as in the reference: BLAS calls threaded, element-wise passes "
            f"single-threaded; SVI off, nn_init off), {n_cells}x{n_cells} cells, {G} genes, {dim}-D, {iters} EM iteration(s) per "
            f"step, {warm}+{steps} steps executed, cost matrix precomputed")
    return pairs / sec, sec, desc, warm + steps


def reference_config(args):
    """What the reference arm really runs: a bounded sample of configs[1] (SURVEY.md 8(d) 'CPU baseline timing')."""
    return {
        "workload": f"bounded CPU sample of the morpho_align pair workload: 2 synthetic {args.dim}-D slices, {args.cpu_cells} cells "
                    f"each, {args.genes} genes, KL, full EM (SVI_mode=False), K=15, nn_init=False; one step = {args.cpu_iters} EM "
                    f"iteration(s) (the 100000-cell pair needs 7 live N x M fp32 temporaries = 280 GB in the reference's "
                    f"get_P_core and does not fit the host; pairs/s is size-independent to first order)",
        "cells_per_slice": args.cpu_cells, "genes": args.genes, "dim": args.dim, "em_iterations_per_step": args.cpu_iters,
        "K": 15, "svi": False, "nn_init": False, "sample_of": "BASELINE configs[1] (100000 cells per slice, 200 iterations)",
    }


def run_reference_arm(args):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return
    cores = os.cpu_count()
    v, sec, desc, executed = cpu_em_sample(args.cpu_cells, args.genes, args.dim, args.cpu_iters, warm=args.warmup,
                                           steps=args.steps)
    line = {
        "impl": "reference",
        "metric": "cell-pairs/sec through morpho_align EM", "value": v, "unit": "cell-pairs/s", "n_gpus": args.gpus,
        "steps": args.steps, "warmup": args.warmup, "steps_executed": executed, "ms_per_step": sec * 1e3,
        "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
        "config": reference_config(args),
        "cpu_baseline": {"value": v, "unit": "cell-pairs/s", "cores": cores, "kind": "port", "sample": desc},
        "e2e": {"value": v, "unit": "cell-pairs/s", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "note": "one CPU process on rank 0 regardless of --gpus: at N > 1 compare per GPU, not the N-GPU aggregate",
    }
    print(json.dumps(line), flush=True)


def workload_config(args):
    mode = "SVI(batch=N_B/10)" if args.svi else "full EM (SVI_mode=False)"
    return {
        "workload": f"morpho_align pair: 2 synthetic {args.dim}-D slices, {args.cells} cells each, {args.genes} genes, "
                    f"KL, {mode}, K={args.K}, nn_init=True, max_iter={args.max_iter}; one pair per GPU",
        "cells_per_slice": args.cells, "genes": args.genes, "dim": args.dim, "max_iter": args.max_iter, "K": args.K,
        "svi": bool(args.svi), "pairs_per_gpu": 1, "parallelism": "independent slice pair per GPU + 1 all-gather",
        "zero_tile_culling": "on (product default; exact: skipped pairs are 0 in fp32) — dense timings under roofline.dense",
        "cache": "inputs_larger_than_L2 (cost matrix %.1f GB per pair)" % (4.0 * args.cells * args.cells / 1e9),
    }


# ---------------------------------------------------------------------------------------------------------------------
def vfc_problem(n, M, D=3, seed=0):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 100, size=(n, D))
    c = X - 50.0
    V = np.zeros_like(X)
    V[:, 0], V[:, 1] = -0.05 * c[:, 1], 0.05 * c[:, 0]
    V += 2.0 * np.exp(-np.sum(c**2, 1, keepdims=True) / (2 * 15.0**2))
    V += rng.normal(0, 0.1, size=V.shape)
    k = n // 10
    V[:k] = rng.uniform(-5, 5, size=(k, D))
    ctrl = rng.permutation(n)[:M]
    return X, V, ctrl


def run_vfc(args):
    """BASELINE configs[4]: SparseVFC on 1M 3-D cells, 500 control points, 50 EM iterations, 1 GPU. Metric: cell x
    control-point pairs per second through the public ``SparseVFC`` call (host arrays in / host arrays out, so the line's
    ``value`` is end to end by construction). Roofline: the wgmma contraction of the normal equations, timed with CUDA
    events inside the call (``timings``), against the measured dense bf16 tensor peak."""
    import torch

    import __graft_entry__ as ge

    ge.build()
    from spateo_release_b200.tdr.sparsevfc import SparseVFC

    n, M, D = args.vfc_cells, args.vfc_M, 3
    X, V, ctrl = vfc_problem(n, M)
    beta = 1.0 / 20.0**2
    sampler = ClockSampler(0)
    from spateo_release_b200 import _capi

    lib = _capi.load_library()

    def arm(gram, n_warm, n_steps, clocks_on):
        times, tms, out = [], [], None
        launches0 = 0
        for s in range(n_warm + n_steps):
            if s == n_warm:
                launches0 = lib.spb_launch_count()
                if clocks_on:
                    sampler.start()
            tm = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = SparseVFC(X, V, Grid=None, M=M, beta=beta, lambda_=0.02, MaxIter=args.vfc_iters, ecr=0.0, ctrl_idx=ctrl,
                            device="0", timings=tm, gram=gram)
            torch.cuda.synchronize()
            if s >= n_warm:
                times.append(time.perf_counter() - t0)
                tms.append(tm)
        return dict(sec=float(np.mean(times)), tms=tms, out=out,
                    launches=int((lib.spb_launch_count() - launches0) // max(n_steps, 1)))

    # the product default (reference-accurate normal equations, fp64 products) is the headline; the opt-in tensor-core
    # contraction is measured beside it together with its deviation from the default's fit
    main = arm("fp64", args.warmup, args.steps, True)
    clocks = sampler.stop()
    tens = arm("tensor", 1, max(1, min(args.steps, 3)), False)
    out, sec, tms = main["out"], main["sec"], tens["tms"]
    iters = int(out["iteration"]) + 1
    units = float(n) * M * iters
    peaks = {}
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            peaks = json.load(f)
    except Exception:
        pass
    peak_tf = float(peaks.get("bf16_tflops_sustained", peaks.get("bf16_tflops", 989.0)))
    tc_ms = float(np.mean([t["gram_tc_ms"].mean() for t in tms])) if "gram_tc_ms" in tms[0] else None
    flop = 2.0 * n * M * (M + D)  # SURVEY 8(d): 2 N M^2 + 2 N M D per iteration (the symmetric half would be N M^2)
    k_out = n // 10
    dev_V = float(np.abs(tens["out"]["V"][k_out:] - out["V"][k_out:]).max() / np.abs(out["V"]).max())
    per_it = lambda T, k: float(np.mean([t[k].mean() for t in T]))
    roofline = None
    if tc_ms is not None:
        ach = flop / (tc_ms * 1e-3) / 1e12
        roofline = {
            "bound": "tensor", "kernel": "gram_tc_kernel (opt-in gram='tensor' arm)", "achieved": ach, "peak": peak_tf,
            "unit": "TFLOP/s", "frac": ach / peak_tf, "traffic": None,
            "peak_source": "MEASURED_PEAKS.json bf16_tflops_sustained (dense bf16)" if peaks else "H100 SXM data sheet, 989 TFLOP/s dense bf16",
            "definition": "algorithmic FLOP of one launch (2 N M (M + D): U^T P U and U^T P Y of one EM iteration) / mean "
                          "CUDA-event duration of spb_gram_tc (wgmma GEMM + 1% fp64 fold) inside the timed calls",
            "note": "TF32 peaks at half the bf16 rate and the fp32-accurate 3xTF32 split issues 3 MMAs per product: "
                    "the ceiling of this formulation is peak / 6; the kernel re-reads its operands (A 128-row and B 256-row "
                    "panels per output tile, 8 B per element as hi/lo fp32), which makes it HBM-bound at this shape",
            "operand_bytes_per_launch": float((6 * 128 + 4 * 256 + 4 * 16) * 8.0 * n),
            "per_iteration_ms": {k: per_it(tms, k) for k in ("estep_ms", "gram_prepare_ms", "gram_tc_ms", "solve_ms")},
        }
    fp64_gram_ms = per_it(main["tms"], "gram_ms")
    fp64_path = {
        "per_iteration_ms": {k: per_it(main["tms"], k) for k in ("estep_ms", "gram_ms", "solve_ms")},
        "gram_kernel": "weighted_gram_kernel (fp64 FMA, block upper triangle)",
        "gram_fp64_TFLOPs": float(n) * M * (M + 32) * 2 / (fp64_gram_ms * 1e-3) / 1e12,
        "fp64_peak_TFLOPs_nominal": 34.0, "eigh_fallbacks": int(main["tms"][-1].get("eigh_fallbacks", 0)),
    }
    tensor_arm = {
        "value": float(n) * M * (int(tens["out"]["iteration"]) + 1) / tens["sec"], "ms_per_step": tens["sec"] * 1e3,
        "iterations_run": int(tens["out"]["iteration"]) + 1, "sigma2": tens["out"]["sigma2"],
        "inlier_field_deviation_vs_default": dev_V,
        "note": "opt-in approximate arm: fp32-level normal equations + ridge above the noise floor (a smoother fit, not the "
                "reference solution); the deviation is max |V_tensor - V_default| over the inlier cells / max |V|",
    }
    cpu = None
    if not args.no_cpu_baseline:
        from oracle.morpho_oracle import sparse_vfc

        try:
            from threadpoolctl import threadpool_limits

            threadpool_limits(limits=os.cpu_count())
        except Exception:
            pass
        tt = []
        for mi in (1, 3):
            t0 = time.perf_counter()
            sparse_vfc(X, V, ctrl, beta, lambda_=0.02, MaxIter=mi, ecr=0.0)
            tt.append(time.perf_counter() - t0)
        per_it = max((tt[1] - tt[0]) / 2.0, 1e-9)
        cpu = {"value": float(n) * M / per_it, "unit": "pairs/s", "cores": os.cpu_count(), "kind": "port",
               "sample": f"float64 numpy restatement of dynamo's SparseVFC (parity unpinned), full size {n} x {M}: runs of 1 and "
                         f"3 EM iterations, per-iteration time from their difference ({per_it:.2f} s/iteration; one-off kernel "
                         f"matrix construction {tt[0] - per_it:.1f} s excluded)"}
    print(json.dumps({
        "metric": "cell x control-point pairs/sec through SparseVFC EM", "value": units / sec, "unit": "pairs/s",
        "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True,
        "scaling": "weak", "vs_baseline": None, "dtype": "f32 kernel matrix, f64 normal equations / solve / posterior",
        "data": "synthetic",
        "config": {"workload": f"SparseVFC: {n} 3-D cells, {M} control points, {iters} EM iterations (ecr=0), lambda=0.02, host "
                               "arrays in/out; parity unpinned vs dynamo (third-party, absent)",
                   "cache": "inputs_larger_than_L2 (kernel matrix 2 GB, split operands 8 GB)"},
        "clocks": clocks,
        "e2e": {"value": units / sec, "unit": "pairs/s", "h2d_bytes_per_step": int(n * D * 8 * 2),
                "d2h_bytes_per_step": int(n * (D + 1) * 8)},
        "gpu_launches": main["launches"],
        "roofline": roofline, "cpu_baseline": cpu, "fp64_path": fp64_path, "tensor_arm": tensor_arm,
        "iterations_run": iters, "sigma2": out["sigma2"],
    }), flush=True)


def make_chain_slice(k, n, G, device):
    """Slice k of a synthetic serial-section chain: the same 2-D tissue (smooth expression programmes) re-sampled with its own
    cells and counts, placed with its own pose (rotation 0.12 k rad, translation (3 k, -2 k)) plus 0.3 positional jitter."""
    import pandas as pd
    import torch

    from spateo_release_b200.anndata_lite import AnnDataLite

    g0 = torch.Generator(device=device)
    g0.manual_seed(4321)  # shared programmes
    W = torch.randn((2, G), generator=g0, device=device, dtype=torch.float64)
    phi = torch.rand((G,), generator=g0, device=device, dtype=torch.float64) * 2 * np.pi
    g = torch.Generator(device=device)
    g.manual_seed(1000 + k)
    base = torch.rand((n, 2), generator=g, device=device, dtype=torch.float64) * 100
    lam = torch.exp(torch.sin(base @ W / 30.0 + phi)).float()
    X = torch.poisson(lam, generator=g)
    th = 0.12 * k
    R = torch.tensor([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]], dtype=torch.float64, device=device)
    tvec = torch.tensor([3.0 * k, -2.0 * k], dtype=torch.float64, device=device)
    coords = base @ R.T + tvec + torch.randn((n, 2), generator=g, device=device, dtype=torch.float64) * 0.3
    var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
    ad = AnnDataLite(X.cpu().numpy(), var=var, obsm={"spatial": coords.cpu().numpy()})
    ad.uns["pose"] = (th, 3.0 * k, -2.0 * k)
    ad.uns["base"] = base.cpu().numpy()
    return ad


def run_chain(args):
    """BASELINE configs[2]: serial chain of ``--chain-slices`` 2-D slices x ``--chain-cells`` cells x ``--genes`` genes;
    consecutive pairs are independent problems sharded round-robin over the ranks (pair p -> rank p mod N), each rank
    software-pipelines its pairs (host preparation + H2D of the next pair under the EM of the current one), ONE NCCL
    all-gather of the 2-D similarities, prefix composition, every rank places its own slices.
    value = (pairs x N_A x N_B x iterations) / max-over-ranks wall time of the whole job, host arrays in / host arrays out."""
    import torch
    import torch.distributed as dist

    import __graft_entry__ as ge

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    import spateo_release_b200 as st
    from spateo_release_b200.alignment.distributed import align_chain_pipelined, shard_pairs

    S, n, G = args.chain_slices, args.chain_cells, args.genes
    n_pairs = S - 1
    mine = shard_pairs(n_pairs, rank, world)
    need = sorted({q for p in mine for q in (p, p + 1)})
    slices = {k: make_chain_slice(k, n, G, dev) for k in need}  # untimed: stands for the slices on this rank's disk
    torch.cuda.empty_cache()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    kw = dict(SVI_mode=bool(args.svi), max_iter=args.max_iter, K=args.K, nn_init=True, verbose=False)
    times, stats = [], {}
    sampler = ClockSampler(local_rank)
    n_run = args.warmup + args.steps
    for s in range(n_run):
        for ad in slices.values():
            ad.obsm.pop("align_spatial", None)
        if s == args.warmup:
            sampler.start()
        barrier()
        t0 = time.perf_counter()
        np.random.seed(rank)
        stats = {}
        placed, tr = align_chain_pipelined(lambda k: slices[k], S, device=str(local_rank), stats=stats, **kw)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if s >= args.warmup:
            times.append(max_over_ranks(dt))
    clocks = sampler.stop()
    # sanity: every placed slice lands on the frame of slice 0 (residual against the common tissue coordinates)
    res = 0.0
    for k, ad in placed.items():
        want = ad.uns["base"]  # slice 0 carries the identity pose: its frame is the tissue's own
        res = max(res, float(np.sqrt(np.mean(np.sum((np.asarray(ad.obsm["align_spatial"]) - want) ** 2, axis=1)))))
    res = max_over_ranks(res)
    sec = float(np.mean(times))
    pairs_per_iter = float(n) * (args.chain_cells // 10 if args.svi else n)
    total = float(n_pairs) * pairs_per_iter * args.max_iter
    busiest = max(len(shard_pairs(n_pairs, r, world)) for r in range(world))
    if rank == 0:
        print(json.dumps({
            "metric": "cell-pairs/sec through morpho_align EM (slice chain)", "value": total / sec, "unit": "cell-pairs/s",
            "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": sec * 1e3, "higher_is_better": True,
            "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"chain of {S} 2-D slices x {n} cells x {G} genes = {n_pairs} independent pairs (KL, "
                                   f"{'SVI' if args.svi else 'full EM'}, K={args.K}, max_iter={args.max_iter}) round-robin over "
                                   f"{world} GPU(s), next pair prepared under the current pair's EM, 1 all-gather, prefix composition",
                       "pairs_on_busiest_gpu": busiest, "load_balance_ceiling": n_pairs / float(busiest * world),
                       "cache": "inputs_larger_than_L2 (cost matrix %.1f GB per pair)" % (4.0 * n * n / 1e9)},
            "clocks": clocks,
            "e2e": {"value": total / sec, "unit": "cell-pairs/s", "h2d_bytes_per_step": int(busiest * 2 * n * G * 4),
                    "d2h_bytes_per_step": int(busiest * n * 2 * 4 * 4),
                    "note": "value is end to end by construction: host arrays in, placed coordinates out, per rank"},
            "gpu_launches": int(stats.get("kernel_launches", 0)),
            "chain": {"seconds_per_pair_rank0": stats.get("seconds_per_pair"), "rms_residual_vs_truth": res,
                      "pairs": n_pairs, "pairs_rank0": stats.get("pairs")},
        }), flush=True)
    if world > 1:
        dist.destroy_process_group()


def run_shard(args):
    """ONE slice pair (BASELINE configs[1] shape) column-sharded over the ranks: strong scaling of a single alignment. Every
    rank holds the moving slice and N_B / world fixed cells; per iteration the only exchange is the sum of 7 fp64 row
    statistics per moving cell, done inside the row-finalize kernel over NVLink peer memory (mode p2p) or by ncclAllReduce.
    value = N_A x N_B x iterations / max-over-ranks device time of the EM loop (cost matrix blocks resident)."""
    import torch
    import torch.distributed as dist

    import __graft_entry__ as ge

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    from spateo_release_b200.alignment.distributed import morpho_align_pair_sharded

    A, B = make_pair_on_device(args.cells, args.genes, args.dim, seed=0, device=dev)  # the SAME pair on every rank
    torch.cuda.empty_cache()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    results = {}
    clocks = None
    for mode in (["p2p", "nccl"] if world > 1 else ["nccl"]):
        np.random.seed(0)
        t0 = time.perf_counter()
        try:
            m = morpho_align_pair_sharded(A, B, mode=mode, device=str(local_rank), max_iter=args.max_iter, K=args.K, nn_init=True,
                                          verbose=False)
        except Exception as e:  # symmetric memory unavailable: report and continue with the collective
            results[mode] = {"unavailable": repr(e)[:300]}
            continue
        barrier()
        t_prep = time.perf_counter() - t0
        ms = []
        sampler = ClockSampler(local_rank) if clocks is None else None  # clocks are sampled during the first mode's timed steps
        for s in range(args.warmup + args.steps):
            m.reset_state()
            if s == args.warmup and sampler is not None:
                sampler.start()
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m.run_em()
            e1.record()
            barrier()
            if s >= args.warmup:
                ms.append(max_over_ranks(e0.elapsed_time(e1)))
        if sampler is not None:
            clocks = sampler.stop()
        m._finish()
        results[mode] = {"ms_per_step": float(np.mean(ms)), "mode_used": m._shard_mode, "prepare_s": max_over_ranks(t_prep),
                         "sigma2_final": float(m.sigma2), "checksum_XAHat": float(np.abs(m.XAHat).sum())}
        del m
        torch.cuda.empty_cache()
    if rank == 0:
        best = min((v for v in results.values() if "ms_per_step" in v), key=lambda v: v["ms_per_step"])
        pairs = float(args.cells) * args.cells * args.max_iter
        print(json.dumps({
            "metric": "cell-pairs/sec through morpho_align EM (one pair, column-sharded)", "value": pairs / (best["ms_per_step"] * 1e-3),
            "unit": "cell-pairs/s", "n_gpus": world, "steps": args.steps, "warmup": args.warmup, "ms_per_step": best["ms_per_step"],
            "higher_is_better": True, "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": {"workload": f"ONE morpho_align pair, {args.cells} x {args.cells} cells, {args.genes} genes, {args.dim}-D, full "
                                   f"EM, K={args.K}, max_iter={args.max_iter}; fixed cells split over {world} GPU(s), row statistics "
                                   "summed once per iteration (7 fp64 per moving cell)",
                       "cache": "inputs_larger_than_L2 (cost-matrix block %.1f GB per GPU)" % (4.0 * args.cells * args.cells / world / 1e9)},
            "clocks": clocks, "modes": results,
            "e2e": None, "gpu_launches": None,
        }), flush=True)
    if world > 1:
        dist.destroy_process_group()


def main():
    args = parse_args()
    if args.impl == "reference":
        run_reference_arm(args)
        return
    if args.workload == "vfc":
        run_vfc(args)
        return
    if args.workload == "chain":
        run_chain(args)
        return
    if args.workload == "shard":
        run_shard(args)
        return
    import torch
    import torch.distributed as dist

    import __graft_entry__ as ge

    rank = int(os.environ.get("RANK", "0"))
    local_rank = int(os.environ.get("LOCAL_RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(local_rank)
    dev = torch.device("cuda", local_rank)
    if world > 1:
        dist.init_process_group("nccl", device_id=dev)
    if rank == 0:
        ge.build()
    if world > 1:
        dist.barrier()
    import spateo_release_b200 as st
    from spateo_release_b200 import _capi

    lib = _capi.load_library()

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()

    def max_over_ranks(x):
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        if world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---- data + host-side preparation (untimed: preprocessing / coarse init are reported separately) ----
    t0 = time.perf_counter()
    A, B = make_pair_on_device(args.cells, args.genes, args.dim, seed=rank, device=dev)
    t_data = time.perf_counter() - t0
    np.random.seed(rank)
    t0 = time.perf_counter()
    m = st.align.Morpho_pairwise(
        sampleA=B, sampleB=A, SVI_mode=bool(args.svi), max_iter=args.max_iter, K=args.K, nn_init=True, verbose=False,
        device=str(local_rank), materialize_P=False, vecfld_key_added="vf",
    )
    t_pre = time.perf_counter() - t0
    t0 = time.perf_counter()
    m.prepare_host()
    torch.cuda.synchronize()
    t_init = time.perf_counter() - t0
    m.pin_inputs()

    NA, NB = m.NA, m.NB
    cols = m.batch_size if args.svi else NB
    pairs_per_step = float(NA) * cols * args.max_iter

    gathered = [torch.zeros(12, dtype=torch.float64, device=dev) for _ in range(world)]

    def consensus_step():
        """closing similarity of this rank's pair + ONE all-gather + serial chain composition (morpho_alignment.py:300)"""
        import ctypes as C

        _capi.check(lib.spb_optimal_rigid(C.byref(m._params), _capi.ptr(m._state["optimal"]), _capi.current_stream_ptr()), "opt")
        if world > 1:
            dist.all_gather(gathered, m._state["optimal"])
        else:
            gathered[0].copy_(m._state["optimal"])

    # ---- end-to-end arm 1: the PUBLIC call on plain host arrays (what a user of the reference types) ----
    from spateo_release_b200.alignment import morpho_class as _mc

    def public_call():
        np.random.seed(rank)
        aligned, pis = st.align.morpho_align(
            [A, B], device=str(local_rank), verbose=False, SVI_mode=bool(args.svi), max_iter=args.max_iter, K=args.K,
            nn_init=True, mode="SN-N", materialize_P=False, iter_key_added=None,
        )
        vf = aligned[1].uns["VecFld_morpho"]
        mine = torch.zeros(12, dtype=torch.float64)
        D_ = vf["optimal_R"].shape[0]
        mine[:9].view(3, 3)[:D_, :D_] = torch.from_numpy(np.asarray(vf["optimal_R"], dtype=np.float64))
        mine[9:9 + D_] = torch.from_numpy(np.asarray(vf["optimal_t"], dtype=np.float64).reshape(-1))
        mine = mine.to(dev)
        if world > 1:  # the chain's single exchange: every pair's closing similarity
            dist.all_gather(gathered, mine)
        else:
            gathered[0].copy_(mine)
        res = np.asarray(aligned[1].obsm["align_spatial"])  # host numpy: the result the caller reads
        assert np.isfinite(res).all()
        return res

    pub_times = []
    pub_h2d = pub_d2h = 0
    m.__dict__.pop("_GT", None)
    m.__dict__.pop("_state", None)
    torch.cuda.empty_cache()
    for s in range(1 + max(args.e2e_steps, 1)):
        _mc.TRANSFER_BYTES["h2d"] = _mc.TRANSFER_BYTES["d2h"] = 0
        torch.cuda.empty_cache()
        barrier()
        t0 = time.perf_counter()
        public_call()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if s >= 1:
            pub_times.append(max_over_ranks(dt))
        pub_h2d, pub_d2h = _mc.TRANSFER_BYTES["h2d"], _mc.TRANSFER_BYTES["d2h"]
    pub_sec = float(np.mean(pub_times))
    torch.cuda.empty_cache()

    # ---- end-to-end arm 2 (narrower, kept for continuity): pre-constructed solver, pinned inputs ----
    e2e_times = []
    h2d = d2h = 0
    for s in range(1 + 2):
        m._prepared = False
        m.__dict__.pop("_GT", None)
        m.__dict__.pop("_state", None)
        torch.cuda.empty_cache()
        m._h2d_bytes = 0
        barrier()
        t0 = time.perf_counter()
        m.prepare_device()          # H2D expression + coords, cost matrix, state
        m.run_em()
        consensus_step()
        m._finish()                 # closing similarity, D2H of coordinates / vectors / scalars
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        if s >= 1:
            e2e_times.append(max_over_ranks(dt))
        h2d = m._h2d_bytes + (NA + NB) * m.D * 4
        d2h = NA * m.D * 4 * 3 + NA * 4 * 5 + cols * 4 + 12 * 8 + 264
        m.SVI_mode = bool(args.svi)
    e2e_sec = float(np.mean(e2e_times))

    # ---- device-resident arms: EM loop only, cost matrix in HBM ----
    # (1) product default: exact zero-tile culling on; (2) dense sweeps (culling off) for the plain 8 B/pair roofline
    def timed_arm(cull, n_warm, n_steps, sample_clocks, events=False):
        """events=False: the product path (iterations replayed from CUDA graphs) -> step times; events=True: the same launch
        sequence enqueued kernel by kernel with CUDA events around the two sweeps of every iteration -> roofline."""
        m.cull_zero_tiles = cull
        sampler = ClockSampler(local_rank)
        step_ms, sweep_ms, visited = [], [], []
        launches0 = 0
        replayed0 = 0
        for s in range(n_warm + n_steps):
            m.reset_state()
            ev = []
            if s == n_warm:
                barrier()
                if sample_clocks:
                    sampler.start()
                launches0 = lib.spb_launch_count()
                replayed0 = getattr(m, "graph_replayed_launches", 0)
            barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            m.run_em(sweep_events=ev if events else None)
            consensus_step()
            e1.record()
            barrier()
            if s >= n_warm:
                step_ms.append(max_over_ranks(e0.elapsed_time(e1)))
                sweep_ms.append([(a.elapsed_time(b), c.elapsed_time(d)) for (a, b, c, d) in ev])
                visited.append(m._state["trace_buf"][:, 7].cpu().numpy().copy())
        # kernels enqueued directly + kernels inside replayed CUDA graphs (counted per captured graph x replays)
        launches = (lib.spb_launch_count() - launches0) + (getattr(m, "graph_replayed_launches", 0) - replayed0)
        clocks = sampler.stop() if sample_clocks else None
        return dict(ms=float(np.mean(step_ms)), sweeps=np.array(sweep_ms, dtype=np.float64), visited=np.array(visited),
                    launches=int(launches), clocks=clocks)

    main_arm = timed_arm(True, args.warmup, args.steps, True)
    if args.dump_outputs is not None and rank == 0:
        dump_outputs(m, args.dump_outputs)
    main_ev = timed_arm(True, 0, max(1, min(args.steps, 2)), False, events=True)   # per-launch sweep timings, same workload
    dense_arm = timed_arm(False, min(args.warmup, 1), max(1, min(args.steps, 2)), False)
    dense_ev = timed_arm(False, 0, 1, False, events=True)
    m.cull_zero_tiles = True
    ms_per_step = main_arm["ms"]
    launches, clocks = main_arm["launches"], main_arm["clocks"]
    value = pairs_per_step * world / (ms_per_step * 1e-3)

    # ---- roofline of the dominant kernels (live CUDA-event timings of every launch in the timed region) ----
    peaks = {}
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            peaks = json.load(f)
    except Exception:
        pass
    peak_gbs = float(peaks.get("hbm_gbs", 3350.0))
    nrb = m.ldx // _capi.ROW_TILE
    tiles_all = float(nrb) * cols
    # algorithmic bytes of one sweep launch = 4 B x (cell pairs the launch has to read): all pairs when dense, the visited
    # (row block x column) tiles x N_A/nrb rows when culling skipped the provably-zero tiles
    sw = main_ev["sweeps"]                                      # [steps, iters, 2] ms
    vis = main_ev["visited"]                                    # [steps, iters] tiles
    bytes_per_launch = 4.0 * vis * (float(NA) / nrb)            # [steps, iters]
    s1_gbs = float(bytes_per_launch.sum() / (sw[..., 0].sum() * 1e-3) / 1e9)
    s2_gbs = float(bytes_per_launch.sum() / (sw[..., 1].sum() * 1e-3) / 1e9)
    dom = "estep_sweep2_kernel" if sw[..., 1].sum() >= sw[..., 0].sum() else "estep_sweep1_kernel"
    dom_gbs = min(s1_gbs, s2_gbs)
    dsw = dense_ev["sweeps"].reshape(-1, 2)
    d1, d2 = float(dsw[:, 0].mean()), float(dsw[:, 1].mean())
    alg_dense = 4.0 * NA * cols
    roofline = {
        "bound": "hbm", "kernel": dom, "achieved": dom_gbs, "peak": peak_gbs, "unit": "GB/s", "frac": dom_gbs / peak_gbs,
        "peak_source": "MEASURED_PEAKS.json hbm_gbs" if "hbm_gbs" in peaks else "H100 SXM data sheet, 3350 GB/s",
        "definition": "sum over the launches of 4 B x cell pairs the launch must read (visited tiles) / sum of CUDA-event "
                      "launch durations; the events are recorded in extra steps of the same workload right after the timed "
                      "ones, kernel by kernel (the timed steps replay whole iterations from CUDA graphs, which leaves no "
                      "room for events between kernels); ms_per_step_with_events shows the two agree",
        "ms_per_step_with_events": main_ev["ms"],
        "sweep1_GBs": s1_gbs, "sweep2_GBs": s2_gbs,
        "visited_pair_fraction": float(vis.sum() / (tiles_all * vis.size)),
        "sweeps_share_of_step": float(sw.sum() / sw.shape[0] / main_ev["ms"]),
        # where the time goes over the run: mean (sweep 1, sweep 2) ms per iteration and visited fraction per quarter
        "by_quarter": [
            {"iterations": f"{a}-{b - 1}", "sweep1_ms": float(sw[:, a:b, 0].mean()), "sweep2_ms": float(sw[:, a:b, 1].mean()),
             "visited_pair_fraction": float(vis[:, a:b].mean() / tiles_all)}
            for a, b in ((q * sw.shape[1] // 4, (q + 1) * sw.shape[1] // 4) for q in range(4)) if b > a
        ],
        "dense": {
            "note": "same kernels with culling off: every launch reads all N_A x N_B pairs (4 B each)",
            "value": pairs_per_step * world / (dense_arm["ms"] * 1e-3), "ms_per_step": dense_arm["ms"],
            "sweep1_ms": d1, "sweep2_ms": d2, "sweep1_GBs": alg_dense / (d1 * 1e-3) / 1e9,
            "sweep2_GBs": alg_dense / (d2 * 1e-3) / 1e9, "frac": alg_dense / (max(d1, d2) * 1e-3) / 1e9 / peak_gbs,
            "em_loop_GBs_8B_per_pair": 8.0 * pairs_per_step / (dense_arm["ms"] * 1e-3) / 1e9,
        },
    }

    # ---- secondary configurations of config 2 (SURVEY.md 8(d)): default SVI mode and K = 200, EM loop only, 1 step each ----
    secondary = None
    if world == 1 and not args.no_secondary and not args.svi:
        secondary = {}
        sig_final, gam_final = float(m.sigma2), float(m.gamma)
        m.__dict__.pop("_GT", None)
        m.__dict__.pop("_state", None)
        torch.cuda.empty_cache()
        for tag, kw in (("svi_default_batch", dict(SVI_mode=True, K=args.K)),
                        ("svi_default_batch_one_iteration_per_graph", dict(SVI_mode=True, K=args.K)),
                        ("full_em_K200", dict(SVI_mode=False, K=200)), ("full_em_K500", dict(SVI_mode=False, K=500))):
            np.random.seed(rank)
            m2 = st.align.Morpho_pairwise(sampleA=B, sampleB=A, max_iter=args.max_iter, nn_init=True, verbose=False,
                                          device=str(local_rank), materialize_P=False, **kw)
            if tag.endswith("one_iteration_per_graph"):
                m2.graph_unroll = 1  # A/B of the product default (8 light iterations per captured graph)
            m2.prepare()
            cols2 = m2.batch_size if m2.SVI_mode else NB
            ms2 = []
            for srep in range(2):
                m2.reset_state()
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                m2.run_em()
                e1.record()
                torch.cuda.synchronize()
                ms2.append(e0.elapsed_time(e1))
            secondary[tag] = {"value": float(NA) * cols2 * args.max_iter / (ms2[-1] * 1e-3), "unit": "cell-pairs/s",
                              "ms_per_step": ms2[-1], "columns_per_iteration": int(cols2), "K": int(m2.K),
                              "iterations_per_graph": int(m2._graph_unroll()),
                              "note": "EM loop only, device-resident, second of two runs"}
            del m2
            torch.cuda.empty_cache()
    else:
        sig_final, gam_final = float(m.sigma2), float(m.gamma)

    if rank == 0:
        cpu = None
        if world == 1 and not args.no_cpu_baseline:
            v, sec, desc, _n = cpu_em_sample(args.cpu_cells, args.genes, args.dim, args.cpu_iters, warm=0,
                                             steps=args.cpu_baseline_steps)
            cpu = {"value": v, "unit": "cell-pairs/s", "cores": os.cpu_count(), "kind": "port", "sample": desc,
                   "seconds_per_step": sec}
        line = {
            "metric": "cell-pairs/sec through morpho_align EM", "value": value, "unit": "cell-pairs/s", "n_gpus": world,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": ms_per_step, "higher_is_better": True,
            "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic",
            "config": workload_config(args),
            "clocks": clocks,
            "value_dense": roofline["dense"]["value"],
            "e2e": {"value": pairs_per_step * world / pub_sec, "unit": "cell-pairs/s", "h2d_bytes_per_step": int(pub_h2d),
                    "d2h_bytes_per_step": int(pub_d2h), "seconds_per_step": pub_sec, "steps": len(pub_times),
                    "call": "st.align.morpho_align([A, B], device=..., SVI_mode=False, max_iter=200, K=15, nn_init=True, "
                            "mode='SN-N', materialize_P=False, iter_key_added=None) on plain (pageable) host arrays",
                    "includes": "slice copies, Morpho_pairwise constructor (gene intersection, dense extraction, "
                                "normalisation, inducing kernel), coarse rigid + variational initialisation, H2D of "
                                "expression and coordinates, expression-cost precompute, EM loop, closing similarity, "
                                "all-gather, D2H of the aligned coordinates and vectors",
                    "device_only": {"value": pairs_per_step * world / e2e_sec, "seconds_per_step": e2e_sec,
                                    "steps": len(e2e_times), "h2d_bytes_per_step": int(h2d), "d2h_bytes_per_step": int(d2h),
                                    "includes": "pre-constructed solver, pinned inputs: H2D, expression-cost precompute, "
                                                "EM loop, closing similarity, all-gather, D2H of results"}},
            "roofline_dense": roofline["dense"],
            "gpu_launches": int(launches),
            "roofline": roofline,
            "cpu_baseline": cpu,
            "aux": {"datagen_s": t_data, "construct_s": t_pre, "coarse_and_variational_init_s": t_init, "init_breakdown": getattr(m, "_timing", None),
                    "sigma2_final": sig_final, "gamma_final": gam_final, "secondary": secondary,
                    "chain_transforms_gathered": world},
        }
        print(json.dumps(line), flush=True)
    if world > 1:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
