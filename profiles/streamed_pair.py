"""Streamed cost matrix: resident vs streamed runs of the 100k-cell pair, and the 160k-cell pair that only fits streamed.

Usage (one H100): python profiles/streamed_pair.py [--out DIR] [--skip-160k]
Prints one JSON document (card, power limit, every figure below); with --out it is also written to DIR/streamed_pair.json.

  100k x 100k x 2000 genes, 3-D: default SVI (200 iterations) and the full EM (--full-iters iterations), resident and
      forced-streamed (one chunk of the SVI batch; the widest chunk the card takes for the full EM), alternating. Seconds per
      alignment (``run()`` after the host preparation), ms per iteration split into cost-kernel and E-step / M-step time
      (CUDA events), and the largest output difference between the two.
  160k x 160k x 2000 genes, 3-D: default SVI through ``st.align.morpho_align`` (total time, peak allocated memory, plan),
      and the full EM for --full-iters-160k iterations (ms per iteration).
Streaming of the 100k pair is forced by patching ``morpho_class._device_budget``.
"""

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make_pair(n, genes=2000, seed=0):
    from spateo_release_b200.synthetic import make_slice_pair

    return make_slice_pair(n, n, genes, dim=3, seed=seed, z_thickness=20.0)


def solver(A, B, **kw):
    import spateo_release_b200 as st

    np.random.seed(0)
    return st.align.Morpho_pairwise(sampleA=B, sampleB=A, device="0", verbose=False, materialize_P=False, nn_init=False, **kw)


def timed_run(m, streamed_width=None):
    """prepare + run with events; returns (outputs, figures)."""
    import torch

    from spateo_release_b200.alignment import morpho_class as mc
    from spateo_release_b200.alignment.distributed import pair_device_bytes

    saved = mc._device_budget
    if streamed_width is not None:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        budget = pair_device_bytes(m.NA, m.NB, m._cost_features(), chunk_cols=streamed_width, n_sms=sms)
        mc._device_budget = lambda dev: budget
    try:
        m.prepare_host()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        m.prepare_device()
        torch.cuda.synchronize()
        t_prep = time.perf_counter() - t0
    finally:
        mc._device_budget = saved
    if m._streamed:
        m.cost_events = []
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    m.run()
    e1.record()
    torch.cuda.synchronize()
    t_run = time.perf_counter() - t0
    iters = max(m.max_iter, 1)
    em_ms = e0.elapsed_time(e1)
    cost_ms = sum(a.elapsed_time(b) for a, b in (getattr(m, "cost_events", None) or []))
    out = {k: np.asarray(getattr(m, k)) for k in ("XAHat", "optimal_RnA", "R", "t", "sigma2", "gamma", "K_NA", "K_NB")}
    fig = dict(plan=m.cost_plan.mode, chunks=m.cost_plan.n_chunks, width=m.cost_plan.width, prepare_device_s=round(t_prep, 3),
               run_s=round(t_run, 3), ms_per_iter=round(em_ms / iters, 3), cost_ms_per_iter=round(cost_ms / iters, 3),
               estep_mstep_ms_per_iter=round((em_ms - cost_ms) / iters, 3))
    return out, fig


def max_diff(a, b):
    return {k: float(np.abs(a[k].astype(np.float64) - b[k].astype(np.float64)).max()) for k in a}


def compare_100k(A, B, svi, iters, reps, widest):
    import torch

    res = {"resident": [], "streamed": []}
    diffs, identical = [], []
    for r in range(reps):
        outs = {}
        for mode in ("resident", "streamed"):
            kw = dict(SVI_mode=svi, max_iter=iters, K=15)
            m = solver(A, B, **kw)
            width = (min(max(int(m.NB / 10), 1000), m.NB) if svi else widest) if mode == "streamed" else None
            outs[mode], fig = timed_run(m, width)
            res[mode].append(fig)
            del m
            torch.cuda.empty_cache()
        diffs.append(max_diff(outs["streamed"], outs["resident"]))
        identical.append(all(np.array_equal(outs["streamed"][k], outs["resident"][k]) for k in outs["resident"]))
    return dict(runs=res, max_abs_diff=diffs, bit_identical=identical)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for streamed_pair.json (default: print only)")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--full-iters", type=int, default=10)
    ap.add_argument("--full-iters-160k", type=int, default=20)
    ap.add_argument("--full-width-100k", type=int, default=25000, help="chunk width of the forced-streamed 100k full EM")
    ap.add_argument("--skip-160k", action="store_true")
    args = ap.parse_args()
    import torch

    import spateo_release_b200 as st

    doc = dict(card=card(), torch=torch.__version__)
    print(doc, flush=True)
    A, B = make_pair(100000)
    doc["100k_svi"] = compare_100k(A, B, True, 200, args.reps, None)
    print(json.dumps(doc["100k_svi"]), flush=True)
    doc["100k_full"] = compare_100k(A, B, False, args.full_iters, args.reps, args.full_width_100k)
    print(json.dumps(doc["100k_full"]), flush=True)
    del A, B
    if not args.skip_160k:
        from spateo_release_b200.alignment import morpho_class as mc

        A, B = make_pair(160000)
        plans = []
        orig = mc.Morpho_pairwise._plan_cost

        def spy(self, nb):
            orig(self, nb)
            plans.append(self.cost_plan._asdict())

        mc.Morpho_pairwise._plan_cost = spy
        torch.cuda.reset_peak_memory_stats()
        np.random.seed(0)
        t0 = time.perf_counter()
        out, _ = st.align.morpho_align([A, B], device="0", verbose=False)
        torch.cuda.synchronize()
        doc["160k_svi_morpho_align"] = dict(seconds=round(time.perf_counter() - t0, 2), plan=plans,
                                            peak_allocated_GiB=round(torch.cuda.max_memory_allocated() / 2**30, 2),
                                            finite=bool(np.isfinite(out[1].obsm["align_spatial"]).all()))
        print(json.dumps(doc["160k_svi_morpho_align"]), flush=True)
        mc.Morpho_pairwise._plan_cost = orig
        del out
        torch.cuda.empty_cache()
        m = solver(A, B, SVI_mode=False, max_iter=args.full_iters_160k, K=15)
        torch.cuda.reset_peak_memory_stats()
        _, fig = timed_run(m)
        fig["peak_allocated_GiB"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
        doc["160k_full"] = fig
        print(json.dumps(fig), flush=True)
    if args.out is not None:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "streamed_pair.json"), "w") as f:
            json.dump(doc, f, indent=1)
    print(json.dumps(doc))


if __name__ == "__main__":
    main()
