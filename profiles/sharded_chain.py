"""``morpho_align_column_sharded`` against ``morpho_align`` on one chain of 3-D slices: wall time and EM time of every pair.

Usage: torchrun --nproc-per-node W profiles/sharded_chain.py [--cells 60000 60000 60000] [--genes 2000] [--iters 200]
                                                             [--reps 2] [--out DIR]
(one process per GPU; W = 1 also runs without torchrun). The slices are serial sections of one synthetic warped tissue
(``make_slice_pair``: each is a re-sampled, rotated, shifted copy), one per ``--cells`` entry. Both arms run in the same
call, alternating which goes first in every repetition: the column-sharded chain on every rank, then (or before it)
``morpho_align`` on rank 0 alone while the other ranks wait. Both use the drivers' defaults (SVI, history of every
iteration under ``iter_spatial``) with ``materialize_P=False``. For every pair: wall time from building the solver to its
outputs (host clock after a device synchronise; the sharded arm's also covers storing them and releasing the pair) and EM
time (CUDA events around ``run_em``); for the chain: the total wall time of the driver call. Rank 0 prints one JSON
document with the card's name and power limit; with --out it also goes to DIR/sharded_chain.json.
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


def make_chain(cells, genes, seed=0):
    from spateo_release_b200.synthetic import make_slice_pair

    n = max(cells)
    return [make_slice_pair(n, c, genes, dim=3, seed=seed, z_thickness=20.0, warp_amplitude=1.0, theta=0.3 * k,
                            shift=4.0 * k)[1] for k, c in enumerate(cells)]


class PairTimer:
    """Per-pair wall time (around ``pair_fn`` of ``module``) and EM time (events around ``Morpho_pairwise.run_em``)."""

    def __init__(self, module, pair_fn):
        import torch

        from spateo_release_b200.alignment.morpho_class import Morpho_pairwise

        self.walls, self.events = [], []
        self._undo = []
        run_em, inner = Morpho_pairwise.run_em, getattr(module, pair_fn)

        def timed_run_em(solver, *a, **k):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = run_em(solver, *a, **k)
            e1.record()
            self.events.append((e0, e1))
            return out

        def timed_pair(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = inner(*a, **k)
            torch.cuda.synchronize()
            self.walls.append(time.perf_counter() - t0)
            return out

        Morpho_pairwise.run_em = timed_run_em
        setattr(module, pair_fn, timed_pair)
        self._undo = [(Morpho_pairwise, "run_em", run_em), (module, pair_fn, inner)]

    def close(self):
        for obj, name, fn in self._undo:
            setattr(obj, name, fn)
        return [dict(wall_s=round(w, 3), em_ms=round(a.elapsed_time(b), 1)) for w, (a, b) in zip(self.walls, self.events)]


def run_arm(arm, models, args, device):
    import torch

    import spateo_release_b200 as st
    from spateo_release_b200.alignment import distributed, morpho_alignment

    kw = dict(max_iter=args.iters, device=device, verbose=False, materialize_P=False, mode="SN-N")
    if arm == "column_sharded":
        timer, fn = PairTimer(distributed, "sharded_chain_pair"), st.align.morpho_align_column_sharded
    else:
        timer, fn = PairTimer(morpho_alignment, "_solve_pair"), st.align.morpho_align
    np.random.seed(0)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    try:
        aligned, _ = fn(models, **kw)
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
    finally:
        pairs = timer.close()
    torch.cuda.empty_cache()
    return dict(total_s=round(total, 3), pairs=pairs), [np.asarray(m.obsm["align_spatial"]) for m in aligned]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cells", type=int, nargs="+", default=[60000, 60000, 60000], help="cells of every slice")
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--out", default=None, help="directory for sharded_chain.json (default: print only)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    if world > 1:
        dist.init_process_group("nccl")
    models = make_chain(args.cells, args.genes)
    runs = {"column_sharded": [], "morpho_align": []}
    diffs = []
    for rep in range(args.reps):
        arms = ("column_sharded", "morpho_align") if rep % 2 == 0 else ("morpho_align", "column_sharded")
        coords = {}
        for arm in arms:
            if arm == "column_sharded" or rank == 0:
                fig, coords[arm] = run_arm(arm, models, args, local)
                runs[arm].append(fig)
            if world > 1:
                dist.barrier()
        if rank == 0:
            diffs.append(max(float(np.abs(a - b).max()) for a, b in zip(coords["column_sharded"], coords["morpho_align"])))
    if rank == 0:
        doc = dict(card=card(), torch=torch.__version__, world=world, cells=args.cells, genes=args.genes,
                   iters=args.iters, runs=runs, max_abs_coord_diff=diffs,
                   coord_scale=float(max(np.abs(np.asarray(m.obsm["spatial"])).max() for m in models)))
        text = json.dumps(doc)
        print(text, flush=True)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "sharded_chain.json"), "w") as f:
                f.write(text + "\n")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
