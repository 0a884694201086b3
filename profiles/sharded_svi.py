"""SVI on a column-sharded pair: ms per iteration of the sharded run against the unsharded resident and streamed runs.

Usage: torchrun --nproc-per-node W profiles/sharded_svi.py [--n 100000] [--iters 200] [--out DIR]
(one process per GPU; W = 1 runs on a single GPU without torchrun as well). Every rank aligns the same synthetic
n x n x 2000-gene 3-D pair with ``morpho_align_pair_sharded(SVI_mode=True)``; rank 0 then times the unsharded solver on
its GPU, resident and forced-streamed (one chunk of the SVI batch). Rank 0 prints one JSON document (card, power limit,
world size, ms per iteration of each run, largest output difference to the resident run); with --out it is also written
to DIR/sharded_svi.json.
"""

import argparse
import gc
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "profiles"))

from streamed_pair import card, make_pair, max_diff, timed_run  # noqa: E402


def sharded_run(A, B, iters, rank):
    """The pair over every rank; returns (outputs, figures) on every rank."""
    import torch

    from spateo_release_b200.alignment.distributed import morpho_align_pair_sharded

    np.random.seed(0)
    t0 = time.perf_counter()
    m = morpho_align_pair_sharded(A, B, device=str(rank), SVI_mode=True, max_iter=iters, K=15, nn_init=False,
                                  verbose=False)
    torch.cuda.synchronize()
    t_prep = time.perf_counter() - t0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0 = time.perf_counter()
    e0.record()
    m.run()
    e1.record()
    torch.cuda.synchronize()
    out = {k: np.asarray(getattr(m, k)) for k in ("XAHat", "optimal_RnA", "R", "t", "sigma2", "gamma", "K_NA", "K_NB")}
    fig = dict(columns=m._col_range(), width=int(m._params.NBb), mode=m._shard_mode, prepare_s=round(t_prep, 3),
               run_s=round(time.perf_counter() - t0, 3), ms_per_iter=round(e0.elapsed_time(e1) / max(iters, 1), 3))
    return out, fig


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=100000, help="cells per slice")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None, help="directory for sharded_svi.json (default: print only)")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist

    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    if world > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", rank)))
        dist.init_process_group("nccl")
    A, B = make_pair(args.n)
    out_sh, fig_sh = sharded_run(A, B, args.iters, int(os.environ.get("LOCAL_RANK", rank)))
    gc.collect()  # the sharded solver's cost matrix goes back to the allocator before the unsharded runs
    torch.cuda.empty_cache()
    figs = [fig_sh]
    if world > 1:
        figs = [None] * world
        dist.all_gather_object(figs, fig_sh)
    if rank == 0:
        import streamed_pair as sp

        doc = dict(card=card(), torch=torch.__version__, world=world, n=args.n, iters=args.iters, sharded=figs)
        for mode in ("resident", "streamed"):
            m = sp.solver(A, B, SVI_mode=True, max_iter=args.iters, K=15)
            width = min(max(int(m.NB / 10), 1000), m.NB) if mode == "streamed" else None
            out, fig = timed_run(m, width)
            doc[mode] = fig
            if mode == "resident":
                ref = out
            del m
            torch.cuda.empty_cache()
        doc["sharded_max_abs_diff_to_resident"] = max_diff(out_sh, ref)
        text = json.dumps(doc)
        print(text, flush=True)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, "sharded_svi.json"), "w") as f:
                f.write(text + "\n")
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
