"""Posterior transfer on the benchmark pair: cost of P @ F_B and P^T @ F_A after a full EM.

Usage (one H100): python profiles/posterior_transfer.py [--out DIR] [--cells N] [--genes G] [--max-iter I] [--reps R]
Prints one JSON document (card, power limit, every figure below); with --out it is also written to
DIR/posterior_transfer.json.

  100k x 100k cells, 3-D, 2000 genes, full EM of 200 iterations (``run_em``, timed with CUDA events). Then, on the final
  state, one E-step and the four transfers: a 32-class one-hot and the 2000 genes, each through P @ F_B (fixed slice's
  features to the moving cells) and P^T @ F_A (moving slice's features to the fixed cells). Per transfer: CUDA-event
  milliseconds (mean of --reps after one warm-up), seconds added relative to the EM, cost-matrix bytes read (visited
  tiles x 512 rows x 4 bytes x panels of 16 features) and the resulting GB/s against the H100's 3.35 TB/s.
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--genes", type=int, default=2000)
    ap.add_argument("--max-iter", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()

    import ctypes as C

    import torch

    import spateo_release_b200 as st
    from spateo_release_b200 import _capi
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(args.cells, args.cells, args.genes, dim=3, seed=0, z_thickness=20.0)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(sampleA=B, sampleB=A, max_iter=args.max_iter, SVI_mode=False, K=15, nn_init=True,
                                 verbose=False, device="0", materialize_P=False)
    m.prepare()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    m.run_em()
    e1.record()
    torch.cuda.synchronize()
    em_s = e0.elapsed_time(e1) / 1e3

    rng = np.random.default_rng(0)
    W = _capi.CONST["SPB_TRANSFER_PANEL"]
    nrb = m.ldx // _capi.ROW_TILE
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    last = m.max_iter - 1
    feats = {
        "labels32": (np.eye(32, dtype=np.float32)[rng.integers(0, 32, m.NB)], np.eye(32, dtype=np.float32)[rng.integers(0, 32, m.NA)]),
        f"genes{args.genes}": (m.exp_layers_B[0], m.exp_layers_A[0]),
    }
    out = {"card": card(), "pair": f"{args.cells} x {args.cells}, 3-D, {args.genes} genes, full EM",
           "max_iter": m.max_iter, "em_s": em_s, "transfers": {}}
    for name, (fb, fa) in feats.items():
        for side in ("rows", "cols"):
            m._FB_host, m._FA_host = (fb, None) if side == "rows" else (None, fa)
            for k in [k for k in m._state if k.startswith("xfer_")]:
                del m._state[k]
            torch.cuda.empty_cache()
            m._allocate_transfer(m._state, m.NB, nrb)
            m._estep_only(last, stream)
            torch.cuda.synchronize()
            visited = float(m._read_scalars().visited)
            F = (fb if side == "rows" else fa).shape[1]
            m._transfer_begin()
            m._transfer_capture(m._params, last, stream)  # warm-up
            torch.cuda.synchronize()
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record()
            for _ in range(args.reps):
                m._transfer_capture(m._params, last, stream)
            t1.record()
            torch.cuda.synchronize()
            sec = t0.elapsed_time(t1) / 1e3 / args.reps
            gt_bytes = visited * _capi.ROW_TILE * 4 * (-(-F // W))
            out["transfers"][f"{name}_{'P@F_B' if side == 'rows' else 'PT@F_A'}"] = {
                "features": F, "ms": sec * 1e3, "added_vs_em": sec / em_s, "gt_bytes": gt_bytes,
                "gt_GBps": gt_bytes / sec / 1e9, "share_of_3.35TBps": gt_bytes / sec / HBM_BYTES_PER_S,
                "visited_tiles": visited, "tiles": float(nrb * m.NB),
            }
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "posterior_transfer.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
