"""st.tdr.morphopath on realistic fields: kernel and whole-call time, and the scipy oracle's per-cell time.

Usage (one H100): python profiles/morphopath.py [--out DIR] [--cells N] [--oracle-cells M] [--reps R]
Prints one JSON document (card, power limit, every figure below); with --out it is also written to
DIR/morphopath.json.

  Fields: the Gaussian-process field of a morpho_align run on a 100k x 100k 3-D pair (``morphofield_gp``), and SparseVFC
  fields fitted to that pair's per-cell displacements with M = 100 and 500 control points (``morphofield_sparsevfc``).
  For each field, at interpolation_num 20 and 250 (t_end 10000, forward): the CUDA-event time of spb_field_integrate
  alone and of the whole ``morphopath`` call (mean of --reps after one warm-up), the accepted / rejected steps per cell,
  and the oracle's (scipy solve_ivp per cell) host time per cell on --oracle-cells cells.
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--cells", type=int, default=100000)
    ap.add_argument("--oracle-cells", type=int, default=200)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--max-iter", type=int, default=200)
    args = ap.parse_args()

    import torch

    import spateo_release_b200 as st
    from oracle import path_oracle as po
    from spateo_release_b200.synthetic import make_slice_pair
    from spateo_release_b200.tdr import morphofield_dg as dg

    A, B = make_slice_pair(args.cells, args.cells, 50, dim=3, seed=0, z_thickness=20.0)
    np.random.seed(0)
    t0 = time.time()
    aligned, _ = st.align.morpho_align([A, B], max_iter=args.max_iter, device="0", verbose=False, SVI_mode=True)
    moving = aligned[1]
    align_s = time.time() - t0
    st.tdr.morphofield_gp(moving, grid_num=[5, 5, 5])
    fields = {"gp": dict(moving.uns["VecFld_morpho"])}
    X = np.asarray(moving.uns["VecFld_morpho"]["X"], dtype=np.float64)
    V = np.asarray(moving.uns["VecFld_morpho"]["V"], dtype=np.float64) * 10000  # displacement per cell
    for M in (100, 500):
        vf = st.tdr.sparsevfc.SparseVFC(X, V, Grid=None, M=M, lambda_=0.02, MaxIter=30, device="0")
        vf["method"], vf["X"] = "sparsevfc", X
        fields[f"sparsevfc_M{M}"] = vf

    class _A:
        def __init__(self, vf):
            self.uns, self.obs_names = {"VecFld_morpho": vf}, [str(i) for i in range(len(X))]

    res = {"card": card(), "cells": len(X), "align_s_incl_compile": round(align_s, 1), "fields": {}}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, vf in fields.items():
        if vf["method"] == "sparsevfc":
            f, z, C = dg._desc_svc(vf, 3, 2), vf["X_ctrl"], vf["C"]
        else:
            f, z, C = dg._desc(vf, 3, False, 2), vf["inducing_variables"], vf["Coff"]
        z, C = (np.ascontiguousarray(np.asarray(a), dtype=np.float64) for a in (z, C))
        row = {"K": int(z.shape[0])}
        for ni in (20, 250):
            # kernel alone: device buffers prepared once
            from spateo_release_b200 import _capi

            lib = _capi.load_library()
            Xd, zd, Cd = (torch.from_numpy(a).cuda() for a in (X, z, C))
            n = len(X)
            out = torch.empty((n, ni + 1, 3), dtype=torch.float64, device="cuda")
            ts = torch.empty(n, dtype=torch.float64, device="cuda")
            steps = torch.empty((n, 2), dtype=torch.int32, device="cuda")
            status = torch.empty(n, dtype=torch.int32, device="cuda")

            def launch():
                _capi.check(lib.spb_field_integrate(f, _capi.ptr(Xd), n, _capi.ptr(zd), _capi.ptr(Cd), 10000.0, ni + 1,
                                                    1e-3, 1e-6, 10000.0 / ni, _capi.ptr(out), _capi.ptr(ts),
                                                    _capi.ptr(steps), _capi.ptr(status), _capi.current_stream_ptr()),
                            "spb_field_integrate")

            launch()
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.reps):
                launch()
            e1.record()
            torch.cuda.synchronize()
            kernel_ms = e0.elapsed_time(e1) / args.reps
            s = steps.cpu().numpy()
            a = _A(vf)
            st.tdr.morphopath(a, t_end=10000, interpolation_num=ni)
            torch.cuda.synchronize()
            e0.record()
            for _ in range(args.reps):
                st.tdr.morphopath(a, t_end=10000, interpolation_num=ni)
            e1.record()
            torch.cuda.synchronize()
            call_ms = e0.elapsed_time(e1) / args.reps
            sample = np.random.default_rng(0).choice(n, args.oracle_cells, replace=False)
            t0 = time.time()
            po.path(X[sample], vf, 10000.0, ni, "forward")
            oracle_s = (time.time() - t0) / args.oracle_cells
            row[f"interp{ni}"] = {
                "kernel_ms": round(kernel_ms, 2), "call_ms": round(call_ms, 2),
                "accepted_mean": round(float(s[:, 0].mean()), 1), "rejected_mean": round(float(s[:, 1].mean()), 2),
                "status": a.uns["fate_morpho"]["status"], "oracle_ms_per_cell": round(oracle_s * 1e3, 2),
                "oracle_s_all_cells_est": round(oracle_s * n, 1),
            }
            print(name, ni, row[f"interp{ni}"], flush=True)
        res["fields"][name] = row
    doc = json.dumps(res, indent=1)
    print(doc)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "morphopath.json"), "w") as fh:
            fh.write(doc)


if __name__ == "__main__":
    main()
