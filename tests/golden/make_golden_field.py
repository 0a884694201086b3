"""Generate tests/golden/case_field_geometry.npz by running the UNMODIFIED reference's GPVectorField functions
(spateo/tdr/morphometrics/morphofield_dg/GPVectorField.py, morphofield/gaussian_process.py) on seeded synthetic
fields. Needs the reference:  SPATEO_REFERENCE=<spateo-release checkout> python tests/golden/make_golden_field.py
"""

import io
import os
import sys
from contextlib import redirect_stderr

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_harness import load_reference_tdr  # noqa: E402


def synthetic_field(D, K, seed):
    rng = np.random.default_rng(seed)
    th = 0.3
    R = np.eye(D)
    R[:2, :2] = [[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]]
    return dict(
        norm_dict=dict(mean_transformed=rng.normal(size=D) * 10, scale_transformed=np.float64(7.3),
                       mean_fixed=rng.normal(size=D) * 10, scale_fixed=np.float64(6.9)),
        kernel_type="euc", inducing_variables=rng.normal(size=(K, D)), beta=0.5,
        Coff=rng.normal(size=(K, D)) * 0.1, R=R, t=rng.normal(size=(1, D)) * 0.1, method="gaussian_process")


class _A:
    pass


def main():
    gp, gv = load_reference_tdr()
    out = {}
    for tag, D, K, n, seed in [("2d", 2, 15, 300, 1), ("3d", 3, 40, 400, 2)]:
        vf = synthetic_field(D, K, seed)
        X = np.random.default_rng(seed + 10).normal(size=(n, D)) * 7 + vf["norm_dict"]["mean_transformed"]
        for k in ("inducing_variables", "Coff", "R", "t"):
            out[f"{tag}_{k}"] = vf[k]
        for k, v in vf["norm_dict"].items():
            out[f"{tag}_nd_{k}"] = np.asarray(v)
        out[f"{tag}_beta"] = np.float64(vf["beta"])
        out[f"{tag}_X"] = X
        for nro in (False, True):
            sfx = "_nro" if nro else ""
            vf["X"], vf["V"] = X, gp._gp_velocity(X, vf, nonrigid_only=nro)
            a = _A()
            a.uns = {"VecFld": vf}
            c = gv.GPVectorField()
            c.from_adata(a, vf_key="VecFld", nonrigid_only=nro)
            with redirect_stderr(io.StringIO()):
                out[f"{tag}_V{sfx}"] = vf["V"]
                acc, acc_mat = c.compute_acceleration()
                out[f"{tag}_acc{sfx}"], out[f"{tag}_acc_mat{sfx}"] = acc, acc_mat
                c2, c2m = c.compute_curvature(formula=2)
                out[f"{tag}_curv2{sfx}"], out[f"{tag}_curv2_mat{sfx}"] = c2, c2m
                out[f"{tag}_curv1{sfx}"] = c.compute_curvature(formula=1)[0]
                if D == 3:
                    out[f"{tag}_torsion{sfx}"] = c.compute_torsion()
                if not nro:
                    out[f"{tag}_J"] = gv.Jacobian_GP_gaussian_kernel(X, vf)
                    out[f"{tag}_J_vec"] = gv.Jacobian_GP_gaussian_kernel(X, vf, vectorize=True)
                    out[f"{tag}_J_single"] = gv.Jacobian_GP_gaussian_kernel(X[3], vf)
                    out[f"{tag}_curl"] = c.compute_curl()
                    out[f"{tag}_div"] = c.compute_divergence()
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "case_field_geometry.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
