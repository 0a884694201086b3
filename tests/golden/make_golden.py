"""Generate the golden fixtures in this directory by EXECUTING THE UNMODIFIED REFERENCE (needs SPATEO_REFERENCE).

    python tests/golden/make_golden.py

Each ``case_*.npz`` holds, for one seeded synthetic slice pair: the solver inputs (raw coordinates, dense expression in
the reference's gene order), the state after ``Morpho_pairwise.__init__`` + coarse init + variational init, full E-step
dumps at a few iterations (inputs and every output of ``_update_assignment_P``), per-iteration scalar trajectories, and
the final outputs of ``run()`` — for the float32 reference and (suffix ``_f64``) the float64 reference.
Reference call sites: spateo/alignment/methods/morpho_class.py:242-313 (run), :1071-1200 (E-step).
"""

import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
warnings.filterwarnings("ignore")

from oracle.ref_harness import load_reference  # noqa: E402
from spateo_release_b200.synthetic import make_slice_pair  # noqa: E402

CASES = {
    # name: (n_moving, n_fixed, genes, dim, SVI, max_iter, K, warp, extra kwargs)
    "2d_full": dict(n_a=260, n_b=240, g=30, dim=2, svi=False, max_iter=120, K=15, warp=0.0, kw={}, dump_exp_dist=True),
    "3d_svi": dict(n_a=1300, n_b=1200, g=24, dim=3, svi=True, max_iter=120, K=15, warp=0.0, kw={}),
    "3d_full_warp": dict(n_a=300, n_b=320, g=30, dim=3, svi=False, max_iter=130, K=30, warp=2.0, kw={}),
    "2d_full_nonn_euc": dict(n_a=220, n_b=250, g=12, dim=2, svi=False, max_iter=100, K=15, warp=0.0,
                             kw=dict(nn_init=False, dissimilarity="euc")),
    # guidance pairs (morpho_class.py:551-587, 1282-1288, 1322-1327, 1360-1363, 1384-1388): 12 landmark correspondences
    "2d_full_guide_both": dict(n_a=300, n_b=280, g=24, dim=2, svi=False, max_iter=110, K=15, warp=1.5,
                               kw=dict(guidance_effect="both", guidance_weight=2.0), guide=True),
    "2d_svi_guide_nonrigid": dict(n_a=1250, n_b=1200, g=20, dim=2, svi=True, max_iter=110, K=15, warp=1.5,
                                  kw=dict(guidance_effect="nonrigid"), guide=True),
    # sparse_calculation_mode (utils.py:1085-1094, morpho_class.py:1187-1198): top-k entries of every column of P
    "2d_full_sparse48": dict(n_a=300, n_b=280, g=24, dim=2, svi=False, max_iter=110, K=15, warp=1.0,
                             kw=dict(sparse_calculation_mode=True, sparse_top_k=48)),
    "3d_svi_sparse32": dict(n_a=1250, n_b=1200, g=20, dim=3, svi=True, max_iter=110, K=15, warp=0.0,
                            kw=dict(sparse_calculation_mode=True, sparse_top_k=32)),
    # kernel_type="geodist" (morpho_class.py:865-871): inducing kernel from shortest paths on the kNN graph of the moving cells
    "2d_full_geodist": dict(n_a=260, n_b=240, g=30, dim=2, svi=False, max_iter=120, K=15, warp=1.5,
                            kw=dict(kernel_type="geodist")),
    # BASELINE configs[0] (SURVEY 8(d) config 1): 2-D, 5000 x 5000 cells, 100 genes, 200 iterations, the reference's default
    # SVI mode (batch 1000) and the full EM; E-step dumps at iterations 0 / 60 / 150 (5 row blocks of 1024 moving cells,
    # several column segments, zero-tile culling active at 150)
    "c1_2d_svi": dict(n_a=5000, n_b=5000, g=100, dim=2, svi=True, max_iter=200, K=15, warp=0.0, kw={},
                      dump_iters=(0, 60, 150)),
    "c1_2d_full_warp": dict(n_a=5000, n_b=5000, g=100, dim=2, svi=False, max_iter=200, K=15, warp=2.0, kw={},
                            dump_iters=(0, 60, 150)),
}
DUMP_ITERS = (0, 3, 60, 95, 110)
P_DUMP_ITERS = (0, 95)


def _dense(P):
    return P.toarray() if hasattr(P, "toarray") else P


def run_reference(cfg, dtype, dump):
    mc, _ = load_reference()
    A, B = make_slice_pair(cfg["n_a"], cfg["n_b"], cfg["g"], dim=cfg["dim"], seed=1, warp_amplitude=cfg["warp"])
    extra = {}
    guide = None
    if cfg.get("guide"):
        from spateo_release_b200.synthetic import _rotation

        pts = np.random.default_rng(5).uniform(10, 90, size=(12, cfg["dim"]))
        guide = [pts, pts @ _rotation(cfg["dim"], 0.5).T + 5.0]  # [X_BI on the fixed slice, X_AI on the moving slice]
        extra["guidance_pair"] = guide
    np.random.seed(0)
    ref = mc.Morpho_pairwise(
        sampleA=B, sampleB=A, device="cpu", dtype=dtype, verbose=False, SVI_mode=cfg["svi"], max_iter=cfg["max_iter"],
        K=cfg["K"], vecfld_key_added="vf", **cfg["kw"], **extra,
    )
    out = {}
    if guide is not None and dump:
        out["guide_fixed"], out["guide_moving"] = guide
    sfx = "" if dtype == "float32" else "_f64"
    if dump:
        out["raw_coords_moving"] = np.asarray(B.obsm["spatial"])
        out["raw_coords_fixed"] = np.asarray(A.obsm["spatial"])
        out["exp_moving"] = np.asarray(ref.exp_layers_A[0])
        out["exp_fixed"] = np.asarray(ref.exp_layers_B[0])
        out["gene_order"] = np.array([int(g[1:]) for g in ref.genes])
    # ---- replicate run() step by step (morpho_class.py:258-313) so intermediate state can be captured ----
    if ref.nn_init:
        ref._coarse_rigid_alignment()
    ref._initialize_variational_variables()
    ref.exp_layer_dist = mc.calc_distance(
        X=ref.exp_layers_A, Y=ref.exp_layers_B, metric=ref.dissimilarity, label_transfer=ref.label_transfer
    )
    pre = dict(
        coordsA=ref.coordsA, coordsB=ref.coordsB, U=ref.U, GammaSparse=ref.GammaSparse,
        inducing_variables=ref.inducing_variables, sigma2_0=ref.sigma2, samples_s=ref.samples_s,
        beta2=np.asarray(ref.probability_parameters[0]), normalize_scales=ref.normalize_scales,
        normalize_means=ref.normalize_means,
    )
    if ref.nn_init:
        pre.update(inlier_A=ref.inlier_A, inlier_B=ref.inlier_B, inlier_P=ref.inlier_P, init_R=ref.init_R, init_t=ref.init_t)
    if ref.SVI_mode:
        pre.update(batch_perm=ref.batch_perm, batch_size=np.asarray(ref.batch_size))
    for k, v in pre.items():
        out[f"pre_{k}{sfx}"] = np.asarray(v)
    if dump and cfg.get("dump_exp_dist"):
        out["exp_dist"] = np.asarray(ref.exp_layer_dist[0])
    traj = {k: [] for k in ("sigma2", "gamma", "Sp", "Sp_spatial", "Sp_sigma2", "sigma2_variance")}
    DUMP_ITERS = cfg.get("dump_iters", globals()["DUMP_ITERS"])
    for it in range(ref.max_iter):
        if ref.SVI_mode:
            ref._update_batch(iter=it)
        if it in DUMP_ITERS:
            e_in = dict(XAHat=ref.XAHat, alpha=ref.alpha, SigmaDiag=ref.SigmaDiag, sigma2=ref.sigma2, gamma=ref.gamma,
                        sigma2_variance=np.asarray(ref.sigma2_variance, dtype=np.float64))
            if ref.SVI_mode:
                e_in["batch_idx"] = ref.batch_idx
            for k, v in e_in.items():
                out[f"it{it}_in_{k}{sfx}"] = np.array(v)
        ref._update_assignment_P()
        if it in DUMP_ITERS:
            e_out = dict(K_NA=ref.K_NA, K_NB=ref.K_NB, K_NA_spatial=ref.K_NA_spatial, K_NA_sigma2=ref.K_NA_sigma2,
                         sigma2_related=ref.sigma2_related, Sp=ref.Sp, Sp_spatial=ref.Sp_spatial, Sp_sigma2=ref.Sp_sigma2)
            if cfg["n_a"] <= 400 and it in P_DUMP_ITERS and dtype == "float32":
                e_out["P"] = _dense(ref.P)
            else:
                YB = ref.coordsB[ref.batch_idx] if ref.SVI_mode else ref.coordsB
                e_out["PXB"] = ref.P @ YB
            for k, v in e_out.items():
                out[f"it{it}_out_{k}{sfx}"] = np.array(v)
        ref._update_gamma()
        ref._update_alpha()
        if (it > ref.nonrigid_start_iter) or ref.nonrigid_flag:
            ref.nonrigid_flag = True
            ref._update_nonrigid()
        ref._update_rigid()
        ref.XAHat = ref.VnA + ref.RnA
        ref._update_sigma2(iter=it)
        if it in DUMP_ITERS:
            m_out = dict(alpha=ref.alpha, R=ref.R, t=ref.t, RnA=ref.RnA, VnA=ref.VnA, XAHat=ref.XAHat,
                         SigmaDiag=ref.SigmaDiag, Coff=ref.Coff, sigma2=ref.sigma2, gamma=ref.gamma)
            if ref.nonrigid_flag:
                m_out["SigmaInv"] = ref.SigmaInv
            for k, v in m_out.items():
                out[f"it{it}_post_{k}{sfx}"] = np.array(v)
        for k in traj:
            traj[k].append(float(getattr(ref, k)))
    ref._get_optimal_R()
    ref._wrap_output()
    for k in traj:
        out[f"traj_{k}{sfx}"] = np.array(traj[k])
    fin = dict(P=_dense(ref.P), optimal_RnA=ref.optimal_RnA, XAHat=ref.XAHat, RnA=ref.RnA, R=ref.R, t=ref.t, Coff=ref.Coff,
               sigma2=ref.sigma2, gamma=ref.gamma, optimal_R=ref.optimal_R, optimal_t=ref.optimal_t)
    if cfg["n_a"] > 400:
        fin.pop("P")
        fin["P_colsum"] = np.asarray(ref.P.sum(0)).reshape(-1)
        fin["P_rowsum"] = np.asarray(ref.P.sum(1)).reshape(-1)
    for k, v in fin.items():
        out[f"final_{k}{sfx}"] = np.asarray(v)
    return out


if __name__ == "__main__":
    only = sys.argv[1:]
    for name, cfg in CASES.items():
        if only and name not in only:
            continue
        data = {}
        data.update(run_reference(cfg, "float32", dump=True))
        data.update(run_reference(cfg, "float64", dump=False))
        data["cfg"] = np.array(repr({k: v for k, v in cfg.items()}))
        path = os.path.join(HERE, f"case_{name}.npz")
        np.savez_compressed(path, **data)
        print(name, "->", path, f"{os.path.getsize(path) / 1e6:.2f} MB", len(data), "arrays")
