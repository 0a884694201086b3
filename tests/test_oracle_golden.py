"""CPU: pins oracle/morpho_oracle.py against golden vectors produced by executing the unmodified reference
(tests/golden/make_golden.py). Bitwise with the host BLAS they were made with; tolerances below allow for a different one."""

import ast
import contextlib

import numpy as np
import pytest

from oracle import morpho_oracle as mo

CASES = ["2d_full", "3d_svi", "3d_full_warp", "2d_full_nonn_euc", "2d_full_guide_both", "2d_svi_guide_nonrigid",
         "2d_full_sparse48", "3d_svi_sparse32"]


def _cfg(g):
    return ast.literal_eval(str(g["cfg"]))


def cfg_sparse(g):
    kw = _cfg(g)["kw"]
    return kw.get("sparse_top_k", 1024) if kw.get("sparse_calculation_mode") else 0


def _relmax(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-30)


def _make_oracle(g, dtype):
    cfg = _cfg(g)
    if "guide_fixed" in g:
        cfg["kw"] = dict(cfg["kw"], guidance_pair=[g["guide_fixed"], g["guide_moving"]])
    np.random.seed(0)
    return mo.MorphoPairOracle(
        np.asfortranarray(g["raw_coords_moving"]), np.asfortranarray(g["raw_coords_fixed"]),
        [g["exp_moving"]], [g["exp_fixed"]], dtype=dtype, SVI_mode=cfg["svi"], max_iter=cfg["max_iter"], K=cfg["K"],
        **cfg["kw"],
    )


def test_calc_distance_kl_matches_reference(golden):
    g = golden("2d_full")
    [d] = mo.calc_distance(g["exp_moving"], g["exp_fixed"], "kl")
    assert d.dtype == np.float32
    assert np.abs(d - g["exp_dist"]).max() <= 2e-6


@pytest.mark.parametrize("case", ["2d_full", "3d_full_warp"])
@pytest.mark.parametrize("it", [0, 95])
def test_get_P_core_matches_reference_dump(golden, case, it):
    g = golden(case)
    XAHat, alpha, SigmaDiag = g[f"it{it}_in_XAHat"], g[f"it{it}_in_alpha"], g[f"it{it}_in_SigmaDiag"]
    sigma2, gamma = g[f"it{it}_in_sigma2"], g[f"it{it}_in_gamma"]
    sv = np.float32(g[f"it{it}_in_sigma2_variance"])
    yb = g["pre_coordsB"]
    [ed] = mo.calc_distance(g["exp_moving"], g["exp_fixed"], "kl")
    P, kns, kn2, s2r = mo.get_P_core(
        Dim=np.float32(yb.shape[1]), spatial_dist=mo.euc_distance(XAHat, yb), exp_dist=[ed], sigma2=sigma2,
        model_mul=(alpha * np.exp(-SigmaDiag / sigma2))[:, None], gamma=gamma, samples_s=g["pre_samples_s"],
        sigma2_variance=sv, probability_type=["gauss"], probability_parameters=[g["pre_beta2"]],
    )
    assert _relmax(P, g[f"it{it}_out_P"]) < 2e-4
    assert _relmax(kns, g[f"it{it}_out_K_NA_spatial"]) < 1e-4
    assert _relmax(kn2, g[f"it{it}_out_K_NA_sigma2"]) < 1e-4
    assert _relmax(P.sum(1), g[f"it{it}_out_K_NA"]) < 1e-4
    assert _relmax(P.sum(0), g[f"it{it}_out_K_NB"]) < 1e-4


@pytest.mark.parametrize("case", CASES)
def test_preparation_matches_reference(golden, case):
    g = golden(case)
    orc = _make_oracle(g, "float32")
    assert _relmax(orc.U, g["pre_U"]) < 1e-5
    assert _relmax(orc.GammaSparse, g["pre_GammaSparse"]) < 1e-5
    orc.prepare()
    assert _relmax(orc.coordsA, g["pre_coordsA"]) < 1e-4
    assert _relmax(orc.coordsB, g["pre_coordsB"]) < 1e-5
    assert _relmax(orc.sigma2, g["pre_sigma2_0"]) < 1e-4
    assert _relmax(orc.probability_parameters[0], g["pre_beta2"]) < 1e-4
    if orc.nn_init:
        assert orc.inlier_P.shape == g["pre_inlier_P"].shape
        assert _relmax(orc.init_R, g["pre_init_R"]) < 1e-4
    if orc.SVI_mode:
        assert np.array_equal(orc.batch_perm, g["pre_batch_perm"])


GOLDEN_BLAS_THREADS = 8  # OpenBLAS threads of the reference runs that made the fixtures


def golden_blas_threads():
    """A threaded BLAS sums in an order that depends on its thread count, and 100+ EM iterations carry that difference
    past the float64 tolerance: run with the thread count the fixtures were made with, whatever the host's core count.
    Without threadpoolctl the BLAS keeps its own thread count."""
    try:
        from threadpoolctl import threadpool_limits
    except ImportError:
        return contextlib.nullcontext()
    return threadpool_limits(limits=GOLDEN_BLAS_THREADS, user_api="blas")


@pytest.mark.parametrize("case", CASES)
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_full_run_matches_reference(golden, case, dtype):
    g = golden(case)
    sfx = "" if dtype == "float32" else "_f64"
    orc = _make_oracle(g, dtype)
    with golden_blas_threads():
        orc.run()
    scale = np.abs(g["final_optimal_RnA" + sfx]).max()
    tol = 2e-4 if dtype == "float32" else 1e-6
    for key in ("optimal_RnA", "XAHat", "RnA"):
        assert np.abs(getattr(orc, key) - g[f"final_{key}{sfx}"]).max() / scale < tol, key
    assert _relmax(orc.sigma2, g["final_sigma2" + sfx]) < 1e-3
    assert _relmax(orc.gamma, g["final_gamma" + sfx]) < 1e-3
    assert _relmax(orc.optimal_R, g["final_optimal_R" + sfx]) < tol
    if "final_P" + sfx in g:
        P = orc.P.toarray() if hasattr(orc.P, "toarray") else orc.P
        if cfg_sparse(g):
            assert (P > 0).sum(0).max() <= cfg_sparse(g)  # at most top_k stored entries per column
        num = np.linalg.norm(P.astype(np.float64) - g["final_P" + sfx])
        assert num / np.linalg.norm(g["final_P" + sfx]) < (2e-2 if dtype == "float32" else 1e-5)


@pytest.mark.parametrize("case", ["2d_full", "3d_svi_sparse32"])
@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_oracle_is_bitwise_equal_to_the_reference(golden, case, dtype):
    """Every final output the reference run stored (posterior or its row / column sums, aligned coordinates, Coff, R, t,
    the closing similarity, sigma2, gamma) is reproduced by the oracle to the last bit: same numpy calls in the same order,
    with the BLAS thread count the fixtures were made with."""
    pytest.importorskip("threadpoolctl", reason="pinning the BLAS thread count needs threadpoolctl")
    g = golden(case)
    sfx = "" if dtype == "float32" else "_f64"
    orc = _make_oracle(g, dtype)
    with golden_blas_threads():
        orc.run()
    # sparse mode stores only the row / column sums, taken like the fixture did (on the sparse matrix)
    derived = {"P_rowsum": np.asarray(orc.P.sum(1)).reshape(-1), "P_colsum": np.asarray(orc.P.sum(0)).reshape(-1),
               "P": orc.P.toarray() if hasattr(orc.P, "toarray") else orc.P}
    keys = [k[len("final_"):len(k) - len(sfx)] for k in g if k.startswith("final_") and k.endswith(sfx)
            and (sfx or not k.endswith("_f64"))]
    assert {"Coff", "R", "t", "optimal_t", "XAHat", "optimal_RnA"} <= set(keys)
    for key in keys:
        got = derived[key] if key in derived else getattr(orc, key)
        assert np.array_equal(np.asarray(got, dtype=np.float64), np.asarray(g[f"final_{key}{sfx}"], dtype=np.float64)), key


def test_ba_transform_reproduces_training_points(golden):
    g = golden("3d_full_warp")
    orc = _make_oracle(g, "float64")
    orc.run()
    XAHat, _, opt = mo.ba_transform(orc.vecfld, g["raw_coords_moving"], dtype="float64")
    assert np.abs(XAHat - orc.XAHat).max() < 1e-6 * np.abs(orc.XAHat).max()
    assert np.abs(opt - orc.optimal_RnA).max() < 1e-6 * np.abs(orc.XAHat).max()


@pytest.mark.parametrize("tag", ["2d", "3d"])
def test_ba_transform_matches_reference_fixture(golden, tag):
    """oracle.ba_transform against outputs of the unmodified reference BA_transform (tests/golden/make_golden_transform.py):
    bit-identical in float64 and float32, both deformation scales."""
    g = golden("ba_transform")
    vf = {k: g[f"{tag}_vf_{k}"] for k in ("R", "t", "optimal_R", "optimal_t", "init_R", "init_t", "Coff", "inducing_variables")}
    vf["beta"] = float(g[f"{tag}_vf_beta"])
    vf["normalize_c"] = bool(g[f"{tag}_vf_normalize_c"])
    vf["norm_dict"] = {k: g[f"{tag}_nd_{k}"] for k in ("mean_transformed", "mean_fixed", "scale_transformed", "scale_fixed")}
    pts = g[f"{tag}_points"]
    for dt in ("float64", "float32"):
        for ds in (1, 0.5):
            X, V, O = mo.ba_transform(vf, pts, deformation_scale=ds, dtype=dt)
            sfx = f"{dt}_{ds}"
            assert np.array_equal(X, g[f"{tag}_XAHat_{sfx}"]) and X.dtype == g[f"{tag}_XAHat_{sfx}"].dtype
            assert np.array_equal(V, g[f"{tag}_vel_{sfx}"]) and np.array_equal(O, g[f"{tag}_opt_{sfx}"])


# ---------------------------------------------------------------------------------------------------------------------
# BASELINE configs[0] scale (5000 x 5000 cells, 100 genes, 2-D): preparation + E-step dumps of the reference
# ---------------------------------------------------------------------------------------------------------------------
C1_CASES = ["c1_2d_svi", "c1_2d_full_warp"]


@pytest.mark.parametrize("case", C1_CASES)
def test_config1_preparation_matches_reference(golden, case):
    g = golden(case)
    orc = _make_oracle(g, "float32")
    orc.prepare()
    assert _relmax(orc.U, g["pre_U"]) < 1e-5
    assert _relmax(orc.coordsA, g["pre_coordsA"]) < 1e-4
    assert _relmax(orc.sigma2, g["pre_sigma2_0"]) < 1e-4
    assert _relmax(orc.probability_parameters[0], g["pre_beta2"]) < 1e-4
    assert orc.inlier_P.shape == g["pre_inlier_P"].shape and _relmax(orc.init_R, g["pre_init_R"]) < 1e-4
    if orc.SVI_mode:
        assert np.array_equal(orc.batch_perm, g["pre_batch_perm"])


@pytest.mark.parametrize("case", C1_CASES)
@pytest.mark.parametrize("it", [0, 150])
def test_config1_estep_matches_reference_dump(golden, case, it):
    """float32 oracle E-step (evaluated in column chunks) on the reference's inputs against the reference's outputs."""
    g = golden(case)
    XAHat, alpha, SD = g[f"it{it}_in_XAHat"], g[f"it{it}_in_alpha"], g[f"it{it}_in_SigmaDiag"]
    sigma2, gamma = g[f"it{it}_in_sigma2"], g[f"it{it}_in_gamma"]
    yb, eB = g["pre_coordsB"], g["exp_fixed"]
    if f"it{it}_in_batch_idx" in g:
        yb, eB = yb[g[f"it{it}_in_batch_idx"]], eB[g[f"it{it}_in_batch_idx"]]
    out = mo.estep_column_chunks(
        Dim=np.float32(yb.shape[1]), XAHat=XAHat, YB=yb, exp_A=[g["exp_moving"]], exp_B=[eB], metric=["kl"], sigma2=sigma2,
        model_mul=(alpha * np.exp(-SD / sigma2))[:, None], gamma=gamma, samples_s=g["pre_samples_s"],
        sigma2_variance=np.float32(g[f"it{it}_in_sigma2_variance"]), probability_type=["gauss"],
        probability_parameters=[g["pre_beta2"]], chunk=1250,
    )
    # chunked accumulation changes the fp32 summation order of the row statistics: tolerance = fp32 noise
    assert _relmax(out["K_NB"], g[f"it{it}_out_K_NB"]) < 1e-4
    assert _relmax(out["K_NA"], g[f"it{it}_out_K_NA"]) < 5e-4
    assert _relmax(out["K_NA_spatial"], g[f"it{it}_out_K_NA_spatial"]) < 5e-4
    assert _relmax(out["K_NA_sigma2"], g[f"it{it}_out_K_NA_sigma2"]) < 5e-4
    assert _relmax(out["PXB"], g[f"it{it}_out_PXB"]) < 5e-4


def test_estep_column_chunks_equals_one_block(golden):
    """The chunked evaluation is the same computation as one get_P_core call over all columns."""
    g = golden("3d_full_warp")
    it = 95
    f8 = lambda k: g[k].astype(np.float64)
    XAHat, alpha, SD = f8(f"it{it}_in_XAHat"), f8(f"it{it}_in_alpha"), f8(f"it{it}_in_SigmaDiag")
    sigma2, gamma = float(g[f"it{it}_in_sigma2"]), float(g[f"it{it}_in_gamma"])
    yb = f8("pre_coordsB")
    common = dict(sigma2=sigma2, model_mul=(alpha * np.exp(-SD / sigma2))[:, None], gamma=gamma,
                  samples_s=float(g["pre_samples_s"]), sigma2_variance=float(g[f"it{it}_in_sigma2_variance"]),
                  probability_type=["gauss"], probability_parameters=[float(g["pre_beta2"])])
    out = mo.estep_column_chunks(Dim=3.0, XAHat=XAHat, YB=yb, exp_A=[f8("exp_moving")], exp_B=[f8("exp_fixed")],
                                 metric=["kl"], chunk=77, keep_P=True, **common)
    [ed] = mo.calc_distance(f8("exp_moving"), f8("exp_fixed"), "kl")
    P, kns, kn2, s2r = mo.get_P_core(Dim=3.0, spatial_dist=mo.euc_distance(XAHat, yb), exp_dist=[ed], **common)
    assert _relmax(out["P"], P) < 1e-12 and _relmax(out["K_NA_spatial"], kns) < 1e-12
    assert _relmax(out["K_NA_sigma2"], kn2) < 1e-12 and abs(out["sigma2_related_num"] - s2r) < 1e-12 * abs(s2r)
