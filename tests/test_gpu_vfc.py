"""GPU: SparseVFC device solver against the float64 numpy restatement (oracle.sparse_vfc — parity unpinned vs dynamo)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import morpho_oracle as mo  # noqa: E402


def _field_data(n, D, seed=0, outliers=0.1):
    rng = np.random.default_rng(seed)
    X = rng.uniform(0, 100, size=(n, D))
    c = X - 50.0
    V = np.zeros_like(X)
    V[:, 0], V[:, 1] = -0.05 * c[:, 1], 0.05 * c[:, 0]  # rotation
    V += 2.0 * np.exp(-np.sum(c**2, 1, keepdims=True) / (2 * 15.0**2)) * np.ones((1, D))  # bump
    V += rng.normal(0, 0.1, size=V.shape)
    k = int(outliers * n)
    V[:k] = rng.uniform(-5, 5, size=(k, D))
    return X, V


@pytest.mark.parametrize("D,n,M", [(3, 6000, 60), (2, 4000, 33)])
def test_sparsevfc_matches_oracle(D, n, M, gram="fp64"):
    """The default path (``gram="fp64"``: normal equations contracted with fp64 products) against the float64 restatement."""
    from spateo_release_b200.tdr.sparsevfc import SparseVFC

    X, V = _field_data(n, D)
    ctrl_idx = np.random.default_rng(1).permutation(n)[:M]
    beta = 1.0 / 25.0**2
    grid = X[:50] + 0.5
    tm = {}
    got = SparseVFC(X, V, Grid=grid, M=M, beta=beta, lambda_=0.02, MaxIter=40, ecr=0.0, ctrl_idx=ctrl_idx, device="0",
                    gram=gram, timings=tm)
    want = mo.sparse_vfc(X, V, ctrl_idx, beta, lambda_=0.02, MaxIter=40, ecr=0.0, Grid=grid)
    assert got["iteration"] == want["iteration"] - 1 and tm["gram"] == gram
    scale = np.abs(want["V"]).max()
    eV = np.abs(got["V"] - want["V"]).max() / scale
    eS = abs(got["sigma2"] - want["sigma2"]) / want["sigma2"]
    eE = np.abs(got["E_traj"] - want["E_traj"]).max() / np.abs(want["E_traj"]).max()
    print(f"\n[vfc {gram} D={D} n={n} M={M}] V {eV:.2e}  sigma2 {eS:.2e}  E {eE:.2e}  P {np.abs(got['P'][:, 0] - want['P']).max():.2e}"
          f"  eigh fallbacks {tm['eigh_fallbacks']}")
    assert eV < 1e-4
    assert np.abs(got["grid_V"] - want["grid_V"]).max() < 1e-4 * scale
    assert eS < 1e-4
    assert np.abs(got["P"][:, 0] - want["P"]).max() < 1e-3
    assert eE < 1e-5
    assert set(["X", "valid_ind", "X_ctrl", "ctrl_idx", "Y", "beta", "V", "C", "P", "VFCIndex", "sigma2", "grid", "grid_V",
                "iteration", "tecr_traj", "E_traj"]) <= set(got)
    # outliers are recognised
    k = int(0.1 * n)
    assert got["P"][:k, 0].mean() < 0.1 and got["P"][k:, 0].mean() > 0.5


def test_sparsevfc_tensor_path_is_a_regularised_fit():
    """``gram="tensor"`` (opt-in): the tensor-core contraction delivers the normal equations with fp32-level relative noise
    (~1e-7). SparseVFC's own regulariser lambda sigma2 K sits at that same relative level of U^T P U, so the tensor path has
    to add a ridge above its noise floor and is therefore a slightly smoother fit, NOT the reference solution: it must
    recover the same inliers / noise level / smooth field, and its distance to the fp64 path is printed."""
    from spateo_release_b200.tdr.sparsevfc import SparseVFC

    X, V = _field_data(20000, 3)
    ctrl_idx = np.random.default_rng(1).permutation(20000)[:300]
    kw = dict(M=300, beta=1.0 / 25.0**2, lambda_=0.02, MaxIter=40, ecr=0.0, ctrl_idx=ctrl_idx, device="0")
    a = SparseVFC(X, V, gram="fp64", **kw)
    b = SparseVFC(X, V, gram="tensor", **kw)
    k = 2000
    dV = np.abs(a["V"][k:] - b["V"][k:]).max() / np.abs(a["V"]).max()
    print(f"\n[vfc tensor vs fp64, 20000 x 300] inlier field deviation {dV:.2e}  sigma2 {b['sigma2']:.4g} vs {a['sigma2']:.4g}")
    assert abs(b["sigma2"] - a["sigma2"]) < 0.2 * a["sigma2"]
    assert np.mean((a["P"][:, 0] > 0.75) == (b["P"][:, 0] > 0.75)) > 0.98
    assert dV < 0.25


def test_morphofield_alias_and_restart_wrapper():
    import spateo_release_b200 as st
    from spateo_release_b200.anndata_lite import AnnDataLite

    X, V = _field_data(3000, 3, seed=3)
    ad = AnnDataLite(np.zeros((3000, 2), dtype=np.float32), obsm={"align_spatial": X, "V_mapping": V})
    assert st.tdr.morphofield is st.tdr.morphofield_sparsevfc
    st.tdr.morphofield(ad, NX=X[:20], M=40, MaxIter=30, device="0")
    vf = ad.uns["VecFld_morpho"]
    assert vf["method"] == "sparsevfc" and vf["grid_V"].shape == (20, 3) and vf["V"].shape == (3000, 3)
    ref, pred = vf["Y"], vf["V"]
    cos = np.sum(ref * pred, 1) / (np.linalg.norm(ref, axis=1) * np.linalg.norm(pred, axis=1) + 1e-20)
    assert np.median(cos[300:]) > 0.9


def test_weighted_gram_matches_numpy():
    import torch

    from spateo_release_b200 import _capi
    from spateo_release_b200._capi import check, ptr

    lib = _capi.load_library()
    rng = np.random.default_rng(0)
    N, K, ld = 5000, 70, 5120
    U = rng.uniform(0, 1, size=(K, N)).astype(np.float32)
    w = rng.uniform(0, 1, size=N).astype(np.float32)
    X3 = rng.normal(size=(3, N)).astype(np.float32)
    dev = torch.device("cuda", 0)
    UT = torch.zeros((K, ld), dtype=torch.float32, device=dev); UT[:, :N] = torch.from_numpy(U).to(dev)
    wd = torch.zeros(ld, dtype=torch.float32, device=dev); wd[:N] = torch.from_numpy(w).to(dev)
    Xd = torch.zeros((3, ld), dtype=torch.float32, device=dev); Xd[:, :N] = torch.from_numpy(X3).to(dev)
    A = torch.empty((K, K), dtype=torch.float64, device=dev)
    B = torch.empty((K, 3), dtype=torch.float64, device=dev)
    check(lib.spb_weighted_gram(ptr(UT), ld, N, K, ptr(wd), ptr(Xd), ptr(A), ptr(B), _capi.current_stream_ptr()), "gram")
    U64 = U.astype(np.float64)
    assert np.abs(A.cpu().numpy() - (U64 * w.astype(np.float64)) @ U64.T).max() < 1e-9 * N
    assert np.abs(B.cpu().numpy() - U64 @ X3.astype(np.float64).T).max() < 1e-9 * N


def test_kernel_interpolation_general_output_dimension():
    """st.tdr.kernel_interpolation (interpolation_sparseVFC.py:13-100): 2-D coordinates -> 5 expression / label columns; the
    device regression equals the float64 numpy restatement run on the same control points, and a smooth gene is recovered."""
    import pandas as pd

    import spateo_release_b200 as st
    from spateo_release_b200.anndata_lite import AnnDataLite

    rng = np.random.default_rng(0)
    n = 4000
    xy = rng.uniform(0, 100, size=(n, 2))
    f = lambda p: np.stack([np.sin(p[:, 0] / 15.0), np.cos(p[:, 1] / 20.0), 0.01 * p[:, 0], np.exp(-((p - 50) ** 2).sum(1) / 800.0)], 1)
    genes = f(xy) + rng.normal(0, 0.02, size=(n, 4))
    lab = (xy[:, 0] > 50).astype(float)
    ad = AnnDataLite(genes.astype(np.float32), var=pd.DataFrame(index=["g0", "g1", "g2", "g3"]), obsm={"spatial": xy},
                     obs=pd.DataFrame({"side": lab}, index=[f"c{i}" for i in range(n)]))
    targets = rng.uniform(5, 95, size=(300, 2))
    ctrl = rng.permutation(n)[:120]
    out = st.tdr.kernel_interpolation(ad, targets, keys=["side", "g0", "g1", "g2", "g3"], beta=1.0 / 7.0**2, M=120,
                                      ctrl_idx=ctrl, MaxIter=30, ecr=0.0, device="0")
    info = np.c_[lab, genes.astype(np.float32).astype(np.float64)]
    want = mo.sparse_vfc(xy, info, ctrl, 1.0 / 7.0**2, lambda_=0.02, MaxIter=30, ecr=0.0, Grid=targets)
    got = np.c_[np.asarray(out.obs["side"]), np.asarray(out.X)]
    assert got.shape == (300, 5) and list(out.var.index) == ["g0", "g1", "g2", "g3"]
    assert np.abs(got - want["grid_V"]).max() < 2e-4 * np.abs(want["grid_V"]).max()
    assert np.median(np.abs(np.asarray(out.X) - f(targets))) < 0.1  # sanity only: 120 narrow kernels on a 100 x 100 field
