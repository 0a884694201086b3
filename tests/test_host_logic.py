"""CPU tests: C-ABI exports, header/ctypes agreement and the host-side helpers against the oracle."""

import numpy as np
import pytest

from oracle import fast_host as FH
from oracle import morpho_oracle as mo
from spateo_release_b200 import _capi
from spateo_release_b200.alignment import utils as U
from spateo_release_b200.alignment.morpho_alignment import compose_transformations
from spateo_release_b200.synthetic import make_slice_pair


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as g

    g.build()
    lib = _capi.load_library()
    names = _capi.declared_functions()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), n
        assert n in lib._spb_signatures, f"{n} has no ctypes signature"
    assert lib.spb_version() >= 100
    assert lib.spb_sizeof_em_params() == _capi.C.sizeof(_capi.SpbEmParams)
    assert lib.spb_sizeof_scalars() == _capi.C.sizeof(_capi.SpbScalars)


def test_no_oracle_import_in_product():
    import os
    import re

    root = os.path.join(_capi.REPO_ROOT, "spateo_release_b200")
    for dp, _, fs in os.walk(root):
        for f in fs:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle", src, re.M), f"{f} imports the oracle"


def test_voxel_data_matches_reference_loop():
    rng = np.random.default_rng(0)
    for D, n in ((2, 1500), (3, 900)):
        coords = rng.uniform(0, 50, size=(n, D)).astype(np.float32)
        ge = rng.poisson(1.0, size=(n, 17)).astype(np.float32)
        c_ref, g_ref = mo.voxel_data(coords, ge, voxel_num=max(min(int(n / 20), 1000), 100))
        c_new, g_new = FH.voxel_data(coords, ge, voxel_num=max(min(int(n / 20), 1000), 100))
        assert c_ref.shape == c_new.shape and np.array_equal(c_ref, c_new)
        assert np.abs(g_ref - g_new).max() < 1e-5


def test_inlier_from_NN_matches_oracle():
    rng = np.random.default_rng(1)
    x = rng.normal(size=(400, 2))
    th = 0.4
    R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    y = x @ R.T + 0.3 + rng.normal(0, 0.02, size=x.shape)
    y[:40] = rng.normal(size=(40, 2)) * 3
    d = rng.uniform(0, 1, size=(400, 1))
    a = mo.inlier_from_NN(x, y, d)
    b = FH.inlier_from_NN(x, y, d)
    for u, v in zip(a, b):
        assert np.allclose(u, v, rtol=1e-9, atol=1e-12)


def test_normalize_coords_matches_oracle():
    rng = np.random.default_rng(2)
    a = rng.uniform(0, 100, size=(300, 3)).astype(np.float32)
    b = rng.uniform(10, 80, size=(280, 3)).astype(np.float32)
    ca, cb, sc, mu = U.normalize_coords(a, b)
    oa, ob, osc, omu = mo.normalize_coords(a, b)
    assert np.abs(ca - oa).max() < 1e-5 and np.abs(cb - ob).max() < 1e-5
    assert np.allclose(sc, osc, rtol=1e-6) and np.allclose(mu, omu, rtol=1e-6)
    assert a[0, 0] != ca[0, 0]  # inputs are not mutated


@pytest.mark.parametrize("case", ["2d_full", "3d_svi", "3d_full_warp", "c1_2d_svi", "c1_2d_full_warp"])
def test_normalisation_is_bitwise_the_references(golden, case):
    """check_spatial_coords + normalize_coords of the PRODUCT reproduce the reference's float32 arrays to the last bit
    (the coarse initialisation's np.arange voxel grid flips between n and n + 1 points on a one-ulp change)."""
    from spateo_release_b200.anndata_lite import AnnDataLite

    g = golden(case)
    A = AnnDataLite(np.zeros((g["raw_coords_moving"].shape[0], 1), np.float32), obsm={"spatial": g["raw_coords_moving"]})
    B = AnnDataLite(np.zeros((g["raw_coords_fixed"].shape[0], 1), np.float32), obsm={"spatial": g["raw_coords_fixed"]})
    ca = U.check_spatial_coords(A).astype(np.float32)
    cb = U.check_spatial_coords(B).astype(np.float32)
    _, nb, sc, mu = U.normalize_coords(ca, cb)
    assert np.array_equal(nb, g["pre_coordsB"])
    assert np.array_equal(sc, g["pre_normalize_scales"]) and np.array_equal(mu, g["pre_normalize_means"])


def test_check_spatial_coords_errors():
    A, _ = make_slice_pair(50, 50, 5, dim=2)
    with pytest.raises(KeyError):
        U.check_spatial_coords(A, "nope")
    A.obsm["flat"] = np.c_[np.arange(50.0), np.zeros(50)]
    with pytest.raises(ValueError):
        U.check_spatial_coords(A, "flat")
    A.obsm["xyz0"] = np.c_[A.obsm["spatial"], np.zeros(50)]
    assert U.check_spatial_coords(A, "xyz0").shape == (50, 2)  # constant axis dropped


def test_common_genes_and_errors():
    assert U.intersect_lsts(["a", "b", "c"], ["c", "a"]) == ["a", "c"]
    with pytest.raises(ValueError):
        U.filter_common_genes(["a"], ["b"])


def test_solve_RT_and_chain_composition():
    rng = np.random.default_rng(3)
    Y = rng.normal(size=(100, 2))
    th = 0.7
    R0 = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
    X = Y @ R0.T + np.array([1.0, -2.0])
    R, t = U.solve_RT_by_correspondence(X, Y)
    assert np.allclose(Y @ R.T + t, X, atol=1e-9)
    # composing two links equals applying them one after the other (morpho_alignment.py:300-303)
    tr = [{"Rotation": R, "Translation": t}, {"Rotation": R0.T, "Translation": np.array([0.5, 0.5])}]
    (R1, t1), (R2, t2) = compose_transformations(tr)
    p = rng.normal(size=(5, 2))
    step = (p @ tr[1]["Rotation"].T + tr[1]["Translation"]) @ tr[0]["Rotation"].T + tr[0]["Translation"]
    assert np.allclose(p @ R2.T + t2, step)


def test_label_transfer_defaults():
    d = U.generate_label_transfer_dict(["x", "y"], ["x", "z"])
    assert abs(sum(d["x"].values()) - 1) < 1e-6 and d["x"]["x"] > d["x"]["z"]
    with pytest.raises(KeyError):
        U.check_label_transfer_dict(["x"], ["x", "q"], {"x": {"x": 1.0}})


def test_field_desc_layout_and_constants():
    """The third parsed struct and the new constants agree with the built library."""
    lib = _capi.load_library()
    assert lib.spb_sizeof_field_desc() == _capi.C.sizeof(_capi.SpbFieldDesc)
    names = [f[0] for f in _capi.SpbFieldDesc._fields_]
    assert names[:4] == ["D", "K", "nonrigid_only", "curvature_formula"] and "mean_transformed" in names
    assert _capi.CONST["SPB_COLMASK_WORDS"] * 32 * _capi.ROW_TILE >= 262144
    em = dict(_capi.SpbEmParams._fields_)
    assert em["colmask"] is _capi.C.c_void_p and em["sparse_k"] is _capi.C.c_int32


def test_argmax_key_decoding_and_transpose():
    """ArgmaxPi.decode inverts the kernels' (float bits << 32 | ~index) key; .T swaps rows and columns."""
    from spateo_release_b200.alignment.mapping import ArgmaxPi

    vals = np.array([0.0, 1.5e-30, 0.25, 1.0], dtype=np.float32)
    idx = np.array([0, 7, 99999, 123], dtype=np.int64)
    keys = (vals.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - idx.astype(np.uint64))
    arg, val = ArgmaxPi.decode(keys)
    assert np.array_equal(arg, idx) and np.array_equal(val, vals)
    # larger value wins; equal values -> lower index wins (what the 64-bit max implements)
    assert keys[3] > keys[2] > keys[1] > keys[0]
    k_lo = (np.uint64(vals[2:3].view(np.uint32)[0]) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.uint64(5))
    assert k_lo > keys[2]
    pi = ArgmaxPi((3, 2), [1, 0, 1], [0.5, 0.2, 0.0], [0, 2], [0.2, 0.5])
    t = pi.T
    assert t.shape == (2, 3) and np.array_equal(t.row_arg, pi.col_arg) and np.array_equal(t.col_val, pi.row_val)


def test_segment_choice_respects_the_column_cap():
    from spateo_release_b200.alignment.morpho_class import Morpho_pairwise

    seg = Morpho_pairwise._choose_segments(98, 100000, 132)  # H100 SXM
    assert (100000 + seg - 1) // seg <= 4096 and seg * 98 >= 296
    seg2 = Morpho_pairwise._choose_segments(98, 100000, 132, max_cols=1024)
    assert seg2 > seg and (100000 + seg2 - 1) // seg2 <= 1024
    assert Morpho_pairwise._choose_segments(1, 240, 132) >= 1


def test_svc_field_descriptor_and_oracle_jacobian():
    """The SparseVFC field rides on the GP kernel as its plain RBF part (unit scales, zero means, velocity not divided);
    the float64 restatement of its Jacobian is the derivative of its velocity (central differences)."""
    from oracle import field_oracle as fo
    from spateo_release_b200.tdr import morphofield_dg as dg

    rng = np.random.default_rng(5)
    vf = {"X_ctrl": rng.uniform(0, 10, (7, 3)), "C": rng.normal(size=(7, 3)), "beta": 0.08, "method": "sparsevfc"}
    f = dg._desc_svc(vf, 3, 2)
    assert (f.D, f.K, f.nonrigid_only, f.velocity_divisor) == (3, 7, 1, 1.0)
    assert f.scale_fixed == f.scale_transformed == 1.0 and list(f.mean_transformed) == [0.0] * 3 and f.beta == 0.08
    assert dg._is_svc(vf) and not dg._is_svc({"inducing_variables": 1, "Coff": 2, "method": "gaussian_process"})
    gp = {"inducing_variables": vf["X_ctrl"], "Coff": vf["C"], "beta": 0.08, "kernel_type": "euc", "R": np.eye(3),
          "t": np.zeros(3), "norm_dict": {"mean_transformed": np.zeros(3), "mean_fixed": np.zeros(3),
                                          "scale_transformed": 1.0, "scale_fixed": 1.0}}
    assert dg._desc(gp, 3, False, 2).velocity_divisor == 10000.0
    X = rng.uniform(0, 10, (6, 3))
    g = fo.svc_geometry(X, vf)
    # with unit scales the GP restatement's non-rigid part is the same field / 10000 and the same Jacobian
    assert np.allclose(fo.gp_velocity(X, gp, nonrigid_only=True) * 10000, g["V"], rtol=1e-12, atol=0)
    assert np.allclose(fo.jacobian(X, gp), g["J"], rtol=1e-12, atol=1e-15)
    h = 1e-5
    for j in range(3):
        e = np.zeros(3); e[j] = h
        fd = (fo.svc_velocity(X + e, vf) - fo.svc_velocity(X - e, vf)) / (2 * h)   # d v_i / d x_j for every point
        assert np.allclose(g["J"][:, j, :].T, fd, rtol=1e-6, atol=1e-9)
    assert np.allclose(g["div"], np.einsum("iin->n", g["J"]))


def test_apply_transformation_matches_reference_driver(golden):
    """morpho_align_apply_transformation / compose_transformations against the UNMODIFIED reference driver's output
    (tests/golden/make_golden_drivers.py; morpho_alignment.py:284-303): host-only code, identical arithmetic order."""
    from driver_helpers import models_from_golden
    from spateo_release_b200.alignment import morpho_alignment as ma

    g = golden("drivers")
    tr = [{"Rotation": g[f"tr{i}_Rotation"], "Translation": g[f"tr{i}_Translation"]} for i in range(3)]
    placed = ma.morpho_align_apply_transformation(models_from_golden(g), transformation=tr, verbose=False)
    for k in range(4):
        assert np.array_equal(np.asarray(placed[k].obsm["align_spatial"]), g[f"placed{k}"]), k
    # every link of the golden is a proper 2-D rotation, and slice 0 is left where it was
    for t in tr:
        assert np.allclose(t["Rotation"] @ t["Rotation"].T, np.eye(2), atol=1e-6) and np.linalg.det(t["Rotation"]) > 0
    assert np.array_equal(g["placed0"], g["in0_spatial"])


def test_solve_RT_by_correspondence_reproduces_reference_links(golden):
    """The link of pair i is solve_RT_by_correspondence(optimal_RnA[:, :2], raw[:, :2]) (morpho_alignment.py:205-207). The
    serial driver's rigid output of slice 1 is the same pair solved on the same coordinates, so the golden's own arrays pin
    our solver: rotating/translating the raw slice with the stored link must land on the stored rigid placement."""
    from spateo_release_b200.alignment import utils as AU

    g = golden("drivers")
    raw1, rigid1 = g["in1_spatial"], g["SNS_1_align_spatial_rigid"]
    R, t = AU.solve_RT_by_correspondence(rigid1, raw1)
    assert np.allclose(R, g["tr0_Rotation"], atol=1e-6) and np.allclose(t, g["tr0_Translation"], atol=1e-4)
    assert np.abs(raw1 @ R.T + t - rigid1).max() < 1e-3


def test_graph_unroll_choice():
    """Iterations per captured CUDA graph: 8 for light iterations (default SVI batch of the 100k pair, small pairs), 1 for
    the heavy full-EM iterations; an explicit ``graph_unroll`` attribute wins."""
    from types import SimpleNamespace

    from spateo_release_b200.alignment.morpho_class import Morpho_pairwise

    f = Morpho_pairwise._graph_unroll
    assert f(SimpleNamespace(graph_unroll=0, SVI_mode=False, NA=100000, NB=100000, batch_size=None)) == 1
    assert f(SimpleNamespace(graph_unroll=0, SVI_mode=True, NA=100000, NB=100000, batch_size=10000)) == 8
    assert f(SimpleNamespace(graph_unroll=0, SVI_mode=False, NA=5000, NB=5000, batch_size=None)) == 8
    assert f(SimpleNamespace(graph_unroll=3, SVI_mode=False, NA=100000, NB=100000, batch_size=None)) == 3


def test_two_125k_cost_matrices_do_not_fit_80_gb():
    """The prefetch estimate of the chain driver: one 125k-cell pair fits an 80 GB H100, two do not."""
    from spateo_release_b200.alignment.distributed import pair_device_bytes

    one = pair_device_bytes(125000, 125000, 2000)
    assert 4 * 125000 * 125440 < one < 80e9 < 2 * one


def test_library_built_with_other_nvcc_flags_is_rebuilt(tmp_path, monkeypatch):
    """A library with no record of its nvcc flags, or built for another target (say sm_100a), is stale."""
    import __graft_entry__ as ge

    lib, stamp = tmp_path / "lib.so", tmp_path / "lib.so.flags"
    lib.write_bytes(b"")
    monkeypatch.setattr(ge, "LIB", str(lib))
    monkeypatch.setattr(ge, "FLAGS_STAMP", str(stamp))
    assert ge._stale()
    stamp.write_text(" ".join(ge.NVCC_FLAGS).replace("sm_90a", "sm_100a"))
    assert ge._stale()
    stamp.write_text(" ".join(ge.NVCC_FLAGS))
    assert not ge._stale()
