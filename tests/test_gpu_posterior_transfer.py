"""Posterior transfer: P @ F_B and P^T @ F_A of the final E-step without forming P (spb_posterior_transfer_rows / _cols).

From an identical device state the transfer is checked against the E-step's own statistics (K_NA, K_NB, P @ XB), against
the device's dense P and the float64 oracle, in sparse mode, streamed in column chunks and column-sharded; and through the
public interface (validation, SVI, the drivers, an unchanged run without it)."""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import morpho_oracle as mo  # noqa: E402
from layout_helpers import force_width, run_sharded, sharded_solvers, stream as _stream, three_chunks  # noqa: E402
from parity_helpers import model_from_golden, poke_golden_estep  # noqa: E402


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def _set_features(m, FB=None, FA=None):
    """Give a prepared solver transfer features (caller's row order) and their device buffers."""
    from spateo_release_b200 import _capi

    m._FB_host = None if FB is None else np.ascontiguousarray(FB, dtype=np.float32)
    m._FA_host = None if FA is None else np.ascontiguousarray(FA, dtype=np.float32)
    for k in [k for k in m._state if k.startswith("xfer_")]:
        del m._state[k]
    c0, c1 = m._col_range()
    m._allocate_transfer(m._state, c1 - c0, m.ldx // _capi.ROW_TILE)


def _transfer(m, it, FB=None, FA=None, cull=None, dense=False):
    """One E-step on the current device state, then the transfer (and optionally the dense P) of its posterior.
    Returns (P_FB, PT_FA, P) with rows in the caller's order."""
    import torch

    from spateo_release_b200._capi import check, ptr

    _set_features(m, FB, FA)
    if cull is not None:
        m._params.cull = int(bool(cull))
    st = _stream()
    m._estep_only(it, st)
    m._transfer_begin()
    m._transfer_capture(m._params, it, st)
    P = None
    if dense:
        Pd = torch.empty((m.NA, m._NBb), dtype=torch.float32, device=m._dev)
        check(m._lib.spb_materialize_P(C.byref(m._params), it, ptr(Pd), m._NBb, st), "spb_materialize_P")
        P = m._unsorted(Pd.cpu().numpy())
    torch.cuda.synchronize()
    m.P_FB = m.PT_FA = None
    m._transfer_results(m._NBb)
    return m.P_FB, m.PT_FA, P


def _device_rows(m, name, d=None):
    t = m._state[name]
    t = t[:, : m.NA].T if d is not None else t[: m.NA]
    if d is not None:
        t = t[:, :d]
    return m._unsorted(t.contiguous().cpu().numpy())


def _within(got, want, scale, bar):
    got, want, scale = (np.asarray(a, dtype=np.float64) for a in (got, want, scale))
    bad = np.abs(got - want) > bar * scale + 1e-30
    assert not bad.any(), (int(bad.sum()), float(np.abs(got - want).max()), float(scale.max()))


def _golden_model(golden, case, it, **over):
    g = golden(case)
    m = model_from_golden(g, probability_parameters=[float(g["pre_beta2"])], **over)
    m.prepare()
    poke_golden_estep(m, g, it)
    return g, m


def _fixed_rows(m, it):
    """Fixed cell of every column of the E-step (the SVI batch of iteration ``it``, or all fixed cells)."""
    if m._params.svi:
        return m._state["batch_idx"][it].cpu().numpy().astype(np.int64)
    return np.arange(m.NB)


# ---------------------------------------------------------------------------------------------------------------------
# 1. self-consistency with the E-step's own statistics
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,it", [("3d_full_warp", 95), ("c1_2d_full_warp", 150)])
def test_ones_and_coordinates_reproduce_estep_statistics(golden, case, it):
    g, m = _golden_model(golden, case, it)
    D = m.D
    yb = np.asarray(g["pre_coordsB"], dtype=np.float32)
    FB = np.concatenate([np.ones((m.NB, 1), np.float32), yb], axis=1)
    P_FB, PT_FA, P = _transfer(m, it, FB=FB, FA=np.ones((m.NA, 1), np.float32), cull=1, dense=True)
    K_NA, PXB = _device_rows(m, "K_NA"), _device_rows(m, "PXB", D)
    K_NB = m._state["K_NB"][: m.NB].cpu().numpy()
    Pabs = np.abs(P.astype(np.float64))
    _within(P_FB[:, 0], K_NA, np.abs(K_NA), 1e-6)
    _within(P_FB[:, 1:], PXB, Pabs @ np.abs(yb.astype(np.float64)), 1e-6)
    _within(PT_FA[:, 0], K_NB, np.abs(K_NB), 1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# 2. against the device's own dense P, every panel edge; culling off and on: P^T @ F_A bit-identical (per column the fold
#    over row blocks adds exact zeros for the dropped tiles, as K_NB), P @ F_B within the bar (the column segments of a
#    culled list hold other columns, as for the E-step's row statistics)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,it", [("3d_full_warp", 60), ("c1_2d_full_warp", 150)])
def test_matches_dense_P_at_panel_edges(golden, case, it):
    g, m = _golden_model(golden, case, it)
    rng = np.random.default_rng(1)
    labels_B = np.eye(7, dtype=np.float32)[rng.integers(0, 7, m.NB)]
    labels_A = np.eye(5, dtype=np.float32)[rng.integers(0, 5, m.NA)]
    for F in (1, 15, 16, 17, 33, 300):
        FB = rng.normal(size=(m.NB, F)).astype(np.float32)
        FA = rng.normal(size=(m.NA, F)).astype(np.float32)
        results = []
        for cull in (0, 1):
            poke_golden_estep(m, g, it)
            P_FB, PT_FA, P = _transfer(m, it, FB=FB, FA=FA, cull=cull, dense=True)
            P64 = P.astype(np.float64)
            _within(P_FB, P64 @ FB, np.abs(P64) @ np.abs(FB), 1e-5)
            _within(PT_FA, P64.T @ FA, np.abs(P64).T @ np.abs(FA), 1e-5)
            results.append((P_FB, PT_FA))
        _within(results[0][0], results[1][0], np.abs(P64) @ np.abs(FB), 1e-5)
        assert np.array_equal(results[0][1], results[1][1]), F
    poke_golden_estep(m, g, it)
    P_FB, PT_FA, P = _transfer(m, it, FB=labels_B, FA=labels_A, cull=1, dense=True)
    P64 = P.astype(np.float64)
    _within(P_FB, P64 @ labels_B, P64 @ labels_B, 1e-5)
    _within(PT_FA, P64.T @ labels_A, P64.T @ labels_A, 1e-5)
    assert m.NA % 512 != 0


# ---------------------------------------------------------------------------------------------------------------------
# 3. against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("it", [0, 95])
def test_matches_float64_oracle(golden, it):
    g, m = _golden_model(golden, "3d_full_warp", it)
    rng = np.random.default_rng(2)
    FB = rng.random((m.NB, 9)).astype(np.float32)
    FA = rng.random((m.NA, 9)).astype(np.float32)
    P_FB, PT_FA, _ = _transfer(m, it, FB=FB, FA=FA, cull=1)
    f8 = lambda k: g[k].astype(np.float64)
    XAHat, alpha, SD = f8(f"it{it}_in_XAHat"), f8(f"it{it}_in_alpha"), f8(f"it{it}_in_SigmaDiag")
    sigma2, gamma = float(g[f"it{it}_in_sigma2"]), float(g[f"it{it}_in_gamma"])
    yb = f8("pre_coordsB")
    spatial = ((XAHat[:, None, :] - yb[None, :, :]) ** 2).sum(-1)
    [ed] = mo.calc_distance(f8("exp_moving"), f8("exp_fixed"), "kl")
    P64 = mo.get_P_core(
        Dim=float(m.D), spatial_dist=spatial, exp_dist=[ed], sigma2=sigma2, model_mul=(alpha * np.exp(-SD / sigma2))[:, None],
        gamma=gamma, samples_s=float(g["pre_samples_s"]), sigma2_variance=float(g[f"it{it}_in_sigma2_variance"]),
        probability_type=["gauss"], probability_parameters=[float(g["pre_beta2"])],
    )[0]
    want_B, want_A = P64 @ FB, P64.T @ FA
    assert np.abs(P_FB - want_B).max() < 1e-4 * np.abs(want_B).max()
    assert np.abs(PT_FA - want_A).max() < 1e-4 * np.abs(want_A).max()


# ---------------------------------------------------------------------------------------------------------------------
# 4. sparse mode: the kept entries w >= tau_j
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case,it", [("2d_full_sparse48", 60), ("3d_svi_sparse32", 60)])
def test_sparse_mode_transfers_the_kept_entries(golden, case, it):
    g, m = _golden_model(golden, case, it)
    rng = np.random.default_rng(3)
    FB = np.concatenate([np.ones((m.NB, 1)), rng.normal(size=(m.NB, 20))], axis=1).astype(np.float32)
    FA = np.concatenate([np.ones((m.NA, 1)), rng.normal(size=(m.NA, 20))], axis=1).astype(np.float32)
    P_FB, PT_FA, _ = _transfer(m, it, FB=FB, FA=FA, cull=1)
    m._capture_P(it, _stream())  # the COO entries of the same posterior
    Ps = m._sparse_P_to_coo(np.float64).tocsr()
    K_NA = _device_rows(m, "K_NA")
    K_NB = m._state["K_NB"][: m._NBb].cpu().numpy()
    _within(P_FB[:, 0], K_NA, np.abs(K_NA), 1e-6)
    _within(PT_FA[:, 0], K_NB, np.abs(K_NB), 1e-6)
    FBc = FB[_fixed_rows(m, it)].astype(np.float64)
    absP = abs(Ps)
    _within(P_FB, Ps @ FBc, absP @ np.abs(FBc), 1e-5)
    _within(PT_FA, Ps.T @ FA.astype(np.float64), absP.T @ np.abs(FA.astype(np.float64)), 1e-5)


# ---------------------------------------------------------------------------------------------------------------------
# 5. determinism and row order
# ---------------------------------------------------------------------------------------------------------------------
def test_reruns_are_bit_identical_and_row_order_is_the_callers(golden):
    it = 150
    g, m = _golden_model(golden, "c1_2d_full_warp", it)
    rng = np.random.default_rng(4)
    FB = rng.normal(size=(m.NB, 20)).astype(np.float32)
    FA = rng.normal(size=(m.NA, 20)).astype(np.float32)
    a = _transfer(m, it, FB=FB, FA=FA, cull=1)
    poke_golden_estep(m, g, it)
    b = _transfer(m, it, FB=FB, FA=FA, cull=1, dense=True)
    assert m._perm is not None
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    _, u = _golden_model(golden, "c1_2d_full_warp", it, spatial_sort=False)
    c = _transfer(u, it, FB=FB, FA=FA, cull=1)
    P64 = b[2].astype(np.float64)
    _within(c[0], b[0], np.abs(P64) @ np.abs(FB), 2e-5)
    _within(c[1], b[1], np.abs(P64).T @ np.abs(FA), 2e-5)


# ---------------------------------------------------------------------------------------------------------------------
# 6. streamed cost matrix
# ---------------------------------------------------------------------------------------------------------------------
def _stream_pair():
    from spateo_release_b200.synthetic import make_slice_pair

    return make_slice_pair(2600, 2400, 24, dim=3, seed=2, z_thickness=15.0, warp_amplitude=1.0)


def _pair_solver(A, B, **kw):
    import spateo_release_b200 as st

    np.random.seed(0)
    opts = dict(max_iter=40, K=15, nn_init=False, verbose=False, device="0", SVI_mode=False, materialize_P=False)
    opts.update(kw)
    return st.align.Morpho_pairwise(sampleA=B, sampleB=A, **opts)


def test_streamed_chunks_match_resident(monkeypatch):
    import torch

    A, B = _stream_pair()
    rng = np.random.default_rng(5)
    FB = rng.normal(size=(A.shape[0], 19)).astype(np.float32)
    FA = rng.normal(size=(B.shape[0], 19)).astype(np.float32)
    res = _pair_solver(A, B)
    res.prepare()
    res.run_em(n_iter=25)
    torch.cuda.synchronize()
    XA = res._unsorted(res._state["XAHat"][: res.D, : res.NA].T.contiguous().cpu().numpy())
    alpha, SD = _device_rows(res, "alpha"), _device_rows(res, "SigmaDiag")
    sc = res._read_scalars()
    from parity_helpers import poke_estep_state

    state = (XA, alpha, SD, float(sc.sigma2), float(sc.gamma), float(sc.sigma2_variance))
    poke_estep_state(res, *state)
    want = _transfer(res, 25, FB=np.concatenate([FB, np.abs(FB)], axis=1), FA=FA, cull=1)
    scale = want[0][:, 19:]  # P @ |F_B|
    want = (want[0][:, :19], want[1])

    cols = res.NB
    force_width(monkeypatch, res.NA, cols, res._cost_features(), three_chunks(cols))
    s = _pair_solver(A, B)
    s.prepare()
    assert s._streamed and s.cost_plan.n_chunks == 3
    poke_estep_state(s, *state)
    _set_features(s, FB, FA)
    st = _stream()
    s._estep_only(25, st, on_chunk=s._capture_begin())
    torch.cuda.synchronize()
    s._transfer_results(cols)
    assert np.array_equal(s.PT_FA, want[1])
    _within(s.P_FB, want[0], scale, 1e-6)


# ---------------------------------------------------------------------------------------------------------------------
# 7. column-sharded pair (lock-step shards of one process)
# ---------------------------------------------------------------------------------------------------------------------
def _sharded_solvers(world, **opts):
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(2600, 2300, 40, dim=3, seed=5, z_thickness=15.0, warp_amplitude=1.0)
    rng = np.random.default_rng(6)
    ones = lambda n: np.ones((n, 1), np.float32)
    kw = dict(max_iter=30, K=15, nn_init=True, verbose=False, device="0", materialize_P=False,
              transfer_B=np.concatenate([ones(A.shape[0]), rng.random((A.shape[0], 17))], axis=1).astype(np.float32),
              transfer_A=np.concatenate([ones(B.shape[0]), rng.random((B.shape[0], 2))], axis=1).astype(np.float32))
    kw.update(opts)
    return sharded_solvers(A, B, world, **kw)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("opts", [dict(SVI_mode=False), dict(SVI_mode=True, return_mapping=True)], ids=["full", "svi_rm"])
def test_column_sharded_transfer_matches_unsharded(world, opts):
    ref, shards = _sharded_solvers(world, **opts)
    ref.run()
    run_sharded(shards)
    m0 = shards[0]
    for m in shards:  # every replica holds the same bits
        assert np.array_equal(m.P_FB, m0.P_FB) and np.array_equal(m.PT_FA, m0.PT_FA)
    assert m0.P_FB.shape == ref.P_FB.shape and m0.PT_FA.shape == ref.PT_FA.shape
    # the gathered columns and the rank-summed rows are the shards' own posterior's: the ones columns are K_NB and K_NA
    _within(m0.PT_FA[:, 0], m0.K_NB, m0.K_NB, 1e-6)
    _within(m0.P_FB[:, 0], m0.K_NA, m0.K_NA, 1e-5)
    # the sharded EM follows the unsharded one to the bars of the whole-run shard tests; the transfer follows it too
    for got, want in ((m0.P_FB, ref.P_FB), (m0.PT_FA, ref.PT_FA)):
        assert np.abs(got - want).max() < 1e-3 * np.abs(want).max()


# ---------------------------------------------------------------------------------------------------------------------
# 8. public interface
# ---------------------------------------------------------------------------------------------------------------------
def test_svi_transfer_is_the_closing_posteriors():
    import torch

    A, B = _stream_pair()
    rng = np.random.default_rng(7)
    FB = rng.random((A.shape[0], 4)).astype(np.float32)
    with pytest.raises(ValueError, match="return_mapping"):
        _pair_solver(A, B, SVI_mode=True, transfer_B=FB)
    m = _pair_solver(A, B, SVI_mode=True, return_mapping=True, transfer_B=FB, max_iter=20)
    m.run()
    assert m.P_FB.shape == (B.shape[0], 4) and m.PT_FA is None and m.P_FB.dtype == np.float32
    # the same E-step (last iteration's index, full columns, final parameters) recomputed with the dense P
    got = _transfer(m, 19, FB=FB, cull=1, dense=True)
    torch.cuda.synchronize()
    assert np.array_equal(got[0], m.P_FB)
    _within(m.P_FB, got[2].astype(np.float64) @ FB, got[2].astype(np.float64) @ FB, 1e-5)


def test_run_without_transfer_is_unchanged_and_launches_only_the_transfer_kernels():
    import torch

    from spateo_release_b200 import _capi

    A, B = _stream_pair()
    lib = _capi.load_library()
    out = []
    for kw in (dict(), dict(transfer_B=np.ones((A.shape[0], 1), np.float32), transfer_A=np.ones((B.shape[0], 1), np.float32))):
        m = _pair_solver(A, B, materialize_P=True, **kw)
        m.prepare()
        torch.cuda.synchronize()
        n0 = lib.spb_launch_count()
        m.run()
        torch.cuda.synchronize()
        out.append((m, lib.spb_launch_count() - n0))
    (a, na), (b, nb) = out
    assert nb - na == 4  # one panel each way: the transfer kernel and its fold
    for k in ("XAHat", "K_NA", "K_NB", "P", "sigma2"):
        assert np.array_equal(getattr(a, k), getattr(b, k)), k
    assert a.P_FB is None and a.PT_FA is None
    _within(b.P_FB[:, 0], b.K_NA, b.K_NA, 1e-6)
    _within(b.PT_FA[:, 0], b.K_NB, b.K_NB, 1e-6)


def test_morpho_align_chain_stores_transferred_labels():
    import pandas as pd

    import spateo_release_b200 as st
    from spateo_release_b200.alignment.morpho_alignment import _normalise_rows
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(1500, 1400, 24, dim=2, seed=8)
    C3, _ = make_slice_pair(1300, 1200, 24, dim=2, seed=9)
    rng = np.random.default_rng(8)
    for sl in (A, B, C3):
        sl.obs["ct"] = pd.Categorical(rng.choice(["a", "b", "c"], sl.shape[0]))
    kw = dict(max_iter=20, K=15, verbose=False, device="0", SVI_mode=False)
    with pytest.raises(ValueError, match="ambiguous"):
        st.align.morpho_align([A, B, C3], transfer_B=np.ones((A.shape[0], 1)), **kw)
    np.random.seed(0)
    aligned, _ = st.align.morpho_align([A, B, C3], transfer_B="ct", transfer_A="ct", **kw)
    assert "ct_from_fixed" in aligned[1].obsm and "ct_from_moving" in aligned[1].obsm  # moving in pair 0, fixed in pair 1
    assert "ct_from_moving" in aligned[0].obsm and "ct_from_fixed" in aligned[2].obsm
    for k in (1, 2):
        lab = aligned[k].obs["ct_from_fixed"]
        assert list(lab.cat.categories) == ["a", "b", "c"]
    # the first pair at the solver level, from the same seed and inputs
    np.random.seed(0)
    from spateo_release_b200.alignment.morpho_alignment import _seed_keys, _working_copy

    fixed, moving = _working_copy(A), _working_copy(B)
    _seed_keys([fixed, moving], "spatial", "align_spatial")
    s = st.align.Morpho_pairwise(sampleA=moving, sampleB=fixed, spatial_key="align_spatial", key_added="align_spatial",
                                 iter_key_added="iter_spatial", vecfld_key_added="VecFld_morpho", materialize_P="auto",
                                 transfer_B="ct", transfer_A="ct", **kw)
    s.run()
    want = _normalise_rows(s.P_FB, s.K_NA)
    assert np.array_equal(aligned[1].obsm["ct_from_fixed"], want)
    assert np.array_equal(aligned[0].obsm["ct_from_moving"], _normalise_rows(s.PT_FA, s.K_NB))
    cats = np.asarray(["a", "b", "c"])
    assert (np.asarray(aligned[1].obs["ct_from_fixed"]) == cats[want.argmax(axis=1)]).all()
