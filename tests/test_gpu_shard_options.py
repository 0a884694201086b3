"""GPU: the options of a column-sharded pair beyond the full EM — SVI, return_mapping, guidance, the sparse posterior and
the cell mapping. One process emulates W ranks on ONE GPU: W solver objects, each holding a block of the fixed cells. The
iterations are driven through the solver's own two halves of a sharded iteration (``_shard_iteration_local`` up to the
fold, ``_shard_iteration_finish`` after it) with the cross-rank sum of the row statistics done here in rank order; the
closing ``_finish`` runs one thread per shard, whose collectives (``_shard_comm``) exchange through host memory."""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from layout_helpers import finish_all, run_sharded, sharded_solvers, stream as _stream  # noqa: E402


def _pair():
    from spateo_release_b200.synthetic import make_slice_pair

    return make_slice_pair(2600, 2300, 40, dim=3, seed=5, z_thickness=15.0, warp_amplitude=1.0)


def _guidance(A, B, n=24):
    rng = np.random.default_rng(3)
    return [np.asarray(A.obsm["spatial"])[rng.choice(A.shape[0], n, replace=False)],
            np.asarray(B.obsm["spatial"])[rng.choice(B.shape[0], n, replace=False)]]


def _solvers(world, **opts):
    """The unsharded solver and W shards with the same host initialisation (the driver broadcasts rank 0's)."""
    A, B = _pair()
    kw = dict(max_iter=110, K=15, nn_init=True, verbose=False, device="0", materialize_P=False)
    kw.update(opts)
    if kw.pop("guide", False):
        kw.update(guidance_pair=_guidance(A, B), guidance_effect="both")
    ref, shards = sharded_solvers(A, B, world, **kw)
    return A, ref, shards


# ---------------------------------------------------------------------------------------------------------------------
# whole runs against the unsharded solver
# ---------------------------------------------------------------------------------------------------------------------
_RUNS = {
    "svi": dict(SVI_mode=True),
    "svi_return_mapping": dict(SVI_mode=True, return_mapping=True),
    "svi_guidance_both": dict(SVI_mode=True, guide=True),
    "full_guidance_both": dict(SVI_mode=False, guide=True),
}


@pytest.mark.parametrize("world", [1, 3])
@pytest.mark.parametrize("case", list(_RUNS))
def test_sharded_run_matches_unsharded(world, case):
    A, ref, shards = _solvers(world, **_RUNS[case])
    ref.run()
    run_sharded(shards)
    scale = np.abs(ref.XAHat).max()
    for m in shards:
        assert np.abs(m.XAHat - ref.XAHat).max() < 2e-5 * scale
        assert np.abs(m.optimal_RnA - ref.optimal_RnA).max() < 2e-5 * scale
        assert abs(float(m.sigma2) - float(ref.sigma2)) < 1e-4 * float(ref.sigma2)
        assert np.abs(m.K_NA - ref.K_NA).max() < 1e-4 * np.abs(ref.K_NA).max()
        assert m.K_NB.shape == ref.K_NB.shape
        assert np.abs(m.K_NB - ref.K_NB).max() < 1e-4 * np.abs(ref.K_NB).max()
        if ref.SVI_mode:
            assert np.array_equal(m.batch_idx, ref.batch_idx)
    for m in shards[1:]:  # replicas are bit-identical
        for key in ("XAHat", "optimal_RnA", "K_NA", "K_NB", "sigma2"):
            assert np.array_equal(getattr(m, key), getattr(shards[0], key)), key


@pytest.mark.parametrize("case", ["svi_sparse_mapping", "svi_return_mapping"])
def test_driver_run_world1_matches_unsharded(case):
    """The path users call: ``morpho_align_pair_sharded(SVI_mode=True).run()`` (the solver's sharded ``_iteration`` and
    ``_finish``) on one GPU without a process group, against the unsharded solver with the same seed."""
    import spateo_release_b200 as st
    from spateo_release_b200.alignment.distributed import morpho_align_pair_sharded

    A, B = _pair()
    kw = dict(SVI_mode=True, max_iter=110, K=15, nn_init=True, verbose=False)
    if case == "svi_sparse_mapping":
        kw.update(sparse_calculation_mode=True, sparse_top_k=32, materialize_P=True, compute_mapping=True)
    else:
        kw.update(return_mapping=True, materialize_P=False)
    np.random.seed(0)
    ref = st.align.Morpho_pairwise(sampleA=B, sampleB=A, device="0", **kw)
    P_ref = ref.run()
    np.random.seed(0)
    m = morpho_align_pair_sharded(A, B, device="0", **kw)
    assert m.column_shard[:2] == (0, 1) and m.SVI_mode
    P = m.run()
    scale = np.abs(ref.XAHat).max()
    assert np.abs(m.XAHat - ref.XAHat).max() < 2e-5 * scale
    assert np.abs(m.optimal_RnA - ref.optimal_RnA).max() < 2e-5 * scale
    assert abs(float(m.sigma2) - float(ref.sigma2)) < 1e-4 * float(ref.sigma2)
    assert np.abs(m.K_NA - ref.K_NA).max() < 1e-4 * np.abs(ref.K_NA).max()
    assert m.K_NB.shape == ref.K_NB.shape and np.abs(m.K_NB - ref.K_NB).max() < 1e-4 * np.abs(ref.K_NB).max()
    assert np.array_equal(m.batch_idx, ref.batch_idx)
    if case == "svi_sparse_mapping":
        assert P.shape == P_ref.shape == (ref.NA, ref.batch_size) and P.nnz == P_ref.nnz == 32 * ref.batch_size
        assert np.array_equal(P.col, P_ref.col) and np.abs(P.data - P_ref.data).max() < 1e-4 * np.abs(P_ref.data).max()
        assert m.mapping.shape == ref.mapping.shape
        for key in ("row_val", "col_val"):
            got, want = getattr(m.mapping, key), getattr(ref.mapping, key)
            assert np.abs(got - want).max() < 1e-4 * np.abs(want).max(), key
    else:
        assert P is None and P_ref is None and m.K_NB.shape == (ref.NB,)


def test_inducing_points_rebuilt_from_another_rank():
    """The sharded driver hands every rank rank 0's inducing points: the kernel matrices rebuilt from them equal those of
    a solver that drew them itself, guidance kernel included."""
    import spateo_release_b200 as st

    A, B = _pair()
    kw = dict(K=15, verbose=False, device="0", guidance_pair=_guidance(A, B), guidance_effect="both")
    np.random.seed(0)
    a = st.align.Morpho_pairwise(sampleA=B, sampleB=A, **kw)
    np.random.seed(1)
    b = st.align.Morpho_pairwise(sampleA=B, sampleB=A, **kw)
    assert not np.array_equal(a.inducing_variables_idx, b.inducing_variables_idx)
    b._construct_kernel(a.inducing_variables_idx)
    assert np.array_equal(a.inducing_variables, b.inducing_variables) and np.array_equal(a.GammaSparse, b.GammaSparse)
    assert np.array_equal(a.U_I, b.U_I) and np.array_equal(a.U, b.U)


# ---------------------------------------------------------------------------------------------------------------------
# one E-step from an identical state
# ---------------------------------------------------------------------------------------------------------------------
_ROW_STATE = ("XAHat", "lm", "mm", "alpha", "SigmaDiag", "VnA", "RnA", "PXB_term", "sc")


def _identical_state(world, it=40, **opts):
    """The unsharded solver after ``it`` iterations, its row state copied into every shard, then the E-step of iteration
    ``it`` on all of them (the shards' row statistics summed in rank order). Returns (ref, shards, ref_rowstat)."""
    import torch

    A, ref, shards = _solvers(world, **opts)
    ref.prepare_device()
    ref.run_em(n_iter=it)
    for m in shards:
        for k in _ROW_STATE:
            m._state[k].copy_(ref._state[k])
    st = _stream()
    ref._estep_local(it, st)
    # the unsharded E-step's row statistics folded in fp64 the same way (spb_row_fold)
    rowstat = torch.zeros((2 * 8 * ref.ldx,), dtype=torch.float64, device=ref._state["XAHat"].device)
    ref._params.rowstat = rowstat.data_ptr()
    from spateo_release_b200._capi import check

    check(ref._lib.spb_row_fold(C.byref(ref._params), 0, st), "fold")
    check(ref._lib.spb_row_finalize(C.byref(ref._params), st), "finalize")
    _lockstep_iterations_estep(shards, it)
    torch.cuda.synchronize()
    return ref, shards, rowstat[: 8 * ref.ldx]


def _lockstep_iterations_estep(shards, it):
    import torch

    st = _stream()
    views = [m._shard_iteration_local(it, st) for m in shards]
    total = torch.zeros_like(views[0])
    for v in views:
        total += v
    for v in views:
        v.copy_(total)
    for m in shards:
        m._shard_finish_rows(st)
    shards[0]._summed_rowstat = total


def _positions(m, it):
    from spateo_release_b200.alignment.distributed import column_block

    if m._shard_pos is not None:
        return m._shard_pos[it]
    return np.arange(*column_block(m.NB, int(m.column_shard[0]), int(m.column_shard[1])), dtype=np.int32)


def test_svi_estep_from_identical_state():
    import torch

    from spateo_release_b200._capi import SpbEmParams, check

    it = 40
    ref, shards, ref_stat = _identical_state(3, it=it, SVI_mode=True)
    knb_ref = ref._state["K_NB"].cpu().numpy()
    cc_ref = ref._state["colconst"].cpu().numpy()
    covered = []
    for m in shards:
        pos = _positions(m, it)
        real = pos >= 0
        covered.append(pos[real])
        # every column's outputs depend only on the row state and fold over the row blocks in a fixed order: same bits
        assert np.array_equal(m._state["K_NB"].cpu().numpy()[: pos.shape[0]][real], knb_ref[pos[real]])
        assert np.array_equal(m._state["colconst"].cpu().numpy()[: pos.shape[0]][real], cc_ref[pos[real]])
    assert np.array_equal(np.sort(np.concatenate(covered)), np.arange(ref.batch_size))
    got = shards[0]._summed_rowstat.cpu().numpy()[: 7 * ref.ldx].reshape(7, ref.ldx)[:, : ref.NA]
    want = ref_stat.cpu().numpy()[: 7 * ref.ldx].reshape(7, ref.ldx)[:, : ref.NA]
    # sweep 2 accumulates each row over the columns of one column segment in fp32 before the fp64 fold, and a shard's
    # segments hold other columns than the unsharded run's: the sums differ at fp32 rounding, not at fp64 rounding. The
    # bound is per row: its own magnitude (statistics 0-3 are sums of non-negative terms; |sum_j P_ij y_j| of P @ XB is
    # at most K_NA_i max |y|), plus a floor at fp64 rounding of the largest row for rows of denormal fp32 terms
    ymax = np.abs(ref.coordsB).max()
    for q in range(7):
        mag = np.abs(want[q]) if q < 4 else want[3] * ymax
        assert (np.abs(got[q] - want[q]) <= 1e-5 * mag + 1e-12 * np.abs(want[q]).max()).all(), q

    # a padded iteration gives the same row partials as its members run without the null column
    st = _stream()
    m, it_pad = next((m, t) for m in shards for t in range(m.max_iter) if (m._shard_pos[t] < 0).any())
    pos = m._shard_pos[it_pad]
    n = int((pos >= 0).sum())
    m._state["rowpart"].zero_()
    m._estep_local(it_pad, st)
    torch.cuda.synchronize()
    padded_rowpart = m._state["rowpart"].clone()
    padded_knb = m._state["K_NB"][:n].clone()
    sched = np.zeros((m.max_iter, max(n, 1)), dtype=np.int32)
    sched[it_pad, :n] = m._state["batch_idx"][it_pad, :n].cpu().numpy()
    sched_d = torch.from_numpy(sched).to(m._state["XAHat"].device)
    q = SpbEmParams.from_buffer_copy(m._params)
    q.NBb, q.batch_idx = n, sched_d.data_ptr()
    m._state["rowpart"].zero_()
    m._state["colgeom"][n:].zero_()  # the record after the last column is the zero pad entry, as in a launch of width n
    m._state["colconst"][n:].zero_()
    for fn, args in (("spb_iter_begin", (it_pad,)), ("spb_gather_cols", (it_pad,)), ("spb_estep_col_lists", ()),
                     ("spb_estep_sweep1", (it_pad,)), ("spb_col_finalize", ()), ("spb_estep_sweep2", (it_pad,))):
        check(getattr(m._lib, fn)(C.byref(q), *args, st), fn)
    torch.cuda.synchronize()
    assert torch.equal(m._state["rowpart"], padded_rowpart)
    assert torch.equal(m._state["K_NB"][:n], padded_knb)


@pytest.mark.parametrize("svi", [True, False])
def test_sparse_posterior_from_identical_state(svi):
    from spateo_release_b200.alignment.distributed import assemble_columns

    it = 40
    k = 32
    ref, shards, _ = _identical_state(3, it=it, SVI_mode=svi, sparse_calculation_mode=True, sparse_top_k=k,
                                      materialize_P=True)
    st = _stream()
    ref._capture_P(it, st)
    n_cols = ref.batch_size if svi else ref.NB
    parts_r, parts_v, positions = [], [], []
    for m in shards:
        m._capture_P(it, st)
        parts_r.append(m._P_rows.cpu().numpy())
        parts_v.append(m._P_vals.cpu().numpy())
        positions.append(_positions(m, it))
    import torch

    rows = torch.from_numpy(assemble_columns(parts_r, positions, n_cols))
    vals = torch.from_numpy(assemble_columns(parts_v, positions, n_cols))
    P = shards[0]._sparse_P_to_coo(np.float32, rows, vals)
    P_ref = ref._sparse_P_to_coo(np.float32)
    assert P.shape == P_ref.shape == (ref.NA, n_cols) and P.nnz == k * n_cols
    assert np.array_equal(np.sort(P.data.reshape(n_cols, k), axis=1), np.sort(P_ref.data.reshape(n_cols, k), axis=1))
    assert np.array_equal(P.toarray(), P_ref.toarray())  # the same (row, value) entries of every column


@pytest.mark.parametrize("svi", [True, False])
def test_sparse_posterior_whole_run(svi):
    k = 32
    A, ref, shards = _solvers(3, SVI_mode=svi, sparse_calculation_mode=True, sparse_top_k=k, materialize_P=True)
    P_ref = ref.run()
    run_sharded(shards)
    n_cols = ref.batch_size if svi else ref.NB
    top = np.abs(P_ref.data).max()
    for m in shards:
        assert m.P.shape == P_ref.shape == (ref.NA, n_cols) and m.P.nnz == k * n_cols
        assert np.array_equal(m.P.col, P_ref.col)
        assert np.abs(m.P.data - P_ref.data).max() < 1e-4 * top
    for m in shards[1:]:
        assert np.array_equal(m.P.data, shards[0].P.data) and np.array_equal(m.P.row, shards[0].P.row)


@pytest.mark.parametrize("svi", [True, False])
def test_mapping_from_identical_state(svi):
    import spateo_release_b200 as st_

    it = 40
    ref, shards, _ = _identical_state(3, it=it, SVI_mode=svi, compute_mapping=True, max_iter=it + 1)
    st = _stream()
    ref._capture_P(it, st)
    for m in shards:
        m._capture_P(it, st)
    # the unmapped entry point and an identity map give the same keys
    import torch

    from spateo_release_b200._capi import check

    rb, cb = torch.zeros_like(ref._rowbest), torch.zeros_like(ref._colbest)
    ident = torch.arange(ref._NBb, dtype=torch.int32, device=rb.device)
    check(ref._lib.spb_posterior_argmax_mapped(C.byref(ref._params), it, C.c_void_p(ident.data_ptr()),
                                               C.c_void_p(rb.data_ptr()), C.c_void_p(cb.data_ptr()), st), "mapped")
    assert torch.equal(rb, ref._rowbest) and torch.equal(cb, ref._colbest)
    ref._finish()
    finish_all(shards)  # merges the row keys (maximum) and gathers the column keys
    Y = np.asarray(_pair()[0].obsm["spatial"])
    Y = Y[ref.batch_idx] if svi else Y
    want = st_.align.get_optimal_mapping_relationship(ref.optimal_RnA, Y, ref.mapping)
    for m in shards:
        mp = m.mapping
        assert mp.shape == ref.mapping.shape
        for key in ("row_arg", "row_val", "col_arg", "col_val"):
            assert np.array_equal(getattr(mp, key), getattr(ref.mapping, key)), key
        got = st_.align.get_optimal_mapping_relationship(m.optimal_RnA, Y, mp)
        for u, v in zip(got, want):
            assert np.array_equal(u, v)


def test_dense_posterior_refused_on_a_shard():
    import spateo_release_b200 as st

    A, B = _pair()
    m = st.align.Morpho_pairwise(sampleA=B, sampleB=A, column_shard=(0, 2, "nccl"), max_iter=5, verbose=False, device="0",
                                 SVI_mode=True, materialize_P=True)
    with pytest.raises(NotImplementedError, match="materialize_P"):
        m.prepare()
