"""GPU: ``morpho_align_column_sharded`` — ``morpho_align``'s serial chain with every pair column-sharded — against
``morpho_align`` on a 3-slice 3-D chain. W = 1 runs the public driver without a process group. W = 3 is emulated in one
process: one thread per rank runs the driver's per-pair routine (``sharded_chain_pair``) with collectives that exchange
through host memory, so every broadcast, sum and gather of a real run takes place between the three shards."""

import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from layout_helpers import LockStep, force_width, three_chunks  # noqa: E402

KEY = "align_spatial"
BASE = dict(max_iter=110, K=15, verbose=False, device="0", iter_key_added=None)


def _chain(n_slices=3):
    """Serial 3-D sections of one warped tissue (2,300-2,600 cells each), each with an ``.obs`` label of its own x band."""
    import pandas as pd

    from spateo_release_b200.synthetic import make_slice_pair

    kw = dict(dim=3, seed=5, z_thickness=15.0, warp_amplitude=1.0)
    A, B = make_slice_pair(2600, 2300, 40, **kw)
    out = [A, B]
    for k, n in zip(range(2, n_slices), (2450, 2400)):
        out.append(make_slice_pair(2600, n, 40, theta=0.5 + 0.3 * (k - 1), shift=5.0 + 3.0 * (k - 1), **kw)[1])
    for sl in out:
        x = np.asarray(sl.obsm["spatial"])[:, 0]
        sl.obs["band"] = pd.Categorical(np.digitize(x, np.quantile(x, [0.25, 0.5, 0.75])).astype(str))
    return out


class Record:
    """What every pair's solver started from and ended with, per (driver, pair): ``"ref"`` for ``morpho_align``, the
    rank for a shard. Taken where the drivers store a pair's outputs."""

    def __init__(self, monkeypatch):
        import torch

        from spateo_release_b200.alignment import distributed, morpho_alignment

        self.rows, lock, store = {}, threading.Lock(), morpho_alignment._store_pair

        def recording_store(target, solver, *args, **kw):
            who = "ref" if solver.column_shard is None else int(solver.column_shard[0])
            with lock:
                pair = sum(1 for w, _ in self.rows if w == who)
                self.rows[(who, pair)] = dict(
                    batch_idx=np.array(getattr(solver, "batch_idx", None)), inducing=solver.inducing_variables_idx.copy(),
                    fixed=np.asarray(solver.sampleB.obsm[solver.spatial_key]).copy(), sigma2=float(solver.sigma2),
                    K_NA=np.asarray(solver.K_NA).copy(), K_NB=np.asarray(solver.K_NB).copy(),
                    allocated=torch.cuda.memory_allocated())
            return store(target, solver, *args, **kw)

        monkeypatch.setattr(morpho_alignment, "_store_pair", recording_store)
        monkeypatch.setattr(distributed, "_store_pair", recording_store)


class Ranks(LockStep):
    """``LockStep`` with the host broadcast of rank 0's objects."""

    def broadcast(self, m, obj):
        if int(m.column_shard[0]) == 0:
            self.obj = obj
        self.bar.wait()
        out = self.obj
        self.bar.wait()
        return out


def _rank_chain(models, rank, world, comm, mode, **kw):
    """One rank's chain, as ``morpho_align_column_sharded`` runs it, through ``sharded_chain_pair``."""
    from spateo_release_b200.alignment.distributed import sharded_chain_pair
    from spateo_release_b200.alignment.morpho_alignment import _seed_keys, _working_copy

    aligned = [_working_copy(m) for m in models]
    _seed_keys(aligned, "spatial", KEY)
    pis = []
    try:
        for i in range(len(aligned) - 1):
            pis.append(sharded_chain_pair(aligned[i], aligned[i + 1], i, rank, world, comm, mode=mode, exchange="nccl",
                                          spatial_key=KEY, key_added=KEY, vecfld_key_added="VecFld_morpho",
                                          materialize_P=False, **kw))
    except BaseException:
        comm.bar.abort()  # the other ranks leave their barriers instead of waiting out the timeout
        raise
    return aligned, pis


def _reference(models, **kw):
    """``morpho_align`` from ``np.random.seed(0)``; returns (aligned, pis, NumPy stream state after the call)."""
    import spateo_release_b200 as st

    np.random.seed(0)
    aligned, pis = st.align.morpho_align(models, **kw)
    return aligned, pis, np.random.get_state()


def _assert_close(got, want, rec=None, who=0):
    """Slices within the tolerances of a sharded pair (tests/test_gpu_shard_options.py); with ``rec`` also each pair's
    σ², K_NA, K_NB and its random draws against ``morpho_align``'s."""
    for k, (g, w) in enumerate(zip(got, want)):
        for suffix in ("", "_rigid", "_nonrigid"):
            a, b = np.asarray(g.obsm[KEY + suffix]), np.asarray(w.obsm[KEY + suffix])
            assert a.shape == b.shape
            assert np.abs(a - b).max() < 2e-5 * np.abs(b).max(), (k, suffix, np.abs(a - b).max())
        if k:
            fg, fw = g.uns["VecFld_morpho"], w.uns["VecFld_morpho"]
            assert set(fg) == set(fw)
            for name in fw:
                assert np.shape(fg[name]) == np.shape(fw[name]), name
    if rec is None:
        return
    for pair in range(len(got) - 1):
        g, w = rec.rows[(who, pair)], rec.rows[("ref", pair)]
        assert np.array_equal(g["batch_idx"], w["batch_idx"]) and np.array_equal(g["inducing"], w["inducing"])
        assert abs(g["sigma2"] - w["sigma2"]) < 1e-4 * w["sigma2"]
        for name in ("K_NA", "K_NB"):
            assert g[name].shape == w[name].shape
            assert np.abs(g[name] - w[name]).max() < 1e-4 * np.abs(w[name]).max(), (pair, name)


# ---------------------------------------------------------------------------------------------------------------------
# W = 1: the public driver without a process group
# ---------------------------------------------------------------------------------------------------------------------
_CASES = {
    "snn_svi": dict(mode="SN-N"),
    "sns_full": dict(mode="SN-S", SVI_mode=False),
    "sparse_top_k": dict(mode="SN-N", sparse_calculation_mode=True, sparse_top_k=32, materialize_P=True),
    "transfer_obs": dict(mode="SN-N", SVI_mode=False, transfer_B="band"),
    "iter_key_added": dict(mode="SN-N", iter_key_added="iter_spatial"),
}


@pytest.mark.parametrize("case", list(_CASES))
def test_world1_matches_morpho_align(case, monkeypatch):
    import spateo_release_b200 as st

    models = _chain()
    kw = dict(BASE, **_CASES[case])
    kw.setdefault("materialize_P", False)
    rec = Record(monkeypatch)
    want, pis_ref, stream_ref = _reference(models, **kw)
    np.random.seed(0)
    got, pis = st.align.morpho_align_column_sharded(models, **kw)
    # the NumPy stream advanced pair by pair exactly as in morpho_align
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), stream_ref))
    assert all("align_spatial_rigid" not in m.obsm for m in models)  # inputs untouched
    _assert_close(got, want, rec)
    if kw.get("sparse_calculation_mode"):
        for P, Q in zip(pis, pis_ref):  # P.T: rows of the transposed matrix are the fixed cells
            assert P.shape == Q.shape and P.nnz == Q.nnz == 32 * Q.shape[0]
            assert np.array_equal(P.row, Q.row)
            assert np.abs(P.data - Q.data).max() < 1e-4 * np.abs(Q.data).max()
    else:
        assert pis == [None, None] and pis_ref == [None, None]
    if "transfer_B" in kw:
        for g, w in zip(got[1:], want[1:]):
            a, b = g.obsm["band_from_fixed"], w.obsm["band_from_fixed"]
            assert np.abs(a - b).max() < 1e-4
            top2 = np.sort(b, axis=1)[:, -2:]
            clear = top2[:, 1] - top2[:, 0] > 1e-3  # rows whose label is not a near tie
            assert clear.mean() > 0.9
            assert (np.asarray(g.obs["band_from_fixed"])[clear] == np.asarray(w.obs["band_from_fixed"])[clear]).all()
    if "iter_key_added" in _CASES[case]:
        for g, w in zip(got[1:], want[1:]):
            hg, hw = g.uns["iter_spatial"], w.uns["iter_spatial"]
            assert set(hg) == set(hw) and set(hg[KEY]) == set(hw[KEY]) == set(range(kw["max_iter"]))
            last = kw["max_iter"] - 1
            assert np.abs(hg[KEY][last] - hw[KEY][last]).max() < 2e-5 * np.abs(hw[KEY][last]).max()


# ---------------------------------------------------------------------------------------------------------------------
# W = 3 emulated in one process
# ---------------------------------------------------------------------------------------------------------------------
def test_world3_emulated_matches_morpho_align(monkeypatch):
    models = _chain()
    kw = dict(BASE, mode="SN-N")
    rec = Record(monkeypatch)
    want, _, stream_ref = _reference(models, materialize_P=False, **kw)
    world, comm = 3, Ranks(3)
    mode = kw.pop("mode")
    np.random.seed(0)
    with ThreadPoolExecutor(world) as ex:
        runs = [ex.submit(_rank_chain, models, r, world, comm, mode, **kw) for r in range(world)]
        results = [f.result() for f in runs]
    # rank 0 drew what morpho_align drew and the other ranks left the (shared) stream where rank 0 left it
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), stream_ref))
    got0 = results[0][0]
    for aligned, pis in results[1:]:  # the replicas are bit-identical
        assert pis == [None, None]
        for k in range(len(models)):
            for suffix in ("", "_rigid", "_nonrigid"):
                assert np.array_equal(aligned[k].obsm[KEY + suffix], got0[k].obsm[KEY + suffix]), (k, suffix)
    for r in range(world):
        _assert_close(results[r][0], want, rec, who=r)
        # pair 2 started from rank 0's pair-1 result, not from morpho_align's
        assert np.array_equal(rec.rows[(r, 1)]["fixed"], got0[1].obsm[KEY])
    assert not np.array_equal(got0[1].obsm[KEY], want[1].obsm[KEY])


# ---------------------------------------------------------------------------------------------------------------------
# refusals and memory
# ---------------------------------------------------------------------------------------------------------------------
def test_dense_posterior_refused_before_any_pair(monkeypatch):
    import spateo_release_b200 as st
    from spateo_release_b200.alignment import morpho_class

    def no_solver(*a, **k):
        raise AssertionError("a solver was built")

    monkeypatch.setattr(morpho_class.Morpho_pairwise, "__init__", no_solver)
    for P in (True, "auto"):
        with pytest.raises(NotImplementedError, match="materialize_P"):
            st.align.morpho_align_column_sharded(_chain(), materialize_P=P, **BASE)


def test_block_that_would_be_streamed_names_the_pair(monkeypatch):
    import spateo_release_b200 as st

    models = _chain()
    # room for pair 0 streamed in three chunks, not resident
    force_width(monkeypatch, models[1].shape[0], models[0].shape[0], models[0].shape[1], three_chunks(models[0].shape[0]))
    with pytest.raises(NotImplementedError, match=r"pair 0 .*column_shard.*More ranks"):
        st.align.morpho_align_column_sharded(models, SVI_mode=False, **BASE)


def test_chain_holds_one_pair_at_a_time(monkeypatch):
    import torch

    import spateo_release_b200 as st

    models = _chain(n_slices=4)
    (torch.ones((64, 64), device="cuda") @ torch.ones((64, 64), device="cuda")).sum().item()  # library handles up
    rec = Record(monkeypatch)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    np.random.seed(0)
    st.align.morpho_align_column_sharded(models, **dict(BASE, max_iter=40))
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() - before < 64 << 20
    held = [rec.rows[(0, p)]["allocated"] - before for p in range(3)]
    assert held[0] > 0 and max(held[1:]) < 1.5 * held[0], held
