"""GPU: pairs whose cost matrix does not fit the device recompute it every iteration in column chunks. Streaming is forced
here by patching the memory budget (``morpho_class._device_budget``) to exactly the footprint of the wanted chunk width."""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from layout_helpers import force_width as _force_width, three_chunks as _three_chunks  # noqa: E402
from parity_helpers import cfg_of, model_from_golden, poke_golden_estep, relmax  # noqa: E402


def _pair(n=2600, nb=2400, genes=24, seed=2):
    from spateo_release_b200.synthetic import make_slice_pair

    return make_slice_pair(n, nb, genes, dim=3, seed=seed, z_thickness=15.0, warp_amplitude=1.0)


def _solver(A, B, **kw):
    import spateo_release_b200 as st

    np.random.seed(0)
    return st.align.Morpho_pairwise(sampleA=B, sampleB=A, device="0", verbose=False, **kw)


def _with_labels(A, B):
    import pandas as pd

    for ad in (A, B):
        x = np.asarray(ad.obsm["spatial"])[:, 0]
        ad.obs["region"] = pd.Categorical(np.where(x < np.median(x), "left", "right"), categories=["left", "right"])
    return A, B


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layers", [dict(dissimilarity="kl"), dict(dissimilarity="sym_kl"), dict(dissimilarity="euc"),
                                    dict(dissimilarity="cos"),
                                    dict(rep_layer=["region"], rep_field=["obs"], dissimilarity=["label"]),
                                    dict(rep_layer=["X", "region"], rep_field=["layer", "obs"], dissimilarity=["kl", "label"]),
                                    dict(rep_layer=["X", "X"], rep_field=["layer", "layer"], dissimilarity=["kl", "cos"])])
def test_cost_rows_of_gathered_columns_equal_the_resident_matrix(monkeypatch, layers):
    import torch

    A, B = _with_labels(*_pair())
    kw = dict(SVI_mode=True, max_iter=20, K=15, materialize_P=False, nn_init=False, **layers)
    ref = _solver(A, B, **kw)
    ref.prepare()
    assert not ref.cost_plan.streamed
    m = _solver(A, B, **kw)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), 1000)
    m.prepare()
    assert m.cost_plan.streamed and m.cost_plan.n_chunks == 1
    NA = m.NA
    for it in (0, 7):
        idx = m._state["chunk_sched"][0][it]
        n = idx.shape[0]
        m._chunk_cost(0, n, idx)
        torch.cuda.synchronize()
        got = m._GT[:n, :NA].cpu().numpy()
        want = ref._GT[idx.long(), :NA].cpu().numpy()
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), relmax(got, want)
    # full-EM chunks address the resident operands by row offset
    m._chunk_cost(200, 333, None)
    torch.cuda.synchronize()
    assert np.array_equal(m._GT[:133, :NA].cpu().numpy(), ref._GT[200:333, :NA].cpu().numpy())


OUTPUTS = ("XAHat", "optimal_RnA", "R", "t", "sigma2", "gamma", "K_NA", "K_NB", "Coff")


def test_svi_one_chunk_is_bit_identical(monkeypatch):
    A, B = _pair()
    kw = dict(SVI_mode=True, max_iter=100, nonrigid_start_iter=60, K=15, materialize_P=False)
    ref = _solver(A, B, **kw)
    ref.run()
    m = _solver(A, B, **kw)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), 1000)
    m.run()
    assert m.cost_plan.streamed and m.cost_plan.chunks == ((0, 1000),)
    assert m.nonrigid_flag
    for k in OUTPUTS:
        a, b = np.asarray(getattr(m, k)), np.asarray(getattr(ref, k))
        assert np.array_equal(a, b), (k, relmax(a, b))


def _assert_close(m, ref):
    scale = np.abs(ref.XAHat).max()
    assert np.abs(m.XAHat - ref.XAHat).max() < 2e-5 * scale
    assert np.abs(m.optimal_RnA - ref.optimal_RnA).max() < 2e-5 * scale
    assert abs(float(m.sigma2) - float(ref.sigma2)) < 1e-4 * float(ref.sigma2)
    assert np.abs(m.K_NA - ref.K_NA).max() < 1e-4 * np.abs(ref.K_NA).max()


@pytest.mark.parametrize("svi", [True, False])
def test_three_ragged_chunks_match_resident_and_reproduce(monkeypatch, svi):
    A, B = _pair()
    kw = dict(SVI_mode=svi, max_iter=100, nonrigid_start_iter=60, K=15, materialize_P=False)
    ref = _solver(A, B, **kw)
    ref.run()
    runs = []
    for _ in range(2):
        m = _solver(A, B, **kw)
        cols = 1000 if svi else m.NB
        w = _three_chunks(cols)
        _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), w)
        m.run()
        assert m.cost_plan.n_chunks == 3 and m.cost_plan.chunks[-1][1] - m.cost_plan.chunks[-1][0] < w
        _assert_close(m, ref)
        runs.append(m)
    for k in OUTPUTS:
        assert np.array_equal(np.asarray(getattr(runs[0], k)), np.asarray(getattr(runs[1], k))), k


def test_one_estep_from_the_same_state(monkeypatch, golden):
    """3d_full_warp, one E-step of the reference's inputs with culling on: K_NB and the visited tiles exactly as resident,
    P (materialised chunk by chunk) and the row statistics within 1e-4 of the float64 oracle."""
    import torch

    from oracle import morpho_oracle as mo
    from spateo_release_b200._capi import check

    g = golden("3d_full_warp")
    it = 95
    ref = model_from_golden(g, probability_parameters=[float(g["pre_beta2"])])
    ref.prepare()
    m = model_from_golden(g, probability_parameters=[float(g["pre_beta2"])], materialize_P=False)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), _three_chunks(m.NB))
    m.prepare()
    assert m.cost_plan.n_chunks == 3
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    NA, NB = m.NA, m.NB
    P = torch.zeros((NA, NB), dtype=torch.float32, device=m._dev)

    def grab(q, it_, c0, c1):
        check(m._lib.spb_materialize_P(C.byref(q), it_, C.c_void_p(P.data_ptr() + 4 * c0), NB, st), "materialize")

    for mm in (ref, m):
        poke_golden_estep(mm, g, it)
        mm._params.cull = 1
    ref._estep_only(it, st)
    m._estep_only(it, st, on_chunk=grab)
    torch.cuda.synchronize()
    assert np.array_equal(m._state["K_NB"][:NB].cpu().numpy(), ref._state["K_NB"][:NB].cpu().numpy())
    assert m._read_scalars().visited == ref._read_scalars().visited
    Pm = m._unsorted(P.cpu().numpy())
    f8 = lambda k: g[k].astype(np.float64)
    XAHat, alpha, SD = f8(f"it{it}_in_XAHat"), f8(f"it{it}_in_alpha"), f8(f"it{it}_in_SigmaDiag")
    sigma2, gamma = float(g[f"it{it}_in_sigma2"]), float(g[f"it{it}_in_gamma"])
    yb = f8("pre_coordsB")
    spatial = ((XAHat[:, None, :] - yb[None, :, :]) ** 2).sum(-1)
    [ed] = mo.calc_distance(f8("exp_moving"), f8("exp_fixed"), "kl")
    P64, kns, kn2, _ = mo.get_P_core(
        Dim=float(m.D), spatial_dist=spatial, exp_dist=[ed], sigma2=sigma2, model_mul=(alpha * np.exp(-SD / sigma2))[:, None],
        gamma=gamma, samples_s=float(g["pre_samples_s"]), sigma2_variance=float(g[f"it{it}_in_sigma2_variance"]),
        probability_type=["gauss"], probability_parameters=[float(g["pre_beta2"])],
    )
    dvec = lambda name: m._unsorted(m._state[name][:NA].cpu().numpy())
    assert np.abs(Pm - P64).max() < 1e-4 * P64.max()
    assert relmax(dvec("K_NA"), P64.sum(1)) < 1e-4
    assert relmax(dvec("K_NA_spatial"), kns) < 1e-4
    assert relmax(dvec("K_NA_sigma2"), kn2) < 1e-4
    pxb = m._unsorted(m._state["PXB"][: m.D, :NA].T.contiguous().cpu().numpy())
    assert relmax(pxb, P64 @ yb) < 1e-4


@pytest.mark.parametrize("case", ["3d_svi", "c1_2d_svi", "2d_full_guide_both", "3d_svi_sparse32", "2d_full_sparse48"])
def test_golden_runs_streamed(monkeypatch, golden, case):
    g = golden(case)
    sparse = "sparse" in case
    m = model_from_golden(g, materialize_P=sparse)
    cols = m.batch_size if m.SVI_mode else m.NB
    if m.SVI_mode and cols is None:
        cols = min(max(int(m.NB / 10), 1000), m.NB)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), _three_chunks(cols))
    P = m.run()
    assert m.cost_plan.streamed and m.cost_plan.n_chunks == 3
    for sfx in ("", "_f64"):
        scale = np.abs(g["final_optimal_RnA" + sfx]).max()
        for key in ("optimal_RnA", "XAHat", "RnA"):
            err = np.abs(getattr(m, key) - g[f"final_{key}{sfx}"]).max() / scale
            ref_noise = np.abs(g[f"final_{key}"].astype(np.float64) - g[f"final_{key}_f64"]).max() / scale
            assert err < (1e-3 if sfx == "" else max(1e-3, 2 * ref_noise)), (key, sfx, err)
        s2_noise = abs(float(g["final_sigma2"]) - float(g["final_sigma2_f64"])) if sfx else 0.0
        gm_noise = abs(float(g["final_gamma"]) - float(g["final_gamma_f64"])) if sfx else 0.0
        assert abs(float(m.sigma2) - float(g["final_sigma2" + sfx])) < max(2e-2 * float(g["final_sigma2" + sfx]), 2 * s2_noise)
        assert abs(float(m.gamma) - float(g["final_gamma" + sfx])) < max(1e-2, 2 * gm_noise)
    assert relmax(m.optimal_R, g["final_optimal_R"]) < 1e-3
    if sparse:
        k = cfg_of(g)["kw"]["sparse_top_k"]
        assert P.shape == (m.NA, cols) and P.nnz == k * cols and P.dtype == np.float32
    else:
        assert P is None


def test_return_mapping_under_svi(monkeypatch):
    A, B = _pair()
    kw = dict(SVI_mode=True, max_iter=60, K=15, materialize_P=False, return_mapping=True)
    ref = _solver(A, B, **kw)
    ref.run()
    m = _solver(A, B, **kw)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), _three_chunks(1000))
    m.run()
    assert m.cost_plan.n_chunks == 3 and m.K_NB.shape == (m.NB,)
    _assert_close(m, ref)
    assert np.abs(m.K_NB - ref.K_NB).max() < 1e-4 * np.abs(ref.K_NB).max()


@pytest.mark.parametrize("opt", [dict(materialize_P=True), dict(compute_mapping=True), dict(column_shard=(0, 1, "nccl"))])
def test_refused_options_when_streamed(monkeypatch, opt):
    A, B = _pair(900, 800)
    kw = dict(SVI_mode=False, max_iter=5, K=15, materialize_P=False)
    kw.update(opt)
    ref = _solver(A, B, **kw)
    if "column_shard" not in opt:
        ref.prepare()
        assert not ref.cost_plan.streamed
    m = _solver(A, B, **kw)
    _force_width(monkeypatch, m.NA, m.NB, m._cost_features(), 256)
    with pytest.raises(NotImplementedError, match=list(opt)[0]):
        m.prepare()


def test_public_call_streamed_matches_resident(monkeypatch):
    import spateo_release_b200 as st
    from spateo_release_b200.alignment import morpho_class as mc

    A, B = _pair(3000, 2800, 24, seed=4)
    np.random.seed(0)
    out_ref, pis_ref = st.align.morpho_align([A.copy(), B.copy()], device="0", verbose=False, max_iter=60)
    plans = []
    orig = mc.Morpho_pairwise._plan_cost

    def spy(self, nb):
        orig(self, nb)
        plans.append(self.cost_plan)

    monkeypatch.setattr(mc.Morpho_pairwise, "_plan_cost", spy)
    _force_width(monkeypatch, 2800, 3000, 24, 1000)
    np.random.seed(0)
    out, pis = st.align.morpho_align([A.copy(), B.copy()], device="0", verbose=False, max_iter=60)
    assert [p.mode for p in plans] == ["streamed"] and plans[0].chunks == ((0, 1000),)
    assert pis_ref[0] is not None and pis[0] is None  # the dense posterior is built only for a resident pair
    for a, b in zip(out_ref, out):
        assert np.array_equal(np.asarray(a.obsm["align_spatial"]), np.asarray(b.obsm["align_spatial"]))
