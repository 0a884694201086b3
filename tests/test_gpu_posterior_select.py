"""The sparse top-k posterior (col_select, sweep 2's threshold, col_emit) and the posterior argmax, kernel by kernel.

Part 1 runs one sparse E-step on real states (the config-1 goldens at iterations 0, 60 and 150, full EM and an SVI batch;
a 20k x 20k 3-D late-sigma2 state) for k = 1, 32, 1024 and 1025 with culling on and off, and compares the COO matrix and
the sums with ``parity_helpers.sparse_posterior_reference`` in float64, fed the device's own cost matrix and state.

Part 2 checks the kernels against an exact replay on the device's own weights w = q g (``replay_weights``): the column
threshold tau bit for bit, the emitted entries, and sweep 2's row sums and K_NB within an fp32 accumulation bound. Most
states are written directly: alpha = 1, SigmaDiag = 0 and sigma2 = 1e30 make every q exactly 1.0, so the written cost
matrix is the weight matrix. They put the selected level-0 bin on both sides of the candidate cap, let level 2 decide,
straddle the k-th position with exact ties, and hold subnormals, zeros and columns with fewer than k non-zero weights.
The argmax keys are compared with the replay bit for bit.

The printed report gives, per case, the path each column took: the selected level-0 bin's candidate count against
kSelCap, whether the row-block mask was on, and the level that decided tau."""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from parity_helpers import (argmax_replay, model_from_golden, poke_estep_state, poke_golden_estep,  # noqa: E402
                            replay_weights, sparse_posterior_reference, topk_replay)

KSEL_CAP = 8192          # col_select_kernel's candidate buffer (estep.cu kSelCap)
MASK_BLOCKS = 512        # row blocks the per-column mask covers (32 * SPB_COLMASK_WORDS)
U32 = 2.0 ** -24         # unit roundoff of fp32


def _torch():
    import torch

    return torch


def _stream():
    return C.c_void_p(_torch().cuda.current_stream().cuda_stream)


def _check(rc, what):
    from spateo_release_b200._capi import check

    check(rc, what)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


# ---------------------------------------------------------------------------------------------------------------------
# running one sparse E-step and reading what it produced (all in device row order)
# ---------------------------------------------------------------------------------------------------------------------
def _set_k(m, k, cull):
    m.sparse_top_k = int(k)
    m._params.sparse_k = int(k)
    m._params.cull = int(bool(cull))


def _outputs(m, k, nbb=None):
    s, NA = m._state, m.NA
    nbb = m._NBb if nbb is None else nbb
    cc = s["colconst"][:nbb].cpu().numpy()
    kk = min(int(k), NA)
    return dict(
        tau=cc[:, 18].copy(), c=cc[:, 10].copy(), Y=cc[:, [0, 2, 4][: m.D]].astype(np.float64),
        K_NB=s["K_NB"][:nbb].cpu().numpy().astype(np.float64),
        K_NA=s["K_NA"][:NA].cpu().numpy().astype(np.float64),
        PXB=s["PXB"][: m.D, :NA].T.cpu().numpy().astype(np.float64),
        rows=m._P_rows[:, :kk].cpu().numpy().astype(np.int64) if getattr(m, "_P_rows", None) is not None else None,
        vals=m._P_vals[:, :kk].cpu().numpy() if getattr(m, "_P_vals", None) is not None else None,
    )


def _sparse_estep(m, it, k, cull):
    torch = _torch()
    _set_k(m, k, cull)
    st = _stream()
    m._estep_only(it, st)
    m._capture_P(it, st)
    torch.cuda.synchronize()
    return _outputs(m, k)


def _paths(W, tau, k, cull, nrb):
    """Per column: the count of the level-0 bin holding tau (the candidates col_select gathers when it fits kSelCap)
    and the level that decided tau: 0, 1 or 2 (the deepest level whose bin still held values other than tau), or "-" when
    the column has fewer than k non-zero weights."""
    key = _bits(W)
    tk = _bits(tau)
    b0 = (key >> 19) == (tk >> 19)[None, :]
    b1 = (key >> 7) == (tk >> 7)[None, :]
    nz = key != 0
    cand = (b0 & nz).sum(0)
    differ = key != tk[None, :]
    level = np.where((b1 & differ & nz).any(0), 2, np.where((b0 & differ & nz).any(0), 1, 0))
    level = np.where(tau > 0, level, -1)
    live = tau > 0
    mask = "on" if (cull and nrb <= MASK_BLOCKS) else "off"
    return (f"mask {mask} ({nrb} row blocks); level-0 candidates max {int(cand[live].max()) if live.any() else 0} "
            f"(> kSelCap in {int((cand[live] > KSEL_CAP).sum())} columns, == kSelCap in {int((cand[live] == KSEL_CAP).sum())}); "
            f"tau decided at level 0/1/2: {int((level == 0).sum())}/{int((level == 1).sum())}/{int((level == 2).sum())}, "
            f"fewer than k non-zero: {int((level < 0).sum())}")


def _check_against_replay(name, W, out, k, cull, nrb):
    """tau bit for bit, the COO's structure and values, K_NB and sweep 2's row sums within the fp32 bound; returns the
    replay."""
    NA, NB = W.shape
    kk = min(int(k), NA)
    r = topk_replay(W, k, out["c"], out["Y"])
    print(f"\n[{name} k={k} cull={int(bool(cull))}] " + _paths(W, r["tau"], k, cull, nrb))
    assert np.array_equal(_bits(out["tau"]), _bits(r["tau"])), "tau differs from the replay"
    if out.get("rows") is not None:
        rows, vals = out["rows"], out["vals"]
        assert rows.shape == (NB, kk)
        srt = np.sort(rows, axis=1)
        assert (srt[:, 1:] > srt[:, :-1]).all() and srt.min() >= 0 and srt.max() < NA, "a column repeats a row"
        w = np.take_along_axis(W.T, rows, axis=1)                          # [NB, kk]
        above = w > r["tau"][:, None]
        assert np.array_equal(above.sum(1), r["n_above"]), "an entry with w > tau is missing"
        assert (w[~above] == np.broadcast_to(r["tau"][:, None], w.shape)[~above]).all(), "an entry below tau"
        assert np.array_equal(_bits(vals), _bits(w * out["c"][:, None])), "COO values are not w c_j"
    # measured (H100 SXM, 700 W): K_NB <= 3.3e-7 and K_NA <= 4.1e-7 relative, far inside these bounds.
    # fp32 sums of non-negative terms: |error| <= (n + 4) u sum|terms| whatever the order (n terms, 4 roundings more);
    # sums in fp32's subnormal range carry an absolute error instead (the 1e-38)
    eK = np.abs(out["K_NB"] - r["K_NB"]) / np.maximum(r["K_NB"], 1e-300)
    assert (np.abs(out["K_NB"] - r["K_NB"]) <= (NA + 4) * U32 * r["K_NB"] + 1e-38).all(), "K_NB"
    absy = topk_replay(W, k, out["c"], np.abs(out["Y"]))["PXB"]    # sum |terms| of P @ XB (c >= 0)
    eA = np.abs(out["K_NA"] - r["K_NA"]) / np.maximum(r["K_NA"], 1e-300)
    assert (np.abs(out["K_NA"] - r["K_NA"]) <= (NB + 4) * U32 * r["K_NA"] + 1e-38).all(), "K_NA"
    assert (np.abs(out["PXB"] - r["PXB"]) <= (NB + 4) * U32 * absy + 1e-38).all(), "P @ XB"
    ties = int((r["n_ties"] > 1).sum())
    gap = np.abs(r["K_NB"] - r["K_NB_k"]) / np.maximum(r["K_NB_k"], 1e-300)
    nK, nA = r["K_NB"] > 1e-30, r["K_NA"] > 1e-30                     # relative errors above the subnormal range
    print(f"  K_NB rel err {eK[nK].max() if nK.any() else 0:.2e} (bound {(NA + 4) * U32:.1e}), K_NA rel err {eA[nA].max() if nA.any() else 0:.2e} "
          f"(bound {(NB + 4) * U32:.1e}); columns with ties at tau {ties}, K_NB vs the k-entry sum up to {gap.max():.2e}")
    return r


def _argmax(m, it, colmap=None):
    torch = _torch()
    from spateo_release_b200._capi import ptr

    rowbest = torch.zeros((m.NA,), dtype=torch.int64, device=m._dev)
    colbest = torch.zeros((m._NBb,), dtype=torch.int64, device=m._dev)
    cm = None if colmap is None else torch.from_numpy(np.asarray(colmap, np.int32)).to(m._dev)
    _check(m._lib.spb_posterior_argmax_mapped(C.byref(m._params), it, ptr(cm), ptr(rowbest), ptr(colbest), _stream()),
           "spb_posterior_argmax_mapped")
    torch.cuda.synchronize()
    return rowbest.cpu().numpy().view(np.uint64), colbest.cpu().numpy().view(np.uint64)


def _check_argmax(name, m, it, W, c, tau, colmap=None):
    rk, ck = _argmax(m, it, colmap)
    wr, wc = argmax_replay(W, c, tau, colmap)
    nrow = (m.NA + 255) // 256
    n_sm = _torch().cuda.get_device_properties(0).multi_processor_count
    nseg = min(max((n_sm * 8 + nrow - 1) // nrow, 1), m._NBb)
    print(f"  [{name} argmax] N_A {m.NA} (mod 256 = {m.NA % 256}), NBb {m._NBb}, row segments {nseg} "
          f"(NBb mod segments {m._NBb % nseg}), map {'none' if colmap is None else 'with -1 / permuted'}")
    assert np.array_equal(ck, wc), "column argmax keys"
    assert np.array_equal(rk, wr), "row argmax keys"


# ---------------------------------------------------------------------------------------------------------------------
# Part 1: real states against float64
# ---------------------------------------------------------------------------------------------------------------------
KS = (1, 32, 1024, 1025)


def _reference_of_device_state(m, it, ks, fp32=False):
    """``sparse_posterior_reference`` on the device's own inputs: fp32 positions, model multipliers, fixed coordinates and
    cost rows of this iteration's columns, widened to fp64 (device row order)."""
    s, NA, D, nbb = m._state, m.NA, m.D, m._NBb
    sc = m._read_scalars()
    XA = s["XAHat"][:D, :NA].T.double().cpu().numpy()
    alpha, SD = s["alpha"][:NA].double().cpu().numpy(), s["SigmaDiag"][:NA].double().cpu().numpy()
    sigma2 = float(sc.sigma2)
    cols = np.arange(nbb) if not m.SVI_mode else s["batch_idx"][it].long().cpu().numpy()
    G = m._GT[_torch().from_numpy(cols).to(m._dev)][:, :NA].cpu().numpy().T   # fp32, widened chunk by chunk
    YB = s["xb4"][cols, :D].double().cpu().numpy()
    kw = dict(Dim=float(D), XAHat=XA, YB=YB, G=G, sigma2=sigma2, model_mul=(alpha * np.exp(-SD / sigma2))[:, None],
              gamma=float(sc.gamma), samples_s=float(m._params.samples_s), sigma2_variance=float(sc.sigma2_variance),
              ks=ks, chunk=1000)
    ref = sparse_posterior_reference(**kw)
    ref32 = sparse_posterior_reference(dtype=np.float32, **kw) if fp32 else None
    return ref, ref32, kw


def _coo_vs_reference(name, out, ref, ref32, NA):
    rows, vals = out["rows"], out["vals"].astype(np.float64)
    NB, kk = rows.shape
    pmax = float(ref["vals"].max())
    # support: compare the sets of rows with a non-zero value; they may differ only where the fp64 k-th and (k+1)-th
    # values of the column agree to fp32 rounding
    dr = np.where(vals > 0, rows, -1)
    rr = np.where(ref["vals"] > 0, ref["rows"], -1)
    o1, o2 = np.argsort(dr, axis=1), np.argsort(rr, axis=1)
    d_sorted, r_sorted = np.take_along_axis(dr, o1, 1), np.take_along_axis(rr, o2, 1)
    same = (d_sorted == r_sorted).all(1)
    gap = (ref["kth"] - ref["kth1"]) / np.maximum(ref["kth"], 1e-300)
    near = (gap <= 2e-5) | (ref["kth"] < 1e-30)           # fp32 rounding, or the k-th value underflows in fp32
    dv, rv = np.take_along_axis(vals, o1, 1), np.take_along_axis(ref["vals"], o2, 1)
    err_v = np.abs(dv - rv)[same].max() / pmax if same.any() else 0.0
    eK_NB = np.abs(out["K_NB"] - ref["K_NB"]).max() / ref["K_NB"].max()
    eK_NA = np.abs(out["K_NA"] - ref["K_NA"]).max() / ref["K_NA"].max()
    ePXB = np.abs(out["PXB"] - ref["PXB"]).max() / np.abs(ref["PXB"]).max()
    emitted_NB = vals.sum(1) * 1.0
    emitted_NA = np.bincount(rows.reshape(-1), weights=vals.reshape(-1), minlength=NA)
    sNB = np.abs(out["K_NB"] - emitted_NB).max() / out["K_NB"].max()
    sNA = np.abs(out["K_NA"] - emitted_NA).max() / out["K_NA"].max()
    f32 = ""
    if ref32 is not None:
        f32 = (f" | fp32 restatement: vals {np.abs(ref32['vals'] - ref['vals']).max() / pmax:.1e} K_NB "
               f"{np.abs(ref32['K_NB'] - ref['K_NB']).max() / ref['K_NB'].max():.1e} K_NA "
               f"{np.abs(ref32['K_NA'] - ref['K_NA']).max() / ref['K_NA'].max():.1e}")
    print(f"  [{name}] support differs in {int((~same).sum())} of {NB} columns (all near-ties: {bool(near[~same].all())}); "
          f"vals {err_v:.1e}  K_NB {eK_NB:.1e}  K_NA {eK_NA:.1e}  PXB {ePXB:.1e}; sums of the emitted matrix: K_NB "
          f"{sNB:.1e} K_NA {sNA:.1e}" + f32)
    # measured on an H100 SXM (700 W), over every state and k: values <= 4.8e-7, K_NB / K_NA / P @ XB <= 4.8e-7 (the fp32
    # restatement: <= 3.3e-7), sums of the emitted matrix <= 3.2e-7
    assert near[~same].all(), "support differs from the fp64 top-k away from a near-tie"
    assert err_v < 1e-4
    assert eK_NB < 1e-4 and eK_NA < 1e-4 and ePXB < 1e-4
    assert sNB < 1e-5 and sNA < 1e-5


def _part1(name, m, it, cull_states, ks=KS, fp32=True, poke=None, replay=None):
    """``replay``: the (k, cull) settings also checked against the exact replay (default all)."""
    ref, ref32, kw = _reference_of_device_state(m, it, ks, fp32=fp32)
    nrb = m.ldx // 512
    for k in ks:
        for cull in cull_states:
            if poke is not None:
                poke()
            out = _sparse_estep(m, it, k, cull)
            if replay is None or (k, cull) in replay:
                _check_against_replay(f"{name} it{it}", replay_weights(m, it), out, k, cull, nrb)
            _coo_vs_reference(f"{name} it{it} k={k} cull={int(cull)}", out, ref[k], None if ref32 is None else ref32[k], m.NA)
    return kw


def _argmax_vs_reference(name, m, it, kw):
    """Dense mode: each chosen entry's fp64 value is within 1e-4 of the fp64 row / column maximum, and the keys equal the
    replay's."""
    from oracle.morpho_oracle import get_P_core

    mode = m.sparse_calculation_mode
    m.sparse_calculation_mode, m._params.sparse_k = False, 0
    try:
        m._estep_only(it, _stream())
        _torch().cuda.synchronize()
        rk, ck = _argmax(m, it)
        W = replay_weights(m, it)
        cc = m._state["colconst"][: m._NBb].cpu().numpy()
        _check_argmax(name, m, it, W, cc[:, 10], cc[:, 18])
    finally:
        m.sparse_calculation_mode = mode
    NA, NB = W.shape
    spatial = ((kw["XAHat"][:, None, :] - kw["YB"][None, :, :]) ** 2).sum(-1)
    P64, _, _, _ = get_P_core(Dim=kw["Dim"], spatial_dist=spatial, exp_dist=[kw["G"].astype(np.float64)], sigma2=kw["sigma2"],
                              model_mul=kw["model_mul"], gamma=kw["gamma"], samples_s=kw["samples_s"],
                              sigma2_variance=kw["sigma2_variance"], probability_type=["prob"])
    ra = (0xFFFFFFFF - (rk & np.uint64(0xFFFFFFFF))).astype(np.int64)
    ca = (0xFFFFFFFF - (ck & np.uint64(0xFFFFFFFF))).astype(np.int64)
    rmax, cmax = P64.max(1), P64.max(0)
    er = np.abs(P64[np.arange(NA), ra] - rmax) / np.maximum(rmax, 1e-300)
    ec = np.abs(P64[ca, np.arange(NB)] - cmax) / np.maximum(cmax, 1e-300)
    er, ec = er[rmax > 0], ec[cmax > 0]
    print(f"  [{name} argmax vs fp64] rows {er.max():.1e}  columns {ec.max():.1e}")
    assert er.max() < 1e-4 and ec.max() < 1e-4    # measured 0 on the config-1 states (H100 SXM, 700 W)


@pytest.mark.parametrize("case,it", [("c1_2d_full_warp", 0), ("c1_2d_full_warp", 60), ("c1_2d_full_warp", 150),
                                     ("c1_2d_svi", 60)])
def test_real_state_sparse_estep_matches_float64(golden, case, it):
    g = golden(case)
    m = model_from_golden(g, probability_parameters=[float(g["pre_beta2"])], sparse_calculation_mode=True)
    m.prepare()
    poke_golden_estep(m, g, it)
    kw = _part1(case, m, it, (False, True), poke=lambda: poke_golden_estep(m, g, it))
    _check_argmax(f"{case} it{it} k=1025", m, it, replay_weights(m, it), *_tau_c(m))
    _argmax_vs_reference(f"{case} it{it} dense", m, it, kw)


def _tau_c(m):
    cc = m._state["colconst"][: m._NBb].cpu().numpy()
    return cc[:, 10].copy(), cc[:, 18].copy()


@pytest.fixture(scope="module")
def late_20k():
    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(20000, 20000, 64, dim=3, seed=7, z_thickness=20.0)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(B, A, device="0", verbose=False, SVI_mode=False, max_iter=200, K=15, nn_init=False,
                                 sparse_calculation_mode=True)
    m.prepare()
    it = 130
    m.sparse_calculation_mode, m._params.sparse_k = False, 0   # the dense EM trajectory of test_gpu_lm_culling.py
    m.run_em(n_iter=it)
    m.sparse_calculation_mode = True
    assert float(m._read_scalars().sigma2) < 9e-3, "expected a late-iteration state"
    s = m._state
    snap = {k: s[k].clone() for k in ("XAHat", "alpha", "SigmaDiag", "mm", "lm", "sc")}
    return m, it, snap


def _restore(m, snap):
    for k, v in snap.items():
        m._state[k].copy_(v)


def test_late_20k_3d_sparse_estep_matches_float64(late_20k):
    m, it, snap = late_20k
    _restore(m, snap)
    _part1("20k 3-D", m, it, (False, True), fp32=False, poke=lambda: _restore(m, snap), replay=((1024, True), (1025, False)))


# ---------------------------------------------------------------------------------------------------------------------
# Part 2: written states against the exact replay
# ---------------------------------------------------------------------------------------------------------------------
def _solver(NA, NB, D, k, svi=False, genes=8, seed=0):
    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(NB, NA, genes, dim=D, seed=seed, **({"z_thickness": 10.0} if D == 3 else {}))
    np.random.seed(0)
    m = st.align.Morpho_pairwise(sampleA=B, sampleB=A, device="0", verbose=False, SVI_mode=svi, max_iter=20, K=15,
                                 nn_init=False, sparse_calculation_mode=True, sparse_top_k=k)
    m.prepare()
    assert (m.NA, m.NB) == (NA, NB)
    return m


def _unit_q(m, sigma2=1e30):
    """alpha = 1, SigmaDiag = 0 (lm = 0) and a huge sigma2: c_q d rounds to a tiny argument, ex2 of it is exactly 1.
    gamma = 1 makes the outlier term omega exactly 0, so the column factors c_j = 1 / (sum_i w_ij + 1e-8) stay non-zero."""
    s, NA, D = m._state, m.NA, m.D
    XA = m._unsorted(s["XAHat"][:D, :NA].T.contiguous().cpu().numpy())
    sc = m._read_scalars()
    poke_estep_state(m, XA, np.ones(NA), np.zeros(NA), sigma2, 1.0, float(sc.sigma2_variance))


def _write_cost(m, G):
    """Cost rows of the fixed cells <- G [N_A, NB] (device row order)."""
    torch = _torch()
    m._GT[: G.shape[1], : m.NA] = torch.from_numpy(np.ascontiguousarray(G.T)).to(m._dev)


def _bin_values(rng, key0, n, span_bits=19, distinct=False):
    if distinct:
        off = rng.choice(1 << span_bits, size=n, replace=False)
    else:
        off = rng.integers(0, 1 << span_bits, size=n)
    return (np.uint32(key0) + off.astype(np.uint32)).view(np.float32)


def _cap_matrix(NA, NB, rng):
    """Columns (k = 1024): 0 / 1: 100 values above and exactly 8192 / 8193 in the level-0 bin of 1.0; 2: all N_A values
    in that one bin; 3: 964 above and 128 values whose keys differ only in the low 7 bits (level 2 decides); 4: 1000
    above and 50 exact copies of 0.75 straddling the k-th position; 5: 600 normal values, 600 subnormals, zeros; 6: 500
    non-zero, the rest zero (fewer than k); 7: all zero; 8: all equal; the rest uniform."""
    G = rng.uniform(0.01, 0.5, size=(NA, NB)).astype(np.float32)
    one, big, mid = 0x3F800000, 0x40800000, 0x3FC00000

    def place(j, vals):
        idx = rng.choice(NA, size=len(vals), replace=False)
        G[idx, j] = vals
        return idx

    for j, n in ((0, KSEL_CAP), (1, KSEL_CAP + 1)):
        place(j, np.concatenate([_bin_values(rng, big, 100, 23, True), _bin_values(rng, one, n)]))
    G[:, 2] = _bin_values(rng, one, NA)
    place(3, np.concatenate([_bin_values(rng, big, 964, 23, True),
                             (np.uint32(mid) + np.arange(128, dtype=np.uint32)).view(np.float32)]))
    place(4, np.concatenate([_bin_values(rng, big, 1000, 23, True), np.full(50, 0.75, np.float32)]))
    G[:, 5] = 0.0
    place(5, np.concatenate([rng.uniform(1.0, 2.0, 600).astype(np.float32),
                             rng.choice(np.arange(1, 1 << 23, dtype=np.uint32), 600, replace=False).view(np.float32)]))
    G[:, 6] = 0.0
    place(6, rng.uniform(0.1, 1.0, 500).astype(np.float32))
    G[:, 7] = 0.0
    G[:, 8] = 1.0
    return G


@pytest.fixture(scope="module")
def cap_state():
    NA, NB = 20480, 16
    m = _solver(NA, NB, 3, 1024)
    G = _cap_matrix(NA, NB, np.random.default_rng(11))
    return m, G


def _written_estep(m, G, it, k, cull):
    _unit_q(m)
    _write_cost(m, G)
    out = _sparse_estep(m, it, k, cull)
    W = replay_weights(m, it)
    assert np.array_equal(_bits(W), _bits(G)), "q is not exactly 1: the written cost matrix is not the weight matrix"
    return out, W


@pytest.mark.parametrize("k,cull", [(1024, True), (1024, False), (1, True), (32, True), (1025, True)])
def test_written_cap_ties_subnormals_against_replay(cap_state, k, cull):
    m, G = cap_state
    out, W = _written_estep(m, G, 0, k, cull)
    r = _check_against_replay("written 20480 x 16", W, out, k, cull, m.ldx // 512)
    if k == 1024:
        key, tk = _bits(W), _bits(r["tau"])
        cand = ((key >> 19) == (tk >> 19)[None, :]).sum(0)
        assert cand[0] == KSEL_CAP and cand[1] == KSEL_CAP + 1 and cand[2] == m.NA
        assert r["tau"][4] == np.float32(0.75) and r["n_ties"][4] == 50 and r["n_above"][4] == 1000
        assert 0 < r["tau"][5] < np.finfo(np.float32).tiny
        assert r["tau"][6] == 0 and r["tau"][7] == 0 and r["tau"][8] == 1.0
        assert ((key[:, 3] >> 7) == (tk[3] >> 7)).sum() == 128
        # the tie rule: exactly k entries in the COO, every copy of tau in K_NB
        assert out["K_NB"][4] > out["vals"][4].astype(np.float64).sum() * (1 + 1e-3)
        _check_argmax("written 20480 x 16", m, 0, W, out["c"], out["tau"])


@pytest.mark.parametrize("k", [4, 3000, 3001, 3002])
def test_written_small_k_around_n_and_argmax(k):
    """N_A = 3001 (not a multiple of 4, 256, 512 or 2048), 200 columns: k = N_A - 1, N_A, N_A + 1, and k = 4 where many
    rows' maxima fall below their column's tau; all-zero rows and columns, non-zero ties along rows and columns, and a
    column map with -1 and permuted entries for the row argmax."""
    NA, NB = 3001, 200
    m = _solver(NA, NB, 2, k)
    rng = np.random.default_rng(k)
    G = rng.uniform(0.0, 1.0, size=(NA, NB)).astype(np.float32)
    G[G == 0] = 0.5
    if k in (4, NA + 1):  # zeros; at k = N_A - 1 and N_A every column holds N_A non-zero weights and the select runs
        G[rng.random(G.shape) < 0.05] = 0.0
        G[17] = 0.0
        G[:, 33] = 0.0
    G[100, 5] = G[100, 150] = G[100, 7] = 4.0        # ties along a row
    G[[5, 900, 2999], 60] = 8.0                      # ties down a column
    out, W = _written_estep(m, G, 0, k, True)
    _check_against_replay(f"written {NA} x {NB}", W, out, k, True, m.ldx // 512)
    _check_argmax(f"written {NA} x {NB} k={k}", m, 0, W, out["c"], out["tau"])
    cmap = rng.permutation(NB + 50)[:NB].astype(np.int32)
    cmap[rng.random(NB) < 0.2] = -1
    _check_argmax(f"written {NA} x {NB} k={k}", m, 0, W, out["c"], out["tau"], colmap=cmap)


def test_culled_columns_with_fewer_than_k_nonzero_weights():
    """A small sigma2: each column's weights are non-zero on a few hundred rows only, so tau = 0 and the COO is filled
    with zeros; culling on, so col_select skips the row blocks the mask rules out."""
    NA, NB, k = 20000, 1000, 1024
    m = _solver(NA, NB, 3, k)
    s = m._state
    XA = m._unsorted(s["XAHat"][:3, :NA].T.contiguous().cpu().numpy()).astype(np.float64)
    area = np.prod(np.ptp(XA[:, :2], axis=0))
    sigma2 = 300.0 * area / (np.pi * 175.0 * NA)          # ~300 rows within the fp32 underflow radius of a column
    sc = m._read_scalars()
    poke_estep_state(m, XA, np.ones(NA), np.zeros(NA), sigma2, float(sc.gamma), float(sc.sigma2_variance))
    out = _sparse_estep(m, 0, k, True)
    W = replay_weights(m, 0)
    r = _check_against_replay(f"culled {NA} x {NB}", W, out, k, True, m.ldx // 512)
    assert (r["tau"] == 0).mean() > 0.9, "expected most columns to have fewer than k non-zero weights"
    _check_argmax(f"culled {NA} x {NB}", m, 0, W, out["c"], out["tau"])


@pytest.mark.parametrize("k", [32, 1024])
def test_mask_off_above_512_row_blocks(k):
    """N_A = 262,657: more row blocks than the column mask covers, so col_select reads every row."""
    NA, NB = 262657, 256
    m = _solver(NA, NB, 2, k, genes=4)
    nrb = m.ldx // 512
    assert nrb > MASK_BLOCKS
    out = _sparse_estep(m, 0, k, True)
    W = replay_weights(m, 0)
    _check_against_replay(f"mask off {NA} x {NB}", W, out, k, True, nrb)
    if k == 32:
        _check_argmax(f"mask off {NA} x {NB}", m, 0, W, out["c"], out["tau"])


def test_streamed_ragged_chunks_against_replay(monkeypatch, golden):
    """3d_full_warp streamed in three column chunks, the last one shorter: per chunk, tau and the COO against the replay
    of the chunk's weights; the folded row sums against the sum of the chunks' replays."""
    from layout_helpers import force_width, three_chunks

    g = golden("3d_full_warp")
    it, k = 95, 32
    m = model_from_golden(g, probability_parameters=[float(g["pre_beta2"])], sparse_calculation_mode=True, sparse_top_k=k,
                          materialize_P=True)
    force_width(monkeypatch, m.NA, m.NB, m._cost_features(), three_chunks(m.NB))
    m.prepare()
    assert m.cost_plan.n_chunks == 3
    poke_golden_estep(m, g, it)
    m._params.cull = 1
    emit = m._capture_begin()
    chunks = []

    def grab(q, it_, c0, c1):
        emit(q, it_, c0, c1)
        W = replay_weights(m, it_, q)
        cc = m._state["colconst"][: c1 - c0].cpu().numpy()
        chunks.append((c0, c1, W, cc[:, 18].copy(), cc[:, 10].copy(), cc[:, [0, 2, 4][: m.D]].astype(np.float64)))

    m._estep_only(it, _stream(), on_chunk=grab)
    _torch().cuda.synchronize()
    assert len(chunks) == 3 and chunks[-1][1] - chunks[-1][0] < chunks[0][1] - chunks[0][0]
    K_NA = np.zeros(m.NA)
    for c0, c1, W, tau, c, Y in chunks:
        out = dict(tau=tau, c=c, Y=Y, K_NB=m._state["K_NB"][c0:c1].cpu().numpy().astype(np.float64),
                   K_NA=np.zeros(m.NA), PXB=np.zeros((m.NA, m.D)),
                   rows=m._P_rows[c0:c1, :k].cpu().numpy().astype(np.int64), vals=m._P_vals[c0:c1, :k].cpu().numpy())
        r = topk_replay(W, k, c, Y)
        out["K_NA"], out["PXB"] = r["K_NA"], r["PXB"]            # the row sums are checked after the fold
        _check_against_replay(f"streamed 3d_full_warp chunk [{c0}, {c1})", W, out, k, True, m.ldx // 512)
        K_NA += r["K_NA"]
    dev = m._state["K_NA"][: m.NA].cpu().numpy().astype(np.float64)
    err = np.abs(dev - K_NA) / np.maximum(K_NA, 1e-300)
    print(f"  folded K_NA rel err {err[K_NA > 0].max():.2e} (bound {(m.NB + 4) * U32:.1e})")
    assert (np.abs(dev - K_NA) <= (m.NB + 4) * U32 * K_NA + 1e-38).all()


# ---------------------------------------------------------------------------------------------------------------------
# Reproducibility
# ---------------------------------------------------------------------------------------------------------------------
def _select_and_sweep2(m, it):
    torch = _torch()
    st = _stream()
    _check(m._lib.spb_estep_col_select(C.byref(m._params), it, st), "spb_estep_col_select")
    _check(m._lib.spb_estep_sweep2(C.byref(m._params), it, st), "spb_estep_sweep2")
    _check(m._lib.spb_row_finalize(C.byref(m._params), st), "spb_row_finalize")
    torch.cuda.synchronize()
    s = m._state
    return dict(tau=s["colconst"][: m._NBb, 18].clone(), K_NB=s["K_NB"][: m._NBb].clone(),
                rowpart=s["rowpart"].clone(), K_NA=s["K_NA"].clone(), PXB=s["PXB"].clone())


def _assert_repeats(m, it, name, runs=3):
    torch = _torch()
    first = _select_and_sweep2(m, it)
    for _ in range(runs - 1):
        again = _select_and_sweep2(m, it)
        diff = {k: int((first[k] != again[k]).sum()) for k in first}
        print(f"\n[{name}] entries that differ from the first run: {diff}")
        for k in first:
            assert torch.equal(first[k], again[k]), k


def test_select_and_sweep2_repeat_bit_for_bit_on_the_cap_state(cap_state):
    m, G = cap_state
    _written_estep(m, G, 0, 1024, True)
    _assert_repeats(m, 0, "written 20480 x 16, k=1024")


def test_select_and_sweep2_repeat_bit_for_bit_at_20k(late_20k):
    m, it, snap = late_20k
    _restore(m, snap)
    _sparse_estep(m, it, 1024, True)
    _assert_repeats(m, it, "20k 3-D late, k=1024")
