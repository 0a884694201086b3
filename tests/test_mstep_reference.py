"""CPU: the float64 M-step reference of tests/parity_helpers.py (``mstep_reference``, built from the E-step's sufficient
statistics) against the oracle's own M-step methods on the same state, to 1e-12. The GPU M-step tests compare the device
with this reference, so it is pinned here to the oracle, which tests/test_oracle_golden.py pins to the reference
implementation."""

import numpy as np
import pytest

from oracle import morpho_oracle as mo
from parity_helpers import mstep_reference, oracle_mstep_inputs

CASES = {
    # name: (dim, SVI_mode, it, extra oracle keyword arguments)
    "2d_full_nn": (2, False, 6, {}),
    "3d_full_nonn": (3, False, 5, dict(nn_init=False)),
    "2d_svi_step_lt_1": (2, True, 14, dict(batch_size=120)),
    "3d_svi_nn_rigid_phase": (3, True, 12, dict(batch_size=120, nonrigid_start_iter=20)),
    "2d_full_guide_rigid": (2, False, 6, dict(guidance_effect="rigid")),
    "2d_svi_guide_nonrigid": (2, True, 13, dict(guidance_effect="nonrigid", batch_size=150)),
    "3d_full_guide_both": (3, False, 6, dict(guidance_effect="both")),
    "2d_full_no_update_R_kappa": (2, False, 6, dict(update_R=False, kappa="array")),
}


def _rotation(dim, a):
    c, s = np.cos(a), np.sin(a)
    if dim == 2:
        return np.array([[c, -s], [s, c]])
    return np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])


def _oracle(dim, svi, kw):
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(300, 280, 24, dim=dim, seed=2, warp_amplitude=2.0)  # B moves onto A
    kw = dict(kw)
    if "guidance_effect" in kw:
        pts = np.random.default_rng(5).uniform(10, 90, size=(12, dim))
        kw["guidance_pair"] = [pts, pts @ _rotation(dim, 0.5).T + 5.0]
    if kw.get("kappa") == "array":
        kw["kappa"] = np.random.default_rng(9).uniform(0.5, 3.0, size=B.X.shape[0])
    kw.setdefault("nonrigid_start_iter", 3)
    np.random.seed(0)
    return mo.MorphoPairOracle(np.asarray(B.obsm["spatial"], np.float64), np.asarray(A.obsm["spatial"], np.float64),
                               [np.asarray(B.X, np.float64)], [np.asarray(A.X, np.float64)], dtype="float64",
                               SVI_mode=svi, max_iter=40, K=15, **kw)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


@pytest.mark.parametrize("case", list(CASES))
def test_mstep_reference_matches_oracle_methods(case):
    dim, svi, it, kw = CASES[case]
    o = _oracle(dim, svi, kw)
    o.prepare()
    for i in range(it):
        o.em_iteration(i)
    s = oracle_mstep_inputs(o, it)
    ref = mstep_reference(s)
    assert (s["step"] < 1) == (svi and it >= 10)
    # the oracle's own M-step on the same state
    o._update_gamma()
    o._update_alpha()
    nonrigid = s["nonrigid"]
    if nonrigid:
        o._update_nonrigid()
    o._update_rigid()
    o.XAHat = o.VnA + o.RnA
    o._update_sigma2(it)
    want = dict(
        gamma=o.gamma, alpha=o.alpha, Sp=o.Sp, Sp_spatial=o.Sp_spatial, Sp_sigma2=o.Sp_sigma2,
        sigma2_related=o.sigma2_related, VnA=o.VnA, SigmaDiag=o.SigmaDiag, R=o.R, t=o.t, RnA=o.RnA, XAHat=o.XAHat,
        sigma2=o.sigma2, sigma2_variance=o.sigma2_variance, mm=o.alpha * np.exp(-o.SigmaDiag / o.sigma2),
        lm=np.log2(o.alpha * np.exp(-o.SigmaDiag / o.sigma2)),
    )
    if nonrigid:
        want.update(Sigma=o.Sigma, Coff=o.Coff)
        if svi:
            want.update(SigmaInv=o.SigmaInv, PXB_term=o.PXB_term)
    if o.guidance:
        want.update(R_AI=o.R_AI)
        if o.guidance_effect in ("nonrigid", "both"):
            want.update(V_AI=o.V_AI)
    for k, v in want.items():
        assert _rel(ref[k], v) <= 1e-12, (k, _rel(ref[k], v))
    # the cases must reach the branches they are named for
    assert nonrigid == (it > o.nonrigid_start_iter)
    if case == "2d_full_no_update_R_kappa":
        assert np.array_equal(ref["R"], s["R"]) and np.ptp(s["kappa"]) > 1.0


def test_pinv_cutoff_is_k_times_eps_in_fp64():
    """An eigenvalue at 0.3x the cutoff K * eps(float32) * max|ev| is dropped, one at 3x is kept: the reference keeps the
    fp32 rule in fp64 arithmetic instead of scipy's fp64 default."""
    from scipy.linalg import pinv

    K, eps = 15, float(np.finfo(np.float32).eps)
    Q, _ = np.linalg.qr(np.random.default_rng(0).normal(size=(K, K)))
    ev = np.geomspace(1.0, 1e-2, K)
    ev[-2], ev[-1] = 3.0 * K * eps, 0.3 * K * eps
    A = (Q * ev) @ Q.T
    got = pinv(A, atol=0.0, rtol=K * eps)
    want = (Q[:, :-1] / ev[:-1]) @ Q[:, :-1].T
    assert _rel(got, want) < 1e-6
    assert _rel(pinv(A), want) > 1e-2  # scipy's default cutoff keeps the small eigenvalue
