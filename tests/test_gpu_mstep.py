"""The M-step on the device against float64, one step at a time.

Part 1 runs the solver to iteration it - 1, runs the E-step of iteration it, reads the device's own E-step outputs and the
M-step's running state, runs ``_mstep`` and compares every M-step output with ``parity_helpers.mstep_reference`` fed with
those same device values widened from fp32 (U, Gamma, coordinates and E-step statistics as the device holds them): the
comparison measures the M-step alone. Part 2 writes the inputs of single M-step kernels directly and checks them at their
edges (spectra around the pseudo-inverse cutoff, Jacobi warm starts, reflections and rank-deficient Procrustes problems,
digamma arguments from 1e-3 to 1e7, underflowing model multipliers, the ordered reductions' grid cap).

Every bar was measured on an H100 SXM; the measured value and the fp32 restatement's own deviation (``mstep_reference``
evaluated in fp32, the scale of what the reference's fp32 run computes) are printed next to each check."""

import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from parity_helpers import mstep_reference  # noqa: E402

EPS32, EPS64 = float(np.finfo(np.float32).eps), float(np.finfo(np.float64).eps)


def _torch():
    import torch

    return torch


def _stream():
    torch = _torch()
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _check(rc, what):
    from spateo_release_b200._capi import check

    check(rc, what)


def _lib():
    from spateo_release_b200._capi import load_library

    return load_library()


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-300))


class _Bars:
    """Collects every comparison of a test, prints them as one table and fails on any over its bar."""

    def __init__(self, title):
        self.title, self.rows = title, []

    def __call__(self, name, got, want, bar, fp32=None):
        err = _rel(got, want)
        self.rows.append((name, err, bar, fp32))
        return err

    def done(self):
        print(f"\n[{self.title}]")
        for name, err, bar, fp32 in self.rows:
            ref = "" if fp32 is None else f"   fp32 restatement {fp32:.2e}"
            print(f"  {name:16s} {err:.2e}  (bar {bar:.0e}){ref}")
        bad = [(n, e, b) for n, e, b, _ in self.rows if not e <= b]
        assert not bad, bad


# ---------------------------------------------------------------------------------------------------------------------
# Part 1: one whole M-step from an identical state
# ---------------------------------------------------------------------------------------------------------------------

N_MOVING, N_FIXED = 2999, 2711  # not a multiple of the 512-row tile, six row blocks


def _solver(D=2, planar=False, svi=False, K=15, nn_init=True, guide=None, update_R=True, kappa=False,
            kernel_type="euc", start=30):
    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(N_MOVING, N_FIXED, 32, dim=D, seed=11, warp_amplitude=2.0, z_thickness=20.0)
    if planar:  # the moving cells within 1e-6 of one z (an exactly constant axis is dropped as a 2-D slice)
        A.obsm["spatial"][:, 2] = 5.0 + 1e-6 * np.random.default_rng(2).uniform(size=N_MOVING)
    kw = dict(SVI_mode=svi, max_iter=120, K=K, nn_init=nn_init, update_R=update_R, nonrigid_start_iter=start,
              kernel_type=kernel_type, verbose=False, device="0", materialize_P=False)
    if guide is not None:
        pts = np.random.default_rng(5).uniform(10, 90, size=(12, D))
        kw.update(guidance_pair=[pts + 2.0, pts], guidance_effect=guide)
    if kappa:
        kw["kappa"] = np.random.default_rng(9).uniform(0.5, 3.0, size=N_MOVING)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(sampleA=A, sampleB=B, **kw)
    m.prepare()
    return m


def _rows(m, name):
    return m._state[name][: m.NA].double().cpu().numpy()


def _rows3(m, name):
    return m._state[name][: m.D, : m.NA].T.double().cpu().numpy()


def _mat(m, name):
    t = m._state.get(name)
    return None if t is None else t.double().cpu().numpy()


def _device_state(m):
    sc = m._read_scalars()
    D = m.D
    out = dict(
        alpha=_rows(m, "alpha"), SigmaDiag=_rows(m, "SigmaDiag"), VnA=_rows3(m, "VnA"), RnA=_rows3(m, "RnA"),
        XAHat=_rows3(m, "XAHat"), PXB_term=_rows3(m, "PXB_term"), mm=_rows(m, "mm"), lm=_rows(m, "lm"),
        SigmaInv=_mat(m, "SigmaInv"), Sigma=_mat(m, "Sigma"), Coff=_mat(m, "Coff")[:, :D],
        Sp=sc.Sp, Sp_spatial=sc.Sp_spatial, Sp_sigma2=sc.Sp_sigma2, sigma2=sc.sigma2, gamma=sc.gamma,
        sigma2_variance=sc.sigma2_variance, sigma2_related=sc.sigma2_related,
        R=np.array(sc.R[:]).reshape(3, 3)[:D, :D], t=np.array(sc.t[:D]), sums=list(sc.sums),
    )
    if "g_VA" in m._state:
        out.update(V_AI=_mat(m, "g_VA")[:, :D], R_AI=_mat(m, "g_RA")[:, :D])
    return out


def _reference_inputs(m, it, pre, post_e):
    """mstep_reference inputs from the device: the running state before the M-step (``pre``), the E-step's outputs and
    the constants as the device holds them, in the device's row order."""
    p, D, K = m._params, m.D, m.K
    sums = post_e["sums"]
    PXB = _rows3(m, "PXB")
    s = dict(
        D=D, it=it, svi=bool(p.svi), step=min(1.0, 10.0 / (it + 1.0)) if p.svi else 1.0,
        nonrigid=it > m.nonrigid_start_iter,
        K_NA=_rows(m, "K_NA"), K_NA_spatial=_rows(m, "K_NA_spatial"), K_NA_sigma2=_rows(m, "K_NA_sigma2"), PXB=PXB,
        # the device forms sum_i (P @ YB)_i for K_NB @ YB (the same number: P's row sums of P @ YB are its column sums)
        KNB_YB=PXB.sum(0), Sp_spatial_new=sums[0], Sp_sigma2_new=sums[1], Sp_new=sums[2], S2=sums[3],
        U=m._UT[:K, : m.NA].T.double().cpu().numpy(), Gamma=_mat(m, "Gamma"), coordsA=_rows3(m, "xa"),
        kappa=_rows(m, "kappa"), gamma_a=p.gamma_a, gamma_b=p.gamma_b, n_gamma=p.NB_total if p.NB_total > 0 else p.NBb,
        lambdaVF=p.lambdaVF, pinv_eps=p.pinv_eps, update_R=bool(p.update_R), nn_init=bool(p.nn_init),
        nn_init_weight=p.nn_init_weight, sigma2_variance_decress=p.sigma2_variance_decress,
        sigma2_variance_end=p.sigma2_variance_end,
    )
    for k in ("alpha", "SigmaInv", "PXB_term", "Sp", "Sp_spatial", "Sp_sigma2", "R", "t", "RnA", "VnA", "SigmaDiag",
              "sigma2", "sigma2_variance", "V_AI", "R_AI"):
        s[k] = pre.get(k)
    if m.nn_init:
        s.update(inlier_A=m.inlier_A, inlier_B=m.inlier_B, inlier_P=m.inlier_P)
    if m.guidance:
        s["guidance"] = dict(X_AI=_mat(m, "g_XA")[:, :D], X_BI=_mat(m, "g_XB")[:, :D], U_I=_mat(m, "g_UI"),
                             weight=m.guidance_weight, effect=m.guidance_effect)
    return s


# (id, solver keywords, it, jacobi warm start, NB_total multiple)
MSTEP_CASES = [
    ("2d_full_rigid_K15_nn", dict(D=2, K=15), 5, "warm", 0),
    ("3d_svi_rigid_K32_nonn", dict(D=3, svi=True, K=32, nn_init=False), 5, "warm", 0),
    ("2d_svi_step_lt1_K33_both_kappa", dict(D=2, svi=True, K=33, guide="both", kappa=True), 60, "warm", 0),
    ("planar_full_K64_rigidguide_noR", dict(D=3, planar=True, K=64, nn_init=False, guide="rigid", update_R=False), 95,
     "cold", 0),
    ("2d_svi_K65_nonrigidguide", dict(D=2, svi=True, K=65, guide="nonrigid"), 95, "warm", 0),
    ("3d_full_K200_nn_nbtotal", dict(D=3, K=200), 60, "warm", 3),
    ("2d_full_K1_cold_nbtotal", dict(D=2, K=1), 60, "cold", 2),
    ("3d_svi_K2_geodist", dict(D=3, svi=True, K=2, kernel_type="geodist", nn_init=False), 60, "warm", 0),
    ("2d_full_K15_floor_side", dict(D=2, K=15, start=80), 105, "warm", 0),
    ("3d_svi_K32_step1_nonrigid", dict(D=3, svi=True, K=32, start=2), 5, "cold", 0),
]


@pytest.mark.parametrize("case", [c[0] for c in MSTEP_CASES])
def test_one_mstep_matches_float64_reference(case):
    torch = _torch()
    _, kw, it, ws, nb_mult = next(c for c in MSTEP_CASES if c[0] == case)
    m = _solver(**kw)
    m.run_em(n_iter=it)
    torch.cuda.synchronize()
    st, p = _stream(), m._params
    if nb_mult:  # a column chunk or shard of the iteration: gamma takes the whole iteration's column count
        p.NB_total = nb_mult * p.NBb
    if ws == "cold" and m._state["jacobi_ws"] is not None:
        m._state["jacobi_ws"].zero_()
    elif m._state["jacobi_ws"] is not None and it > m.nonrigid_start_iter + 1 and m.K <= 64:
        assert float(m._state["jacobi_ws"][0]) == m.K  # the previous iteration's eigenbasis
    pre = _device_state(m)
    m._estep_only(it, st)
    torch.cuda.synchronize()
    post_e = _device_state(m)
    s = _reference_inputs(m, it, pre, post_e)
    m._mstep(it, st)
    torch.cuda.synchronize()
    got = _device_state(m)
    ref = mstep_reference(s)
    r32 = mstep_reference(s, dtype=np.float32)
    nonrigid = s["nonrigid"]
    large_K = m.K > 64
    b = _Bars(f"one M-step {case}, it {it}, step {s['step']:.3f}, sigma2 {ref['sigma2']:.3e}")

    def chk(name, bar, gkey=None):
        g = got[gkey or name]
        f32 = _rel(r32[name], ref[name]) if isinstance(r32.get(name), np.ndarray) else None
        b(name, g, ref[name], bar, f32)

    # fp64 scalars from fp64 sums of the device's E-step: rounding only (measured: 0 to 2e-16)
    for k in ("Sp", "Sp_spatial", "Sp_sigma2", "sigma2_related", "gamma", "sigma2_variance"):
        chk(k, 1e-13)
    # per-row fp32 results of fp64 arithmetic: one rounding to fp32 (measured <= 6e-8)
    chk("alpha", 3 * EPS32)
    if nonrigid:
        # U^T diag(K_NA) U takes the products u * K_NA rounded to fp32 like the reference's fp32 product: fp64 gram up to
        # 32 inducing points (measured <= 1.1e-9), 3xTF32 tensor-core gram above (measured <= 3.4e-8; its own bar is 5e-7)
        chk("SigmaInv", 1e-8 if m.K <= 32 else 5e-7)
        chk("PXB_term", 4 * EPS32)  # measured <= 4.1e-8
        # the pseudo-inverse multiplies SigmaInv's relative error by the condition number of the kept spectrum (1e2 to
        # 1e5 here), and Coff also carries the cancellation in PXB_term: measured Sigma <= 4.8e-6, Coff <= 3.8e-5, while
        # the fp32 restatement is 2e-4 to 3e-3 off
        chk("Sigma", 5e-5)
        chk("Coff", 1e-4)
        chk("VnA", 1e-5)  # measured <= 2.0e-6
        chk("SigmaDiag", 1e-5)  # measured <= 4.1e-6
        if "V_AI" in got and m.guidance_effect in ("nonrigid", "both"):
            chk("V_AI", 1e-5)  # measured <= 1.3e-6
    # rigid phase: fp64 throughout (measured R <= 4e-16, t <= 8e-15); non-rigid phase: the field's error moves the
    # moments (measured R <= 2.9e-8, t <= 7.0e-7)
    chk("R", 2e-7 if nonrigid else 1e-12)
    chk("t", 3e-6 if nonrigid else 1e-12)
    chk("RnA", 4 * EPS32)  # measured <= 4.7e-8
    chk("XAHat", 1e-6 if nonrigid else 4 * EPS32)  # measured <= 4.3e-7
    # non-rigid phase: sum K_NA_sigma2 SigmaDiag / Sp_sigma2 carries SigmaDiag's error (measured <= 3.6e-9)
    chk("sigma2", 1e-7 if nonrigid else 1e-13)
    chk("mm", 4 * EPS32)  # measured <= 8.9e-8
    chk("lm", 4 * EPS32)  # measured <= 4.4e-8
    if m.guidance:
        chk("R_AI", 3e-6 if nonrigid else 1e-12)  # R_AI R^T + t: the error of t
    b.done()
    if large_K:  # the low-rank factor and the full Sigma give the same field
        lo = (_rows3(m, "VnA"), _rows(m, "SigmaDiag"))
        _check(m._lib.spb_field_apply(C.byref(p), st), "spb_field_apply")
        torch.cuda.synchronize()
        assert _rel(lo[0], _rows3(m, "VnA")) < 1e-6 and _rel(lo[1], _rows(m, "SigmaDiag")) < 1e-6
    if kw.get("planar"):
        assert np.allclose(ref["R"] @ ref["R"].T, np.eye(3), atol=1e-12)


def _snapshot(m):
    torch = _torch()
    return {k: v.clone() for k, v in m._state.items() if isinstance(v, torch.Tensor)}


def _restore(m, snap):
    for k, v in snap.items():
        m._state[k].copy_(v)


_OUTPUTS = ("alpha", "SigmaDiag", "VnA", "RnA", "XAHat", "mm", "lm", "PXB_term", "SigmaInv", "Sigma", "Coff", "sc",
            "jacobi_ws", "K_NA", "PXB", "moments")


@pytest.mark.parametrize("it", [20, 60])
def test_fused_split_and_replay_iterations_are_bit_identical(it):
    """The fused spb_em_iteration, the split E-step + _mstep, and spb_em_iteration_ex(iter=-1) with the device counter
    at it - 1 (the launch sequence graph replay uses) give the same bits from the same state."""
    torch = _torch()
    m = _solver(D=2, svi=True, K=33 if it == 60 else 15, guide="both", start=30)
    m.run_em(n_iter=it)
    torch.cuda.synchronize()
    st, p, lib = _stream(), m._params, m._lib
    snap = _snapshot(m)
    assert m._read_scalars().iter == it - 1
    outs = []
    for path in ("fused", "split", "replay"):
        _restore(m, snap)
        if path == "fused":
            _check(lib.spb_em_iteration(C.byref(p), it, st), "spb_em_iteration")
        elif path == "split":
            m._estep_only(it, st)
            m._mstep(it, st)
        else:
            _check(lib.spb_em_iteration_ex(C.byref(p), -1, int(it > m.nonrigid_start_iter), st), "spb_em_iteration_ex")
        torch.cuda.synchronize()
        outs.append({k: m._state[k].clone() for k in _OUTPUTS if m._state.get(k) is not None})
    for k in outs[0]:
        assert torch.equal(outs[0][k], outs[1][k]), ("split", k)
        assert torch.equal(outs[0][k], outs[2][k]), ("replay", k)


# ---------------------------------------------------------------------------------------------------------------------
# Part 2: single kernels from directly written state
# ---------------------------------------------------------------------------------------------------------------------


class _Params:
    """An spb_em_params with its own device buffers (fp64 unless given as tensors); only what a kernel reads is set."""

    def __init__(self, NA=1, D=3, K=1, **scalars):
        from spateo_release_b200._capi import SpbEmParams, SpbScalars

        torch = _torch()
        self.dev = torch.device("cuda:0")
        self.p = SpbEmParams()
        self.p.NA, self.p.D, self.p.K = NA, D, K
        self.p.ldx = ((NA + 511) // 512) * 512
        self.bufs = {}
        self.sc = SpbScalars()
        for q in range(9):
            self.sc.R[q] = 1.0 if q in (0, 4, 8) else 0.0
        for k, v in scalars.items():
            setattr(self.p, k, v)
        self.set("sc", torch.zeros((C.sizeof(SpbScalars),), dtype=torch.uint8))
        self.set("red_scratch", torch.zeros((592 * 29 + 64,), dtype=torch.float64))
        self.p.red_scratch_doubles = 592 * 29 + 64
        self.set("red_counter", torch.zeros((8,), dtype=torch.int32))

    def set(self, name, arr, dtype=None):
        torch = _torch()
        t = arr if isinstance(arr, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(arr, dtype=dtype or np.float64))
        t = t.to(self.dev).contiguous()
        self.bufs[name] = t
        setattr(self.p, name, t.data_ptr())
        return t

    def rows(self, name, arr, n3=False):
        """Per-row fp32 vector [ldx] or SoA [3][ldx] (arr [NA] or [NA, <=3])."""
        a = np.asarray(arr, np.float32)
        if n3:
            buf = np.zeros((3, self.p.ldx), np.float32)
            buf[: a.shape[1], : a.shape[0]] = a.T
        else:
            buf = np.zeros((self.p.ldx,), np.float32)
            buf[: a.shape[0]] = a
        return self.set(name, buf, np.float32)

    def push_sc(self):
        torch = _torch()
        self.bufs["sc"].copy_(torch.from_numpy(np.frombuffer(bytes(self.sc), dtype=np.uint8).copy()))

    def pull_sc(self):
        from spateo_release_b200._capi import SpbScalars

        return SpbScalars.from_buffer_copy(self.bufs["sc"].cpu().numpy().tobytes())

    def get(self, name, n=None):
        t = self.bufs[name]
        return t.double().cpu().numpy() if n is None else t.double().cpu().numpy()[..., :n]

    def call(self, fn, *args):
        torch = _torch()
        self.push_sc()
        _check(getattr(_lib(), fn)(C.byref(self.p), *args, _stream()), fn)
        torch.cuda.synchronize()
        return self.pull_sc()


def _spectrum_matrix(K, spectrum, rng):
    Q, _ = np.linalg.qr(rng.normal(size=(K, K)))
    if spectrum == "well":
        ev = np.geomspace(1e3, 1e1, K)
    elif spectrum == "cond1e10":
        ev = np.geomspace(1.0, 1e-10, K)
    elif spectrum == "cutoff_straddle":  # around K * eps(float32) * max: nothing closer to the cutoff than 0.3x / 3x
        cut = K * EPS32
        ev = np.concatenate([np.geomspace(1.0, 30 * cut, K - 2 * (K // 3)), np.full(K // 3, 3 * cut),
                             np.full(K // 3, 0.3 * cut)]) if K >= 3 else np.array([1.0, 0.3 * cut][:K])
    else:  # SigmaInv of inducing points that nearly coincide (beta small against their spread): a dense low-rank tail
        pts = rng.uniform(-1, 1, size=(K, 2))
        pts[1::4] = pts[0::4][: len(pts[1::4])] + 1e-4
        x = rng.uniform(-1.5, 1.5, size=(4000, 2))
        U = np.exp(-0.5 * ((x[:, None, :] - pts[None]) ** 2).sum(-1))
        G = np.exp(-0.5 * ((pts[:, None, :] - pts[None]) ** 2).sum(-1)).astype(np.float32).astype(np.float64)
        A = 0.05 * 100.0 * G + U.T @ (U * rng.uniform(0, 1, size=(4000, 1)))
        return 0.5 * (A + A.T)
    return (Q * ev) @ Q.T


def _pinv64(A, eps):
    from scipy.linalg import pinv

    return pinv(A, atol=0.0, rtol=A.shape[0] * eps)


def _solve(A, rhs, start, eps, rng):
    """spb_nonrigid_solve of SigmaInv = A (UtWU = A, lambdaVF = 0, full EM) from the given warm start."""
    K = A.shape[0]
    P = _Params(K=K, svi=0, lambdaVF=0.0, pinv_eps=eps)
    P.set("UtWU", A)
    P.set("Gamma", np.zeros((K, K), np.float32), np.float32)
    P.set("SigmaInv", np.zeros((K, K)))
    P.set("Sigma", np.zeros((K, K)))
    P.set("UtPXB", rhs)
    P.set("Coff", np.zeros((K, 3)))
    ws = np.zeros(1 + K * K)
    if start == "warm_true":
        ws[0] = K
        ws[1:] = np.linalg.eigh(A)[1].reshape(-1)
    elif start == "warm_random":
        ws[0] = K
        ws[1:] = np.linalg.qr(rng.normal(size=(K, K)))[0].reshape(-1)
    elif start == "ws_other_K":  # a basis of another size must be ignored (cold start)
        ws[0] = K + 1
        ws[1:] = rng.normal(size=K * K)
    P.set("jacobi_ws", ws)
    P.sc.sigma2, P.sc.step = 1.0, 1.0
    P.call("spb_nonrigid_solve")
    return P.get("Sigma"), P.get("Coff"), P.get("jacobi_ws")


SPECTRA = ["well", "cond1e10", "cutoff_straddle", "clustered"]


@pytest.mark.parametrize("K", [15, 40, 64])
@pytest.mark.parametrize("spectrum", SPECTRA)
def test_nonrigid_solve_spectrum_and_warm_starts(spectrum, K):
    rng = np.random.default_rng(K)
    A = _spectrum_matrix(K, spectrum, rng)
    # the cond-1e10 matrix is inverted whole under the geodesic kernel's eps(float64) cutoff
    eps = EPS64 if spectrum == "cond1e10" else EPS32
    want = _pinv64(A, eps)
    rhs = rng.normal(size=(K, 3))
    ev = np.abs(np.linalg.eigvalsh(A))
    cut = ev.max() * K * eps
    kept = ev[ev > cut]
    cond = kept.max() / kept.min()
    if spectrum == "cutoff_straddle":
        assert (ev > 3 * cut * 0.99).sum() + (ev < 0.3 * cut * 1.01).sum() == K
    # backward-stable eigensolver: relative error of the pseudo-inverse ~ cond(kept) * eps(float64)
    bar = max(1e-13, 64 * cond * EPS64)
    b = _Bars(f"nonrigid solve K {K} {spectrum}, kept {kept.size}/{K}, cond {cond:.1e}")
    for start in ("cold", "warm_true", "warm_random", "ws_other_K"):
        S, Cf, ws = _solve(A, rhs, start, eps, rng)
        b(f"Sigma {start}", S, want, bar)
        b(f"Coff {start}", Cf, want @ rhs, bar)
        assert np.array_equal(S, S.T), start
        V = ws[1:].reshape(K, K)
        assert ws[0] == K
        off = V.T @ A @ V
        assert np.abs(off - np.diag(np.diag(off))).max() <= 1e-12 * ev.max(), start  # the saved basis diagonalises A
    b.done()


def test_nonrigid_solve_svi_blend_and_guidance():
    K, NI = 21, 7
    rng = np.random.default_rng(3)
    Gm = _spectrum_matrix(K, "well", rng) / 1e3
    G32 = Gm.astype(np.float32)
    UtWU = _spectrum_matrix(K, "well", rng)
    prev = _spectrum_matrix(K, "well", rng)
    UI = rng.uniform(0, 1, size=(NI, K))
    XB, RA = rng.normal(size=(NI, 3)), rng.normal(size=(NI, 3))
    rhs = rng.normal(size=(K, 3))
    P = _Params(K=K, svi=1, lambdaVF=100.0, pinv_eps=EPS32, g_on=1, g_nonrigid=1, g_NI=NI, g_weight=0.7)
    P.set("UtWU", UtWU)
    P.set("Gamma", G32, np.float32)
    P.set("SigmaInv", prev)
    P.set("Sigma", np.zeros((K, K)))
    P.set("UtPXB", rhs)
    P.set("Coff", np.zeros((K, 3)))
    P.set("jacobi_ws", np.zeros(1 + K * K))
    for name, v in (("g_UI", UI), ("g_G1", UI.T @ UI), ("g_XB", XB), ("g_RA", RA), ("g_VA", np.zeros((NI, 3)))):
        P.set(name, v)
    P.sc.sigma2, P.sc.step, P.sc.Sp = 0.05, 0.3, 812.5
    P.call("spb_nonrigid_solve")
    cg = 0.05 * 0.7 * 812.5 / NI
    SI = 0.3 * (0.05 * 100.0 * G32.astype(np.float64) + UtWU) + 0.7 * prev + cg * UI.T @ UI
    UP = rhs + cg * UI.T @ (XB - RA)
    S = _pinv64(0.5 * (SI + SI.T), EPS32)
    b = _Bars("nonrigid solve: SVI blend + nonrigid guidance")
    b("SigmaInv", P.get("SigmaInv"), SI, 1e-15)
    b("UtPXB", P.get("UtPXB"), UP, 1e-15)
    b("Sigma", P.get("Sigma"), S, 1e-13)
    b("Coff", P.get("Coff"), S @ UP, 1e-13)
    b("V_AI", P.get("g_VA"), UI @ (S @ UP), 1e-13)
    b.done()


@pytest.mark.parametrize("rank,ldg", [(0, 40), (13, 13), (13, 40), (16, 16), (37, 45)])
def test_field_apply_lowrank_matches_float64(rank, ldg):
    K, NA = 37, 1500
    rng = np.random.default_rng(rank + ldg)
    U = rng.uniform(0, 1, size=(NA, K)).astype(np.float32)
    Cf = rng.normal(size=(K, 3))
    G = np.zeros((K, ldg))
    G[:, :rank] = rng.normal(size=(K, rank))
    P = _Params(NA=NA, K=K)
    ut = np.zeros((K, P.p.ldx), np.float32)
    ut[:, :NA] = U.T
    P.set("UT", ut, np.float32)
    P.set("Coff", Cf)
    P.rows("VnA", np.zeros((NA, 3)), n3=True)
    P.rows("SigmaDiag", np.zeros(NA))
    Gd = P.set("G", G)
    rk = P.set("rank", np.array([rank], np.int32), np.int32)
    P.sc.sigma2 = 0.37
    P.push_sc()
    _check(_lib().spb_field_apply_lowrank(C.byref(P.p), C.c_void_p(Gd.data_ptr()), ldg, C.c_void_p(rk.data_ptr()),
                                          _stream()), "spb_field_apply_lowrank")
    _torch().cuda.synchronize()
    U64 = U.astype(np.float64)
    b = _Bars(f"low-rank field apply rank {rank} ldg {ldg}")
    b("VnA", P.get("VnA")[:, :NA].T, U64 @ Cf, 2 * EPS32)
    sd = 0.37 * ((U64 @ G[:, :rank]) ** 2).sum(1)
    if rank == 0:
        assert not P.get("SigmaDiag")[:NA].any()
    else:
        b("SigmaDiag", P.get("SigmaDiag")[:NA], sd, 2 * EPS32)
    b.done()


def _rigid_params(A, D, scale=1.0, nn_init=False, svi=0):
    """Moments whose first sums are zero, so that both kernels' cross-covariance is A itself: spb_rigid_solve forms
    A[d2][d1] from m[18 + d1 * 3 + d2], spb_optimal_rigid forms A[d1][d2] from m[18 + d2 * 3 + d1]."""
    m = np.zeros(32)
    for d1 in range(D):
        for d2 in range(D):
            m[18 + d1 * 3 + d2] = A[d2, d1] * scale
    m[28] = 100.0
    P = _Params(D=D, svi=svi, update_R=1, nn_init=int(nn_init), inl_SP=1.0, sigma2_variance_decress=1.0,
                sigma2_variance_end=1.0)
    P.set("moments", m)
    P.sc.Sp, P.sc.Sp_sigma2, P.sc.sigma2, P.sc.sigma2_related, P.sc.sigma2_variance, P.sc.step = 100, 100, 1, 0.5, 1, 1
    return P


def _kabsch(A):
    U, _, Vh = np.linalg.svd(A)
    Cm = np.eye(A.shape[0])
    Cm[-1, -1] = np.linalg.det(U @ Vh)
    return U @ Cm @ Vh


def _with_singular_values(D, s, det_sign, rng):
    U = np.linalg.qr(rng.normal(size=(D, D)))[0]
    V = np.linalg.qr(rng.normal(size=(D, D)))[0]
    A = (U * np.asarray(s, float)) @ V.T
    if np.sign(np.linalg.det(U @ V.T)) != det_sign:
        U[:, -1] *= -1
        A = (U * np.asarray(s, float)) @ V.T
    return A


RIGID_CASES = {
    "3d_proper": (3, [3.0, 2.0, 1.0], 1),
    "3d_reflection": (3, [3.0, 2.0, 1.0], -1),
    "3d_two_equal": (3, [2.0, 2.0, 0.5], 1),
    "3d_two_equal_reflection": (3, [2.0, 2.0, 0.5], -1),
    "3d_planar_rank2": (3, [3.0, 1.0, 0.0], 1),
    "3d_planar_equal": (3, [1.5, 1.5, 0.0], -1),
    "2d_proper": (2, [2.0, 1.0], 1),
    "2d_reflection": (2, [2.0, 1.0], -1),
    "2d_rank1": (2, [2.0, 0.0], 1),
}


@pytest.mark.parametrize("scale", [1e-6, 1.0, 1e6])
@pytest.mark.parametrize("case", list(RIGID_CASES))
def test_rigid_solve_and_optimal_rigid_rotation_edges(case, scale):
    D, s, sign = RIGID_CASES[case]
    rng = np.random.default_rng(len(case))
    A = _with_singular_values(D, s, sign, rng)
    want = _kabsch(A)
    P = _rigid_params(A, D, scale * scale)  # the moments are quadratic in the coordinates
    sc = P.call("spb_rigid_solve", 50)
    R = np.array(sc.R[:]).reshape(3, 3)[:D, :D]
    Pt = _rigid_params(A, D, scale * scale)
    out = Pt.set("optimal", np.zeros(12))
    Pt.push_sc()
    _check(_lib().spb_optimal_rigid(C.byref(Pt.p), C.c_void_p(out.data_ptr()), _stream()), "spb_optimal_rigid")
    _torch().cuda.synchronize()
    Ro = out.cpu().numpy()[:9].reshape(3, 3)[:D, :D]
    for name, got in (("rigid_solve", R), ("optimal_rigid", Ro)):
        assert np.abs(got - want).max() <= 1e-12, (name, np.abs(got - want).max())  # R is unique for rank >= D - 1
        assert np.abs(got @ got.T - np.eye(D)).max() <= 1e-13, name
        assert abs(np.linalg.det(got) - 1.0) <= 1e-13, name
    assert np.abs(np.array(sc.t[:D])).max() == 0.0


def _rigid_from_points(rng, D, NA, svi, step, it, nn_init, sigma2_target=None):
    """Random moving cells, weights and targets: the moments the device would sum, and the mstep_reference inputs."""
    x = rng.uniform(-1, 1, size=(NA, D))
    w = rng.uniform(0.1, 1.0, size=NA)
    v = 0.01 * rng.normal(size=(NA, D))
    Rt = _kabsch(rng.normal(size=(D, D)))
    px = w[:, None] * (x @ Rt.T + 0.3 + 0.02 * rng.normal(size=(NA, D)))
    k2 = rng.uniform(0.1, 1.0, size=NA)
    sd = rng.uniform(0, 1e-3, size=NA)
    X3 = lambda a: np.pad(a, ((0, 0), (0, 3 - D)))
    m = np.zeros(32)
    m[0:3], m[3:6], m[6:9] = w @ X3(x), w @ X3(v), X3(px).sum(0)
    m[9:18] = ((X3(x) * w[:, None]).T @ X3(v)).reshape(-1)
    m[18:27] = (X3(x).T @ X3(px)).reshape(-1)
    m[27], m[28] = k2 @ sd, w.sum()
    Sp = 1.3 * w.sum() if svi else w.sum()  # SVI: the running average differs from this batch's sum
    Sp_sigma2 = 0.9 * k2.sum()
    S2 = (sigma2_target - m[27] / Sp_sigma2) * D * Sp_sigma2 if sigma2_target else 0.02 * D * Sp_sigma2
    R0, t0 = _kabsch(rng.normal(size=(D, D))), rng.normal(size=D)
    s = dict(D=D, it=it, svi=svi, step=step, nonrigid=False, K_NA=w, K_NA_spatial=w, K_NA_sigma2=k2, PXB=px,
             KNB_YB=px.sum(0), Sp_new=Sp, Sp_spatial_new=Sp, Sp_sigma2_new=Sp_sigma2, S2=S2, U=np.zeros((NA, 1)),
             Gamma=np.zeros((1, 1)), coordsA=x, kappa=np.ones(NA), gamma_a=1.0, gamma_b=1.0, n_gamma=1000,
             lambdaVF=100.0, pinv_eps=EPS32, update_R=True, nn_init=nn_init, nn_init_weight=0.8,
             sigma2_variance_decress=1.02, sigma2_variance_end=10.0, alpha=np.ones(NA), SigmaInv=None, PXB_term=None,
             Sp=Sp, Sp_spatial=Sp, Sp_sigma2=Sp_sigma2, R=R0, t=t0, RnA=x, VnA=v, SigmaDiag=sd, sigma2=0.04,
             sigma2_variance=3.0)
    if svi:  # make the running sums equal to Sp (the blend is checked by the gamma / alpha test)
        s.update(Sp_new=Sp, Sp_spatial_new=Sp, Sp_sigma2_new=Sp_sigma2)
    if nn_init:
        n = 40
        iA = rng.uniform(-1, 1, size=(n, D))
        s.update(inlier_A=iA, inlier_B=iA @ Rt.T + 0.3, inlier_P=rng.uniform(0.2, 1, size=(n, 1)))
    return s, m


@pytest.mark.parametrize("D", [2, 3])
@pytest.mark.parametrize("svi,step,nn_init", [(False, 1.0, True), (True, 0.25, True), (True, 0.25, False)])
@pytest.mark.parametrize("it", [99, 100])
def test_rigid_solve_matches_reference_from_moments(D, svi, step, nn_init, it):
    """R, t and sigma2 from moments of random weighted cells, with the nn_init prior (whose weight uses the running Sp,
    not this batch's sum of K_NA), the SVI blend and sigma2 just under the 1e-2 floor on both sides of it = 100."""
    rng = np.random.default_rng(D * 10 + it)
    s, m = _rigid_from_points(rng, D, 300, svi, step, it, nn_init, sigma2_target=4e-3)
    ref = mstep_reference(s)
    P = _Params(D=D, svi=int(svi), update_R=1, nn_init=int(nn_init), nn_init_weight=0.8,
                sigma2_variance_decress=1.02, sigma2_variance_end=10.0)
    P.set("moments", m)
    if nn_init:
        Pn, a, bb = s["inlier_P"][:, 0], np.pad(s["inlier_A"], ((0, 0), (0, 3 - D))), np.pad(s["inlier_B"], ((0, 0), (0, 3 - D)))
        P.p.inl_SP = float(Pn.sum())
        for d in range(3):
            P.p.inl_Sa[d], P.p.inl_Sb[d] = float(Pn @ a[:, d]), float(Pn @ bb[:, d])
        for q, v in enumerate(((a * Pn[:, None]).T @ bb).reshape(-1)):
            P.p.inl_Mab[q] = float(v)
    else:
        P.p.inl_SP = 1.0
    sc = P.sc
    sc.Sp, sc.Sp_sigma2, sc.sigma2, sc.step = ref["Sp"], ref["Sp_sigma2"], s["sigma2"], step
    sc.sigma2_related, sc.sigma2_variance = ref["sigma2_related"], s["sigma2_variance"]
    for q in range(9):
        sc.R[q] = s["R"][q // 3, q % 3] if (q // 3 < D and q % 3 < D) else float(q in (0, 4, 8))
    for d in range(D):
        sc.t[d] = s["t"][d]
    out = P.call("spb_rigid_solve", it)
    b = _Bars(f"rigid solve D {D} svi {svi} step {step} nn_init {nn_init} it {it}")
    b("R", np.array(out.R[:]).reshape(3, 3)[:D, :D], ref["R"], 1e-12)
    b("t", np.array(out.t[:D]), ref["t"], 1e-12)
    b("sigma2", out.sigma2, ref["sigma2"], 1e-13)
    b("sigma2_variance", out.sigma2_variance, ref["sigma2_variance"], 1e-15)
    b.done()
    assert ref["sigma2"] == (1e-2 if it < 100 else pytest.approx(4e-3, rel=1e-9))


@pytest.mark.parametrize("svi", [False, True])
def test_update_gamma_alpha_digamma_sweep(svi):
    from scipy.special import psi

    NA = 4096
    rng = np.random.default_rng(1)
    # digamma arguments kappa + K_NA_spatial from 1e-3 to 1e7 (kappa alone, then with K_NA_spatial on top)
    kap = np.geomspace(1e-3, 1e7, NA).astype(np.float32)
    kns = np.where(np.arange(NA) % 2 == 0, 0.0, rng.uniform(0, 50, NA)).astype(np.float32)
    prev = rng.uniform(0.1, 2.0, NA).astype(np.float32)
    step = 0.3 if svi else 1.0
    b = _Bars(f"gamma / alpha svi {svi}")
    # Sp_spatial and the column count chosen for both gamma clamps and the open range in between
    for Sp_sp_new, nbb, nbt in ((50.0, 1000, 0), (900.0, 1000, 3000), (1e-3, 100000, 0), (999.5, 1000, 0), (2e5, 1000, 0)):
        P = _Params(NA=NA, D=2, svi=int(svi), gamma_a=1.0, gamma_b=1.0, NBb=nbb, NB_total=nbt)
        P.rows("kappa", kap)
        P.rows("K_NA_spatial", kns)
        P.rows("alpha", prev)
        sc = P.sc
        sc.step, sc.Sp_spatial, sc.Sp, sc.Sp_sigma2 = step, 400.0, 410.0, 380.0
        sc.sums[0], sc.sums[1], sc.sums[2], sc.sums[3] = Sp_sp_new, 0.8 * Sp_sp_new + 1, 1.1 * Sp_sp_new, 3.7
        out = P.call("spb_update_gamma_alpha")
        bl = (lambda new, old: step * new + (1 - step) * old) if svi else (lambda new, old: new)
        Sp_sp = bl(Sp_sp_new, 400.0)
        n = nbt if nbt > 0 else nbb
        g = float(np.clip(np.exp(psi(1.0 + Sp_sp) - psi(2.0 + n)), 0.01, 0.99))
        b(f"gamma Sp {Sp_sp_new:g} n {n}", out.gamma, g, 1e-14)
        b("Sp_spatial", out.Sp_spatial, Sp_sp, 1e-15)
        b("Sp", out.Sp, bl(1.1 * Sp_sp_new, 410.0), 1e-15)
        b("sigma2_related", out.sigma2_related, 3.7 / (2 * bl(0.8 * Sp_sp_new + 1, 380.0)), 1e-15)
        k64 = kap.astype(np.float64)
        a = np.exp(psi(k64 + kns) - psi(k64 * NA + Sp_sp))
        a = bl(a, prev.astype(np.float64))
        # fp64 digamma (series above 10, recurrence below), one rounding to fp32
        b("alpha", P.get("alpha", NA), a, 2 * EPS32)
    b.done()


def test_row_update_mm_lm_in_ulps():
    NA = 3000
    rng = np.random.default_rng(4)
    x = rng.uniform(-2, 2, size=(NA, 3)).astype(np.float32)
    v = (0.05 * rng.normal(size=(NA, 3))).astype(np.float32)
    alpha = np.geomspace(1e-30, 3.0, NA).astype(np.float32)
    rng.shuffle(alpha)
    s2 = 2.3e-3
    # SigmaDiag / sigma2 up to 300: exp(-300) underflows fp32, lm stays finite
    sd = (rng.uniform(0, 300, NA) * s2).astype(np.float32)
    R = _kabsch(rng.normal(size=(3, 3)))
    t = rng.normal(size=3)
    P = _Params(NA=NA, D=3)
    P.rows("xa", x, n3=True)
    P.rows("VnA", v, n3=True)
    P.rows("alpha", alpha)
    P.rows("SigmaDiag", sd)
    for name in ("RnA", "XAHat"):
        P.rows(name, np.zeros((NA, 3)), n3=True)
    for name in ("mm", "lm"):
        P.rows(name, np.zeros(NA))
    P.sc.sigma2 = s2
    for q in range(9):
        P.sc.R[q] = R[q // 3, q % 3]
    for d in range(3):
        P.sc.t[d] = t[d]
    P.call("spb_row_update")
    a64, sd64 = alpha.astype(np.float64), sd.astype(np.float64)
    mm = a64 * np.exp(-sd64 / s2)
    lm = np.log2(a64) - sd64 / s2 * np.log2(np.e)
    rna = x.astype(np.float64) @ R.T + t
    got_lm, got_mm = P.get("lm", NA), P.get("mm", NA)
    ulp_lm = np.abs(got_lm - lm) / np.spacing(np.abs(lm).astype(np.float32)).astype(np.float64)
    print(f"\n[row update] lm {ulp_lm.max():.2f} ulp, {int((got_mm == 0).sum())} mm underflow to 0")
    assert ulp_lm.max() <= 0.5 + 1e-3  # fp64 arithmetic, one rounding: lm is the correctly rounded fp32 value
    assert (got_mm == 0).any() and np.isfinite(got_lm).all()
    ok = mm > np.finfo(np.float32).tiny
    ulp_mm = np.abs(got_mm[ok] - mm[ok]) / np.spacing(mm[ok].astype(np.float32)).astype(np.float64)
    print(f"  mm {ulp_mm.max():.2f} ulp")
    assert ulp_mm.max() <= 1.0
    assert np.abs(P.get("RnA")[:, :NA].T - rna).max() <= 0.5 * np.spacing(np.float32(np.abs(rna).max()))
    assert np.array_equal(P.get("XAHat")[:, :NA], (P.bufs["VnA"] + P.bufs["RnA"]).double().cpu().numpy()[:, :NA])


@pytest.mark.parametrize("NA", [1, 255, 256, 257, 151553, 160001])
def test_rigid_moments_match_float64_and_repeat_bitwise(NA):
    rng = np.random.default_rng(NA)
    k = rng.uniform(0, 1, NA).astype(np.float32)
    x = rng.uniform(-3, 3, size=(NA, 3)).astype(np.float32)
    v = (0.1 * rng.normal(size=(NA, 3))).astype(np.float32)
    px = (k[:, None] * rng.uniform(-3, 3, size=(NA, 3))).astype(np.float32)
    k2 = rng.uniform(0, 1, NA).astype(np.float32)
    sd = rng.uniform(0, 1e-2, NA).astype(np.float32)
    P = _Params(NA=NA, D=3)
    for name, a in (("xa", x), ("VnA", v), ("PXB", px)):
        P.rows(name, a, n3=True)
    for name, a in (("K_NA", k), ("K_NA_sigma2", k2), ("SigmaDiag", sd)):
        P.rows(name, a)
    P.set("moments", np.zeros(32))
    P.call("spb_rigid_moments")
    got = P.get("moments")[:29].copy()
    P.bufs["moments"].zero_()
    P.call("spb_rigid_moments")
    again = P.get("moments")[:29]
    assert np.array_equal(got, again)  # ordered grid reduction: the same bits every time
    K, X, V, PX = (a.astype(np.float64) for a in (k, x, v, px))
    want = np.concatenate([K @ X, K @ V, PX.sum(0), ((X * K[:, None]).T @ V).reshape(-1), (X.T @ PX).reshape(-1),
                           [k2.astype(np.float64) @ sd.astype(np.float64), K.sum()]])
    mag = np.concatenate([np.abs(K) @ np.abs(X), np.abs(K) @ np.abs(V), np.abs(PX).sum(0),
                          ((np.abs(X) * K[:, None]).T @ np.abs(V)).reshape(-1), (np.abs(X).T @ np.abs(PX)).reshape(-1),
                          [k2.astype(np.float64) @ sd.astype(np.float64), K.sum()]])
    # fp64 products of fp32 inputs, fp64 sums: error bound ~ n eps(float64) of the sum of magnitudes (log-depth tree)
    err = (np.abs(got - want) / mag).max()
    print(f"\n[rigid moments NA {NA}] max error / sum of magnitudes {err:.2e}")
    assert err <= 1e-14
