"""Shared helpers of the GPU parity tests: build the CUDA ``Morpho_pairwise`` from a golden fixture, overwrite its device
state with the reference's E-step inputs, and evaluate the float64 oracle on the same inputs."""

import ast
import ctypes as C

import numpy as np


def adata_from_golden(g):
    import pandas as pd

    from spateo_release_b200.anndata_lite import AnnDataLite

    G = g["exp_moving"].shape[1]
    var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
    mov = AnnDataLite(np.asarray(g["exp_moving"], dtype=np.float32), var=var.copy(), obsm={"spatial": g["raw_coords_moving"]})
    fix = AnnDataLite(np.asarray(g["exp_fixed"], dtype=np.float32), var=var.copy(), obsm={"spatial": g["raw_coords_fixed"]})
    return mov, fix


def cfg_of(g):
    return ast.literal_eval(str(g["cfg"]))


def model_from_golden(g, **over):
    import spateo_release_b200 as st

    cfg = cfg_of(g)
    mov, fix = adata_from_golden(g)
    kw = dict(SVI_mode=cfg["svi"], max_iter=cfg["max_iter"], K=cfg["K"], verbose=False, device="0", vecfld_key_added="vf")
    kw.update(cfg["kw"])
    if "guide_fixed" in g:
        kw["guidance_pair"] = [g["guide_fixed"], g["guide_moving"]]
    kw.update(over)
    np.random.seed(0)
    return st.align.Morpho_pairwise(sampleA=mov, sampleB=fix, **kw)


def relF(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300)


def relmax(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def poke_estep_state(m, XAHat, alpha, SigmaDiag, sigma2, gamma, sigma2_variance, coordsB=None, samples_s=None):
    """Overwrite the device state with given E-step inputs (arrays in the CALLER's row order)."""
    import torch

    s, NA, D = m._state, m.NA, m.D
    dev = m._dev
    XAHat = m._sorted(np.asarray(XAHat, dtype=np.float32))  # device rows are in processing order
    alpha = m._sorted(np.asarray(alpha, dtype=np.float64))
    SigmaDiag = m._sorted(np.asarray(SigmaDiag, dtype=np.float64))
    s["XAHat"][:D, :NA] = torch.from_numpy(np.ascontiguousarray(XAHat.T)).to(dev)
    s["alpha"][:NA] = torch.from_numpy(alpha.astype(np.float32)).to(dev)
    s["SigmaDiag"][:NA] = torch.from_numpy(SigmaDiag.astype(np.float32)).to(dev)
    mmv = alpha * np.exp(-SigmaDiag / sigma2)
    s["mm"][:NA] = torch.from_numpy(mmv.astype(np.float32)).to(dev)
    s["lm"][:NA] = torch.from_numpy(np.log2(mmv).astype(np.float32)).to(dev)
    if coordsB is not None:
        s["xb4"][:, :D] = torch.from_numpy(np.asarray(coordsB, dtype=np.float32)).to(dev)
    sc = m._read_scalars()
    sc.sigma2, sc.gamma, sc.sigma2_variance = float(sigma2), float(gamma), float(sigma2_variance)
    s["sc"].copy_(torch.from_numpy(np.frombuffer(bytes(sc), dtype=np.uint8).copy()))
    if samples_s is not None:
        m._params.samples_s = float(samples_s)


def poke_golden_estep(m, g, it, sfx=""):
    """Device state <- the reference's E-step inputs at iteration ``it`` of a golden fixture."""
    poke_estep_state(
        m, g[f"it{it}_in_XAHat{sfx}"], g[f"it{it}_in_alpha{sfx}"], g[f"it{it}_in_SigmaDiag{sfx}"],
        float(g[f"it{it}_in_sigma2{sfx}"]), float(g[f"it{it}_in_gamma{sfx}"]), float(g[f"it{it}_in_sigma2_variance{sfx}"]),
        coordsB=g["pre_coordsB" + sfx], samples_s=float(g["pre_samples_s" + sfx]),
    )


def run_estep(m, it, cull=None):
    """One E-step on the current device state (through the C ABI); returns the dense posterior in the caller's row order."""
    import torch

    from spateo_release_b200._capi import check, ptr

    if cull is not None:
        m._params.cull = int(bool(cull))
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    m._estep_only(it, st)
    Pd = torch.empty((m.NA, m._NBb), dtype=torch.float32, device=m._dev)
    check(m._lib.spb_materialize_P(C.byref(m._params), it, ptr(Pd), m._NBb, st), "materialize")
    torch.cuda.synchronize()
    return m._unsorted(Pd.cpu().numpy())


def mstep_reference(s, dtype=np.float64):
    """float64 M-step of one EM iteration from the E-step's sufficient statistics (no dense posterior).

    Restates ``MorphoPairOracle._update_gamma / _update_alpha / _update_nonrigid / _update_rigid / _update_sigma2`` one
    statement at a time, with every product through the dense P rewritten through ``PXB = P @ YB`` and ``KNB_YB = K_NB @
    YB``: ``P @ YB`` is PXB and ``XA_hat^T P XB_hat = XA_hat^T PXB - (XA_hat^T K_NA) mu_XB^T``. The pseudo-inverse keeps
    scipy's cutoff rule ``rtol = K * pinv_eps`` in fp64 arithmetic (pinv_eps: eps(float32) for the reference's fp32
    SigmaInv, eps(float64) for the geodesic kernel or an fp64 run).

    ``s`` holds
      E-step outputs   K_NA, K_NA_spatial, K_NA_sigma2 [NA]; PXB [NA, D]; KNB_YB [D]; Sp_new, Sp_spatial_new,
                       Sp_sigma2_new (sums of this E-step), S2 (sum of P_sigma2 * squared distance)
      previous state   alpha [NA], SigmaInv [K, K], PXB_term [NA, D], Sp, Sp_spatial, Sp_sigma2, R [D, D], t [D], RnA,
                       VnA [NA, D], SigmaDiag [NA], sigma2, sigma2_variance; V_AI, R_AI [NI, D] with guidance
      constants        it, svi, step, nonrigid, U [NA, K], Gamma [K, K], coordsA [NA, D], kappa [NA], gamma_a, gamma_b,
                       n_gamma (columns of the whole iteration), lambdaVF, pinv_eps, update_R, nn_init (+ inlier_A,
                       inlier_B [n, D], inlier_P [n], nn_init_weight), guidance (None or dict X_AI, X_BI, U_I, weight,
                       effect), sigma2_variance_decress, sigma2_variance_end
    Returns every M-step output. ``dtype=np.float32`` evaluates the arrays in fp32 like the reference's own fp32 run (its
    deviation from the fp64 result is the scale the GPU tests print next to theirs)."""
    from scipy.linalg import pinv
    from scipy.special import psi

    f = lambda v: np.asarray(v, dtype=dtype)
    D, it, step, svi = int(s["D"]), int(s["it"]), float(s["step"]), bool(s["svi"])
    K_NA, K_NA_spatial, K_NA_sigma2 = f(s["K_NA"]), f(s["K_NA_spatial"]), f(s["K_NA_sigma2"])
    PXB_rows, coordsA, U = f(s["PXB"]), f(s["coordsA"]), f(s["U"])
    NA, K = coordsA.shape[0], U.shape[1]
    sigma2 = float(s["sigma2"])
    o = {}
    # running sums of the E-step (_update_assignment_P, morpho_class.py:1178-1200)
    if svi:
        o["Sp_spatial"] = step * s["Sp_spatial_new"] + (1 - step) * s["Sp_spatial"]
        o["Sp"] = step * s["Sp_new"] + (1 - step) * s["Sp"]
        o["Sp_sigma2"] = step * s["Sp_sigma2_new"] + (1 - step) * s["Sp_sigma2"]
    else:
        o["Sp_spatial"], o["Sp"], o["Sp_sigma2"] = s["Sp_spatial_new"], s["Sp_new"], s["Sp_sigma2_new"]
    o["Sp_spatial"], o["Sp"], o["Sp_sigma2"] = float(o["Sp_spatial"]), float(o["Sp"]), float(o["Sp_sigma2"])
    Sp = o["Sp"]
    o["sigma2_related"] = float(s["S2"]) / (D * o["Sp_sigma2"])
    # _update_gamma
    g = np.exp(psi(s["gamma_a"] + o["Sp_spatial"]) - psi(s["gamma_a"] + s["gamma_b"] + s["n_gamma"]))
    o["gamma"] = float(np.maximum(np.minimum(g, 0.99), 0.01))
    # _update_alpha
    kappa = f(s["kappa"])
    new = np.exp(psi(kappa + K_NA_spatial) - psi(kappa * NA + o["Sp_spatial"]))
    o["alpha"] = step * new + (1 - step) * f(s["alpha"]) if svi else new
    # _update_nonrigid
    gd = s.get("guidance")
    g_nonrigid = gd is not None and gd["effect"] in ("nonrigid", "both")
    g_rigid = gd is not None and gd["effect"] in ("rigid", "both")
    V_AI = None if gd is None else f(s["V_AI"])
    RnA_prev = f(s["RnA"])
    if s["nonrigid"]:
        SigmaInv = sigma2 * s["lambdaVF"] * f(s["Gamma"]) + U.T @ (U * K_NA[:, None])
        PXB_term = PXB_rows - RnA_prev * K_NA[:, None]
        if svi:
            SigmaInv = step * SigmaInv + (1 - step) * f(s["SigmaInv"])
            PXB_term = step * PXB_term + (1 - step) * f(s["PXB_term"])
        UPXB = U.T @ PXB_term
        if g_nonrigid:
            cg = sigma2 * gd["weight"] * Sp / gd["U_I"].shape[0]
            SigmaInv = SigmaInv + cg * (f(gd["U_I"]).T @ f(gd["U_I"]))
            UPXB = UPXB + cg * (f(gd["U_I"]).T @ (f(gd["X_BI"]) - f(s["R_AI"])))
        Sigma = pinv(SigmaInv, atol=0.0, rtol=K * s["pinv_eps"])
        o["SigmaInv"], o["PXB_term"], o["UPXB"], o["Sigma"] = SigmaInv, PXB_term, UPXB, Sigma
        o["Coff"] = Sigma @ UPXB
        VnA = U @ o["Coff"]
        if g_nonrigid:
            V_AI = f(gd["U_I"]) @ o["Coff"]
        SigmaDiag = sigma2 * np.einsum("ij,ji->i", U, Sigma @ U.T)
    else:
        VnA, SigmaDiag = f(s["VnA"]), f(s["SigmaDiag"])
    o["VnA"], o["SigmaDiag"], o["V_AI"] = VnA, SigmaDiag, V_AI
    # _update_rigid (P @ YB = PXB, K_NB @ YB = KNB_YB)
    PXA = K_NA @ coordsA
    PVA = K_NA @ VnA
    PXB = f(s["KNB_YB"]).copy()
    mu_X_deno = mu_Vn_deno = Sp
    if g_rigid:
        cg = sigma2 * gd["weight"] * Sp / gd["X_BI"].shape[0]
        PXB += cg * f(gd["X_BI"]).mean()  # the mu_* arrays alias the P* arrays (reference quirk)
        PXA += cg * f(gd["X_AI"]).mean()
        PVA += cg * V_AI.mean()
        mu_X_deno += cg * gd["X_BI"].shape[0]
        mu_Vn_deno += cg * gd["X_BI"].shape[0]
    if s["nn_init"]:
        iP, iA, iB = f(s["inlier_P"]).reshape(-1), f(s["inlier_A"]), f(s["inlier_B"])
        c = sigma2 * s["nn_init_weight"] * Sp / iP.sum()
        PXB += c * (iP @ iB)
        PXA += c * (iP @ iA)
        mu_X_deno += c * iP.sum()
    mu_XB, mu_XA, mu_Vn = PXB / mu_X_deno, PXA / mu_X_deno, PVA / mu_Vn_deno
    XA_hat = coordsA - mu_XA
    XAP_XBhat = XA_hat.T @ PXB_rows - np.outer(XA_hat.T @ K_NA, mu_XB)
    A = -((XA_hat.T @ ((VnA - mu_Vn) * K_NA[:, None])) - XAP_XBhat).T
    if g_rigid:
        A -= cg * ((f(gd["X_AI"]) - mu_XA).T @ ((V_AI - mu_Vn) - (f(gd["X_BI"]) - mu_XB))).T
    if s["nn_init"]:
        A -= c * (((iA - mu_XA) * iP[:, None]).T @ -(iB - mu_XB)).T
    o["A"] = A
    svdU, _, svdV = np.linalg.svd(A)
    Cm = np.eye(D)
    Cm[-1, -1] = np.linalg.det(svdU @ svdV)
    R = f(s["R"]).copy()
    if s["update_R"]:
        Rn = svdU @ Cm @ svdV
        R = step * Rn + (1 - step) * R if (svi and step < 1) else Rn
    t_num = PXB - PVA - PXA @ R.T
    t_den = Sp
    if g_rigid:
        t_num += cg * np.sum(f(gd["X_BI"]) - V_AI - f(gd["X_AI"]) @ R.T, axis=0)
        t_den += cg * gd["X_BI"].shape[0]
    if s["nn_init"]:
        t_num += c * (iP @ (iB - iA @ R.T))
        t_den += c * iP.sum()
    t = t_num / t_den
    if svi and step < 1:
        t = step * t + (1 - step) * f(s["t"])
    o["R"], o["t"] = R, t
    o["RnA"] = coordsA @ R.T + t
    if gd is not None:
        o["R_AI"] = f(s["R_AI"]) @ R.T + t
    o["XAHat"] = VnA + o["RnA"]
    # _update_sigma2
    s2 = max(o["sigma2_related"] + float(K_NA_sigma2 @ SigmaDiag) / o["Sp_sigma2"], 1e-3)
    o["sigma2_variance"] = min(s["sigma2_variance"] * s["sigma2_variance_decress"], s["sigma2_variance_end"])
    if it < 100:
        s2 = max(s2, 1e-2)
    o["sigma2"] = s2
    # the next E-step's model multiplier alpha exp(-SigmaDiag / sigma2) and its log2 (morpho_class.py:1087)
    o["mm"] = o["alpha"] * np.exp(-SigmaDiag / s2)
    o["lm"] = np.log2(o["alpha"]) - SigmaDiag / s2 * np.log2(np.e)
    return o


def oracle_mstep_inputs(o, it):
    """The ``mstep_reference`` inputs of iteration ``it`` of a float64 ``MorphoPairOracle`` whose iterations before ``it``
    have run: runs the oracle's own E-step (``_update_batch`` + ``_update_assignment_P``) and collects its outputs with
    the state the M-step starts from."""
    import copy

    if o.SVI_mode:
        o._update_batch(it)
    prev = {k: copy.deepcopy(getattr(o, k)) for k in ("Sp", "Sp_spatial", "Sp_sigma2", "alpha", "R", "t", "RnA", "VnA",
                                                      "SigmaDiag", "sigma2", "sigma2_variance")}
    for k in ("SigmaInv", "PXB_term", "V_AI", "R_AI"):
        prev[k] = copy.deepcopy(getattr(o, k, None))
    o._update_assignment_P()
    YB = o.coordsB[o.batch_idx, :] if o.SVI_mode else o.coordsB
    s = dict(prev)
    s.update(
        D=o.D, it=it, svi=o.SVI_mode, step=float(o.step_size) if o.SVI_mode else 1.0,
        nonrigid=(it > o.nonrigid_start_iter) or o.nonrigid_flag,
        K_NA=o.K_NA, K_NA_spatial=o.K_NA_spatial, K_NA_sigma2=o.K_NA_sigma2, PXB=o.P @ YB, KNB_YB=o.K_NB @ YB,
        Sp_new=float(o.P.sum()), Sp_spatial_new=float(o.K_NA_spatial.sum()), Sp_sigma2_new=float(o.K_NA_sigma2.sum()),
        U=o.U, Gamma=o.GammaSparse, coordsA=o.coordsA, kappa=o.kappa, gamma_a=float(o.gamma_a), gamma_b=float(o.gamma_b),
        n_gamma=o.batch_size if o.SVI_mode else o.NB, lambdaVF=o.lambdaVF, pinv_eps=np.finfo(o.dt).eps,
        update_R=o.update_R, nn_init=o.nn_init, nn_init_weight=o.nn_init_weight,
        sigma2_variance_decress=float(o.sigma2_variance_decress), sigma2_variance_end=float(o.sigma2_variance_end),
    )
    # the oracle keeps sigma2_related = S2 / (D Sp_sigma2) (running Sp_sigma2), not S2 itself
    s["S2"] = float(o.sigma2_related) * o.D * float(o.Sp_sigma2)
    if o.nn_init:
        s.update(inlier_A=o.inlier_A, inlier_B=o.inlier_B, inlier_P=o.inlier_P)
    if o.guidance:
        s["guidance"] = dict(X_AI=o.X_AI, X_BI=o.X_BI, U_I=o.U_I, weight=o.guidance_weight, effect=o.guidance_effect)
    return s


def device_rows(m, name):
    return m._unsorted(m._state[name][: m.NA].cpu().numpy())


def device_pxb(m):
    return m._unsorted(m._state["PXB"][: m.D, : m.NA].T.contiguous().cpu().numpy())


# ---------------------------------------------------------------------------------------------------------------------
# The sparse top-k posterior and the posterior argmax
# ---------------------------------------------------------------------------------------------------------------------
def replay_weights(m, it, q=None):
    """The device's own pair weights w = q g, [N_A, NBb] float32 in DEVICE row order, for the E-step that has just run
    (``q``: the parameters of one streamed column chunk; default the solver's). ``spb_materialize_P`` writes
    ex2(c_q d + lm) * g * c_j; with every c_j replaced by 1.0 the last product is exact and it writes w itself."""
    import torch

    from spateo_release_b200._capi import SpbEmParams, check, ptr

    p = SpbEmParams.from_buffer_copy(m._params if q is None else q)
    cc = m._state["colconst"].clone()
    cc[:, 10] = 1.0
    p.colconst = cc.data_ptr()
    W = torch.empty((m.NA, p.NBb), dtype=torch.float32, device=m._dev)
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    check(m._lib.spb_materialize_P(C.byref(p), it, ptr(W), p.NBb, st), "spb_materialize_P")
    torch.cuda.synchronize()
    return W.cpu().numpy()


def topk_replay(W, k, c, Y=None, block=1024):
    """What the sparse top-k kernels compute from the weights ``W`` [N_A, NB] (float32), the column factors ``c`` [NB]
    (float32) and the fixed coordinates ``Y`` [NB, D]:
      tau        per column the k-th largest w (k clamped to N_A), 0 when the column has fewer non-zero weights (float32)
      n_above    number of w > tau; n_ties: number of w == tau (tau > 0), else 0
      K_NB       c_j * sum_{w >= tau} w in fp64 (every copy of tau counts)
      K_NB_k     c_j * (sum of exactly k entries: every w > tau, then ties at tau) in fp64, the reference's column sum
      K_NA, PXB  the row sums sweep 2 forms, sum_j c_j w_ij [w_ij >= tau_j] and the same weighted by y_j (fp64)."""
    W = np.asarray(W, dtype=np.float32)
    NA, NB = W.shape
    kk = min(int(k), NA)
    c64 = np.asarray(c, np.float64)
    out = dict(tau=np.zeros(NB, np.float32), n_above=np.zeros(NB, np.int64), n_ties=np.zeros(NB, np.int64),
               K_NB=np.zeros(NB), K_NB_k=np.zeros(NB), K_NA=np.zeros(NA))
    if Y is not None:
        out["PXB"] = np.zeros((NA, np.shape(Y)[1]))
    for j0 in range(0, NB, block):  # column blocks bound the fp64 temporaries
        j1 = min(NB, j0 + block)
        Wb = W[:, j0:j1]
        tau = -np.partition(-Wb, kk - 1, axis=0)[kk - 1]
        tau = np.where(tau > 0, tau, np.float32(0)).astype(np.float32)
        kept = np.where(Wb >= tau[None, :], Wb.astype(np.float64), 0.0)
        above = Wb > tau[None, :]
        n_above = above.sum(0)
        n_ties = np.where(tau > 0, (Wb == tau[None, :]).sum(0), 0)
        mass_above = np.where(above, kept, 0.0).sum(0)
        out["tau"][j0:j1], out["n_above"][j0:j1], out["n_ties"][j0:j1] = tau, n_above, n_ties
        out["K_NB"][j0:j1] = c64[j0:j1] * kept.sum(0)
        out["K_NB_k"][j0:j1] = c64[j0:j1] * (mass_above + np.minimum(n_ties, kk - n_above) * tau.astype(np.float64))
        out["K_NA"] += kept @ c64[j0:j1]
        if Y is not None:
            out["PXB"] += kept @ (c64[j0:j1, None] * np.asarray(Y, np.float64)[j0:j1])
    return out


def argmax_keys(v, idx):
    """64-bit argmax keys of ``row_argmax`` / ``col_argmax``: the float bits of the value above the complemented index, so
    the unsigned maximum is the largest value and, among equal values, the lowest index."""
    v = np.ascontiguousarray(v, dtype=np.float32)
    return (v.view(np.uint32).astype(np.uint64) << np.uint64(32)) | (np.uint64(0xFFFFFFFF) - np.asarray(idx).astype(np.uint64))


def argmax_replay(W, c, tau, colmap=None, block=64):
    """Row and column argmax keys of the posterior P = w c (fp32 products) from the weights ``W`` [N_A, NB] (device row
    order): a row's key skips entries below their column's ``tau`` (sparse mode; tau = 0 keeps all) and carries the column
    index ``colmap[j]`` (-1: column skipped; default j); a column's key carries the device row index."""
    W = np.asarray(W, dtype=np.float32)
    NA, NB = W.shape
    c = np.asarray(c, dtype=np.float32)
    colmap = np.arange(NB) if colmap is None else np.asarray(colmap)
    rowkey = np.zeros(NA, dtype=np.uint64)
    colkey = np.zeros(NB, dtype=np.uint64)
    rows = np.arange(NA)
    for j0 in range(0, NB, block):
        j1 = min(NB, j0 + block)
        P = W[:, j0:j1] * c[None, j0:j1]
        ck = argmax_keys(P, rows[:, None]).max(0)
        colkey[j0:j1] = ck
        live = colmap[j0:j1] >= 0
        if live.any():
            Ps = np.where(W[:, j0:j1] >= tau[None, j0:j1], W[:, j0:j1], np.float32(0)) * c[None, j0:j1]
            rk = argmax_keys(Ps[:, live], colmap[j0:j1][live][None, :]).max(1)
            rowkey = np.maximum(rowkey, rk)
    return rowkey, colkey


def sparse_posterior_reference(Dim, XAHat, YB, G, sigma2, model_mul, gamma, samples_s, sigma2_variance, ks, chunk=1000,
                               dtype=np.float64):
    """``get_P_core`` followed by ``dense_to_sparse_topk`` on a given cost matrix ``G`` [N_A, NB] (the product of the
    expression terms, passed as a "prob" term), evaluated in column chunks: every normalisation and the top-k are per
    column. For each k in ``ks``: the COO entries ``rows`` / ``vals`` [NB, k] (descending within a column), the row sums
    K_NA, the column sums K_NB, P @ YB, and each column's k-th and (k+1)-th largest values (``kth``, ``kth1``; 0 past N_A).
    ``dtype=np.float32`` restates it in fp32 (the scale of what an fp32 evaluation of the reference computes)."""
    from oracle.morpho_oracle import get_P_core

    f = lambda a: np.asarray(a, dtype=dtype)
    XAHat, YB, G, model_mul = f(XAHat), f(YB), np.asarray(G), f(model_mul)
    NA, NB = G.shape
    ks = [int(k) for k in ks]
    out = {k: dict(rows=np.zeros((NB, min(k, NA)), np.int64), vals=np.zeros((NB, min(k, NA)), dtype), K_NA=np.zeros(NA, dtype),
                   K_NB=np.zeros(NB, dtype), PXB=np.zeros((NA, YB.shape[1]), dtype), kth=np.zeros(NB, dtype),
                   kth1=np.zeros(NB, dtype)) for k in ks}
    top = min(max(ks) + 1, NA)
    for j0 in range(0, NB, chunk):
        j1 = min(NB, j0 + chunk)
        spatial = ((XAHat[:, None, :] - YB[None, j0:j1, :]) ** 2).sum(-1)
        P, _, _, _ = get_P_core(Dim=Dim, spatial_dist=spatial, exp_dist=[f(G[:, j0:j1])], sigma2=sigma2, model_mul=model_mul,
                                gamma=gamma, samples_s=samples_s, sigma2_variance=sigma2_variance, probability_type=["prob"])
        P = f(P)
        # descending with the lowest row first among equal values, like the reference's stable argsort of -P
        part = np.argpartition(-P, top - 1, axis=0)[:top] if top < NA else np.broadcast_to(np.arange(NA)[:, None], P.shape)
        pv = np.take_along_axis(P, part, axis=0)
        order = np.lexsort((part, -pv), axis=0)
        idx, val = np.take_along_axis(part, order, axis=0), np.take_along_axis(pv, order, axis=0)
        for k in ks:
            kk = min(k, NA)
            o = out[k]
            o["rows"][j0:j1], o["vals"][j0:j1] = idx[:kk].T, val[:kk].T
            o["kth"][j0:j1] = val[kk - 1]
            if kk < NA:
                o["kth1"][j0:j1] = val[kk]
            Ps = np.zeros_like(P)
            np.put_along_axis(Ps, idx[:kk], val[:kk], axis=0)
            o["K_NA"] += Ps.sum(1)
            o["K_NB"][j0:j1] = Ps.sum(0)
            o["PXB"] += Ps @ YB[j0:j1]
    return out
