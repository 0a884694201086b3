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
