"""SparseVFC on the GPU — the solver behind ``st.tdr.morphofield_sparsevfc`` / ``st.tdr.morphofield``.

The reference delegates to third-party ``dynamo.vectorfield.scVectorField.SparseVFC`` (``dynamo-release>=1.4.1``,
requirements.txt:7; call sites spateo/tdr/morphometrics/morphofield/sparsevfc.py:167,189-198), which is not vendored:
**parity unpinned** — this module restates the published algorithm (Ma et al., Pattern Recognition 2013, as implemented
by dynamo; SURVEY.md Appendix E) and is checked against ``oracle.morpho_oracle.sparse_vfc`` only.

Device work per EM iteration: ``spb_vfc_estep`` (V = U C, inlier posterior P, energy sums — one pass over U^T) and
``spb_weighted_gram`` (U^T P U and U^T P Y, fp64 accumulation). The M x M normal equations are solved on the device as the
minimum-norm least-squares solution (symmetric eigen-decomposition with lstsq's eps*M singular-value cutoff — what the
reference's ``lstsq_method="scipy"`` computes; both ``lstsq_method`` values map to it); sigma^2 follows from the accumulated
blocks (sum P|Y - UC|^2 = sum P|Y|^2 - 2 tr(C^T U^T P Y) + tr(C^T U^T P U C)), so U is streamed twice per iteration and the
host synchronises once per iteration (the convergence test of the reference needs the energy on the host).
"""

from __future__ import annotations

from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .. import _capi
from .._capi import check, ptr
from ..alignment.morpho_class import _round_up, resolve_device
from ..alignment.transform import field_eval


def bandwidth_selector(X: np.ndarray) -> float:
    """dynamo's kernel bandwidth: sqrt(2) * mean kNN distance (k = max(2, 0.2 n)) / 1.5."""
    from sklearn.neighbors import NearestNeighbors

    n = X.shape[0]
    k = min(max(2, int(0.2 * n)), n)
    nbrs = NearestNeighbors(n_neighbors=k, algorithm="kd_tree").fit(X)
    dist, _ = nbrs.kneighbors(X)
    return float(np.sqrt(2) * np.mean(dist[:, 1:]) / 1.5)


def sample_by_velocity(V: np.ndarray, n: int, seed: int = 19491001) -> np.ndarray:
    """Control points drawn without replacement with probability proportional to |V| (dynamo's default sampler)."""
    rng = np.random.RandomState(seed)
    mag = np.linalg.norm(V, axis=1)
    p = mag / mag.sum() if mag.sum() > 0 else None
    nz = int((mag > 0).sum()) if p is not None else len(V)
    if p is not None and nz < n:  # not enough non-zero weights for a draw without replacement
        p = None
    return rng.choice(np.arange(len(V)), size=n, p=p, replace=False)


def SparseVFC(
    X: np.ndarray,
    Y: np.ndarray,
    Grid: Optional[np.ndarray] = None,
    M: int = 100,
    a: float = 5,
    beta: Optional[float] = None,
    ecr: float = 1e-5,
    gamma: float = 0.9,
    lambda_: float = 3,
    minP: float = 1e-5,
    MaxIter: int = 500,
    theta: float = 0.75,
    div_cur_free_kernels: bool = False,
    velocity_based_sampling: bool = True,
    sigma: float = 0.8,
    eta: float = 0.5,
    seed: int = 0,
    lstsq_method: str = "drouin",
    verbose: int = 1,
    ctrl_idx: Optional[np.ndarray] = None,
    device=None,
    gram: str = "auto",
    timings: Optional[dict] = None,
) -> dict:
    """Sparse vector-field consensus (same signature as dynamo's ``SparseVFC``; ``ctrl_idx`` / ``device`` / ``gram`` /
    ``timings`` are extras).

    ``gram``: how the normal-equation blocks U^T P U and U^T P Y are contracted — ``"fp64"`` (= ``"auto"``, the default) =
    SIMT kernels with fp64 products, the reference-accurate path; ``"tensor"`` (opt-in) = wgmma kernel (3xTF32 on the
    row-centred kernel matrix, fp64 fold). The tensor path's products carry fp32-level relative noise (~1e-7), which is the
    relative size of SparseVFC's own regulariser lambda sigma2 K against U^T P U at the default lambda: it therefore solves with
    a ridge just above that noise floor and returns a slightly SMOOTHER fit than the reference solution (7x faster at
    1M x 500; deviation measured in tests/test_gpu_vfc.py and reported by bench.py). ``timings``: dict that receives CUDA-event timings of the
    EM loop (bench.py).

    Returns the dictionary documented at sparsevfc.py:139-157: X, valid_ind, X_ctrl, ctrl_idx, Y, beta, V, C, P, VFCIndex,
    sigma2, grid, grid_V, iteration, tecr_traj, E_traj.
    """
    if div_cur_free_kernels:
        raise NotImplementedError("divergence/curl-free kernels are not implemented")
    lib = _capi.load_library()
    dev = resolve_device(device)
    X_full, Y_full = np.asarray(X, dtype=np.float64), np.asarray(Y, dtype=np.float64)
    valid_ind = np.where(np.isfinite(Y_full.sum(1)))[0]
    Xv, Yv = X_full[valid_ind], Y_full[valid_ind]
    N, D = Yv.shape
    if D > 3 or Xv.shape[1] != D:
        # learn a map R^dx -> R^dy with dy != dx or dy > 3 (kernel_interpolation): same EM, column blocks of three
        return _sparse_vfc_general(X_full, Y_full, valid_ind, Grid, M, a, beta, ecr, gamma, lambda_, minP, MaxIter, theta,
                                   velocity_based_sampling, seed, ctrl_idx, dev, lib)
    if ctrl_idx is None:
        tmp_X, uid = np.unique(Xv, axis=0, return_index=True)
        M = min(M, tmp_X.shape[0])
        if velocity_based_sampling:
            idx = sample_by_velocity(Yv[uid], M, seed)
        else:
            idx = np.random.RandomState(seed).permutation(tmp_X.shape[0])[:M]
        ctrl_idx = uid[idx]
    ctrl_idx = np.asarray(ctrl_idx)
    ctrl = Xv[ctrl_idx]
    M = ctrl.shape[0]
    if beta is None:
        h = bandwidth_selector(ctrl)
        beta = 1.0 / h**2
    d2c = ((ctrl[:, None, :] - ctrl[None, :, :]) ** 2).sum(-1)
    Kc = np.exp(-beta * d2c)

    with torch.cuda.device(dev):
        st = _capi.current_stream_ptr()
        ldn = _round_up(N, 1024)
        centre = Xv.mean(axis=0)  # centring keeps the fp32 coordinate rounding negligible
        x_soa = torch.zeros((3, ldn), dtype=torch.float32, device=dev)
        x_soa[:D, :N] = torch.from_numpy(np.ascontiguousarray((Xv - centre).T, dtype=np.float32)).to(dev)
        z = torch.zeros((M, 3), dtype=torch.float32, device=dev)
        z[:, :D] = torch.from_numpy((ctrl - centre).astype(np.float32)).to(dev)
        UT = torch.empty((M, ldn), dtype=torch.float32, device=dev)
        check(lib.spb_rbf_kernel_T(ptr(x_soa), N, ldn, ptr(z), M, float(beta), ptr(UT), st), "spb_rbf_kernel_T")
        Yd = torch.from_numpy(np.ascontiguousarray(Yv)).to(dev)
        P = torch.empty((ldn,), dtype=torch.float64, device=dev)
        V = torch.zeros((N, D), dtype=torch.float64, device=dev)
        Pf = torch.zeros((ldn,), dtype=torch.float32, device=dev)
        PY3 = torch.zeros((3, ldn), dtype=torch.float32, device=dev)
        sums = torch.zeros((5,), dtype=torch.float64, device=dev)
        A_d = torch.empty((M, M), dtype=torch.float64, device=dev)
        B_d = torch.empty((M, 3), dtype=torch.float64, device=dev)
        Cd = torch.zeros((M, 3), dtype=torch.float64, device=dev)
        use_tc = gram == "tensor"  # "auto" = the fp64 products: SparseVFC's regulariser lives at the fp32 noise level (see docstring)
        if gram not in ("auto", "tensor", "fp64"):
            raise ValueError("gram must be 'auto', 'tensor' or 'fp64'")
        if use_tc:
            import ctypes as C_

            A_hi, A_lo = torch.empty_like(UT), torch.empty_like(UT)
            u_mean = torch.empty((M,), dtype=torch.float32, device=dev)
            check(lib.spb_gram_center(ptr(UT), ldn, N, M, ptr(u_mean), ptr(A_hi), ptr(A_lo), st), "spb_gram_center")
            B_hi = torch.zeros((M + 4, ldn), dtype=torch.float32, device=dev)
            B_lo = torch.zeros((M + 4, ldn), dtype=torch.float32, device=dev)
            need = C_.c_int64(0)
            check(lib.spb_gram_tc_scratch_floats(M, 3, N, C_.byref(need)), "spb_gram_tc_scratch_floats")
            g_scratch = torch.empty((need.value,), dtype=torch.float32, device=dev)
            g_sums = torch.zeros((4,), dtype=torch.float64, device=dev)

        Kd = torch.from_numpy(Kc).to(dev)
        sigma2 = max(float((Yv**2).sum() / (N * D)), 1e-7)
        E, tecr, it = 1.0, 1.0, 0
        tecr_traj, E_traj = [], []
        Y2 = (Yd**2).sum(1)  # |Y_i|^2, reused for sum P |Y|^2
        reg_energy = 0.0     # tr(C^T K C) of the current coefficients
        rcond = np.finfo(np.float64).eps * M
        ev_pairs = [] if timings is not None else None
        n_fallback = 0
        while it < MaxIter and tecr > ecr and sigma2 > 1e-8:
            E_old = E
            if ev_pairs is not None:
                evs = [torch.cuda.Event(enable_timing=True) for _ in range(5)]
                evs[0].record()
            check(
                lib.spb_vfc_estep(ptr(UT), ldn, N, M, D, ptr(Cd), ptr(Yd), sigma2, gamma, float(a), float(minP),
                                  float(theta), ptr(P), ptr(V), ptr(Pf), ptr(PY3), ptr(sums), st),
                "spb_vfc_estep",
            )
            if ev_pairs is not None:
                evs[1].record()
            if use_tc:
                check(lib.spb_gram_prepare(ptr(UT), ldn, N, M, ptr(u_mean), ptr(Pf), ptr(PY3), ldn, 3, ptr(B_hi), ptr(B_lo),
                                           ptr(g_sums), st), "spb_gram_prepare")
                if ev_pairs is not None:
                    evs[4].record()
                check(lib.spb_gram_tc(ptr(A_hi), ptr(A_lo), ptr(B_hi), ptr(B_lo), ldn, N, M, 3, ptr(u_mean), ptr(g_sums),
                                      ptr(g_scratch), g_scratch.numel(), ptr(A_d), ptr(B_d), st), "spb_gram_tc")
            else:
                check(lib.spb_weighted_gram(ptr(UT), ldn, N, M, ptr(Pf), ptr(PY3), ptr(A_d), ptr(B_d), st), "spb_weighted_gram")
            if ev_pairs is not None:
                evs[2].record()
            # M-step on the device: (lambda sigma2 K + U^T P U) C = U^T P Y (the reference calls scipy.linalg.lstsq,
            # sparsevfc.py:189). A Cholesky solve is the same solution whenever the system is numerically positive definite;
            # its status flag rides along with the iteration's single host read, and the minimum-norm solution through the
            # symmetric eigen-decomposition with lstsq's eps*M cutoff is the fallback.
            Areg = lambda_ * sigma2 * Kd + 0.5 * (A_d + A_d.T)
            if use_tc:
                # The tensor-core blocks carry fp32-level noise (~1e-7 relative per entry, spectral norm ~1e-5 of a diagonal
                # entry at M = 500), which makes the numerically rank-deficient normal matrix indefinite. A ridge just above
                # that noise floor restores positive definiteness; it perturbs a direction of eigenvalue lambda_i by
                # delta / lambda_i — the same order as the unavoidable effect of the noise itself.
                Areg = Areg + (2e-5 * torch.diagonal(Areg).mean()) * torch.eye(M, dtype=torch.float64, device=dev)
            L, info = torch.linalg.cholesky_ex(Areg)
            Cn = torch.cholesky_solve(B_d, L)
            stats = torch.stack([
                (P[:N] * Y2).sum(), (Cn * B_d).sum(), (Cn * (A_d @ Cn)).sum(), (Cn * (Kd @ Cn)).sum(), info.to(torch.float64),
            ])
            s = torch.cat([sums, stats]).cpu().numpy()  # the one host synchronisation of the iteration
            if s[9] != 0 or not np.isfinite(s[5:9]).all():
                n_fallback += 1
                ev, Q = torch.linalg.eigh(Areg)
                cut = max(rcond, 1e-6 if use_tc else 0.0)
                inv = torch.where(ev > cut * ev.abs().max(), 1.0 / ev, torch.zeros_like(ev)) if use_tc else \
                    torch.where(ev.abs() > rcond * ev.abs().max(), 1.0 / ev, torch.zeros_like(ev))
                Cn = (Q * inv) @ (Q.T @ B_d)
                stats = torch.stack([(P[:N] * Y2).sum(), (Cn * B_d).sum(), (Cn * (A_d @ Cn)).sum(), (Cn * (Kd @ Cn)).sum()])
                s[5:9] = stats.cpu().numpy()
            if ev_pairs is not None:
                evs[3].record()
                ev_pairs.append(evs)
            E = s[0] / (2 * sigma2) + s[1] * np.log(sigma2) * D / 2 + lambda_ / 2 * reg_energy
            tecr = abs((E - E_old) / E)
            tecr_traj.append(tecr)
            E_traj.append(E)
            Cd.copy_(Cn)
            reg_energy = float(s[8])
            resid = s[5] - 2.0 * s[6] + s[7]
            sigma2 = float(max(resid, 0.0) / (s[3] * D))
            gamma = float(min(max(s[4] / N, 0.05), 0.95))
            it += 1
        if timings is not None:
            torch.cuda.synchronize()
            t = np.array([[e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3])] for e in ev_pairs])
            timings.update(estep_ms=t[:, 0], gram_ms=t[:, 1], solve_ms=t[:, 2], gram="tensor" if use_tc else "fp64",
                           eigh_fallbacks=n_fallback)
            if use_tc:  # split of gram_ms: operand preparation | tensor-core contraction + fp64 fold
                timings["gram_prepare_ms"] = np.array([e[1].elapsed_time(e[4]) for e in ev_pairs])
                timings["gram_tc_ms"] = np.array([e[4].elapsed_time(e[2]) for e in ev_pairs])
        C = Cd[:, :D].cpu().numpy()
        # final field on the cells and on the grid
        # scratch outputs of the final evaluation are bound to names so they outlive the (asynchronous) launch
        P_scratch, Pf_scratch, PY3_scratch = sums.new_empty(ldn), torch.empty_like(Pf), torch.empty_like(PY3)
        check(
            lib.spb_vfc_estep(ptr(UT), ldn, N, M, D, ptr(Cd), ptr(Yd), max(sigma2, 1e-300), gamma, float(a), float(minP),
                              float(theta), ptr(P_scratch), ptr(V), ptr(Pf_scratch), ptr(PY3_scratch), ptr(sums), st),
            "spb_vfc_estep(final)",
        )
        V_host = V.cpu().numpy()
        P_host = P[:N].cpu().numpy()
    out = {
        "X": X_full, "valid_ind": valid_ind, "X_ctrl": ctrl, "ctrl_idx": ctrl_idx, "Y": Y_full, "beta": beta,
        "V": V_host, "C": C, "P": P_host[:, None], "VFCIndex": np.where(P_host > theta)[0], "sigma2": sigma2,
        "grid": Grid, "grid_V": None, "iteration": it - 1, "tecr_traj": np.array(tecr_traj), "E_traj": np.array(E_traj),
    }
    if Grid is not None:
        out["grid_V"] = field_eval(np.asarray(Grid, dtype=np.float64), ctrl, C, beta, device=dev)
    return out


def _sparse_vfc_general(X_full, Y_full, valid_ind, Grid, M, a, beta, ecr, gamma, lambda_, minP, MaxIter, theta,
                        velocity_based_sampling, seed, ctrl_idx, dev, lib) -> dict:
    """SparseVFC for a general output dimension (the expression / label interpolation of ``kernel_interpolation``,
    spateo/tdr/interpolations/interpolation_sparseVFC.py:64): inputs live in R^dx (dx <= 3), outputs in R^dy. The posterior
    couples the output columns only through the squared residual, so the normal-equation blocks U^T P U and U^T P Y are
    contracted by the same device kernels three output columns at a time; the O(N dy) element-wise steps and the field
    evaluation V = U C of this secondary path use torch tensor ops."""
    Xv, Yv = X_full[valid_ind], Y_full[valid_ind]
    N, Dy = Yv.shape
    Dx = Xv.shape[1]
    if Dx > 3:
        raise ValueError("SparseVFC: the input coordinates must have at most 3 dimensions")
    if ctrl_idx is None:
        tmp_X, uid = np.unique(Xv, axis=0, return_index=True)
        M = min(M, tmp_X.shape[0])
        idx = sample_by_velocity(Yv[uid], M, seed) if velocity_based_sampling else \
            np.random.RandomState(seed).permutation(tmp_X.shape[0])[:M]
        ctrl_idx = uid[idx]
    ctrl_idx = np.asarray(ctrl_idx)
    ctrl = Xv[ctrl_idx]
    M = ctrl.shape[0]
    if beta is None:
        beta = 1.0 / bandwidth_selector(ctrl) ** 2
    Kc = np.exp(-beta * ((ctrl[:, None, :] - ctrl[None, :, :]) ** 2).sum(-1))
    f64 = torch.float64
    with torch.cuda.device(dev):
        st = _capi.current_stream_ptr()
        ldn = _round_up(N, 1024)
        centre = Xv.mean(axis=0)
        x_soa = torch.zeros((3, ldn), dtype=torch.float32, device=dev)
        x_soa[:Dx, :N] = torch.from_numpy(np.ascontiguousarray((Xv - centre).T, dtype=np.float32)).to(dev)
        z = torch.zeros((M, 3), dtype=torch.float32, device=dev)
        z[:, :Dx] = torch.from_numpy((ctrl - centre).astype(np.float32)).to(dev)
        UT = torch.empty((M, ldn), dtype=torch.float32, device=dev)
        check(lib.spb_rbf_kernel_T(ptr(x_soa), N, ldn, ptr(z), M, float(beta), ptr(UT), st), "spb_rbf_kernel_T")
        U64 = UT[:, :N].T.to(f64)  # [N, M] for the field evaluation of this secondary path
        Yd = torch.from_numpy(np.ascontiguousarray(Yv)).to(dev)
        Kd = torch.from_numpy(Kc).to(dev)
        Cd = torch.zeros((M, Dy), dtype=f64, device=dev)
        V = torch.zeros((N, Dy), dtype=f64, device=dev)
        Pf = torch.zeros((ldn,), dtype=torch.float32, device=dev)
        PY3 = torch.zeros((3, ldn), dtype=torch.float32, device=dev)
        A_d = torch.empty((M, M), dtype=f64, device=dev)
        B3 = torch.empty((M, 3), dtype=f64, device=dev)
        Bd = torch.empty((M, Dy), dtype=f64, device=dev)
        sigma2 = max(float(((Yd - V) ** 2).sum().item() / (N * Dy)), 1e-7)
        E, tecr, it = 1.0, 1.0, 0
        tecr_traj, E_traj = [], []
        rcond = np.finfo(np.float64).eps * M
        P = torch.ones((N,), dtype=f64, device=dev)
        while it < MaxIter and tecr > ecr and sigma2 > 1e-8:
            E_old = E
            r = ((Yd - V) ** 2).sum(1)
            t1 = torch.exp(-r / (2 * sigma2))
            t2 = (2 * np.pi * sigma2) ** (Dy / 2) * (1 - gamma) / (gamma * a)
            P = t1 / (t1 + t2)
            E = float(((P * r).sum() / (2 * sigma2) + P.sum() * np.log(sigma2) * Dy / 2).item()) \
                + lambda_ / 2 * float((Cd * (Kd @ Cd)).sum().item())
            tecr = abs((E - E_old) / E)
            tecr_traj.append(tecr)
            E_traj.append(E)
            P = torch.clamp(P, min=minP)
            Pf[:N] = P.float()
            for c0 in range(0, Dy, 3):
                c1 = min(Dy, c0 + 3)
                PY3.zero_()
                PY3[: c1 - c0, :N] = (P[:, None] * Yd[:, c0:c1]).T.float()
                check(lib.spb_weighted_gram(ptr(UT), ldn, N, M, ptr(Pf), ptr(PY3), ptr(A_d), ptr(B3), st), "spb_weighted_gram")
                Bd[:, c0:c1] = B3[:, : c1 - c0]
            Areg = lambda_ * sigma2 * Kd + 0.5 * (A_d + A_d.T)
            L, info = torch.linalg.cholesky_ex(Areg)
            if int(info.item()) == 0:
                Cn = torch.cholesky_solve(Bd, L)
            else:
                ev, Q = torch.linalg.eigh(Areg)
                inv = torch.where(ev.abs() > rcond * ev.abs().max(), 1.0 / ev, torch.zeros_like(ev))
                Cn = (Q * inv) @ (Q.T @ Bd)
            Cd.copy_(Cn)
            V = U64 @ Cd
            Sp = P.sum()
            sigma2 = float(((P * ((Yd - V) ** 2).sum(1)).sum() / (Sp * Dy)).item())
            gamma = float(min(max(float((P > theta).sum().item()) / N, 0.05), 0.95))
            it += 1
        C = Cd.cpu().numpy()
        V_host, P_host = V.cpu().numpy(), P.cpu().numpy()
        grid_V = None
        if Grid is not None:
            g = torch.from_numpy(np.ascontiguousarray(np.asarray(Grid, dtype=np.float64) - centre)).to(dev)
            zc = torch.from_numpy(np.ascontiguousarray(ctrl - centre)).to(dev)
            grid_V = (torch.exp(-beta * torch.cdist(g, zc) ** 2) @ Cd).cpu().numpy()
    return {
        "X": X_full, "valid_ind": valid_ind, "X_ctrl": ctrl, "ctrl_idx": ctrl_idx, "Y": Y_full, "beta": beta, "V": V_host,
        "C": C, "P": P_host[:, None], "VFCIndex": np.where(P_host > theta)[0], "sigma2": sigma2, "grid": Grid, "grid_V": grid_V,
        "iteration": it - 1, "tecr_traj": np.array(tecr_traj), "E_traj": np.array(E_traj),
    }


def morphofield_sparsevfc_core(
    X: np.ndarray,
    V: np.ndarray,
    NX: Optional[np.ndarray] = None,
    grid_num: Optional[List[int]] = None,
    M: int = 100,
    lambda_: float = 0.02,
    lstsq_method: str = "scipy",
    min_vel_corr: float = 0.8,
    restart_num: int = 10,
    restart_seed: Union[List[int], Tuple[int], np.ndarray] = (0, 100, 200, 300, 400),
    **kwargs,
) -> dict:
    """Restart wrapper of the reference (sparsevfc.py:103-238): retry with new seeds until the cosine correlation between
    input and learned vectors reaches ``min_vel_corr``, else keep the best trial."""
    from .morphofield import _grid_from_points

    if NX is not None:
        predict_X = NX
    else:
        if grid_num is None:
            grid_num = [50, 50, 50]
        predict_X = _grid_from_points(X, grid_num[: X.shape[1]])

    def corr(vf):
        ref, pred = vf["Y"][vf["valid_ind"]], vf["V"]
        tn = ref / (np.linalg.norm(ref, axis=1).reshape(-1, 1) + 1e-20)
        pn = pred / (np.linalg.norm(pred, axis=1).reshape(-1, 1) + 1e-20)
        return np.mean(tn * pn) * pred.shape[1]

    if restart_num > 0:
        restart_seed = np.asarray(restart_seed)
        if len(restart_seed) != restart_num:
            restart_seed = np.arange(restart_num) * 100
        trials, scores = [], []
        counter = 0
        while True:
            cur = SparseVFC(X=X, Y=V, Grid=predict_X, M=M, lstsq_method=lstsq_method, lambda_=lambda_,
                            seed=int(restart_seed[counter]), **kwargs)
            res = corr(cur)
            trials.append(cur)
            scores.append(res)
            if res < min_vel_corr:
                counter += 1
            else:
                vf_dict = cur
                break
            if counter > restart_num - 1:
                vf_dict = trials[int(np.argmax(np.array(scores)))]
                break
    else:
        vf_dict = SparseVFC(X=X, Y=V, Grid=predict_X, M=M, lstsq_method=lstsq_method, lambda_=lambda_, **kwargs)
    vf_dict["method"] = "sparsevfc"
    return vf_dict
