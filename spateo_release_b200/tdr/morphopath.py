"""Cell trajectories through the morphometric vector field (reference: spateo/tdr/morphometrics/morphofield/trajectory.py).

The reference's ``morphopath`` (trajectory.py:11-61) hands the field to dynamo's ``fate``, which calls
``scipy.integrate.solve_ivp`` once per cell in a Python loop. Here one CUDA kernel (``spb_field_integrate``,
csrc/field.cu) integrates every cell at once, one thread per cell, in fp64, restating ``solve_ivp(method="RK45")`` step
for step: Dormand-Prince 5(4) with FSAL, scipy's first-step rule, RMS error norm and step controller, and the same
dense output, terminal event and ``t_eval`` sampling.
"""

from __future__ import annotations

import warnings

import numpy as np

from .. import _capi
from .morphofield_dg import _desc, _desc_svc

_DIRECTIONS = ("forward", "backward", "both")


def _integrate(f, X0, z, C, t_bound, interpolation_num, device):
    """One direction for every cell: samples [n, n_out, D] (after a cell's stop, its state at the stop), stop times,
    step counts [n, 2] and statuses, as numpy arrays."""
    import torch

    n, D = X0.shape
    n_out = interpolation_num + 1
    with torch.cuda.device(device):
        dev = torch.device(device)
        Xd = torch.from_numpy(X0).to(dev)
        zd = torch.from_numpy(z).to(dev)
        Cd = torch.from_numpy(C).to(dev)
        out = torch.empty((n, n_out, D), dtype=torch.float64, device=dev)
        t_stop = torch.empty(n, dtype=torch.float64, device=dev)
        steps = torch.empty((n, 2), dtype=torch.int32, device=dev)
        status = torch.empty(n, dtype=torch.int32, device=dev)
        _capi.check(_capi.load_library().spb_field_integrate(
            f, _capi.ptr(Xd), n, _capi.ptr(zd), _capi.ptr(Cd), float(t_bound), n_out, 1e-3, 1e-6,
            abs(t_bound) / interpolation_num, _capi.ptr(out), _capi.ptr(t_stop), _capi.ptr(steps), _capi.ptr(status),
            _capi.current_stream_ptr()), "spb_field_integrate")
        return out.cpu().numpy(), t_stop.cpu().numpy(), steps.cpu().numpy(), status.cpu().numpy()


def morphopath(
    adata,
    vf_key: str = "VecFld_morpho",
    key_added: str = "fate_morpho",
    direction: str = "forward",
    interpolation_num: int = 250,
    t_end=None,
    average: bool = False,
    nonrigid_only: bool = False,
    inplace: bool = True,
    device=None,
    cores: int = 1,
    **kwargs,
):
    """trajectory.py:11-61 — integrate every cell's trajectory dx/dt = v(x) from ``adata.uns[vf_key]["X"]``.

    The field is chosen by ``uns[vf_key]["method"]``: ``"gaussian_process"`` (the field of ``morphofield_gp``: rigid part,
    normalisation and the /10000 included; ``nonrigid_only`` drops the rigid part) or ``"sparsevfc"`` (K(x, X_ctrl) C, as
    ``SvcVectorField`` evaluates it). Each cell is integrated in fp64 exactly as ``scipy.integrate.solve_ivp(v, (0, ±t_end),
    x0, method="RK45", max_step=t_end / interpolation_num)`` at scipy's default tolerances (rtol 1e-3, atol 1e-6), and
    stops where every component of |v| first falls below 1e-5 (dynamo's terminal event). ``direction="backward"``
    integrates to -t_end; ``"both"`` stores the backward path reversed, then the forward path, with the initial point once.

    Results go to ``adata.uns[key_added]`` in the schema of dynamo's ``fate``: ``init_states``, ``init_cells``,
    ``average``, ``t`` (one array of times per cell) and ``prediction`` (one [D, n_t] array per cell), plus ``status``:
    how many cell integrations reached t_end, were stopped by the event and failed (hit 100 * interpolation_num accepted
    steps, or a step below scipy's minimum; a warning names the count). With ``"both"`` every cell counts once per
    direction. With ``average=True``, ``t`` and ``prediction`` hold one entry each: the mean state over all cells at
    every grid time, where a cell that stopped contributes its state at the stop.

    Differences from the reference: each trajectory is sampled at ``interpolation_num + 1`` evenly spaced times from the
    RK45 dense output (as ``t_eval`` does), on the same curve; dynamo resamples by arc length by default, and that
    resampling is not done here. ``t_end`` must be given (dynamo derives a default from the data; that rule is not
    restated). dynamo is third-party and absent, so parity with it is unpinned; the integration is checked against
    ``solve_ivp`` itself. ``cores`` is accepted and ignored (one kernel launch covers every cell); other ``fate`` options
    are not supported.
    """
    if kwargs:
        raise TypeError(f"morphopath() does not support the dynamo.fate option(s) {sorted(kwargs)}")
    adata = adata if inplace else adata.copy()
    if vf_key not in adata.uns.keys() or "X" not in adata.uns[vf_key]:
        raise Exception(
            f"The initial states ``anndata.uns['{vf_key}']['X']`` are missing. "
            f"Please run ``st.tdr.morphofield_gp(adata, vf_key='{vf_key}')`` or "
            f"``st.tdr.morphofield_sparsevfc(adata, key_added='{vf_key}')`` before running this function."
        )
    vf = adata.uns[vf_key]
    method = vf.get("method")
    if method not in ("gaussian_process", "sparsevfc"):
        raise ValueError(f"``anndata.uns['{vf_key}']['method']`` is {method!r}; expected 'gaussian_process' or 'sparsevfc'.")
    if t_end is None:
        raise ValueError("t_end is required: the default dynamo derives from the data is not implemented.")
    t_end = float(t_end)
    if not np.isfinite(t_end) or t_end <= 0:
        raise ValueError(f"t_end must be a positive finite number, not {t_end}.")
    if direction not in _DIRECTIONS:
        raise ValueError(f"direction must be one of {_DIRECTIONS}, not {direction!r}.")
    if int(interpolation_num) != interpolation_num or interpolation_num < 1:
        raise ValueError(f"interpolation_num must be a positive integer, not {interpolation_num!r}.")
    interpolation_num = int(interpolation_num)
    if interpolation_num + 1 > np.iinfo(np.int32).max // 100:
        raise ValueError(f"interpolation_num {interpolation_num} is too large.")

    X0 = np.ascontiguousarray(np.asarray(vf["X"], dtype=np.float64))
    if X0.ndim != 2 or X0.shape[1] not in (2, 3):
        raise ValueError("X has incorrect dimensions.")
    n, D = X0.shape
    if method == "gaussian_process":
        if vf["kernel_type"] != "euc":
            if vf["kernel_type"] == "geodist":
                raise NotImplementedError("geodist is not implemented yet")
            raise ValueError("current only support euc and geodist")
        f = _desc(vf, D, nonrigid_only, 2)
        zk, ck = "inducing_variables", "Coff"
    else:
        f = _desc_svc(vf, D, 2)
        zk, ck = "X_ctrl", "C"
    z = np.ascontiguousarray(np.asarray(vf[zk], dtype=np.float64))
    C = np.ascontiguousarray(np.asarray(vf[ck], dtype=np.float64))
    if z.ndim != 2 or C.shape != z.shape or z.shape[1] != D:
        raise ValueError("X has incorrect dimensions.")

    _capi.require_cuda()
    dev = "cuda" if device in (None, "cuda") else (f"cuda:{device}" if str(device).isdigit() else str(device))
    bounds = {"forward": [t_end], "backward": [-t_end], "both": [-t_end, t_end]}[direction]
    runs = []
    for t_bound in bounds:
        grid = np.linspace(0.0, t_bound, interpolation_num + 1)
        out, t_stop, _, status = _integrate(f, X0, z, C, t_bound, interpolation_num, dev)
        # samples emitted: the grid times at or before each cell's stop
        n_emit = np.count_nonzero(np.sign(t_bound) * (grid[None, :] - t_stop[:, None]) <= 0, axis=1)
        runs.append((grid, out, n_emit, status))

    def join(parts):  # "both": backward reversed, then forward without its initial point
        return parts[0] if len(parts) == 1 else np.concatenate([parts[0][::-1], parts[1][1:]])

    if average:
        t_all = [join([g for g, _, _, _ in runs])]
        pred = [join([o.mean(axis=0) for _, o, _, _ in runs]).T.copy()]
    else:
        t_all, pred = [], []
        for i in range(n):
            t_all.append(join([g[: m[i]] for g, _, m, _ in runs]))
            pred.append(join([o[i, : m[i]] for _, o, m, _ in runs]).T.copy())
    statuses = np.concatenate([s for _, _, _, s in runs])
    counts = {"reached_t_end": int((statuses == 0).sum()), "stopped_by_event": int((statuses == 1).sum()),
              "failed": int((statuses == -1).sum())}
    if counts["failed"]:
        warnings.warn(f"morphopath: {counts['failed']} cell integration(s) failed (step cap of "
                      f"{100 * interpolation_num} accepted steps or a step below the minimum); their paths end early.")
    obs_names = adata.obs_names if hasattr(adata, "obs_names") else adata.obs.index
    adata.uns[key_added] = {
        "init_states": X0,
        "init_cells": list(obs_names),
        "average": average,
        "t": t_all,
        "prediction": pred,
        "status": counts,
    }
    return None if inplace else adata
