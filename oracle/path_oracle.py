"""TEST INFRASTRUCTURE ONLY — float64 host restatement of ``st.tdr.morphopath``.

The reference (spateo/tdr/morphometrics/morphofield/trajectory.py:11-61) hands the field to dynamo's ``fate``, which runs
``scipy.integrate.solve_ivp`` once per cell with a terminal event that fires once every velocity component is below
1e-5 (dynamo's ``integrate_vf_ivp``). dynamo is third-party and absent, so PARITY WITH DYNAMO IS UNPINNED; the integrator
itself is scipy's and is called here unchanged: ``solve_ivp(RK45, max_step=t_end / interpolation_num, t_eval=...,
events=...)`` per cell, over ``field_oracle``'s ``gp_velocity`` / ``svc_velocity``. The samples are at evenly spaced
times (``t_eval``), not dynamo's arc-length resampling. Only tests and profiles may import this module.
"""

import numpy as np
from scipy.integrate import RK45, solve_ivp

from oracle.field_oracle import gp_velocity, svc_velocity


class _CountingRK45(RK45):
    """scipy's RK45 unchanged, counting accepted steps (the rejected ones follow from nfev = 2 + 6 * attempts)."""

    last = None

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.n_accepted = 0
        _CountingRK45.last = self

    def _step_impl(self):
        ok, message = super()._step_impl()
        self.n_accepted += bool(ok)
        return ok, message


def field_function(vf, nonrigid_only=False):
    """v(x) for one state x [D], chosen by ``vf["method"]`` as ``morphopath`` chooses it."""
    method = vf.get("method")
    if method == "gaussian_process":
        vf = dict(vf, R=np.asarray(vf["R"], dtype=np.float64), t=np.asarray(vf["t"], dtype=np.float64))
        return lambda x: gp_velocity(np.asarray(x, dtype=np.float64)[None], vf, nonrigid_only)[0]
    if method == "sparsevfc":
        vf = {"X_ctrl": np.asarray(vf["X_ctrl"], dtype=np.float64), "C": np.asarray(vf["C"], dtype=np.float64),
              "beta": vf["beta"]}
        return lambda x: svc_velocity(np.asarray(x, dtype=np.float64)[None], vf)[0]
    raise ValueError(f"unknown vector field method {method!r}")


def integrate_one(f, x0, t_bound, interpolation_num, rtol=1e-3, atol=1e-6):
    """One cell, one direction (the sign of ``t_bound``). Returns the samples at the ``t_eval`` grid up to the stop,
    the stop time and state, nfev, the accepted / rejected step counts and the status (0 reached t_bound, 1 event, -1 failed)."""

    def event(t, x):
        return np.all(np.abs(f(x)) < 1e-5) - 1

    event.terminal = True
    t_eval = np.linspace(0.0, t_bound, interpolation_num + 1)
    sol = solve_ivp(lambda t, x: f(x), (0.0, t_bound), np.asarray(x0, dtype=np.float64), method=_CountingRK45,
                    max_step=abs(t_bound) / interpolation_num, t_eval=t_eval, events=event, rtol=rtol, atol=atol)
    solver = _CountingRK45.last
    attempts = (sol.nfev - 2) // 6
    if sol.status == 1:
        t_stop, y_stop = float(sol.t_events[0][0]), sol.y_events[0][0]
    else:
        t_stop, y_stop = float(solver.t), solver.y
    return {"t": sol.t, "y": sol.y.T, "t_stop": t_stop, "y_stop": y_stop, "nfev": int(sol.nfev),
            "accepted": solver.n_accepted,
            "rejected": attempts - solver.n_accepted, "status": int(sol.status)}


def path(X0, vf, t_end, interpolation_num=250, direction="forward", nonrigid_only=False, rtol=1e-3, atol=1e-6):
    """Every cell of X0 [n, D]: a list of {"t": [n_t], "y": [n_t, D], "runs": [one ``integrate_one`` result per
    direction integrated, backward first]}. ``"both"`` is the backward path reversed, then the forward path without its
    repeated initial point."""
    if direction not in ("forward", "backward", "both"):
        raise ValueError(f"direction must be 'forward', 'backward' or 'both', not {direction!r}")
    f = field_function(vf, nonrigid_only)
    bounds = {"forward": [t_end], "backward": [-t_end], "both": [-t_end, t_end]}[direction]
    out = []
    for x0 in np.asarray(X0, dtype=np.float64):
        runs = [integrate_one(f, x0, tb, interpolation_num, rtol, atol) for tb in bounds]
        if direction == "both":
            b, fw = runs
            t = np.concatenate([b["t"][::-1], fw["t"][1:]])
            y = np.concatenate([b["y"][::-1], fw["y"][1:]])
        else:
            t, y = runs[0]["t"], runs[0]["y"]
        out.append({"t": t, "y": y, "runs": runs})
    return out
