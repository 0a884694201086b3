"""GPU: st.tdr.morphopath / spb_field_integrate against scipy's solve_ivp (oracle/path_oracle.py), cell by cell."""

import numpy as np
import pytest

from field_helpers import load_field
from oracle import path_oracle as po

pytestmark = pytest.mark.gpu


class _Adata:
    def __init__(self, n):
        import pandas as pd

        self.uns, self.obsm, self.obs = {}, {}, pd.DataFrame(index=[f"c{i}" for i in range(n)])


def _gp(golden, tag):
    vf, X = load_field(golden("field_geometry"), tag)  # fields of a real 2-D / 3-D morpho_align run
    return vf, X


def _svc(D, n, seed=5):
    """A SparseVFC-style field rotating and drifting outwards: the step controller rejects steps."""
    rng = np.random.default_rng(seed)
    ctrl = rng.uniform(0, 50, (60, D))
    c = ctrl - 25.0
    C = 0.05 * c
    C[:, 0] += -0.2 * c[:, 1]
    C[:, 1] += 0.2 * c[:, 0]
    C += rng.normal(0, 0.3, (60, D))
    vf = {"method": "sparsevfc", "X_ctrl": ctrl, "C": C, "beta": 1.0 / 12.0**2}
    X = rng.uniform(-10, 60, (n, D))
    X[:5] = 200.0 + rng.uniform(0, 1, (5, D))  # already in the slow region: stopped at t = 0
    return vf, X


def _bump(D, n, seed=7):
    """A few control points pushing along +x: every path runs out of the bump and stops where |v| < 1e-5."""
    rng = np.random.default_rng(seed)
    C = rng.normal(0, 0.2, (4, D))
    C[:, 0] += 1.0
    vf = {"method": "sparsevfc", "X_ctrl": rng.normal(0, 0.5, (4, D)), "C": C, "beta": 0.25}
    return vf, rng.uniform(-3, 3, (n, D))


def _gp_large_K(D, n, K, seed=9):
    """A GP field with more inducing points than one shared-memory tile (1024)."""
    rng = np.random.default_rng(seed)
    vf = {"method": "gaussian_process", "kernel_type": "euc", "beta": 2.0,
          "inducing_variables": rng.uniform(-1.5, 1.5, (K, D)), "Coff": rng.normal(0, 0.02, (K, D)),
          "R": np.eye(D), "t": np.zeros(D),
          "norm_dict": {"mean_transformed": np.full(D, 5.0), "scale_transformed": 4.0, "mean_fixed": np.full(D, 5.5),
                        "scale_fixed": 4.2}}
    return vf, rng.uniform(0, 10, (n, D))


def _run(vf, X, t_end, interpolation_num, direction, nonrigid_only=False, average=False):
    from spateo_release_b200 import tdr

    a = _Adata(len(X))
    a.uns["VecFld_morpho"] = dict(vf, X=X)
    tdr.morphopath(a, t_end=t_end, interpolation_num=interpolation_num, direction=direction, average=average,
                   nonrigid_only=nonrigid_only)
    return a.uns["fate_morpho"]


def _kernel_runs(vf, X, t_end, interpolation_num, direction, nonrigid_only=False):
    """The per-cell counts, stop times and statuses of each direction (backward first), straight from the kernel."""
    import importlib

    from spateo_release_b200.tdr import morphofield_dg as dg

    mp = importlib.import_module("spateo_release_b200.tdr.morphopath")  # the package exports the function by that name
    D = X.shape[1]
    if vf["method"] == "sparsevfc":
        f, z, C = dg._desc_svc(vf, D, 2), vf["X_ctrl"], vf["C"]
    else:
        f, z, C = dg._desc(vf, D, nonrigid_only, 2), vf["inducing_variables"], vf["Coff"]
    bounds = {"forward": [t_end], "backward": [-t_end], "both": [-t_end, t_end]}[direction]
    return [mp._integrate(f, np.ascontiguousarray(X, dtype=np.float64), np.ascontiguousarray(z, dtype=np.float64),
                          np.ascontiguousarray(C, dtype=np.float64), tb, interpolation_num, "cuda") for tb in bounds]


def _check(vf, X, t_end, interpolation_num, direction, nonrigid_only=False, label=""):
    n, D = X.shape
    got = _run(vf, X, t_end, interpolation_num, direction, nonrigid_only)
    runs = _kernel_runs(vf, X, t_end, interpolation_num, direction, nonrigid_only)
    want = po.path(X, vf, t_end, interpolation_num, direction, nonrigid_only)
    # the uns schema of dynamo's fate
    assert set(got) == {"init_states", "init_cells", "average", "t", "prediction", "status"}
    assert got["init_cells"] == [f"c{i}" for i in range(n)] and got["average"] is False
    assert np.array_equal(got["init_states"], X) and len(got["t"]) == n and len(got["prediction"]) == n
    assert sum(got["status"].values()) == n * len(runs)
    mismatched, worst_y, worst_t = 0, 0.0, 0.0
    for i in range(n):
        same = True
        for (out, t_stop, steps, status), w in zip(runs, want[i]["runs"]):
            if (steps[i, 0], steps[i, 1]) != (w["accepted"], w["rejected"]):
                same = False
                continue
            assert status[i] == w["status"]
            worst_t = max(worst_t, abs(t_stop[i] - w["t_stop"]) / t_end)
        if not same:
            mismatched += 1
            continue
        t, y = want[i]["t"], want[i]["y"]
        assert np.array_equal(got["t"][i], t) and got["prediction"][i].shape == (D, len(t))
        extent = max(float(np.ptp(y, axis=0).max()), 1e-300)
        worst_y = max(worst_y, float(np.abs(got["prediction"][i].T - y).max()) / extent)
    stats = {s: int(sum((r[3] == s).sum() for r in runs)) for s in (0, 1, -1)}
    print(f"{label}: {n} cells, step counts differ for {mismatched} (knife-edge accept/reject), states {worst_y:.2e} of "
          f"extent, stop times {worst_t:.2e} of t_end, statuses {stats}")
    assert mismatched <= int(0.001 * n)
    assert worst_y < 1e-9 and worst_t < 1e-9
    assert got["status"] == {"reached_t_end": stats[0], "stopped_by_event": stats[1], "failed": stats[-1]}
    return runs


@pytest.mark.parametrize("tag", ["2d", "3d"])
@pytest.mark.parametrize("nonrigid_only", [False, True])
def test_gp_field_from_alignment(golden, tag, nonrigid_only):
    vf, X = _gp(golden, tag)  # 300 / 400 cells: not a multiple of the 128-thread block
    _check(vf, X, 10000.0, 20, "forward", nonrigid_only, f"gp {tag} nonrigid_only={nonrigid_only}")


@pytest.mark.parametrize("direction", ["forward", "backward", "both"])
def test_directions(golden, direction):
    vf, X = _gp(golden, "3d")
    _check(vf, X[:150], 10000.0, 20, direction, label=f"gp 3d {direction}")


def test_interpolation_num_250(golden):
    vf, X = _gp(golden, "2d")
    _check(vf, X[:100], 10000.0, 250, "both", label="gp 2d 250")


@pytest.mark.parametrize("D", [2, 3])
def test_sparsevfc_field(D):
    vf, X = _svc(D, 200)
    runs = _check(vf, X, 100.0, 20, "both", label=f"svc {D}d")
    assert sum((r[2][:, 1] > 0).sum() for r in runs) >= 100  # rejected steps are exercised
    assert all((r[3][:5] == 1).all() and (r[1][:5] == 0.0).all() for r in runs)  # cells that start slow stop at t = 0


@pytest.mark.parametrize("D", [2, 3])
def test_event_stops(D):
    vf, X = _bump(D, 150)
    runs = _check(vf, X, 1e5, 50, "both", label=f"bump {D}d")
    assert all((r[3] == 1).all() and (r[1] != 0).all() for r in runs)


def test_inducing_points_above_the_shared_memory_tile():
    vf, X = _gp_large_K(3, 130, 2500)
    _check(vf, X, 10000.0, 20, "forward", label="gp K=2500")


def test_average():
    vf, X = _svc(3, 200, seed=6)
    got = _run(vf, X, 100.0, 20, "both", average=True)
    want = po.path(X, vf, 100.0, 20, "both")
    grid = np.linspace(-100.0, 100.0, 41)
    assert got["average"] is True and len(got["t"]) == 1 and len(got["prediction"]) == 1
    assert np.allclose(got["t"][0], grid, rtol=0, atol=1e-12) and got["prediction"][0].shape == (3, 41)

    def full(run, t_bound):  # every grid time; after a stop, the state at the stop
        g = np.linspace(0, t_bound, 21)
        y = np.repeat(run["y_stop"][None], 21, axis=0)
        y[: len(run["t"])] = run["y"]
        return g, y

    paths = []
    for w in want:
        (_, yb), (_, yf) = full(w["runs"][0], -100.0), full(w["runs"][1], 100.0)
        paths.append(np.concatenate([yb[::-1], yf[1:]]))
    mean = np.mean(paths, axis=0).T
    assert np.abs(got["prediction"][0] - mean).max() < 1e-9 * np.ptp(mean, axis=1).max()
