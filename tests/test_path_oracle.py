"""CPU: the float64 trajectory oracle (oracle/path_oracle.py) and st.tdr.morphopath's argument checks."""

import numpy as np
import pytest
from scipy.linalg import expm

from oracle import path_oracle as po


def test_linear_field_matches_matrix_exponential():
    A = np.array([[-0.1, 1.0, 0.0], [-1.0, -0.1, 0.0], [0.0, 0.0, 0.05]])
    x0 = np.array([1.0, 0.5, 2.0])
    for t_bound in (10.0, -10.0):
        r = po.integrate_one(lambda x: A @ x, x0, t_bound, 40)
        assert r["status"] == 0 and r["t_stop"] == t_bound
        assert np.array_equal(r["t"], np.linspace(0, t_bound, 41))
        exact = np.stack([expm(A * t) @ x0 for t in r["t"]])
        # rtol 1e-3 / atol 1e-6 per step: the global error stays well inside 1 % of the state's size here
        assert np.abs(r["y"] - exact).max() < 1e-2 * np.abs(exact).max()
        assert r["y"][0].tolist() == x0.tolist()
        assert r["nfev"] == 2 + 6 * (r["accepted"] + r["rejected"]) and r["accepted"] >= 40


def test_decaying_field_stops_where_velocity_falls_below_threshold():
    # one Gaussian bump at the origin pushing along +x: |v| = exp(-beta x^2) < 1e-5 beyond x* = sqrt(ln(1e5) / beta)
    beta = 1.0 / 4.0
    vf = {"method": "sparsevfc", "X_ctrl": np.zeros((1, 2)), "C": np.array([[1.0, 0.0]]), "beta": beta}
    f = po.field_function(vf)
    x_star = np.sqrt(np.log(1e5) / beta)
    r = po.integrate_one(f, np.array([0.5, 0.0]), 1e5, 50)
    assert r["status"] == 1 and 0 < r["t_stop"] < 1e5
    assert np.all(np.abs(f(r["y_stop"])) < 1e-5)
    assert abs(r["y_stop"][0] - x_star) < 0.05 * x_star and r["y_stop"][1] == 0.0
    # only grid times up to the stop are emitted
    assert r["t"][-1] <= r["t_stop"] < r["t"][-1] + 1e5 / 50 and len(r["t"]) < 51
    # a cell already in the slow region stops at t = 0 and emits its initial state only
    r0 = po.integrate_one(f, np.array([3 * x_star, 1.0]), 1e5, 50)
    assert r0["status"] == 1 and r0["t_stop"] == 0.0 and r0["t"].tolist() == [0.0]
    assert r0["y"][0].tolist() == [3 * x_star, 1.0]


def test_both_is_reversed_backward_then_forward():
    rng = np.random.default_rng(4)
    vf = {"method": "sparsevfc", "X_ctrl": rng.uniform(0, 10, (6, 3)), "C": rng.normal(size=(6, 3)), "beta": 0.1}
    X0 = rng.uniform(0, 10, (4, 3))
    both = po.path(X0, vf, 5.0, 10, "both")
    fw = po.path(X0, vf, 5.0, 10, "forward")
    bw = po.path(X0, vf, 5.0, 10, "backward")
    for b, f, w in zip(both, fw, bw):
        assert np.array_equal(b["t"], np.concatenate([w["t"][::-1], f["t"][1:]]))
        assert np.array_equal(b["y"], np.concatenate([w["y"][::-1], f["y"][1:]]))
        assert np.count_nonzero(b["t"] == 0.0) == 1 and b["t"][0] == -5.0 and b["t"][-1] == 5.0
    with pytest.raises(ValueError):
        po.path(X0, vf, 5.0, 10, "sideways")


class _Adata:
    def __init__(self, n):
        import pandas as pd

        self.uns, self.obsm, self.obs = {}, {}, pd.DataFrame(index=[str(i) for i in range(n)])


def test_morphopath_argument_errors():
    from spateo_release_b200 import tdr

    a = _Adata(3)
    with pytest.raises(Exception, match="morphofield_gp"):
        tdr.morphopath(a, t_end=10)
    a.uns["VecFld_morpho"] = {"method": "sparsevfc", "X_ctrl": np.zeros((1, 2)), "C": np.ones((1, 2)), "beta": 1.0}
    with pytest.raises(Exception, match="morphofield_gp"):
        tdr.morphopath(a, t_end=10)
    a.uns["VecFld_morpho"]["X"] = np.zeros((3, 2))
    with pytest.raises(ValueError, match="t_end"):
        tdr.morphopath(a)
    with pytest.raises(ValueError, match="t_end"):
        tdr.morphopath(a, t_end=-1.0)
    with pytest.raises(ValueError, match="direction"):
        tdr.morphopath(a, t_end=10, direction="sideways")
    with pytest.raises(ValueError, match="interpolation_num"):
        tdr.morphopath(a, t_end=10, interpolation_num=0)
    with pytest.raises(TypeError, match="fate"):
        tdr.morphopath(a, t_end=10, arc_sample=True)
    a.uns["VecFld_morpho"]["method"] = "kernel_interpolation"
    with pytest.raises(ValueError, match="method"):
        tdr.morphopath(a, t_end=10)
    del a.uns["VecFld_morpho"]["method"]
    with pytest.raises(ValueError, match="method"):
        tdr.morphopath(a, t_end=10)
    assert "fate_morpho" not in a.uns
