"""CPU: the references of the sparse top-k posterior and the posterior argmax (tests/parity_helpers.py) pinned to the oracle
and to brute force, so that the GPU tests in test_gpu_posterior_select.py compare the kernels with something known right.

- ``sparse_posterior_reference`` (column chunks, cost matrix as input) equals ``oracle.morpho_oracle.get_P_core`` with
  ``sparse_calculation_mode`` (``dense_to_sparse_topk``) to 1e-12, for k from 1 to past N_A.
- ``topk_replay`` (threshold, ties, the column and row sums the kernels form) and ``argmax_replay`` (keys with the
  lowest-index tie rules, the sparse-mode threshold and a column map) equal a per-column / per-row brute force on weights
  with exact ties, zeros, subnormals and columns with fewer than k non-zero weights."""

import numpy as np
import pytest

from oracle import morpho_oracle as mo
from parity_helpers import argmax_keys, argmax_replay, sparse_posterior_reference, topk_replay


def _state(rng, NA, NB, D):
    XA = rng.normal(size=(NA, D)) * 3.0
    YB = rng.normal(size=(NB, D)) * 3.0
    G = rng.uniform(0.05, 1.0, size=(NA, NB))
    G[rng.random(G.shape) < 0.1] = 0.0
    mm = rng.uniform(0.5, 1.5, size=(NA, 1))
    return XA, YB, G, mm


@pytest.mark.parametrize("D", [2, 3])
def test_sparse_posterior_reference_equals_oracle(D):
    rng = np.random.default_rng(D)
    NA, NB = 300, 280
    XA, YB, G, mm = _state(rng, NA, NB, D)
    kw = dict(sigma2=2.5, model_mul=mm, gamma=0.6, samples_s=0.01, sigma2_variance=1.7)
    ks = (1, 7, 48, NA - 1, NA, NA + 1)
    got = sparse_posterior_reference(float(D), XA, YB, G, ks=ks, chunk=64, **kw)
    spatial = ((XA[:, None, :] - YB[None, :, :]) ** 2).sum(-1)
    for k in ks:
        P, _, _, _ = mo.get_P_core(Dim=float(D), spatial_dist=spatial, exp_dist=[G], probability_type=["prob"],
                                   sparse_calculation_mode=True, top_k=k, **kw)
        want = P.toarray()
        o = got[k]
        kk = min(k, NA)
        mine = np.zeros((NA, NB))
        np.put_along_axis(mine, o["rows"].T, o["vals"].T, axis=0)
        scale = np.abs(want).max()
        assert np.abs(mine - want).max() <= 1e-12 * scale, k
        assert (np.diff(o["vals"], axis=1) <= 0).all()
        assert all(len(set(r)) == kk for r in o["rows"])
        assert np.abs(o["K_NA"] - want.sum(1)).max() <= 1e-12 * want.sum(1).max()
        assert np.abs(o["K_NB"] - want.sum(0)).max() <= 1e-12 * want.sum(0).max()
        assert np.abs(o["PXB"] - want @ YB).max() <= 1e-12 * np.abs(want @ YB).max()
        dense, _, _, _ = mo.get_P_core(Dim=float(D), spatial_dist=spatial, exp_dist=[G], probability_type=["prob"], **kw)
        srt = -np.sort(-dense, axis=0)
        assert np.array_equal(o["kth"], srt[kk - 1])
        assert np.array_equal(o["kth1"], srt[kk] if kk < NA else np.zeros(NB))


def test_sparse_posterior_reference_float32_restatement_is_close():
    rng = np.random.default_rng(5)
    XA, YB, G, mm = _state(rng, 200, 150, 2)
    kw = dict(sigma2=2.5, model_mul=mm, gamma=0.6, samples_s=0.01, sigma2_variance=1.0, ks=(16,), chunk=50)
    a = sparse_posterior_reference(2.0, XA, YB, G, **kw)[16]
    b = sparse_posterior_reference(2.0, XA, YB, G, dtype=np.float32, **kw)[16]
    assert b["vals"].dtype == np.float32
    assert np.abs(a["K_NB"] - b["K_NB"]).max() < 1e-5 * a["K_NB"].max()


def _weights():
    """Columns: random; ties straddling the 5th position; subnormals and zeros; fewer than 5 non-zero; all zero; all
    equal; values one bit apart."""
    rng = np.random.default_rng(0)
    NA = 23
    W = rng.uniform(0.1, 1.0, size=(NA, 7)).astype(np.float32)
    W[:, 1] = np.float32(0.25)
    W[:3, 1] = [0.9, 0.8, 0.7]
    W[10:, 1] = 0.1
    sub = np.float32(1e-40)
    W[:, 2] = 0.0
    W[:8, 2] = sub * np.arange(1, 9, dtype=np.float32)
    W[8, 2] = 3.0
    W[:, 3] = 0.0
    W[[4, 9, 17], 3] = [0.5, 0.25, 0.5]
    W[:, 4] = 0.0
    W[:, 5] = 0.5
    W[:, 6] = (np.float32(1.0).view(np.uint32) + np.arange(NA, dtype=np.uint32)[::-1] % 7).view(np.float32)
    return W


@pytest.mark.parametrize("k", [1, 5, 22, 23, 24])
def test_topk_replay_equals_brute_force(k):
    W = _weights()
    NA, NB = W.shape
    c = np.linspace(0.5, 2.0, NB).astype(np.float32)
    Y = np.arange(2 * NB, dtype=np.float64).reshape(NB, 2)
    r = topk_replay(W, k, c, Y)
    kk = min(k, NA)
    for j in range(NB):
        col = sorted(W[:, j].tolist(), reverse=True)
        tau = col[kk - 1] if col[kk - 1] > 0 else 0.0
        assert r["tau"][j] == np.float32(tau)
        keep = [w for w in W[:, j].tolist() if w >= tau]
        assert r["K_NB"][j] == pytest.approx(float(c[j]) * sum(keep), rel=1e-15)
        assert r["K_NB_k"][j] == pytest.approx(float(c[j]) * sum(col[:kk]), rel=1e-15)
        assert r["n_above"][j] == sum(w > tau for w in col)
        assert r["n_ties"][j] == (sum(w == tau for w in col) if tau > 0 else 0)
    kept = np.where(W >= r["tau"][None, :], W.astype(np.float64), 0.0)
    assert np.allclose(r["K_NA"], [sum(kept[i, j] * float(c[j]) for j in range(NB)) for i in range(NA)], rtol=1e-15)
    assert np.allclose(r["PXB"], kept @ (c[:, None].astype(np.float64) * Y), rtol=1e-15)
    # the column of subnormals: the k-th largest is a subnormal for k = 5
    if k == 5:
        assert r["tau"][2] == np.float32(1e-40) * 5
    # fewer than k non-zero weights, or a column of zeros: nothing is cut
    if k >= 3:
        assert r["tau"][3] == 0 and r["tau"][4] == 0


@pytest.mark.parametrize("k", [1, 3, 23])
def test_argmax_replay_equals_brute_force(k):
    W = _weights()
    W[7] = 0.0                      # an all-zero row
    W[11, :] = W[12, :]             # rows with equal values: ties down a column
    W[13, 6] = W[13, 0] = 2.0       # a non-zero tie along a row
    NA, NB = W.shape
    c = np.full(NB, 1.0, np.float32)
    c[1] = 0.75
    tau = topk_replay(W, k, c)["tau"]
    rowkey, colkey = argmax_replay(W, c, tau, block=3)
    P = W * c[None, :]
    for j in range(NB):
        i = int(np.argmax(P[:, j]))                               # first (lowest) row among equal maxima
        assert colkey[j] == argmax_keys(P[i, j], i)
    Ps = np.where(W >= tau[None, :], W, np.float32(0)) * c[None, :]
    for i in range(NA):
        j = int(np.argmax(Ps[i]))
        assert rowkey[i] == argmax_keys(Ps[i, j], j)
    assert rowkey[7] == argmax_keys(np.float32(0), 0)
    assert rowkey[13] == argmax_keys(np.float32(2.0), 0)
    # a column map: -1 skips a column, the key carries the mapped index
    cmap = np.array([5, -1, 0, 3, 2, 1, 4])
    rk, _ = argmax_replay(W, c, tau, colmap=cmap)
    for i in range(NA):
        best = max((int(argmax_keys(Ps[i, j], cmap[j])[0]) for j in range(NB) if cmap[j] >= 0))
        assert int(rk[i]) == best
