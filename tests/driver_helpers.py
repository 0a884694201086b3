"""Inputs shared by tests/golden/make_golden_drivers.py and the driver parity tests: a seeded 4-slice 2-D chain."""

import numpy as np

# keyword arguments handed to the reference drivers and to ours (full EM so that the non-rigid phase runs: 120 > 80)
KW = dict(SVI_mode=False, max_iter=120, K=12)


def driver_chain(n_slices=4, g=24, seed=7):
    """Serial sections of one 2-D tissue: every slice has its own cells (different counts per slice), counts and pose."""
    import pandas as pd

    from spateo_release_b200.anndata_lite import AnnDataLite

    rng = np.random.default_rng(seed)
    W = rng.normal(size=(2, g))
    phi = rng.uniform(0, 2 * np.pi, size=g)
    var = pd.DataFrame(index=[f"g{i}" for i in range(g)])
    out, poses = [], []
    for k in range(n_slices):
        n = 420 + 30 * k
        c = rng.uniform(0, 60, size=(n, 2))
        lam = np.exp(np.sin(c @ W / 18.0 + phi))
        X = rng.poisson(lam).astype(np.float32)
        th, sh = 0.2 * k, np.array([2.5 * k, -1.5 * k])
        R = np.array([[np.cos(th), -np.sin(th)], [np.sin(th), np.cos(th)]])
        raw = c @ R.T + sh + rng.normal(0, 0.15, size=c.shape)
        out.append(AnnDataLite(X, var=var.copy(), obsm={"spatial": raw, "truth": c}))
        poses.append((R, sh))
    return out, poses


def models_from_golden(g, n_slices=4):
    """The same chain rebuilt from the fixture (no RNG-order dependence on this helper)."""
    import pandas as pd

    from spateo_release_b200.anndata_lite import AnnDataLite

    G = g["in0_X"].shape[1]
    var = pd.DataFrame(index=[f"g{i}" for i in range(G)])
    return [AnnDataLite(np.array(g[f"in{k}_X"]), var=var.copy(), obsm={"spatial": np.array(g[f"in{k}_spatial"])})
            for k in range(n_slices)]
