"""TEST INFRASTRUCTURE ONLY — pins ``oracle/morpho_oracle.py`` against the unmodified reference.

Runs ``Morpho_pairwise`` from the reference checkout named by ``SPATEO_REFERENCE`` (oracle/ref_harness.py) and ``MorphoPairOracle`` on identical seeded inputs and prints the maximum
deviation of every output. Expected: bitwise or ~1 ulp agreement (same numpy calls in the same order).

    SPATEO_REFERENCE=<spateo-release checkout> python oracle/check_oracle_vs_reference.py
"""

import os
import sys
import warnings

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
warnings.filterwarnings("ignore")

from oracle.morpho_oracle import MorphoPairOracle  # noqa: E402
from oracle.ref_harness import load_reference  # noqa: E402
from spateo_release_b200.synthetic import make_slice_pair  # noqa: E402


def run_case(name, n_a, n_b, g, dim, dtype, svi, max_iter, K=15, seed=0, **kw):
    mc, _ = load_reference()
    A, B = make_slice_pair(n_a, n_b, g, dim=dim, seed=seed, warp_amplitude=kw.pop("warp", 0.0))
    if kw.pop("guide", False):  # a few (fixed, moving) landmark pairs: exact correspondences of the synthetic pair
        rng = np.random.default_rng(5)
        from spateo_release_b200.synthetic import _rotation

        pts = rng.uniform(10, 90, size=(12, dim))
        kw["guidance_pair"] = [pts, pts @ _rotation(dim, 0.5).T + 5.0]
    np.random.seed(0)
    ref = mc.Morpho_pairwise(
        sampleA=B, sampleB=A, device="cpu", dtype=dtype, verbose=False, SVI_mode=svi, max_iter=max_iter, K=K,
        vecfld_key_added="vf", **kw,
    )
    P_ref = ref.run()
    # the reference hands the solver column-major coordinates (fancy-indexing in check_spatial_coords, utils.py:103)
    rawA = np.asfortranarray(B.obsm["spatial"])
    rawB = np.asfortranarray(A.obsm["spatial"])
    np.random.seed(0)
    # feed the oracle the gene-ordered dense matrices the reference extracted (set() order is process dependent)
    orc = MorphoPairOracle(
        rawA, rawB, [np.asarray(e) for e in ref.exp_layers_A], [np.asarray(e) for e in ref.exp_layers_B],
        dtype=dtype, SVI_mode=svi, max_iter=max_iter, K=K, **kw,
    )
    P_orc = orc.run()
    worst = 0.0
    for key in ["P", "optimal_RnA", "XAHat", "RnA", "R", "t", "Coff", "sigma2", "gamma", "optimal_R", "optimal_t"]:
        a, b = getattr(ref, key), getattr(orc, key)
        if hasattr(a, "toarray"):  # sparse_calculation_mode returns scipy COO
            a, b = a.toarray(), b.toarray()
        a = np.asarray(a, dtype=np.float64)
        b = np.asarray(b, dtype=np.float64)
        d = np.abs(a - b).max() / max(np.abs(a).max(), 1e-30)
        worst = max(worst, d)
        print(f"  {key:12s} shape={a.shape} max-rel-dev={d:.3e}")
    print(f"[{name}] worst={worst:.3e}  P.shape={P_ref.shape}")
    return worst


if __name__ == "__main__":
    w = 0.0
    w = max(w, run_case("2d-full-f32", 400, 380, 40, 2, "float32", False, 120))
    w = max(w, run_case("2d-svi-f32", 1500, 1400, 40, 2, "float32", True, 120))
    w = max(w, run_case("3d-full-f64", 400, 420, 40, 3, "float64", False, 120, K=30, warp=2.0))
    w = max(w, run_case("3d-svi-f32-nonn", 1300, 1200, 30, 3, "float32", True, 100, nn_init=False))
    w = max(w, run_case("2d-full-f32-guide-both", 400, 380, 40, 2, "float32", False, 110, guide=True, guidance_effect="both", guidance_weight=2.0))
    w = max(w, run_case("2d-svi-f64-guide-nonrigid", 1300, 1250, 30, 2, "float64", True, 110, guide=True, guidance_effect="nonrigid"))
    w = max(w, run_case("3d-full-f32-guide-rigid", 380, 400, 30, 3, "float32", False, 100, guide=True, guidance_effect="rigid", nn_init=False))
    w = max(w, run_case("2d-full-f32-sparse64", 400, 380, 40, 2, "float32", False, 110, sparse_calculation_mode=True, sparse_top_k=64))
    w = max(w, run_case("3d-svi-f32-sparse32", 1300, 1200, 30, 3, "float32", True, 100, sparse_calculation_mode=True, sparse_top_k=32))
    print("WORST", w)
    sys.exit(0 if w == 0.0 else 1)
