"""Processing order of the moving cells (``kd_order``): a permutation into compact 512-row blocks of compact 128-row
quarters, which is what makes the exact zero-tile culling of the E-step sweeps effective.

The visited fractions are counted on the host the way ``build_col_lists_kernel`` decides them: a (rows, column) tile is
read when the column lies within the culling radius of the bounding box of those rows."""

import numpy as np

from spateo_release_b200.alignment.morpho_class import kd_order


def _morton_order(c):
    """Z-order curve over an isotropic 10-bit grid (the row order the k-d split replaces), for comparison."""
    n, D = c.shape
    lo = c.min(axis=0)
    ext = float((c.max(axis=0) - lo).max())
    q = np.minimum(((c - lo) / ext * 1023).astype(np.uint64), np.uint64(1023))
    code = np.zeros(n, dtype=np.uint64)
    for b in range(10):
        for d in range(D):
            code |= ((q[:, d] >> np.uint64(b)) & np.uint64(1)) << np.uint64(b * D + d)
    return np.argsort(code, kind="stable")


def _visited_fraction(A, B, rows, r):
    """Fraction of the (moving, fixed) pairs read when every group of ``rows`` consecutive moving cells reads exactly the
    fixed cells within distance r of the group's bounding box."""
    tot = 0
    for k in range(0, A.shape[0], rows):
        blk = A[k:k + rows]
        g = np.maximum(np.maximum(blk.min(axis=0) - B, B - blk.max(axis=0)), 0.0)
        tot += np.count_nonzero((g * g).sum(axis=1) <= r * r) * blk.shape[0]
    return tot / (A.shape[0] * B.shape[0])


def _slab(n, seed=0):
    """Fixed cells uniform in a 100 x 100 x 20 slab, moving cells = fixed cells + N(0, 0.3) (an aligned pair)."""
    rng = np.random.default_rng(seed)
    B = rng.random((n, 3)) * np.array([100.0, 100.0, 20.0])
    return B + rng.normal(0.0, 0.3, (n, 3)), B


def test_kd_order_is_a_permutation_of_whole_blocks():
    A, _ = _slab(10_000 + 77)
    o = kd_order(A, 512, 128)
    assert o.shape == (A.shape[0],)
    assert np.array_equal(np.sort(o), np.arange(A.shape[0]))
    assert np.array_equal(o, kd_order(A.copy(), 512, 128))  # deterministic
    # a 512-row block is the union of its four 128-row quarters and is at least as compact as any Morton block of 512
    ext = lambda P: (P.max(axis=0) - P.min(axis=0)).prod()
    kd_vol = np.median([ext(A[o[k:k + 512]]) for k in range(0, A.shape[0] - 511, 512)])
    m = _morton_order(A)
    mo_vol = np.median([ext(A[m[k:k + 512]]) for k in range(0, A.shape[0] - 511, 512)])
    assert kd_vol < mo_vol


def test_kd_order_in_2d():
    rng = np.random.default_rng(3)
    A = rng.random((3000, 2)) * np.array([50.0, 10.0])
    o = kd_order(A, 512, 128)
    assert np.array_equal(np.sort(o), np.arange(3000))
    # 3000 = 5 whole blocks + 440 rows: each whole block spans about a sixth of the long axis
    spans = [np.ptp(A[o[k:k + 512], 0]) for k in range(0, 2560, 512)]
    assert max(spans) < 50.0 / 3


def test_kd_quarters_cut_visited_pairs_on_the_bench_slab():
    """The bench geometry (100k cells): culling radius 55 (sigma2 on its early floor) and 17.3 (late floor)."""
    A, B = _slab(100_000)
    kd, mort = A[kd_order(A, 512, 128)], A[_morton_order(A)]
    for r, bound in ((17.3, 0.6), (55.0, 0.9)):
        f_kd = _visited_fraction(kd, B, 128, r)
        f_mo = _visited_fraction(mort, B, 512, r)
        print(f"\nr={r}: visited k-d/128 {f_kd:.3f}  Morton/512 {f_mo:.3f}  ratio {f_kd / f_mo:.3f}")
        assert f_kd <= bound * f_mo, (r, f_kd, f_mo)
