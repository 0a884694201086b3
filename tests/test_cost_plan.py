"""CPU: resident / streamed choice of the expression cost matrix (``plan_cost``) and the per-chunk SVI schedules."""

import numpy as np
import pytest

GIB = 1 << 30


def _plan(n, cols, budget=80 * GIB, genes=2000):
    from spateo_release_b200.alignment.morpho_class import plan_cost

    return plan_cost(n, n, genes, cols, budget)


def test_benchmark_pair_stays_resident():
    for cols in (100000, 10000):  # full EM, default SVI batch
        p = _plan(100000, cols)
        assert not p.streamed and p.n_chunks == 1 and p.chunks == ((0, cols),)


def test_160k_pair_streams():
    svi = _plan(160000, 16000)
    assert svi.streamed and svi.chunks == ((0, 16000),) and svi.width == 16000
    full = _plan(160000, 160000)
    assert full.streamed and full.n_chunks >= 2


@pytest.mark.parametrize("n,cols,budget", [(160000, 160000, 80 * GIB), (200000, 200000, 40 * GIB), (160000, 16003, 12 * GIB),
                                           (30000, 30000, 3 * GIB), (5000, 1234, GIB + (300 << 20))])
def test_chunks_tile_the_columns_within_the_budget(n, cols, budget):
    from spateo_release_b200.alignment.distributed import pair_device_bytes

    p = _plan(n, cols, budget)
    assert p.streamed
    assert p.chunks[0][0] == 0 and p.chunks[-1][1] == cols
    assert all(a[1] == b[0] for a, b in zip(p.chunks, p.chunks[1:]))
    assert all((c1 - c0) % 8 == 0 for c0, c1 in p.chunks[:-1])
    assert all(0 < c1 - c0 <= p.width for c0, c1 in p.chunks)
    assert p.width % 8 == 0 or p.n_chunks == 1
    for c0, c1 in p.chunks:
        assert pair_device_bytes(n, n, 2000, chunk_cols=c1 - c0) <= budget
    assert p.need <= budget < pair_device_bytes(n, n, 2000)


def test_chunk_footprint_grows_with_the_width():
    from spateo_release_b200.alignment.distributed import pair_device_bytes

    sizes = [pair_device_bytes(160000, 160000, 2000, chunk_cols=c) for c in (8, 800, 8000, 80000)]
    assert sizes == sorted(sizes) and len(set(sizes)) == 4
    # the resident figure is unchanged by the new keyword
    assert pair_device_bytes(100000, 100000, 2000) == 4 * 100000 * 100352 + 12 * 200000 * 2016 + GIB


def test_budget_below_the_fixed_part_raises():
    with pytest.raises(MemoryError, match="bytes needed"):
        _plan(160000, 16000, budget=4 * GIB)


def test_chunk_schedules_concatenate_to_the_resident_schedule():
    from spateo_release_b200.alignment.morpho_class import svi_chunk_schedules, svi_schedule

    rng = np.random.default_rng(3)
    nb, nbb, max_iter = 1000, 312, 17
    perm = rng.permutation(nb)
    sched = svi_schedule(perm, max_iter, nbb)
    assert np.array_equal(sched[0], perm[:nbb]) and np.array_equal(sched[1], np.roll(perm, nbb)[:nbb])
    chunks = ((0, 104), (104, 208), (208, 312))
    parts = svi_chunk_schedules(sched, chunks)
    assert [q.shape for q in parts] == [(max_iter, 104)] * 3
    assert all(q.flags.c_contiguous and q.dtype == np.int32 for q in parts)
    assert np.array_equal(np.concatenate(parts, axis=1), sched)
