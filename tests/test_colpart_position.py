"""CPU: sweep 1 stores a row block's partial column sums by position in the block's work list, and col_finalize finds
column j's partial from the list builder's per-word data (keep bits, spatially live bits, and the list positions of the
first live and first dead listed column of each 32-column word). This mirrors the builder's compaction (live columns
first, then the dead ones, each in column order) and checks the position formula against the list on random masks. It
checks the formula only: that the device list builder and col_finalize agree is checked on the GPU
(test_gpu_colpart_position.py)."""

import numpy as np
import pytest


def _popc(x: np.ndarray) -> np.ndarray:
    return np.array([bin(int(v)).count("1") for v in x], dtype=np.int64)


def _build(keep: np.ndarray, live: np.ndarray):
    """collist and the per-word (off_live, off_dead) of build_col_lists_kernel for one row block."""
    nb = keep.shape[0]
    cols = np.arange(nb)
    collist = np.concatenate([cols[live], cols[keep & ~live]])
    words = (nb + 31) // 32
    kbits = np.zeros(words, dtype=np.uint64)
    lbits = np.zeros(words, dtype=np.uint64)
    for j in cols[keep]:
        kbits[j // 32] |= np.uint64(1) << np.uint64(j % 32)
    for j in cols[live]:
        lbits[j // 32] |= np.uint64(1) << np.uint64(j % 32)
    n_live = _popc(lbits)
    n_dead = _popc(kbits & ~lbits)
    off_live = np.concatenate([[0], np.cumsum(n_live)[:-1]])
    off_dead = int(n_live.sum()) + np.concatenate([[0], np.cumsum(n_dead)[:-1]])
    return collist, kbits, lbits, off_live, off_dead


def _position(j: int, kbits, lbits, off_live, off_dead) -> int:
    """col_finalize_kernel's list position of a listed column j."""
    w, lane = j // 32, j % 32
    below = np.uint64((1 << lane) - 1)
    bits, lb = kbits[w], lbits[w]
    if (int(lb) >> lane) & 1:
        return int(off_live[w]) + bin(int(lb & below)).count("1")
    return int(off_dead[w]) + bin(int(bits & ~lb & below)).count("1")


@pytest.mark.parametrize("nb,p_keep,p_live,seed", [(1, 1.0, 1.0, 0), (37, 0.5, 0.3, 1), (1000, 0.2, 0.5, 2),
                                                    (4099, 0.9, 0.1, 3), (4096, 0.05, 0.9, 4), (777, 1.0, 0.0, 5)])
def test_list_position_formula_matches_the_list(nb, p_keep, p_live, seed):
    rng = np.random.default_rng(seed)
    keep = rng.random(nb) < p_keep
    live = keep & (rng.random(nb) < p_live)  # a spatially live column is always listed
    collist, kbits, lbits, off_live, off_dead = _build(keep, live)
    assert collist.shape[0] == int(keep.sum())
    pos = [_position(j, kbits, lbits, off_live, off_dead) for j in np.flatnonzero(keep)]
    assert sorted(pos) == list(range(collist.shape[0]))  # every listed column has its own position
    for j, q in zip(np.flatnonzero(keep), pos):
        assert collist[q] == j
        assert (q < int(live.sum())) == bool(live[j])  # positions below colsplit are exactly the spatially live columns
