"""Sweep 1 stores each row block's partial column sums by position in the block's work list (one aligned 32-byte sector per
stage and sum) and leaves the two spatial sums of spatially dead columns unwritten; col_finalize turns column j into its
list position from the builder's keep bits, live bits and per-word offsets. On a late-iteration 20k x 20k state, where
culling has shortened the lists and split them into live and dead groups, the device position data must reproduce every
work list, and the column constants and K_NB of one E-step must equal, bit for bit, a fold written here from the partials
scattered back to their columns in the kernel's order (per warp over row blocks w, w + 8, ..., then over the 8 warps)."""

import ctypes as C

import numpy as np
import pytest

from spateo_release_b200 import _capi  # noqa: E402

pytestmark = pytest.mark.gpu


def _bits(words: np.ndarray) -> np.ndarray:
    """[..., nwords] uint32 -> [..., nwords * 32] bool, column 32 w + l = bit l of word w."""
    b = (words[..., None] >> np.arange(32, dtype=np.uint32)) & np.uint32(1)
    return b.reshape(*words.shape[:-1], -1).astype(bool)


@pytest.mark.parametrize("dim,svi", [(3, False), (3, True), (2, False)])
def test_partials_by_list_position_fold_bit_identically(dim, svi):
    """Full EM in 3-D and 2-D, and the default SVI batch (whose lists are built from the gathered batch coordinates)."""
    import torch

    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    kw = dict(z_thickness=20.0) if dim == 3 else {}
    A, B = make_slice_pair(20000, 20000, 64, dim=dim, seed=7, **kw)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(B, A, device="0", verbose=False, SVI_mode=svi, max_iter=200, K=15, nn_init=False,
                                 materialize_P=False)
    m.prepare()
    it = 130
    m.run_em(n_iter=it)
    m._estep_only(it, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    s, NB = m._state, m._NBb  # columns of this E-step: all fixed cells, or the SVI batch
    nrb = m.ldx // _capi.ROW_TILE
    count = s["colcount"].cpu().numpy().astype(np.int64)
    split = s["colsplit"].cpu().numpy().astype(np.int64)
    collist = s["collist"].cpu().numpy().astype(np.int64)
    part = s["colpart"].cpu().numpy()                           # [nrb][4][nbb_pad], by list position
    keep = _bits(s["keepmask"].cpu().numpy().view(np.uint32))[:, :NB]
    live = _bits(s["livemask"].cpu().numpy().view(np.uint32))[:, :NB]
    off = s["keepoff"].cpu().numpy().astype(np.int64)           # [nrb][nwords][2]
    assert bool((split < count).any()) and bool((split > 0).any()), "expected spatially live and dead list groups"
    assert bool((count < NB).any()), "expected culled lists"

    # position of every listed column: its group's offset in its word + the listed columns of the group below it
    dead = keep & ~live
    nw = off.shape[1]
    pad = nw * 32 - NB
    excl = lambda b: (np.cumsum(np.pad(b, ((0, 0), (0, pad))).reshape(nrb, nw, 32), axis=2) -
                      np.pad(b, ((0, 0), (0, pad))).reshape(nrb, nw, 32)).reshape(nrb, -1)[:, :NB]
    word = np.arange(NB) // 32
    pos = np.where(live, off[:, word, 0] + excl(live), off[:, word, 1] + excl(dead))
    scat = np.zeros((nrb, 4, NB), dtype=np.float32)             # the partials as a column-indexed store would hold them
    for rb in range(nrb):
        n, sp = int(count[rb]), int(split[rb])
        cols = np.flatnonzero(keep[rb])
        assert cols.shape[0] == n and np.array_equal(np.sort(collist[rb, :n]), cols)
        assert np.array_equal(collist[rb, pos[rb, cols]], cols)
        assert np.array_equal(pos[rb, cols] < sp, live[rb, cols])
        lst = collist[rb, :n]
        scat[rb, 2:, lst] = part[rb, 2:, :n].T
        scat[rb, :2, lst[:sp]] = part[rb, :2, :sp].T

    Cw = np.zeros((8, 4, NB))
    for rb in range(nrb):
        Cw[rb % 8] += scat[rb].astype(np.float64)
    Cs = np.zeros((4, NB))
    for w in range(8):
        Cs += Cw[w]
    omega = float(m._read_scalars().omega)
    inl = 1.0 - omega / (omega + Cs[0])
    a = 1.0 / (omega + Cs[1])
    b = inl / (Cs[2] + 1e-8)
    c = inl / (Cs[3] + 1e-8)
    cc = s["colconst"][:NB].cpu().numpy()
    assert np.array_equal(cc[:, 6], a.astype(np.float32))
    assert np.array_equal(cc[:, 8], b.astype(np.float32))
    assert np.array_equal(cc[:, 10], c.astype(np.float32))
    assert np.array_equal(s["K_NB"][:NB].cpu().numpy(), (c * Cs[3]).astype(np.float32))
