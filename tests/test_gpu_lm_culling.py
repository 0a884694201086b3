"""Culling with each quarter's row term: the E-step list builder drops a (128-row quarter, column) pair from the weights q
when c_q dmin^2 + max lm < -127 and from the spatial weights s when c_s dmin^2 < -127. On a late-iteration 20k x 20k
state, every pair it drops must have an fp32 ex2 argument below -126 (an exact +0 weight), it must read clearly fewer
cost-matrix bytes than the test without lm, and one E-step with culling on must give the column sums of one with culling
off bit for bit."""

import ctypes as C

import numpy as np
import pytest

from spateo_release_b200 import _capi  # noqa: E402

pytestmark = pytest.mark.gpu

from parity_helpers import device_pxb, device_rows, relmax  # noqa: E402


def _estep(m, it, cull):
    import torch

    m._params.cull = int(cull)
    m._estep_only(it, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    s = m._state
    return dict(
        colconst=s["colconst"][: m.NB].clone(), K_NB=s["K_NB"][: m.NB].clone(),
        K_NA=device_rows(m, "K_NA"), K_NA_spatial=device_rows(m, "K_NA_spatial"),
        K_NA_sigma2=device_rows(m, "K_NA_sigma2"), PXB=device_pxb(m), sums=list(m._read_scalars().sums),
    )


def test_lm_culling_drops_only_exact_zeros_and_keeps_column_sums_bit_identical():
    import torch

    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(20000, 20000, 64, dim=3, seed=7, z_thickness=20.0)
    np.random.seed(0)
    m = st.align.Morpho_pairwise(B, A, device="0", verbose=False, SVI_mode=False, max_iter=200, K=15, nn_init=False,
                                 materialize_P=False)
    m.prepare()
    it = 130
    m.run_em(n_iter=it)
    assert float(m._read_scalars().sigma2) < 9e-3, "expected a late-iteration state"

    on = _estep(m, it, True)
    s, NA, NB = m._state, m.NA, m.NB
    sc = m._read_scalars()
    cq, cs = float(sc.c_q), float(sc.c_s)
    nrb = m.ldx // _capi.ROW_TILE
    count = s["colcount"].cpu()
    collist, qbits, sbits = s["collist"], s["colquarters"].long(), s["colspatial"].long()
    bbox = s["bbox"].double()                                   # [nrb][4][8]
    X = s["XAHat"][:3].double()                                 # [3][ldx]
    lm = s["lm"].double()
    Y = s["colgeom"][:NB, 0:6:2].double()                       # [NB][3]
    assert int(qbits.max()) <= 0xF and int(sbits.max()) <= 0xF

    worst_q = worst_s = -np.inf
    read = blind = 0
    for rb in range(nrb):
        n = int(count[rb])
        cols = collist[rb, :n].long()
        # per quarter and column: the masks the builder wrote; unlisted columns have both bits clear
        qm = torch.zeros((4, NB), dtype=torch.bool, device=X.device)
        sm = torch.zeros((4, NB), dtype=torch.bool, device=X.device)
        for q in range(4):
            qm[q, cols] = ((qbits[rb, :n] >> q) & 1).bool()
            sm[q, cols] = ((sbits[rb, :n] >> q) & 1).bool()
        read += int(qm.sum())
        # the lm-blind test of the previous builder: c_q dmin^2 >= -127 against each quarter's box
        lo, hi = bbox[rb, :, 0:3], bbox[rb, :, 3:6]             # [4][3]
        gap = torch.clamp(torch.maximum(lo[:, None, :] - Y[None], Y[None] - hi[:, None, :]), min=0.0)
        d2q = (gap * gap).sum(-1)                               # [4][NB]
        blind += int((cq * (1.0 - 1e-5) * d2q >= -127.0).sum())
        for q in range(4):
            r0 = rb * _capi.ROW_TILE + q * 128
            r1 = min(r0 + 128, NA)
            if r1 <= r0:
                assert not bool(qm[q].any()) and not bool(sm[q].any())
                continue
            d = ((X[:, r0:r1, None] - Y.T[:, None, :]) ** 2).sum(0)   # [rows][NB]
            if bool((~qm[q]).any()):
                arg = cq * d[:, ~qm[q]] + lm[r0:r1, None]
                worst_q = max(worst_q, float(arg.max()))
            if bool((~sm[q]).any()):
                worst_s = max(worst_s, float((cs * d[:, ~sm[q]]).max()))
    visited = float(sc.visited)
    print(f"\n[20k it{it}] largest dropped ex2 argument: q {worst_q:.2f}  s {worst_s:.2f};  quarters read "
          f"{read / (4 * nrb * NB):.3f} of all, {read / blind:.3f} of the lm-blind test")
    assert worst_q < -126.0 and worst_s < -126.0
    assert visited == read / 4.0
    assert read <= 0.95 * blind, (read, blind)

    off = _estep(m, it, False)
    assert torch.equal(on["colconst"], off["colconst"])
    assert torch.equal(on["K_NB"], off["K_NB"])
    for k in ("K_NA", "K_NA_spatial", "K_NA_sigma2", "PXB"):
        assert relmax(on[k], off[k]) < 1e-5, k
    for a, b in zip(on["sums"], off["sums"]):
        assert abs(a - b) <= 1e-6 * abs(b)
