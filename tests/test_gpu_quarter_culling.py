"""Quarter-level culling of the E-step sweeps: inside a listed (row block, column) tile, each 128-row quarter whose bounding
box is out of reach of the column is neither read nor computed. On a late-iteration 20k x 20k state this must read
clearly fewer bytes than whole tiles would, and one E-step must still meet the chunked float64 oracle bars."""

import ctypes as C

import numpy as np
import pytest

from spateo_release_b200 import _capi  # noqa: E402

pytestmark = pytest.mark.gpu

from oracle import morpho_oracle as mo  # noqa: E402
from parity_helpers import device_pxb, device_rows, poke_estep_state, relmax  # noqa: E402


def test_quarter_culling_reads_less_and_matches_chunked_float64_oracle():
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
    NA, D = m.NA, m.D
    XAHat32 = m._unsorted(m._state["XAHat"][:D, :NA].T.contiguous().cpu().numpy())
    alpha32, SD32 = device_rows(m, "alpha"), device_rows(m, "SigmaDiag")
    sc = m._read_scalars()
    sigma2, gamma, var = float(sc.sigma2), float(sc.gamma), float(sc.sigma2_variance)
    assert sigma2 < 9e-3, f"expected a late-iteration sigma2 below the 1e-2 early floor, got {sigma2}"
    alpha, SD = alpha32.astype(np.float64), SD32.astype(np.float64)
    want = mo.estep_column_chunks(
        Dim=float(D), XAHat=XAHat32.astype(np.float64), YB=m.coordsB.astype(np.float64),
        exp_A=[m.exp_layers_A[0].astype(np.float64)], exp_B=[m.exp_layers_B[0].astype(np.float64)], metric=["kl"],
        sigma2=sigma2, model_mul=(alpha * np.exp(-SD / sigma2))[:, None], gamma=gamma, samples_s=float(m.samples_s),
        sigma2_variance=var, probability_type=["gauss"], probability_parameters=[float(m.probability_parameters[0])],
        chunk=1000,
    )
    poke_estep_state(m, XAHat32, alpha32, SD32, sigma2, gamma, var)
    m._params.cull = 1
    m._estep_only(it, C.c_void_p(torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()

    nrb = m.ldx // _capi.ROW_TILE
    count = m._state["colcount"].cpu().numpy()
    quarters = m._state["colquarters"].cpu().numpy()
    live = sum(int(np.unpackbits(quarters[rb, : count[rb]]).sum()) for rb in range(nrb))
    assert all(int(quarters[rb, : count[rb]].max(initial=0)) <= 0xF for rb in range(nrb))
    visited = float(m._read_scalars().visited)
    assert visited == live / 4.0  # the trace counts live quarters, in whole tiles
    tiles = float(count.sum())
    print(f"\n[20k it{it}] sigma2 {sigma2:.4g}  listed tiles {tiles / (nrb * m.NB):.3f}  read {visited / (nrb * m.NB):.3f}")
    assert visited < 0.9 * tiles, (visited, tiles)

    errs = dict(
        K_NA=relmax(device_rows(m, "K_NA"), want["K_NA"]),
        K_NB=relmax(m._state["K_NB"][: m.NB].cpu().numpy(), want["K_NB"]),
        K_NA_spatial=relmax(device_rows(m, "K_NA_spatial"), want["K_NA_spatial"]),
        K_NA_sigma2=relmax(device_rows(m, "K_NA_sigma2"), want["K_NA_sigma2"]),
        PXB=relmax(device_pxb(m), want["PXB"]),
    )
    s = m._read_scalars()
    errs["Sp"] = abs(s.sums[2] - want["Sp"]) / want["Sp"]
    errs["sigma2_related"] = abs(s.sums[3] - want["sigma2_related_num"]) / abs(want["sigma2_related_num"])
    print("  ".join(f"{k} {v:.2e}" for k, v in errs.items()))
    for k, v in errs.items():
        assert v < 1e-4, (k, v)
