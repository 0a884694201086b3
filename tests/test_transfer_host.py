"""Host side of the posterior transfer: resolving keys and one-hot labels, the validation errors, the panel and footprint
arithmetic (no GPU needed)."""

import numpy as np
import pandas as pd
import pytest

from spateo_release_b200 import _capi
from spateo_release_b200.alignment.distributed import pair_device_bytes, transfer_device_bytes
from spateo_release_b200.alignment.morpho_alignment import _normalise_rows, _transfer_keys
from spateo_release_b200.alignment.morpho_class import Morpho_pairwise, plan_cost, resolve_transfer
from spateo_release_b200.anndata_lite import AnnDataLite


def _slice(n=6):
    rng = np.random.default_rng(0)
    obs = pd.DataFrame({"ct": pd.Categorical(["b", "a", "c", "a", None, "b"][:n])}, index=[f"c{i}" for i in range(n)])
    return AnnDataLite(rng.random((n, 4)).astype(np.float32), obs=obs,
                       var=pd.DataFrame(index=[f"g{i}" for i in range(4)]),
                       obsm={"spatial": rng.random((n, 2)), "emb": rng.normal(size=(n, 3)),
                             "emb_df": pd.DataFrame(rng.normal(size=(n, 2)))})


def test_obs_key_is_one_hot_in_category_order():
    F, cats = resolve_transfer(_slice(), "ct", 6, "transfer_B")
    assert cats == ["a", "b", "c"]
    assert F.dtype == np.float32 and F.shape == (6, 3)
    assert np.array_equal(F.argmax(axis=1)[[0, 1, 2, 3, 5]], [1, 0, 2, 0, 1])
    assert np.array_equal(F.sum(axis=1), [1, 1, 1, 1, 0, 1])  # a missing label is an all-zero row


def test_obsm_key_and_array():
    sl = _slice()
    F, cats = resolve_transfer(sl, "emb", 6, "transfer_A")
    assert cats is None and np.array_equal(F, sl.obsm["emb"].astype(np.float32))
    F, _ = resolve_transfer(sl, "emb_df", 6, "transfer_A")
    assert F.shape == (6, 2)
    F, _ = resolve_transfer(sl, np.arange(12, dtype=np.int64).reshape(6, 2), 6, "transfer_A")
    assert F.dtype == np.float32 and F[5, 1] == 11


@pytest.mark.parametrize("spec,match", [
    ("nope", "neither"),
    (np.ones((5, 2)), "5 rows"),
    (np.ones((6, 0)), "F = 0"),
    (np.array([[1.0], [np.nan], [1], [1], [1], [1]]), "non-finite"),
    (np.array([[1.0], [np.inf], [1], [1], [1], [1]]), "non-finite"),
    (np.ones(6), "matrix"),
])
def test_validation_errors(spec, match):
    with pytest.raises(ValueError, match=match):
        resolve_transfer(_slice(), spec, 6, "transfer_B")


def test_constructor_validates_before_touching_the_device():
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(300, 280, 12, dim=2, seed=1)
    with pytest.raises(ValueError, match="return_mapping"):
        Morpho_pairwise(sampleA=A, sampleB=B, SVI_mode=True, transfer_B=np.ones((280, 2)), verbose=False)
    with pytest.raises(ValueError, match="rows"):
        Morpho_pairwise(sampleA=A, sampleB=B, SVI_mode=False, transfer_B=np.ones((300, 2)), verbose=False)
    with pytest.raises(ValueError, match="neither"):
        Morpho_pairwise(sampleA=A, sampleB=B, SVI_mode=False, transfer_A="missing", verbose=False)


def test_driver_keywords_are_keys_only_and_rows_normalise():
    assert _transfer_keys({"transfer_B": "ct"}) == ("ct", None)
    with pytest.raises(ValueError, match="ambiguous"):
        _transfer_keys({"transfer_A": np.ones((3, 1))})
    x = np.array([[1.0, 3.0], [0.0, 0.0], [2.0, 2.0]], np.float32)
    got = _normalise_rows(x, np.array([4.0, 0.0, 8.0], np.float32))
    assert np.array_equal(got, np.array([[0.25, 0.75], [0, 0], [0.25, 0.25]], np.float32))


def test_pair_device_bytes_without_transfer_is_unchanged():
    # values of the formula before the transfer term existed
    assert pair_device_bytes(100000, 100000, 2000) == 46052941824
    assert pair_device_bytes(100000, 100000, 2000, chunk_cols=20000) == 14374275224
    assert pair_device_bytes(150000, 140000, 64, chunk_cols=4096, n_sms=132) == 3793855464
    assert pair_device_bytes(5000, 4000, 33) == 1162573824
    assert pair_device_bytes(5000, 4000, 33, transfer=None) == 1162573824


def test_transfer_footprint_and_panels():
    W = _capi.CONST["SPB_TRANSFER_PANEL"]
    assert W == 16
    n_moving, n_fixed, width = 100000, 100000, 100000
    ldx = -(-n_moving // 512) * 512
    nrb = ldx // 512
    seg = Morpho_pairwise._choose_segments(nrb, width, 132)
    # 32 labels on the fixed slice: two panels; 2000 genes on the moving slice: 125 panels
    want_B = 4 * (n_fixed + 1) * 32 + 8 * 32 * ldx + 4 * seg * W * ldx
    assert transfer_device_bytes(n_moving, n_fixed, (32, 0), width) == want_B
    pad = width + 8
    want_A = 4 * 2000 * ldx + 4 * nrb * W * pad + 4 * n_fixed * 2000
    assert transfer_device_bytes(n_moving, n_fixed, (0, 2000), width) == want_A
    assert transfer_device_bytes(n_moving, n_fixed, (17, 0), width) == transfer_device_bytes(n_moving, n_fixed, (32, 0), width)
    base = pair_device_bytes(n_moving, n_fixed, 2000)
    assert pair_device_bytes(n_moving, n_fixed, 2000, transfer=(32, 2000)) == base + want_A + want_B


def test_plan_picks_a_narrower_chunk_that_still_fits_with_the_transfer():
    n_moving, n_fixed, genes = 150000, 140000, 64
    budget = pair_device_bytes(n_moving, n_fixed, genes, chunk_cols=40000)
    plain = plan_cost(n_moving, n_fixed, genes, n_fixed, budget)
    xfer = plan_cost(n_moving, n_fixed, genes, n_fixed, budget, transfer=(32, 2000))
    assert plain.streamed and xfer.streamed
    assert pair_device_bytes(n_moving, n_fixed, genes, chunk_cols=plain.width, transfer=(32, 2000)) > budget
    assert xfer.width < plain.width
    assert xfer.need <= budget
    assert pair_device_bytes(n_moving, n_fixed, genes, chunk_cols=xfer.width, transfer=(32, 2000)) == xfer.need
