"""Expression-cost kernels against float64: the row pre-passes, the tensor-core contraction at its tile edges and at the
benchmark's gene count (G = 2,000, several tiles per CTA), the accumulate epilogue, the public cost matrix of a pair, and
the label layer with more fixed cells than a grid dimension of 65,535 blocks.

The float64 reference is ``oracle.morpho_oracle.calc_distance`` / ``calc_probability``. Where a bar is relative to fp32,
the same oracle fed float32 inputs (the reference's own fp32 path) gives the scale; both deviations are printed.
"""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from oracle import morpho_oracle as mo  # noqa: E402

# Max abs error on e allowed of the contraction, from the G = 2,000 pair of test_gene_cost_persistent_g2000 on an
# H100 80GB HBM3 (700 W power limit), with the fp32 reference's own error on the same data:
#   kl      kernel 2.26e-5, fp32 reference 3.27e-5; without the fixed-side centring 5.40e-5, without the log G
#           shift 2.34e-5 (so the shift is within fp32 noise at this G: its pre-pass is checked directly instead)
#   sym_kl  kernel 3.96e-5, fp32 reference 2.67e-5 (126 k-blocks)
#   cos     kernel 1.28e-5, fp32 reference 5.7e-7: positive terms only, so nothing cancels the rounding of the tensor-core
#           fp32 accumulators over 2,000 features
# These are not fp32-accurate dot products: the KL bar separates the centred kernel from the uncentred one, no more.
E_BAR = {"kl": 3e-5, "sym_kl": 5e-5, "cos": 2e-5}
# euc / square_euc: this many times the fp32 reference's own max error, or 8 ulp of the largest distance
FP32_RATIO = 4.0
# __expf on the Gaussian probability, relative
EXP_RTOL = 2e-6
KL_BAR = E_BAR["kl"]
TM, TN = 128, 256  # the contraction's tile: fixed cells x moving cells


def _lib():
    from spateo_release_b200 import _capi

    return _capi.load_library()


def _dev():
    import torch

    return torch.device("cuda", 0)


def _gc():
    from spateo_release_b200.alignment.morpho_class import GeneCostBuilder

    return GeneCostBuilder(_lib(), _dev())


def _round_up(x, m):
    return (x + m - 1) // m * m


def _t(a):
    import torch

    return torch.from_numpy(np.ascontiguousarray(a)).to(_dev())


def _stream():
    from spateo_release_b200 import _capi

    return _capi.current_stream_ptr()


def _oracle(XA, XB, metric):
    """(float64 e, fp32-reference e) of moving rows XA against fixed rows XB, both [NA, NB]."""
    [e64] = mo.calc_distance(XA.astype(np.float64), XB.astype(np.float64), metric)
    [e32] = mo.calc_distance(XA.astype(np.float32), XB.astype(np.float32), metric)
    return e64, e32.astype(np.float64)


def _beta2_rule(e64):
    """The reference's Gaussian width: the 5 % quantile of every moving cell's nearest cost, over 5 (at least 0.01)."""
    mn = e64.min(1)
    return max(mn[np.argsort(mn)[int(e64.shape[0] * 0.05)]] / 5, 0.01)


def _cost(XA, XB, metric, prob, beta2, ldx, prefill=None):
    """GT of the pair through GeneCostBuilder, written into an [NB + 1][ldx] buffer pre-filled with NaN (or ``prefill``
    with ``accumulate``). Asserts the kernel wrote every cell of the first NB rows (pad columns exactly 0) and nothing of
    the extra row. Returns GT[:NB, :NA] transposed to [NA, NB]."""
    import torch

    NA, NB = XA.shape[0], XB.shape[0]
    gc = _gc()
    opA, rtA, opB, rtB, G = gc.prepare_pair(_t(XA), _t(XB), metric)
    GT = torch.full((NB + 1, ldx), float("nan"), dtype=torch.float32, device=_dev())
    if prefill is not None:
        GT[:NB] = _t(prefill)
    gc.cost(opA, rtA, opB, rtB, NA, NB, G, metric, prob, beta2, prefill is not None, GT, ldx)
    torch.cuda.synchronize()
    out = GT.cpu().numpy()
    assert np.isnan(out[NB]).all(), "the kernel wrote past row NB"
    assert not np.isnan(out[:NB]).any(), "cells of GT[:NB, :ldx] were not written"
    assert np.all(out[:NB, NA:] == 0.0), "pad columns NA..ldx must be exactly 0"
    return out[:NB, :NA].T.astype(np.float64)


def _check(got, e64, e32, metric, prob, beta2, what):
    """Kernel (``got``, [NA, NB]) against float64 at the bars above; prints both deviations."""
    if prob == "gauss":
        want = mo.calc_probability(e64, "gauss", beta2)
        ref = mo.calc_probability(e32.astype(np.float32), "gauss", np.float32(beta2))
        err, err32 = np.max(np.abs(got - want) / want), np.max(np.abs(ref - want) / want)
        bar = KL_BAR / (2 * beta2) + EXP_RTOL
        print(f"{what}: rel err of prob: kernel {err:.3e}, fp32 reference {err32:.3e} (bar {bar:.3e}, beta2 {beta2:.4f})")
    else:
        err, err32 = np.max(np.abs(got - e64)), np.max(np.abs(e32 - e64))
        if metric in E_BAR:
            bar = E_BAR[metric]
        else:
            bar = max(FP32_RATIO * err32, 8 * 2.0**-24 * max(1.0, np.abs(e64).max()))
        print(f"{what}: abs err of e: kernel {err:.3e}, fp32 reference {err32:.3e} (bar {bar:.3e})")
    assert err < bar, f"{what}: kernel {err:.3e} vs float64, bar {bar:.3e} (fp32 reference {err32:.3e})"


def _counts(rng, n, G):
    return rng.poisson(1.5, size=(n, G)).astype(np.float32)


# ---------------------------------------------------------------------------------------------------------------------
# (a) row pre-passes
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("G", [1, 33, 2000])
def test_kl_prepare_rows(G):
    """spb_kl_prepare_rows on a row pitch wider than G: the moving side (Xn and sum Xn (log Xn + log G)), the fixed side
    centred by a profile w (log Yn + log G - c_j and c_j) and uncentred (no row term), zero tail up to the pitch."""
    import torch

    from spateo_release_b200._capi import check, ptr

    lib, st = _lib(), _stream()
    rng = np.random.default_rng(G)
    NA, NB, ldin, Gp = 37, 53, G + 3, _round_up(G, 32)
    wide = {s: _counts(rng, n, ldin) for s, n in (("A", NA), ("B", NB))}
    XA, XB = wide["A"][:, :G], wide["B"][:, :G]
    dA, dB = _t(wide["A"]), _t(wide["B"])

    def run(d, n, fixed, centre, want_rt):
        out = torch.full((n, Gp), float("nan"), dtype=torch.float32, device=_dev())
        rt = torch.full((n,), float("nan"), dtype=torch.float32, device=_dev()) if want_rt else None
        check(lib.spb_kl_prepare_rows(ptr(d), n, G, ldin, ptr(out), Gp, ptr(rt), int(fixed), ptr(centre), st),
              "spb_kl_prepare_rows")
        torch.cuda.synchronize()
        o = out.cpu().numpy()
        assert np.all(o[:, G:] == 0.0), "tail G..Gp must be exactly 0"
        return o[:, :G].astype(np.float64), (rt.cpu().numpy().astype(np.float64) if want_rt else None)

    def norm(X):
        X = X.astype(np.float64) + 0.01
        return X / X.sum(1, keepdims=True)

    Xn, Yn = norm(XA), norm(XB)
    LX, LY = np.log(Xn + 1e-8) + np.log(G), np.log(Yn + 1e-8) + np.log(G)
    # moving side
    o, rt = run(dA, NA, False, None, True)
    assert np.max(np.abs(o - Xn) / Xn) < 2e-6
    assert np.max(np.abs(rt - (Xn * LX).sum(1))) < 2e-6
    # fixed side centred by the mean moving profile
    w = torch.from_numpy(Xn.mean(0).astype(np.float32)).to(_dev())
    c = LY @ w.cpu().numpy().astype(np.float64)
    o, rt = run(dB, NB, True, w, True)
    assert np.max(np.abs(rt - c)) < 2e-6
    assert np.max(np.abs(o - (LY - c[:, None]))) < 4e-6
    # fixed side, uncentred
    o, _ = run(dB, NB, True, None, False)
    assert np.max(np.abs(o - LY)) < 4e-6


@pytest.mark.parametrize("G", [1, 33, 2000])
def test_rows_normalize_and_sqnorm(G):
    """spb_rows_normalize (X / max(|X|, 1e-8): an all-zero row comes out zero, not NaN; zero tail) and spb_rows_sqnorm."""
    import torch

    from spateo_release_b200._capi import check, ptr

    lib, st = _lib(), _stream()
    rng = np.random.default_rng(7 + G)
    ldin, Gp = G + 5, _round_up(G, 32)
    for n in (41, 29):  # both sides of a pair: NA != NB
        X = rng.normal(size=(n, ldin)).astype(np.float32)
        X[3] = 0.0
        d = _t(X)
        out = torch.full((n, Gp), float("nan"), dtype=torch.float32, device=_dev())
        check(lib.spb_rows_normalize(ptr(d), n, G, ldin, ptr(out), Gp, st), "spb_rows_normalize")
        rt = torch.full((n,), float("nan"), dtype=torch.float32, device=_dev())
        check(lib.spb_rows_sqnorm(ptr(d), n, G, ldin, ptr(rt), st), "spb_rows_sqnorm")
        torch.cuda.synchronize()
        o, r = out.cpu().numpy(), rt.cpu().numpy().astype(np.float64)
        assert not np.isnan(o).any(), "rows_normalize produced NaN (the all-zero row)"
        assert np.all(o[3] == 0.0) and np.all(o[:, G:] == 0.0)
        x64 = X[:, :G].astype(np.float64)
        nrm = np.sqrt((x64**2).sum(1, keepdims=True))
        want = x64 / np.maximum(nrm, 1e-8)
        assert np.max(np.abs(o[:, :G] - want)) < 1e-6
        sq = (x64**2).sum(1)
        assert r[3] == 0.0
        assert np.max(np.abs(r - sq) / np.maximum(sq, 1e-30)) < 2e-6


def test_split_tf32_bitwise():
    """spb_split_tf32 bit for bit over more elements than one grid-stride pass: hi is x with its low 13 mantissa bits
    cleared, lo = x - hi exactly, for +-0, negatives, subnormals and values at and around a tf32 rounding boundary."""
    import torch

    from spateo_release_b200._capi import check, ptr

    rng = np.random.default_rng(3)
    base = np.array([1.0, 1.5, -2.75, 3.1e7, -7.2e-30], dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    edges = (base[:, None] | np.array([0x0FFF, 0x1000, 0x1001, 0x1FFF, 0x0001], dtype=np.uint32)[None, :]).ravel()
    special = np.concatenate([
        np.array([0.0, -0.0, 1e-45, -1e-45, 1.1754942e-38, -5.9e-39, 1.17549435e-38, 3.4e38, -3.4e38], np.float32),
        edges.view(np.float32),
    ])
    n = 1184 * 256 * 2 + 37  # the kernel runs 1,184 x 256 threads: this takes three strides
    x = (rng.normal(size=n) * np.exp(rng.uniform(-30, 30, size=n))).astype(np.float32)
    x[rng.choice(n, special.size, replace=False)] = special
    x[-special.size:] = special
    d = _t(x)
    hi, lo = torch.full_like(d, float("nan")), torch.full_like(d, float("nan"))
    check(_lib().spb_split_tf32(ptr(d), ptr(hi), ptr(lo), n, _stream()), "spb_split_tf32")
    torch.cuda.synchronize()
    h, l = hi.cpu().numpy(), lo.cpu().numpy()
    hb = h.view(np.uint32)
    assert np.all(hb & np.uint32(0x1FFF) == 0), "hi keeps bits a tf32 operand drops"
    assert np.array_equal(hb, x.view(np.uint32) & np.uint32(0xFFFFE000)), "hi is not x truncated to tf32"
    assert np.all(h.astype(np.float64) + l.astype(np.float64) == x.astype(np.float64)), "hi + lo != x"


# ---------------------------------------------------------------------------------------------------------------------
# (b) contraction edges: k-blocks (ring fill, no wrap, one wrap), partial tiles, the second warpgroup out of range, pitches
# ---------------------------------------------------------------------------------------------------------------------
EDGE_CASES = [  # G, NB, NA, ldx rounding, metric, probability
    (1, 1, 1, 4, "euc", "prob"),
    (1, 63, 256, 512, "euc", "prob"),
    (32, 63, 255, 512, "kl", "prob"),
    (33, 64, 256, 4, "cos", "prob"),
    (64, 65, 257, 512, "kl", "gauss"),
    (65, 129, 257, 4, "kl", "prob"),
    (96, 1, 1, 512, "cos", "prob"),
    (96, 129, 255, 4, "kl", "gauss"),
]


@pytest.mark.parametrize("G,NB,NA,rnd,metric,prob", EDGE_CASES)
def test_gene_cost_tile_edges(G, NB, NA, rnd, metric, prob):
    """Every cell of GT[:NB, :ldx] written once (no NaN left, pad columns exactly 0), the row past NB untouched, values
    within the bars of the G = 2,000 test. NB % 128 < 64 leaves the second warpgroup without rows; ldx = roundup(NA, 4)
    cuts the last moving tile (the i >= ldx guard)."""
    rng = np.random.default_rng(G * 1000 + NB + NA)
    if metric == "kl":
        XA, XB = _counts(rng, NA, G), _counts(rng, NB, G)
    else:
        XA, XB = rng.normal(size=(NA, G)).astype(np.float32), rng.normal(size=(NB, G)).astype(np.float32)
    e64, e32 = _oracle(XA, XB, metric)
    beta2 = 0.05 if prob == "gauss" else None
    got = _cost(XA, XB, metric, prob, beta2, _round_up(NA, rnd))
    _check(got, e64, e32, metric, prob, beta2, f"G={G} NB={NB} NA={NA} ldx={_round_up(NA, rnd)} {metric}/{prob}")


# ---------------------------------------------------------------------------------------------------------------------
# (c) persistent tiles at the benchmark's gene count
# ---------------------------------------------------------------------------------------------------------------------
BIG_NA, BIG_NB, BIG_G = 4100, 2600, 2000


@pytest.fixture(scope="module")
def big_pair():
    """The benchmark's generative model at G = 2,000, with the float64 and fp32-reference costs of every metric."""
    from spateo_release_b200.synthetic import make_slice_pair

    (_, XA), (_, XB) = make_slice_pair(BIG_NA, BIG_NB, BIG_G, dim=3, z_thickness=20.0, as_anndata=False)
    cache = {}

    def oracle(metric):
        if metric not in cache:
            cache[metric] = _oracle(XA, XB, metric)
        return cache[metric]

    return XA, XB, oracle


@pytest.mark.parametrize("ldx", [BIG_NA, _round_up(BIG_NA, 512)])
@pytest.mark.parametrize("metric,prob", [("kl", "prob"), ("kl", "gauss"), ("sym_kl", "prob"), ("cos", "prob"),
                                         ("euc", "prob")])
def test_gene_cost_persistent_g2000(big_pair, metric, prob, ldx):
    """4100 x 2600 cells at G = 2,000: 63 k-blocks (an odd count: each CTA's next tile starts on the other ring stage
    and parity; sym_kl has 126), 21 fixed-cell tile rows (a partial band of 5 after 16, NB % 128 = 40), a last moving
    tile 4 columns wide at ldx = 4100, and more tiles than SMs, so every CTA runs several."""
    import torch

    XA, XB, oracle = big_pair
    tiles = (-(-ldx // TN)) * (-(-BIG_NB // TM))
    assert tiles > torch.cuda.get_device_properties(0).multi_processor_count, "every CTA must run several tiles"
    e64, e32 = oracle(metric)
    beta2 = _beta2_rule(e64) if prob == "gauss" else None
    got = _cost(XA, XB, metric, prob, beta2, ldx)
    _check(got, e64, e32, metric, prob, beta2, f"G=2000 ldx={ldx} {metric}/{prob}")


# ---------------------------------------------------------------------------------------------------------------------
# (d) accumulate
# ---------------------------------------------------------------------------------------------------------------------
def test_gene_cost_accumulate_g2000(big_pair):
    """accumulate = 1 multiplies into GT: Q * prob, bit for bit the fp32 product of Q with the written matrix, and within
    the KL bar of float64; pad columns (pre-filled with Q too) come out 0."""
    XA, XB, oracle = big_pair
    ldx = _round_up(BIG_NA, 512)
    e64, e32 = oracle("kl")
    beta2 = _beta2_rule(e64)
    Q = np.random.default_rng(11).uniform(0.5, 2.0, size=(BIG_NB, ldx)).astype(np.float32)
    plain = _cost(XA, XB, "kl", "gauss", beta2, ldx)
    got = _cost(XA, XB, "kl", "gauss", beta2, ldx, prefill=Q)
    QT = Q[:, :BIG_NA].T
    assert np.array_equal(got.astype(np.float32), plain.astype(np.float32) * QT), "accumulate != Q * (written matrix)"
    _check(got / QT, e64, e32, "kl", "gauss", beta2, "G=2000 accumulate kl/gauss")


def test_label_cost_accumulate():
    """spb_label_cost writes LT[labA[i], labB[j]] and with accumulate = 1 multiplies it into GT, exactly; pad columns 0."""
    import torch

    from spateo_release_b200._capi import check, ptr

    rng = np.random.default_rng(5)
    NA, NB, ldx = BIG_NA, BIG_NB, _round_up(BIG_NA, 512)
    la, lb = rng.integers(0, 4, NA).astype(np.int32), rng.integers(0, 6, NB).astype(np.int32)
    LT = rng.uniform(0.1, 10.0, size=(4, 6)).astype(np.float32)
    Q = rng.uniform(0.5, 2.0, size=(NB, ldx)).astype(np.float32)
    want = LT[la][:, lb].T
    dla, dlb, dLT = _t(la), _t(lb), _t(LT)  # held until the kernel has run
    for acc in (0, 1):
        GT = _t(Q) if acc else torch.full((NB, ldx), float("nan"), dtype=torch.float32, device=_dev())
        check(_lib().spb_label_cost(ptr(dla), ptr(dlb), ptr(dLT), 6, NA, NB, acc, ptr(GT), ldx, _stream()),
              "spb_label_cost")
        torch.cuda.synchronize()
        got = GT.cpu().numpy()
        assert np.all(got[:, NA:] == 0.0)
        assert np.array_equal(got[:, :NA], want * Q[:, :NA] if acc else want)


# ---------------------------------------------------------------------------------------------------------------------
# (e) the public path at 2,000 genes
# ---------------------------------------------------------------------------------------------------------------------
def test_pair_cost_matrix_g2000():
    """Morpho_pairwise.prepare() at G = 2,000: the resident GT (moving cells in k-d processing order, pitch
    roundup(NA, 512), fixed side centred by centre_of, the tf32 split kept for the run) against float64
    exp(-KL / (2 beta^2)), and its beta^2 against the reference's rule on the same cells (no sub-sample below 20k)."""
    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(3000, 2800, BIG_G, dim=3, z_thickness=20.0, seed=1)
    m = st.align.Morpho_pairwise(A, B, device="0", nn_init=False, materialize_P=False, verbose=False)
    m.prepare()
    NA, NB = m.NA, m.NB
    assert m._perm is not None, "the moving cells must be processed in k-d order here"
    GT = m._GT[:NB, : m.ldx].cpu().numpy()
    assert np.all(GT[:, NA:] == 0.0)
    got = np.empty((NA, NB))
    got[m._perm] = GT[:, :NA].T
    e64, e32 = _oracle(m.exp_layers_A[0], m.exp_layers_B[0], "kl")
    beta2 = float(m.probability_parameters[0])
    want_beta2 = _beta2_rule(e64)
    print(f"G=2000 pair: beta2 {beta2:.6f}, reference rule in float64 {want_beta2:.6f}")
    assert abs(beta2 - want_beta2) < KL_BAR / 5 + 1e-7
    _check(got, e64, e32, "kl", "gauss", beta2, "G=2000 Morpho_pairwise GT kl/gauss")


# ---------------------------------------------------------------------------------------------------------------------
# (f) more fixed cells than a grid dimension of 65,535 blocks
# ---------------------------------------------------------------------------------------------------------------------
LABEL_ROWS = [0, 65534, 65535, 65536]


def test_label_cost_past_65535_fixed_cells():
    """spb_label_cost with NB = 70,000 fixed cells: every row, including those past 65,535, written (and with accumulate
    multiplied) exactly; the row past NB untouched."""
    import torch

    from spateo_release_b200._capi import check, ptr

    rng = np.random.default_rng(9)
    NA, NB, ldx = 1000, 70000, 1024
    la, lb = rng.integers(0, 3, NA).astype(np.int32), rng.integers(0, 5, NB).astype(np.int32)
    LT = rng.uniform(0.1, 10.0, size=(3, 5)).astype(np.float32)
    dla, dlb, dLT = _t(la), _t(lb), _t(LT)
    want = dLT[dla.long()][:, dlb.long()].T.contiguous()  # [NB][NA]
    Q = torch.rand((NB, ldx), dtype=torch.float32, device=_dev()) + 0.5
    for acc in (0, 1):
        GT = torch.full((NB + 1, ldx), float("nan"), dtype=torch.float32, device=_dev())
        if acc:
            GT[:NB] = Q
        check(_lib().spb_label_cost(ptr(dla), ptr(dlb), ptr(dLT), 5, NA, NB, acc, ptr(GT), ldx, _stream()),
              "spb_label_cost")
        torch.cuda.synchronize()
        exp = want * Q[:, :NA] if acc else want
        for j in LABEL_ROWS + [NB - 1]:
            row = LT[la, lb[j]] * (Q[j, :NA].cpu().numpy() if acc else 1.0)
            assert np.array_equal(GT[j, :NA].cpu().numpy(), row), f"row {j}"
        assert torch.equal(GT[:NB, :NA], exp), "rows of the label cost differ"
        assert bool((GT[:NB, NA:] == 0).all()), "pad columns must be 0"
        assert bool(torch.isnan(GT[NB]).all()), "the kernel wrote past row NB"


def test_pair_with_label_layer_past_65535_fixed_cells():
    """Morpho_pairwise.prepare() with a KL layer and a label layer (accumulated into the KL probabilities) against 70,000
    fixed cells: rows around 65,535 match the float64 product of the two layers."""
    import pandas as pd

    import spateo_release_b200 as st
    from spateo_release_b200.synthetic import make_slice_pair

    A, B = make_slice_pair(600, 70000, 24, dim=2, seed=4)
    for ad in (A, B):
        x = np.asarray(ad.obsm["spatial"])[:, 0]
        ad.obs["region"] = pd.Categorical(np.where(x < 30, "a", np.where(x < 60, "b", "c")), categories=["a", "b", "c"])
    m = st.align.Morpho_pairwise(A, B, rep_layer=["X", "region"], rep_field=["layer", "obs"],
                                 dissimilarity=["kl", "label"], probability_type=["gauss", "prob"], device="0",
                                 nn_init=False, materialize_P=False, verbose=False)
    m.prepare()
    assert not m.cost_plan.streamed
    NA, NB = m.NA, m.NB
    rows = np.array(LABEL_ROWS + [NB - 1] + list(np.random.default_rng(0).choice(NB, 20, replace=False)))
    GT = m._GT[rows.tolist(), :NA].cpu().numpy().astype(np.float64)
    got = np.empty((NA, rows.size))
    got[m._perm] = GT.T
    beta2 = float(m.probability_parameters[0])
    [e64] = mo.calc_distance(m.exp_layers_A[0].astype(np.float64), m.exp_layers_B[0][rows].astype(np.float64), "kl")
    lab = np.asarray(m.label_transfer, dtype=np.float64)[m.exp_layers_A[1]][:, m.exp_layers_B[1][rows]]
    want = mo.calc_probability(e64, "gauss", beta2) * lab
    err = np.max(np.abs(got - want) / want)
    bar = KL_BAR / (2 * beta2) + EXP_RTOL
    print(f"70k fixed cells, KL x label rows: rel err {err:.3e} (bar {bar:.3e})")
    assert err < bar
