"""TEST INFRASTRUCTURE ONLY — CPU (numpy) restatement of Spateo's pairwise morpho-alignment EM.

This module is the *oracle*: it restates, on plain numpy arrays, the arithmetic the reference executes on its
NumpyBackend CPU path. It is NOT part of the product: only ``tests/``, ``__graft_entry__.smoke()`` and the
``cpu_baseline`` / ``--impl reference`` legs of ``bench.py`` may import it, and only as the checker / the timed CPU
baseline. The product path (``spateo_release_b200``) never imports it and has no CPU fallback.

Parity status: PINNED. ``tests/test_oracle_golden.py`` checks every function below against golden vectors produced by
executing the unmodified reference (``tests/golden/make_golden.py`` via ``oracle/ref_harness.py``) — per-call
(``calc_distance``, ``get_P_core``, ``con_K``, ``inlier_from_NN``, ``voxel_data``) and end-to-end
(``MorphoPairOracle.run`` vs ``Morpho_pairwise.run``: 2-D/3-D, SVI/full, float32/float64).
Exception: ``sparse_vfc`` restates third-party ``dynamo-release>=1.4.1`` (``scVectorField.SparseVFC``), which is not in
the reference tree and not installed: **parity unpinned** for that function (see its docstring).

All ``file:line`` citations are relative to the spateo-release tree.
"""

from __future__ import annotations

import numpy as np
from scipy.linalg import pinv as _scipy_pinv
from scipy.special import psi as _psi

# ---------------------------------------------------------------------------------------------------------------------
# Expression / spatial dissimilarities            spateo/alignment/methods/utils.py:647-941
# ---------------------------------------------------------------------------------------------------------------------


def kl_distance(X, Y, eps=1e-8):
    """Pairwise KL(X_i || Y_j) with +0.01 pseudo-count and row normalisation (utils.py:679-699)."""
    Xp = X + 0.01
    Yp = Y + 0.01
    Xp = Xp / Xp.sum(axis=1, keepdims=True)
    Yp = Yp / Yp.sum(axis=1, keepdims=True)
    logX = np.log(Xp + eps)
    logY = np.log(Yp + eps)
    self_term = (Xp * logX).sum(axis=1, keepdims=True)
    return self_term - np.dot(Xp, logY.T)


def euc_distance(X, Y, squared=True):
    """|x|^2 + |y|^2 - 2 x.y clamped at 0; sqrt when ``squared`` is False (utils.py:775-788)."""
    D = np.sum(X**2, 1)[:, None] + np.sum(Y**2, 1)[None, :] - 2 * np.dot(X, Y.T)
    D = np.maximum(D, 0.0)
    return D if squared else np.sqrt(D)


def cosine_distance(X, Y, eps=1e-8):
    """0.5 - 0.5 * cos(x, y) (utils.py:730-744)."""
    Xn = X / np.maximum(np.sqrt((X**2).sum(1, keepdims=True)), eps)
    Yn = Y / np.maximum(np.sqrt((Y**2).sum(1, keepdims=True)), eps)
    return -np.dot(Xn, Yn.T) * 0.5 + 0.5


def label_distance(X, Y, label_transfer):
    """Gather label_transfer[X_i, Y_j] (utils.py:818-832)."""
    return label_transfer[X, :][:, Y]


def calc_distance(X, Y, metric="euc", label_transfer=None):
    """List-in/list-out dispatcher; NB "euc" is SQUARED and "square_euc" is the sqrt (utils.py:900-941)."""
    Xs = X if isinstance(X, list) else [X]
    Ys = Y if isinstance(Y, list) else [Y]
    ms = metric if isinstance(metric, list) else [metric]
    out = []
    for x, y, m in zip(Xs, Ys, ms):
        if m == "label":
            assert label_transfer is not None
            out.append(label_distance(x, y, label_transfer))
        elif m in ("euc", "euclidean"):
            out.append(euc_distance(x, y, squared=True))
        elif m in ("square_euc", "square_euclidean"):
            out.append(euc_distance(x, y, squared=False))
        elif m == "kl":
            out.append(kl_distance(x, y))
        elif m == "sym_kl":
            out.append((kl_distance(x, y) + kl_distance(y, x).T) / 2)
        elif m in ("cos", "cosine"):
            out.append(cosine_distance(x, y))
    return out


def calc_probability(dist, probability_type="gauss", probability_parameter=None):
    """gauss: exp(-d / (2 p)); cos: 1 - d; prob: d (utils.py:974-985)."""
    t = probability_type.lower()
    if t in ("gauss", "gaussian"):
        if probability_parameter is None:
            raise ValueError("probability_parameter must be provided for 'Gauss' probability type.")
        return np.exp(-dist / (2 * probability_parameter))
    if t in ("cos", "cosine"):
        return 1 - dist
    if t == "prob":
        return dist
    raise ValueError(f"Unsupported probability type: {probability_type}")


# ---------------------------------------------------------------------------------------------------------------------
# E-step core                                    spateo/alignment/methods/utils.py:993-1096
# ---------------------------------------------------------------------------------------------------------------------


def get_P_core(
    Dim,
    spatial_dist,
    exp_dist,
    sigma2,
    model_mul,
    gamma,
    samples_s,
    sigma2_variance=1,
    probability_type=("gauss",),
    probability_parameters=None,
    eps=1e-8,
    sparse_calculation_mode=False,
    top_k=-1,
):
    """Three column-normalised posteriors sharing one spatial distance block (utils.py:1049-1083).

    ``sparse_calculation_mode`` keeps the ``top_k`` largest entries of every column of the full posterior as a scipy COO
    matrix (utils.py:1085-1094 -> _dense_to_sparse, utils.py:1369-1404); the other two posteriors stay dense.

    Returns (P, K_NA_spatial, K_NA_sigma2, sigma2_related_numerator).
    """
    sp = calc_probability(spatial_dist, "gauss", sigma2 / sigma2_variance)
    outlier_s = samples_s * spatial_dist.shape[0]
    omega = np.power((2 * np.pi * sigma2), Dim / 2) * (1 - gamma) / (gamma * outlier_s)
    inlier = 1 - omega / (omega + sp.sum(axis=0, keepdims=True))
    sp = sp * model_mul
    P = sp / (omega + sp.sum(axis=0, keepdims=True))
    K_NA_spatial = P.sum(1)

    sp = calc_probability(spatial_dist, "gauss", sigma2)
    sp = sp * model_mul
    P = inlier * sp / (sp.sum(axis=0, keepdims=True) + eps)
    K_NA_sigma2 = P.sum(1)
    sigma2_related = (P * spatial_dist).sum()

    if probability_parameters is None:
        probability_parameters = [None] * len(exp_dist)
    for e_d, p_t, p_p in zip(exp_dist, probability_type, probability_parameters):
        sp *= calc_probability(e_d, p_t, p_p)
    P = inlier * sp / (sp.sum(axis=0, keepdims=True) + eps)
    if sparse_calculation_mode:
        P = dense_to_sparse_topk(P, top_k)
    return P, K_NA_spatial, K_NA_sigma2, sigma2_related


def estep_column_chunks(
    Dim, XAHat, YB, exp_A, exp_B, metric, sigma2, model_mul, gamma, samples_s, sigma2_variance, probability_type,
    probability_parameters, chunk=1000, label_transfer=None, keep_P=False,
):
    """One full E-step evaluated in COLUMN CHUNKS (for sizes whose N_A x N_B temporaries do not fit the host).

    Every normalisation inside ``get_P_core`` is a per-column sum over the moving cells (utils.py:1053-1083), so a block of
    columns is an independent sub-problem as long as ``outlier_s`` keeps the full N_A (it does: spatial_dist.shape[0]).
    Each chunk goes through the very same ``calc_distance`` / ``get_P_core`` as ``MorphoPairOracle._update_assignment_P``
    (morpho_class.py:1147-1176); row statistics are accumulated across chunks.

    Returns a dict with K_NA, K_NB, K_NA_spatial, K_NA_sigma2, PXB, sigma2_related_num, Sp (and P when ``keep_P``).
    """
    XAHat = np.asarray(XAHat)
    NA, NB = XAHat.shape[0], YB.shape[0]
    out = dict(
        K_NA=np.zeros(NA), K_NB=np.zeros(NB), K_NA_spatial=np.zeros(NA), K_NA_sigma2=np.zeros(NA),
        PXB=np.zeros((NA, YB.shape[1])), sigma2_related_num=0.0,
    )
    blocks = []
    for j0 in range(0, NB, chunk):
        j1 = min(NB, j0 + chunk)
        spatial = euc_distance(XAHat, YB[j0:j1], squared=True)
        ed = calc_distance(exp_A, [e[j0:j1] for e in exp_B], metric, label_transfer)
        P, kns, kn2, s2r = get_P_core(
            Dim=Dim, spatial_dist=spatial, exp_dist=ed, sigma2=sigma2, model_mul=model_mul, gamma=gamma,
            samples_s=samples_s, sigma2_variance=sigma2_variance, probability_type=probability_type,
            probability_parameters=probability_parameters,
        )
        out["K_NA"] += P.sum(1)
        out["K_NB"][j0:j1] = P.sum(0)
        out["K_NA_spatial"] += kns
        out["K_NA_sigma2"] += kn2
        out["PXB"] += P @ YB[j0:j1]
        out["sigma2_related_num"] += float(s2r)
        if keep_P:
            blocks.append(P)
    out["Sp"] = float(out["K_NA"].sum())
    if keep_P:
        out["P"] = np.concatenate(blocks, axis=1)
    return out


def dense_to_sparse_topk(mat, threshold):
    """utils.py:1369-1404 with sparse_method="topk", axis=0, descending=True (numpy backend: sort2 of the negated matrix,
    backend.py:1138-1142; COO assembly utils.py:1506-1510 with float column indices from ``nx.arange(type_as=mat)``)."""
    import scipy.sparse as sp

    NA, NB = mat.shape
    threshold = int(threshold)
    sorted_mat, sorted_idx = -np.sort(-mat, axis=0), np.argsort(-mat, axis=0)
    if threshold > NA:
        threshold = NA
    col = np.repeat(np.arange(NB).astype(mat.dtype), threshold, axis=0)
    row = sorted_idx[:threshold, :].T.reshape(-1)
    val = sorted_mat[:threshold, :].T.reshape(-1)
    return sp.coo_matrix((val, (row, col)), shape=(NA, NB))


def _dot(a, b):
    """NumpyBackend.dot (backend.py:1082-1091): scipy-sparse aware."""
    import scipy.sparse as sp

    if sp.issparse(a):
        return a.dot(b)
    if sp.issparse(b):
        return b.T.dot(a.T).T
    return np.dot(a, b)


def con_K(X, Y, beta=0.01):
    """Squared-exponential kernel exp(-beta |x-y|^2) through the expanded squared distance (utils.py:1149-1158)."""
    return np.exp(-beta * euc_distance(X, Y, squared=True))


# ---------------------------------------------------------------------------------------------------------------------
# Coarse rigid initialisation helpers            spateo/alignment/methods/utils.py:1220-1354
# ---------------------------------------------------------------------------------------------------------------------


def inlier_from_NN(train_x, train_y, distance):
    """100-iteration robust weighted Procrustes with annealed expression weight (utils.py:1225-1280)."""
    N, D = train_x.shape
    alpha = 1
    distance = np.maximum(0, distance)
    distance = distance / (np.max(distance) / (np.log(10) * 2))
    y_hat = train_x
    sigma2 = np.sum((y_hat - train_y) ** 2) / (D * N)
    weight = np.exp(-distance * alpha)
    init_weight = weight
    P = np.ones((N, 1)) * weight
    max_iter = 100
    alpha_decrease = np.power(0.1 / alpha, 1 / (max_iter - 20))
    gamma = 0.5
    a = np.maximum(
        np.prod(train_x.max(axis=0) - train_x.min(axis=0)),
        np.prod(train_y.max(axis=0) - train_y.min(axis=0)),
    )
    Sp = P.sum()
    R, t = np.eye(D), np.ones((D, 1))
    for it in range(max_iter):
        mu_x = (train_x * P).sum(0) / Sp
        mu_y = (train_y * P).sum(0) / Sp
        Xc, Yc = train_x - mu_x, train_y - mu_y
        A = Yc.T @ (Xc * P)
        U, _, Vh = np.linalg.svd(A)
        C = np.eye(D)
        C[-1, -1] = np.linalg.det(U @ Vh)
        R = U @ C @ Vh
        t = mu_y - mu_x @ R.T
        y_hat = train_x @ R.T + t
        term1 = np.exp(-np.sum((train_y - y_hat) ** 2, 1, keepdims=True) / (2 * sigma2)) * weight
        outlier = np.max(weight) * (1 - gamma) * np.power(2 * np.pi * sigma2, D / 2) / (gamma * a)
        P = term1 / (term1 + outlier)
        Sp = P.sum()
        gamma = np.minimum(np.maximum(Sp / N, 0.01), 0.99)
        P = np.maximum(P, 1e-6)
        sigma2 = np.sum((y_hat - train_y) ** 2 * P) / (D * Sp)
        if it > 20:
            alpha = alpha * alpha_decrease
            weight = np.exp(-distance * alpha)
            weight = weight / np.max(weight)
    fix_sigma2, fix_gamma = 1e-2, 0.1
    term1 = np.exp(-np.sum((train_y - y_hat) ** 2, 1, keepdims=True) / (2 * fix_sigma2)) * weight
    outlier = np.max(weight) * (1 - fix_gamma) * np.power(2 * np.pi * fix_sigma2, D / 2) / (fix_gamma * a)
    P = term1 / (term1 + outlier)
    gamma = np.minimum(np.maximum(P.sum() / N, 0.01), 0.99)
    return P, R, t, init_weight, sigma2, gamma


def voxel_data(coords, gene_exp, voxel_size=None, voxel_num=10000):
    """Radius-membership (overlapping) voxel averaging on an int(sqrt(voxel_num))-per-axis grid (utils.py:1310-1336)."""
    N, D = coords.shape
    lo, hi = coords.min(axis=0), coords.max(axis=0)
    if voxel_size is None:
        voxel_size = np.sqrt(np.prod(hi - lo)) / (np.sqrt(N) / 5)
    steps = (hi - lo) / int(np.sqrt(voxel_num))
    axes = [np.arange(a, b, s) for a, b, s in zip(lo, hi, steps)]
    grid = np.stack(np.meshgrid(*axes), axis=-1).reshape(-1, D)
    means = np.zeros((grid.shape[0], gene_exp.shape[1]))
    used = np.zeros((grid.shape[0],))
    for i, g in enumerate(grid):
        mask = np.sqrt(np.sum((coords - g) ** 2, axis=1)) < voxel_size / 2
        if np.any(mask):
            means[i] = np.mean(gene_exp[mask], axis=0)
            used[i] = 1
    return grid[used == 1, :], means[used == 1, :]


def init_guess_sigma2(XA, XB, subsample=20000):
    """sum(d^4) / (D * nA * nA) on a <=20k subsample — squares the already squared distance (utils.py:1344-1354)."""
    NA, NB, D = XA.shape[0], XB.shape[0], XA.shape[1]
    sa = np.random.choice(NA, subsample, replace=False) if NA > subsample else np.arange(NA)
    sb = np.random.choice(NB, subsample, replace=False) if NB > subsample else np.arange(NB)
    d = euc_distance(XA[sa, :], XB[sb, :], squared=True)
    d = d**2
    return d.sum() / (D * sa.shape[0] * sa.shape[0])


def normalize_coords(coordsA, coordsB, separate_mean=True, separate_scale=False):
    """Per-slice mean, RMS scale (shared = mean of both unless separate_scale) (morpho_class.py:603-635)."""
    dt = coordsA.dtype
    coords = [coordsA.copy(order="K"), coordsB.copy(order="K")]
    D = coordsA.shape[1]
    scales = np.zeros((2,), dtype=dt)
    means = np.zeros((2, D), dtype=dt)
    for i in range(2):
        means[i] = np.einsum("ij->j", coords[i]) / coords[i].shape[0]
    if not separate_mean:
        gm = means.mean(axis=0)
        means = np.repeat(gm, 2, axis=0)  # reference quirk (morpho_class.py:615): repeat on a 1-D vector
    for i in range(2):
        coords[i] -= means[i]
        scales[i] = np.sqrt(np.einsum("ij->", np.einsum("ij,ij->ij", coords[i], coords[i])) / coords[i].shape[0])
    if not separate_scale:
        scales = np.full((2,), scales.mean(), dtype=dt)
    for i in range(2):
        coords[i] /= scales[i]
    return coords[0], coords[1], scales, means


# ---------------------------------------------------------------------------------------------------------------------
# The pairwise EM                               spateo/alignment/methods/morpho_class.py:242-313, 683-1528
# ---------------------------------------------------------------------------------------------------------------------


class MorphoPairOracle:
    """Array-level restatement of ``Morpho_pairwise`` (morpho_class.py:54) — moving slice A, fixed slice B.

    Inputs are what ``_align_preprocess`` hands to the solver: raw coordinates and dense representation matrices
    (one per rep layer) in the solver dtype. ``init_rep_A/B`` are the ``init_layer`` representations used by the coarse
    rigid initialisation (default: layer 0). Uses the global ``np.random`` stream in the reference's call order
    (SURVEY.md Appendix D) so ``np.random.seed(s)`` right before construction reproduces the reference draws.

    Not restated (the product raises NotImplementedError for them in round 1): sparse top-k mode, geodesic kernel
    (chunked mode is a memory work-around with identical results).
    """

    def __init__(
        self,
        coordsA,
        coordsB,
        exp_layers_A,
        exp_layers_B,
        dissimilarity="kl",
        probability_type="gauss",
        probability_parameters=None,
        label_transfer=None,
        init_rep_A=None,
        init_rep_B=None,
        init_metric="kl",
        nn_init=True,
        init_transform=True,
        allow_flip=False,
        nn_init_top_K=10,
        nn_init_weight=1.0,
        max_iter=200,
        nonrigid_start_iter=80,
        SVI_mode=True,
        batch_size=None,
        pre_compute_dist=True,
        lambdaVF=1e2,
        beta=0.01,
        K=15,
        sigma2_init_scale=0.1,
        sigma2_end=None,
        gamma_a=1.0,
        gamma_b=1.0,
        kappa=1.0,
        partial_robust_level=10,
        normalize_c=True,
        separate_mean=True,
        separate_scale=False,
        dtype="float32",
        return_mapping=False,
        update_R=True,
        guidance_pair=None,
        guidance_effect=False,
        guidance_weight=1.0,
        trace=None,
        sparse_calculation_mode=False,
        sparse_top_k=1024,
    ):
        self.sparse_calculation_mode, self.sparse_top_k = sparse_calculation_mode, sparse_top_k
        self.dt = np.float32 if dtype == "float32" else np.float64
        dt = self.dt
        self.f = lambda v: np.asarray(v, dtype=dt)  # the reference's _data(nx, v, type_as)
        n_layers = len(exp_layers_A)
        self.dissimilarity = [dissimilarity] * n_layers if isinstance(dissimilarity, str) else list(dissimilarity)
        self.probability_type = (
            [probability_type] * n_layers if isinstance(probability_type, str) else list(probability_type)
        )
        self.probability_parameters = (
            [None] * n_layers if probability_parameters is None else list(probability_parameters)
        )
        self.label_transfer = label_transfer
        self.exp_layers_A = [np.asarray(e, dtype=dt) if e.dtype.kind == "f" else e for e in exp_layers_A]
        self.exp_layers_B = [np.asarray(e, dtype=dt) if e.dtype.kind == "f" else e for e in exp_layers_B]
        self.init_rep_A = self.exp_layers_A[0] if init_rep_A is None else np.asarray(init_rep_A, dtype=dt)
        self.init_rep_B = self.exp_layers_B[0] if init_rep_B is None else np.asarray(init_rep_B, dtype=dt)
        self.init_metric = init_metric
        self.nn_init, self.init_transform, self.allow_flip = nn_init, init_transform, allow_flip
        self.nn_init_top_K, self.nn_init_weight = nn_init_top_K, nn_init_weight
        self.max_iter, self.nonrigid_start_iter = max_iter, nonrigid_start_iter
        self.SVI_mode, self.batch_size, self.pre_compute_dist = SVI_mode, batch_size, pre_compute_dist
        if sparse_calculation_mode:  # morpho_class.py:439-440
            self.pre_compute_dist = False
        self.lambdaVF, self.beta, self.K = lambdaVF, beta, K
        self.sigma2_init_scale, self.sigma2_end = sigma2_init_scale, sigma2_end
        self.gamma_a, self.gamma_b, self.kappa = gamma_a, gamma_b, kappa
        self.partial_robust_level = partial_robust_level
        self.normalize_c = normalize_c
        self.return_mapping, self.update_R = return_mapping, update_R
        self.guidance_pair, self.guidance_effect, self.guidance_weight = guidance_pair, guidance_effect, guidance_weight
        self.trace = trace

        # astype keeps the caller's memory order: the reference's coordinates come out of a fancy-indexed
        # (column-major) array (utils.py:103) and numpy's reductions round differently per layout.
        self.coordsA = np.asarray(coordsA).astype(dt, order="K", copy=True)
        self.coordsB = np.asarray(coordsB).astype(dt, order="K", copy=True)
        assert self.coordsA.shape[1] == self.coordsB.shape[1]
        self.NA, self.NB, self.D = self.coordsA.shape[0], self.coordsB.shape[0], self.coordsA.shape[1]
        if normalize_c:
            self.coordsA, self.coordsB, self.normalize_scales, self.normalize_means = normalize_coords(
                self.coordsA, self.coordsB, separate_mean, separate_scale
            )
        # guidance pairs [X_BI (fixed), X_AI (moving)], normalised with the slices' parameters (morpho_class.py:551-587)
        self.guidance = (guidance_pair is not None) and (guidance_effect is not False) and (guidance_weight > 0)
        if self.guidance:
            if not isinstance(guidance_pair, list) or len(guidance_pair) != 2:
                raise ValueError("guidance_pair must be a list with two elements: [X_BI, X_AI].")
            self.X_BI = np.asarray(guidance_pair[0]).astype(dt)
            self.X_AI = np.asarray(guidance_pair[1]).astype(dt)
            self.V_AI = np.zeros(self.X_AI.shape, dtype=dt)
            self.R_AI = np.zeros(self.X_AI.shape, dtype=dt)
            if normalize_c:
                self.X_AI = (self.X_AI - self.normalize_means[0]) / self.normalize_scales[0]
                self.X_BI = (self.X_BI - self.normalize_means[1]) / self.normalize_scales[1]
        self._construct_kernel()

    # -- morpho_class.py:845-875 ------------------------------------------------------------------------------------
    def _construct_kernel(self):
        uniq, uniq_idx = np.unique(self.coordsA, return_index=True, axis=0)
        if uniq.shape[0] > self.K:
            pick = np.random.choice(uniq.shape[0], self.K, replace=False)
        else:
            pick = np.arange(uniq.shape[0])
        self.inducing_idx = uniq_idx[pick]
        self.inducing_variables = self.coordsA[self.inducing_idx, :]
        self.GammaSparse = con_K(self.inducing_variables, self.inducing_variables, self.beta)
        self.U = con_K(self.coordsA, self.inducing_variables, self.beta)
        self.U_I = (
            con_K(self.X_AI, self.inducing_variables, self.beta) if self.guidance_effect in ["nonrigid", "both"] else None
        )
        self.K = self.inducing_variables.shape[0]

    # -- morpho_class.py:920-1035 -----------------------------------------------------------------------------------
    def _coarse_rigid_alignment(self, n_sampling=20000):
        top_K = self.nn_init_top_K
        ia = np.random.choice(self.NA, n_sampling, replace=False) if self.NA > n_sampling else np.arange(self.NA)
        ib = np.random.choice(self.NB, n_sampling, replace=False) if self.NB > n_sampling else np.arange(self.NB)
        cA, cB = self.coordsA[ia, :], self.coordsB[ib, :]
        N, M, D = cA.shape[0], cB.shape[0], cA.shape[1]
        XA, XB = self.init_rep_A[ia], self.init_rep_B[ib]
        cA, XA = voxel_data(cA, XA, voxel_num=max(min(int(N / 20), 1000), 100))
        cB, XB = voxel_data(cB, XB, voxel_num=max(min(int(M / 20), 1000), 100))
        [exp_dist] = calc_distance(XA, XB, self.init_metric)
        while True:
            try:
                item2 = np.argpartition(exp_dist, top_K, axis=0)[:top_K, :].T
                item1 = np.repeat(np.arange(exp_dist.shape[1])[:, None], top_K, axis=1)
                NN1 = np.dstack((item1, item2)).reshape((-1, 2))
                d1 = exp_dist.T[NN1[:, 0], NN1[:, 1]]
                item1 = np.argpartition(exp_dist, top_K, axis=1)[:, :top_K]
                item2 = np.repeat(np.arange(exp_dist.shape[0])[:, None], top_K, axis=1)
                NN2 = np.dstack((item1, item2)).reshape((-1, 2))
                d2 = exp_dist.T[NN2[:, 0], NN2[:, 1]]
                break
            except Exception as e:  # same retry policy as morpho_class.py:987-995
                top_K -= 1
                if top_K == 0:
                    raise RuntimeError("Failed to perform coarse rigid alignment after reducing top_K.") from e
        NN = np.vstack((NN1, NN2))
        dist = np.r_[d1, d2]
        train_x, train_y = cA[NN[:, 1], :], cB[NN[:, 0], :]
        P, R, t, _, sigma2, gamma = inlier_from_NN(train_x, train_y, dist[:, None])
        if self.allow_flip:
            Rf = np.eye(D)
            Rf[-1, -1] = -1
            P2, R2, t2, _, s2, g2 = inlier_from_NN(train_x @ Rf, train_y, dist[:, None])
            if g2 > gamma:
                P, R, t, sigma2 = P2, R2 @ Rf, t2, s2
        thr = min(P[np.argsort(-P[:, 0])[20], 0], 0.5)
        keep = np.where(P[:, 0] > thr)[0]
        dt = self.dt
        self.inlier_A = train_x[keep, :].astype(dt)
        self.inlier_B = train_y[keep, :].astype(dt)
        self.inlier_P = P[keep, :].astype(dt)
        self.init_R = R.astype(dt)
        self.init_t = t.astype(dt)
        if self.init_transform:
            self.inlier_A = np.dot(self.inlier_A, self.init_R.T) + self.init_t
            self.coordsA = np.dot(self.coordsA, self.init_R.T) + self.init_t

    # -- morpho_class.py:701-760, 788-817 -------------------------------------------------------------------------
    def _initialize_variational_variables(self):
        f, dt = self.f, self.dt
        self.sigma2 = self.sigma2_init_scale * init_guess_sigma2(self.coordsA, self.coordsB)
        for i, (eA, eB, d_s, p_t, p_p) in enumerate(
            zip(self.exp_layers_A, self.exp_layers_B, self.dissimilarity, self.probability_type, self.probability_parameters)
        ):
            if p_p is not None or p_t.lower() != "gauss":
                continue
            sa = np.random.choice(self.NA, 20000, replace=False) if self.NA > 20000 else np.arange(self.NA)
            sb = np.random.choice(self.NB, 20000, replace=False) if self.NB > 20000 else np.arange(self.NB)
            [ed] = calc_distance(eA[sa], eB[sb], d_s)
            mn = ed.min(1)
            self.probability_parameters[i] = np.maximum(mn[np.argsort(mn)[int(sa.shape[0] * 0.05)]] / 5, f(0.01))
        self.sigma2_variance = 1
        self.sigma2_variance_end = self.partial_robust_level
        self.sigma2_variance_decress = np.power(f(self.sigma2_variance_end / self.sigma2_variance), 1 / 100)
        if isinstance(self.kappa, float):
            self.kappa = np.ones((self.NA,), dtype=dt) * self.kappa
        else:
            self.kappa = np.asarray(self.kappa, dtype=dt)
        self.alpha = np.ones((self.NA,), dtype=dt)
        self.gamma, self.gamma_a, self.gamma_b = f(0.5), f(self.gamma_a), f(self.gamma_b)
        self.VnA = np.zeros(self.coordsA.shape, dtype=dt)
        self.XAHat, self.RnA = self.coordsA.copy(), self.coordsA.copy()
        self.Coff = np.zeros(self.K, dtype=dt)
        self.SigmaDiag = np.zeros((self.NA,), dtype=dt)
        self.R = np.identity(self.D, dtype=dt)
        self.nonrigid_flag = False
        self.Dim = f(self.D)
        self.samples_s = np.maximum(
            np.prod(self.coordsA.max(axis=0) - self.coordsA.min(axis=0)),
            np.prod(self.coordsB.max(axis=0) - self.coordsB.min(axis=0)),
        )
        self.C = np.identity(self.D, dtype=dt)
        if self.SVI_mode:
            self.SVI_deacy = f(10.0)
            if self.batch_size is None:
                self.batch_size = min(max(int(self.NB / 10), 1000), self.NB)
            else:
                self.batch_size = min(self.batch_size, self.NB)
            self.batch_perm = np.random.permutation(self.NB)
            self.Sp, self.Sp_spatial, self.Sp_sigma2 = 0, 0, 0
            self.SigmaInv = np.zeros((self.K, self.K), dtype=dt)
            self.PXB_term = np.zeros((self.NA, self.D), dtype=dt)

    # -- morpho_class.py:894-896 ----------------------------------------------------------------------------------
    def _update_batch(self, it):
        self.step_size = np.minimum(self.f(1.0), self.SVI_deacy / (it + 1.0))
        self.batch_idx = self.batch_perm[: self.batch_size]
        self.batch_perm = np.roll(self.batch_perm, self.batch_size)

    # -- morpho_class.py:1087-1200 --------------------------------------------------------------------------------
    def _update_assignment_P(self):
        model_mul = (self.alpha * np.exp(-self.SigmaDiag / self.sigma2))[:, None]
        YB = self.coordsB[self.batch_idx, :] if self.SVI_mode else self.coordsB
        spatial_dist = euc_distance(self.XAHat, YB, squared=True)
        if self.pre_compute_dist:
            exp_dist = [e[:, self.batch_idx] for e in self.exp_layer_dist] if self.SVI_mode else self.exp_layer_dist
        else:
            exp_dist = calc_distance(
                self.exp_layers_A,
                [e[self.batch_idx] if self.SVI_mode else e for e in self.exp_layers_B],
                self.dissimilarity,
                self.label_transfer,
            )
        self.P, self.K_NA_spatial, self.K_NA_sigma2, s2r = get_P_core(
            Dim=self.Dim,
            spatial_dist=spatial_dist,
            exp_dist=exp_dist,
            sigma2=self.sigma2,
            model_mul=model_mul,
            gamma=self.gamma,
            samples_s=self.samples_s,
            sigma2_variance=self.sigma2_variance,
            probability_type=self.probability_type,
            probability_parameters=self.probability_parameters,
            sparse_calculation_mode=self.sparse_calculation_mode,
            top_k=self.sparse_top_k,
        )
        Sp = self.P.sum()
        Sp_sigma2 = self.K_NA_sigma2.sum()
        Sp_spatial = self.K_NA_spatial.sum()
        self.K_NA = self.P.sum(axis=1)
        self.K_NB = self.P.sum(axis=0)
        if self.sparse_calculation_mode:  # morpho_class.py:1187-1198 (scipy returns np.matrix)
            self.K_NA = np.asarray(self.K_NA).squeeze(-1)
            self.K_NB = np.asarray(self.K_NB).squeeze(0)
        if self.SVI_mode:
            s = self.step_size
            self.Sp_spatial = s * Sp_spatial + (1 - s) * self.Sp_spatial
            self.Sp = s * Sp + (1 - s) * self.Sp
            self.Sp_sigma2 = s * Sp_sigma2 + (1 - s) * self.Sp_sigma2
        else:
            self.Sp_spatial, self.Sp, self.Sp_sigma2 = Sp_spatial, Sp, Sp_sigma2
        self.sigma2_related = s2r / (self.Dim * self.Sp_sigma2)

    # -- morpho_class.py:1214-1252 --------------------------------------------------------------------------------
    def _update_gamma(self):
        n = self.batch_size if self.SVI_mode else self.NB
        g = np.exp(_psi(self.gamma_a + self.Sp_spatial) - _psi(self.gamma_a + self.gamma_b + n))
        self.gamma = np.maximum(np.minimum(g, self.f(0.99)), self.f(0.01))

    def _update_alpha(self):
        new = np.exp(_psi(self.kappa + self.K_NA_spatial) - _psi(self.kappa * self.NA + self.Sp_spatial))
        if self.SVI_mode:
            self.alpha = self.step_size * new + (1 - self.step_size) * self.alpha
        else:
            self.alpha = new

    # -- morpho_class.py:1266-1298 --------------------------------------------------------------------------------
    def _update_nonrigid(self):
        SigmaInv = self.sigma2 * self.lambdaVF * self.GammaSparse + np.dot(
            self.U.T, np.einsum("ij,i->ij", self.U, self.K_NA)
        )
        YB = self.coordsB[self.batch_idx, :] if self.SVI_mode else self.coordsB
        PXB_term = _dot(self.P, YB) - np.einsum("ij,i->ij", self.RnA, self.K_NA)
        if self.SVI_mode:
            s = self.step_size
            self.SigmaInv = s * SigmaInv + (1 - s) * self.SigmaInv
            self.PXB_term = s * PXB_term + (1 - s) * self.PXB_term
        else:
            self.SigmaInv, self.PXB_term = SigmaInv, PXB_term
        UPXB = np.dot(self.U.T, self.PXB_term)
        g_nonrigid = self.guidance and (self.guidance_effect in ("nonrigid", "both"))
        if g_nonrigid:  # morpho_class.py:1282-1288 (in SVI mode the += lands in the running average — reference quirk)
            cg = self.sigma2 * self.guidance_weight * self.Sp / self.U_I.shape[0]
            self.SigmaInv += cg * np.dot(self.U_I.T, self.U_I)
            UPXB += cg * np.dot(self.U_I.T, self.X_BI - self.R_AI)
        Sigma = _scipy_pinv(self.SigmaInv)
        self.Sigma = Sigma
        self.Coff = np.dot(Sigma, UPXB)
        self.VnA = np.dot(self.U, self.Coff)
        if g_nonrigid:
            self.V_AI = np.dot(self.U_I, self.Coff)
        self.SigmaDiag = self.sigma2 * np.einsum("ij->i", np.einsum("ij,ji->ij", self.U, np.dot(Sigma, self.U.T)))

    # -- morpho_class.py:1312-1408 --------------------------------------------------------------------------------
    def _update_rigid(self):
        YB = self.coordsB[self.batch_idx, :] if self.SVI_mode else self.coordsB
        PXA = np.dot(self.K_NA, self.coordsA)[None, :]
        PVA = np.dot(self.K_NA, self.VnA)[None, :]
        PXB = np.dot(self.K_NB, YB)[None, :]
        # mu_* alias the P* arrays: the in-place += below also changes PXB / PXA used in the translation (quirk B-5)
        mu_XB, mu_XA, mu_Vn = PXB, PXA, PVA
        mu_X_deno, mu_Vn_deno = np.copy(self.Sp), np.copy(self.Sp)
        g_rigid = self.guidance and (self.guidance_effect in ("rigid", "both"))
        if g_rigid:  # morpho_class.py:1322-1327: SCALAR means of the guidance points, added in place (aliases!)
            cg = self.sigma2 * self.guidance_weight * self.Sp / self.X_BI.shape[0]
            mu_XB += cg * self.X_BI.mean()
            mu_XA += cg * self.X_AI.mean()
            mu_Vn += cg * self.V_AI.mean()
            mu_X_deno += cg * self.X_BI.shape[0]
            mu_Vn_deno += cg * self.X_BI.shape[0]
        if self.nn_init:
            c = self.sigma2 * self.nn_init_weight * self.Sp / np.sum(self.inlier_P)
            mu_XB += c * np.dot(self.inlier_P.T, self.inlier_B)
            mu_XA += c * np.dot(self.inlier_P.T, self.inlier_A)
            mu_X_deno += c * np.sum(self.inlier_P)
        mu_XB = mu_XB / mu_X_deno
        mu_XA = mu_XA / mu_X_deno
        mu_Vn = mu_Vn / mu_Vn_deno
        XA_hat = self.coordsA - mu_XA
        VnA_hat = self.VnA - mu_Vn
        XB_hat = YB - mu_XB
        A = -(
            np.dot(XA_hat.T, np.einsum("ij,i->ij", VnA_hat, self.K_NA)) - np.dot(_dot(XA_hat.T, self.P), XB_hat)
        ).T
        if g_rigid:  # morpho_class.py:1347-1350, 1360-1363
            A -= cg * np.dot((self.X_AI - mu_XA).T, (self.V_AI - mu_Vn) - (self.X_BI - mu_XB)).T
        if self.nn_init:
            iA_hat = self.inlier_A - mu_XA
            iB_hat = self.inlier_B - mu_XB
            A -= c * np.dot((iA_hat * self.inlier_P).T, -iB_hat).T
        svdU, _, svdV = np.linalg.svd(A)
        self.C[-1, -1] = np.linalg.det(np.dot(svdU, svdV))
        if self.update_R:
            R = np.dot(np.dot(svdU, self.C), svdV)
            if self.SVI_mode and self.step_size < 1:
                self.R = self.step_size * R + (1 - self.step_size) * self.R
            else:
                self.R = R
        t_num = PXB - PVA - np.dot(PXA, self.R.T)
        t_den = np.copy(self.Sp)
        if g_rigid:  # morpho_class.py:1384-1388
            t_num += cg * np.sum(self.X_BI - self.V_AI - np.dot(self.X_AI, self.R.T), axis=0)
            t_den += cg * self.X_BI.shape[0]
        if self.nn_init:
            t_num += c * np.dot(self.inlier_P.T, self.inlier_B - np.dot(self.inlier_A, self.R.T))
            t_den += c * np.sum(self.inlier_P)
        t = t_num / t_den
        if self.SVI_mode and self.step_size < 1:
            self.t = self.step_size * t + (1 - self.step_size) * self.t
        else:
            self.t = t
        self.RnA = np.dot(self.coordsA, self.R.T) + self.t
        if self.guidance:  # morpho_class.py:1407-1408: iterates R_AI itself (starts at zeros), not X_AI — reference quirk
            self.R_AI = np.dot(self.R_AI, self.R.T) + self.t

    # -- morpho_class.py:1426-1435 --------------------------------------------------------------------------------
    def _update_sigma2(self, it):
        self.sigma2 = np.maximum(
            self.sigma2_related + np.einsum("i,i", self.K_NA_sigma2, self.SigmaDiag) / self.Sp_sigma2, self.f(1e-3)
        )
        self.sigma2_variance = np.minimum(self.sigma2_variance * self.sigma2_variance_decress, self.sigma2_variance_end)
        if it < 100:
            self.sigma2 = np.maximum(self.sigma2, self.f(1e-2))

    # -- morpho_class.py:1451-1469 --------------------------------------------------------------------------------
    def _get_optimal_R(self):
        YB = self.coordsB[self.batch_idx, :] if self.SVI_mode else self.coordsB
        mu_A = np.dot(self.K_NA, self.coordsA) / self.Sp
        mu_B = np.dot(self.K_NB, YB) / self.Sp
        A = np.dot(_dot(self.P, YB - mu_B).T, self.coordsA - mu_A)
        svdU, _, svdV = np.linalg.svd(A)
        self.C[-1, -1] = np.linalg.det(np.dot(svdU, svdV))
        self.optimal_R = np.dot(np.dot(svdU, self.C), svdV)
        self.optimal_t = mu_B - np.dot(mu_A, self.optimal_R.T)
        self.optimal_RnA = np.dot(self.coordsA, self.optimal_R.T) + self.optimal_t

    # -- morpho_class.py:242-313 ----------------------------------------------------------------------------------
    def prepare(self):
        """Everything ``run`` does before the EM loop (coarse init, variational init, cost precompute)."""
        if self.nn_init:
            self._coarse_rigid_alignment()
        self._initialize_variational_variables()
        if (not self.SVI_mode) or self.pre_compute_dist:
            self.exp_layer_dist = calc_distance(
                self.exp_layers_A, self.exp_layers_B, self.dissimilarity, self.label_transfer
            )

    def em_iteration(self, it):
        if self.SVI_mode:
            self._update_batch(it)
        self._update_assignment_P()
        self._update_gamma()
        self._update_alpha()
        if (it > self.nonrigid_start_iter) or self.nonrigid_flag:
            self.nonrigid_flag = True
            self._update_nonrigid()
        self._update_rigid()
        self.XAHat = self.VnA + self.RnA
        self._update_sigma2(it)

    def finish(self):
        if self.sigma2_end is not None:
            self.sigma2 = self.f(self.sigma2_end)
        if self.return_mapping and self.SVI_mode:
            self.SVI_mode = False
            self._update_assignment_P()
        self._get_optimal_R()
        if self.normalize_c:  # de-normalise with the FIXED slice's scale / mean (morpho_class.py:1484-1486)
            s, m = self.normalize_scales[1], self.normalize_means[1]
            self.XAHat = self.XAHat * s + m
            self.RnA = self.RnA * s + m
            self.optimal_RnA = self.optimal_RnA * s + m
        self.vecfld = self._vecfld()
        return self.P

    def run(self):
        self.prepare()
        for it in range(self.max_iter):
            if self.trace is not None:
                self.trace(self, it, "pre")
            self.em_iteration(it)
            if self.trace is not None:
                self.trace(self, it, "post")
        return self.finish()

    # -- morpho_class.py:1499-1528 --------------------------------------------------------------------------------
    def _vecfld(self):
        D = self.D
        norm_dict = None
        if self.normalize_c:
            norm_dict = {
                "mean_transformed": self.normalize_means[0],
                "mean_fixed": self.normalize_means[1],
                "scale": self.normalize_scales[0],
                "scale_transformed": self.normalize_scales[0],
                "scale_fixed": self.normalize_scales[1],
            }
        return {
            "R": self.R,
            "t": self.t,
            "optimal_R": self.optimal_R,
            "optimal_t": self.optimal_t,
            "init_R": self.init_R if self.nn_init else np.eye(D),
            "init_t": self.init_t if self.nn_init else np.zeros(D),
            "beta": self.beta,
            "Coff": self.Coff,
            "inducing_variables": self.inducing_variables,
            "normalize_scales": self.normalize_scales if self.normalize_c else None,
            "normalize_means": self.normalize_means if self.normalize_c else None,
            "normalize_c": self.normalize_c,
            "dissimilarity": self.dissimilarity,
            "sigma2": self.sigma2,
            "gamma": self.gamma,
            "NA": self.NA,
            "sigma2_variance": self.sigma2_variance,
            "method": "Spateo",
            "norm_dict": norm_dict,
            "kernel_type": "euc",
        }


# ---------------------------------------------------------------------------------------------------------------------
# Field evaluation                                spateo/alignment/transform.py:61-116; gaussian_process.py:102-127
# ---------------------------------------------------------------------------------------------------------------------


def ba_transform(vecfld, query_points, deformation_scale=1, dtype="float64"):
    """Apply the learned field + rigid maps to arbitrary points (transform.py:83-116)."""
    dt = np.float32 if dtype == "float32" else np.float64
    f = lambda v: np.asarray(v, dtype=dt)
    scale = f(vecfld["norm_dict"]["scale_transformed"])
    mean_ref = f(vecfld["norm_dict"]["mean_fixed"])
    mean_q = f(vecfld["norm_dict"]["mean_transformed"])
    XA = f(query_points)
    if vecfld["normalize_c"]:
        XA = (XA - mean_q) / scale
    ker = con_K(XA, f(vecfld["inducing_variables"]), vecfld["beta"])
    XA = XA @ f(vecfld["init_R"]).T + f(vecfld["init_t"])
    vel = (ker @ f(vecfld["Coff"])) * deformation_scale
    sim = XA @ f(vecfld["R"]).T + f(vecfld["t"])
    opt = XA @ f(vecfld["optimal_R"]).T + f(vecfld["optimal_t"])
    XAHat = vel + sim
    if vecfld["normalize_c"]:
        XAHat = XAHat * scale + mean_ref
        vel = vel * scale
        opt = opt * scale + mean_ref
    return XAHat, vel, opt


def gp_velocity(X, vf, nonrigid_only=False):
    """morphofield_gp's field evaluation (gaussian_process.py:107-127): exp(-beta*cdist^2) @ Coff + rigid, /10000."""
    nd = vf["norm_dict"]
    nx_ = (X - nd["mean_transformed"]) / nd["scale_transformed"]
    d2 = ((nx_[:, None, :] - np.asarray(vf["inducing_variables"])[None, :, :]) ** 2).sum(-1)
    ker = np.exp(-vf["beta"] * d2)
    vel = ker @ vf["Coff"]
    if nonrigid_only:
        out = vel * nd["scale_fixed"] + (nd["scale_fixed"] - nd["scale_transformed"]) * nx_
    else:
        rigid = nx_ @ np.asarray(vf["R"]).T + vf["t"]
        out = (vel + rigid) * nd["scale_fixed"] + nd["mean_fixed"] - X
    return out / 10000


# ---------------------------------------------------------------------------------------------------------------------
# SparseVFC — PARITY UNPINNED (third-party dynamo-release>=1.4.1, not in the reference tree; SURVEY.md Appendix E)
# ---------------------------------------------------------------------------------------------------------------------


def sparse_vfc(
    X,
    Y,
    ctrl_idx,
    beta,
    lambda_=0.02,
    a=5.0,
    gamma=0.9,
    ecr=1e-5,
    minP=1e-5,
    MaxIter=500,
    theta=0.75,
    Grid=None,
):
    """float64 restatement of dynamo ``SparseVFC`` (Ma et al. 2013) with the control points given explicitly.

    PARITY UNPINNED: the algorithm lives in ``dynamo.vectorfield.scVectorField.SparseVFC`` (requirements.txt:7,
    call sites spateo/tdr/morphometrics/morphofield/sparsevfc.py:167,189-198); dynamo is neither vendored nor
    installed, and the reference has no test pinning results at that boundary. Control-point sampling and the default
    bandwidth are left to the caller so this function only restates the EM itself.
    """
    X = np.asarray(X, dtype=np.float64)
    Y = np.asarray(Y, dtype=np.float64)
    N, D = Y.shape
    ctrl = X[ctrl_idx]
    sq = lambda A, B: np.maximum((A**2).sum(1)[:, None] + (B**2).sum(1)[None, :] - 2 * A @ B.T, 0)
    Kc = np.exp(-beta * sq(ctrl, ctrl))
    U = np.exp(-beta * sq(X, ctrl))
    M = ctrl.shape[0]
    V = np.zeros((N, D))
    C = np.zeros((M, D))
    sigma2 = max(((Y - V) ** 2).sum() / (N * D), 1e-7)
    E, tecr, it = 1.0, 1.0, 0
    tecr_traj, E_traj = [], []
    P = np.ones(N)
    while it < MaxIter and tecr > ecr and sigma2 > 1e-8:
        E_old = E
        r = ((Y - V) ** 2).sum(1)
        t1 = np.exp(-r / (2 * sigma2))
        t2 = (2 * np.pi * sigma2) ** (D / 2) * (1 - gamma) / (gamma * a)
        if (t1 == 0).any() and (t1 > 0).any():
            t1[t1 == 0] = t1[t1 > 0].min()
        P = t1 / (t1 + t2)
        E = (P * r).sum() / (2 * sigma2) + P.sum() * np.log(sigma2) * D / 2 + lambda_ / 2 * np.trace(C.T @ Kc @ C)
        tecr = abs((E - E_old) / E)
        tecr_traj.append(tecr)
        E_traj.append(E)
        P = np.maximum(P, minP)
        UP = U.T * P
        C = np.linalg.lstsq(lambda_ * sigma2 * Kc + UP @ U, UP @ Y, rcond=None)[0]
        V = U @ C
        Sp = P.sum()
        sigma2 = (P * ((Y - V) ** 2).sum(1)).sum() / (Sp * D)
        gamma = min(max((P > theta).sum() / N, 0.05), 0.95)
        it += 1
    out = dict(X=X, X_ctrl=ctrl, ctrl_idx=np.asarray(ctrl_idx), Y=Y, beta=beta, V=V, C=C, P=P,
               VFCIndex=np.where(P > theta)[0], sigma2=sigma2, iteration=it, tecr_traj=np.array(tecr_traj),
               E_traj=np.array(E_traj), gamma=gamma)
    if Grid is not None:
        out["grid"] = Grid
        out["grid_V"] = np.exp(-beta * sq(np.asarray(Grid, dtype=np.float64), ctrl)) @ C
    return out
