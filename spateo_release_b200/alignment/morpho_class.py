"""``Morpho_pairwise`` — drop-in for ``spateo.alignment.methods.morpho_class.Morpho_pairwise`` (morpho_class.py:54)
whose EM runs as hand-written sm_90a CUDA kernels behind the C ABI in ``include/spateo_b200.h``.

Host side (this file): validation, gene intersection, dense extraction, coordinate normalisation, inducing-point choice,
coarse rigid initialisation bookkeeping and output wrapping — same names, argument meaning, RNG call order
(SURVEY.md Appendix D), result attributes and exceptions as the reference. Device side: expression-cost matrix,
fused two-sweep E-step (P never materialised), gamma/alpha, non-rigid solve, rigid Procrustes, sigma2; all scalar state
stays on the device, there is no host synchronisation inside the iteration loop and no CPU fallback.
"""

from __future__ import annotations

import ctypes as C
from typing import List, NamedTuple, Optional, Union

import numpy as np
import torch

from .. import _capi
from .._capi import SpbEmParams, SpbScalars, check, ptr
from . import utils as U

_METRIC_CODE = {
    "kl": _capi.CONST["SPB_METRIC_KL"],
    "euc": _capi.CONST["SPB_METRIC_EUC"],
    "euclidean": _capi.CONST["SPB_METRIC_EUC"],
    "square_euc": _capi.CONST["SPB_METRIC_SQRT_EUC"],
    "square_euclidean": _capi.CONST["SPB_METRIC_SQRT_EUC"],
    "cos": _capi.CONST["SPB_METRIC_COS"],
    "cosine": _capi.CONST["SPB_METRIC_COS"],
    "sym_kl": _capi.CONST["SPB_METRIC_SYMKL"],
}
_PROB_CODE = {
    "gauss": _capi.CONST["SPB_PROB_GAUSS"],
    "gaussian": _capi.CONST["SPB_PROB_GAUSS"],
    "cos": _capi.CONST["SPB_PROB_COS"],
    "cosine": _capi.CONST["SPB_PROB_COS"],
    "prob": _capi.CONST["SPB_PROB_PROB"],
}


# bytes moved between host and device by the big transfers of an alignment (expression matrices, coordinate / result
# arrays); bench.py reads and resets it around the public call for the end-to-end line
TRANSFER_BYTES = {"h2d": 0, "d2h": 0}


def _count_h2d(t) -> None:
    TRANSFER_BYTES["h2d"] += int(t.numel()) * int(t.element_size())


def _count_d2h(t) -> None:
    TRANSFER_BYTES["d2h"] += int(t.numel()) * int(t.element_size())


_STAGE_FLOATS = 16 << 20  # two reusable 64 MB pinned staging buffers
_stage = {}
_stage_lock = __import__("threading").Lock()


def staged_to_device(host: np.ndarray, dev: torch.device) -> torch.Tensor:
    """Pageable host array -> device through two reusable pinned staging buffers (chunk k is copied into pinned memory
    while chunk k-1 is on the wire), which avoids both a slow pageable ``.to()`` and the first-use cost of ``pin_memory()`` on
    a large array. Counts the bytes in ``TRANSFER_BYTES``."""
    t = torch.from_numpy(np.ascontiguousarray(host, dtype=np.float32))
    _count_h2d(t)
    if t.is_pinned() or t.numel() < (2 << 20):
        return t.to(dev, non_blocking=t.is_pinned())
    events = [torch.cuda.Event(), torch.cuda.Event()]
    out = torch.empty(t.shape, dtype=torch.float32, device=dev)
    src, dst = t.view(-1), out.view(-1)
    n = src.numel()
    with _stage_lock, torch.cuda.device(dev):
        if "bufs" not in _stage:
            _stage["bufs"] = [torch.empty((_STAGE_FLOATS,), dtype=torch.float32).pin_memory() for _ in range(2)]
        bufs = _stage["bufs"]
        for k, o in enumerate(range(0, n, _STAGE_FLOATS)):
            b = k & 1
            m = min(_STAGE_FLOATS, n - o)
            if k >= 2:
                events[b].synchronize()
            bufs[b][:m].copy_(src[o:o + m])
            dst[o:o + m].copy_(bufs[b][:m], non_blocking=True)
            events[b].record()
        for e in events[: min(2, (n + _STAGE_FLOATS - 1) // _STAGE_FLOATS)]:
            e.synchronize()  # the staging buffers are reused by the next call
    return out


def _round_up(x: int, m: int) -> int:
    return ((x + m - 1) // m) * m


def _kd_groups(c: np.ndarray, idx: np.ndarray, unit: int) -> list:
    """Split the points ``idx`` (columns of the [D][n] coordinates ``c``) into consecutive groups of ``unit`` rows (the last one may be shorter): each cut goes across the
    longest extent of the points it splits, after floor(groups / 2) whole groups (a stable sort makes it deterministic)."""
    out, stack = [], [idx]
    while stack:  # depth first, left part before right part
        ix = stack.pop()
        groups = -(-ix.shape[0] // unit)
        if groups <= 1:
            out.append(ix)
            continue
        p = c[:, ix]
        axis = int(np.argmax(p.max(axis=1) - p.min(axis=1)))
        ix = ix[np.argsort(p[axis], kind="stable")]
        cut = (groups // 2) * unit
        stack.append(ix[cut:])
        stack.append(ix[:cut])
    return out


def kd_order(coords: np.ndarray, tile: int = 512, quarter: int = 128) -> np.ndarray:
    """Row permutation into compact row blocks: a balanced k-d split of the points into blocks of ``tile`` rows, then of every
    block into ``quarter``-row parts the same way. Row block k is rows [k tile, (k + 1) tile) of the permuted order; only the
    last block can be short."""
    c = np.ascontiguousarray(np.asarray(coords, dtype=np.float64).T)
    blocks = _kd_groups(c, np.arange(c.shape[1], dtype=np.int64), tile)
    return np.concatenate([q for b in blocks for q in _kd_groups(c, b, quarter)])


def _device_budget(dev) -> int:
    """Bytes the next allocations on ``dev`` can use: driver-free memory plus what the caching allocator holds unused."""
    free, _ = torch.cuda.mem_get_info(dev)
    return free + torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)


class CostPlan(NamedTuple):
    """How a pair holds its expression cost matrix. ``resident``: the whole [N_B][ldx] matrix is built once and kept.
    ``streamed``: every iteration recomputes it in column chunks ``chunks`` (``[c0, c1)`` ranges over the iteration's
    ``cols`` columns, ``width`` columns wide except the last) that fit the device next to the rest of the pair."""

    mode: str
    width: int
    chunks: tuple
    need: int
    budget: int

    @property
    def streamed(self) -> bool:
        return self.mode == "streamed"

    @property
    def n_chunks(self) -> int:
        return len(self.chunks)


def plan_cost(n_moving: int, n_fixed: int, n_genes: int, cols: int, budget: int, n_sms: int = 132,
              transfer: Optional[tuple] = None) -> CostPlan:
    """Resident when ``pair_device_bytes`` fits ``budget``; otherwise the widest multiple of 8 columns (at most ``cols``,
    the columns of one iteration) whose streamed footprint fits, balanced over the chunks it takes. Raises MemoryError
    when not even 8 columns fit. ``transfer``: the feature counts (F_B, F_A) of a posterior transfer (``pair_device_bytes``)."""
    from .distributed import pair_device_bytes

    need = pair_device_bytes(n_moving, n_fixed, n_genes, transfer=transfer, n_sms=n_sms, cols=cols)
    if need <= budget:
        return CostPlan("resident", cols, ((0, cols),), need, budget)

    def need_at(c):
        return pair_device_bytes(n_moving, n_fixed, n_genes, chunk_cols=c, n_sms=n_sms, transfer=transfer)

    if need_at(min(8, cols)) > budget:
        raise MemoryError(
            f"the pair ({n_moving} x {n_fixed} cells, {n_genes} features) does not fit the device even with its cost matrix "
            f"streamed 8 columns at a time: {need_at(min(8, cols))} bytes needed, {budget} bytes available")
    if need_at(cols) <= budget:
        width = cols
    else:
        lo, hi = 1, (cols - 1) // 8  # 8 lo fits; find the largest multiple of 8 below cols that fits
        while lo < hi:
            mid = (lo + hi + 1) // 2
            if need_at(8 * mid) <= budget:
                lo = mid
            else:
                hi = mid - 1
        width = 8 * lo
    n = -(-cols // width)
    width = min(cols, _round_up(-(-cols // n), 8))  # same chunk count, widths as even as multiples of 8 allow
    chunks = tuple((c0, min(cols, c0 + width)) for c0 in range(0, cols, width))
    return CostPlan("streamed", width, chunks, need_at(width), budget)


def resolve_transfer(adata, spec, n_rows: int, name: str):
    """Features of a posterior transfer on one slice: ``spec`` is a float array [n_rows, F] in the slice's row order, the
    name of an ``.obsm`` matrix, or the name of an ``.obs`` column, one-hot encoded in ``pd.Categorical(...).categories``
    order (a missing value is an all-zero row). Returns (float32 [n_rows, F], categories or None); ``ValueError`` for a
    missing key, a row count other than ``n_rows``, F = 0 or a non-finite value."""
    import pandas as pd

    cats = None
    if isinstance(spec, str):
        if spec in adata.obsm:
            arr = adata.obsm[spec]
            arr = arr.values if isinstance(arr, pd.DataFrame) else (arr.toarray() if hasattr(arr, "toarray") else arr)
        elif spec in adata.obs.columns:
            cat = pd.Categorical(adata.obs[spec])
            cats = list(cat.categories)
            codes = np.asarray(cat.codes)
            arr = np.zeros((codes.shape[0], len(cats)), dtype=np.float32)
            arr[np.flatnonzero(codes >= 0), codes[codes >= 0]] = 1.0
        else:
            raise ValueError(f"{name}: '{spec}' is neither an .obsm matrix nor an .obs column of the slice")
    else:
        arr = spec
    try:
        arr = np.asarray(arr, dtype=np.float64)
    except (TypeError, ValueError) as e:
        raise ValueError(f"{name}: the features must be numeric ({e})") from None
    if arr.ndim != 2:
        raise ValueError(f"{name}: expected a [cells, features] matrix, got shape {arr.shape}")
    if arr.shape[0] != n_rows:
        raise ValueError(f"{name}: {arr.shape[0]} rows for a slice of {n_rows} cells")
    if arr.shape[1] == 0:
        raise ValueError(f"{name}: no features (F = 0)")
    if not np.isfinite(arr).all():
        raise ValueError(f"{name}: the features hold non-finite values")
    return arr.astype(np.float32), cats


def svi_schedule(batch_perm: np.ndarray, max_iter: int, nbb: int) -> np.ndarray:
    """[max(max_iter, 1)][nbb] fixed cells of every SVI iteration: a deterministic function of the initial permutation
    (morpho_class.py:894-896)."""
    sched = np.empty((max(max_iter, 1), nbb), dtype=np.int32)
    perm = batch_perm.copy()
    for it in range(max_iter):
        sched[it] = perm[:nbb]
        perm = np.roll(perm, nbb)
    return sched


def svi_chunk_schedules(sched: np.ndarray, chunks) -> list:
    """Every column chunk's own [max_iter][c1 - c0] slice of the SVI schedule: the chunks of iteration ``it`` together
    cover the same fixed cells, in the same order, as row ``it`` of ``sched``."""
    return [np.ascontiguousarray(sched[:, c0:c1]) for c0, c1 in chunks]


def shard_svi_schedule(sched: np.ndarray, n_fixed: int, rank: int, world: int):
    """One rank's fixed-width share of the SVI schedule ``sched`` of a column-sharded pair. Returns ``(local, pos)``, both
    [max_iter][w]: ``local[it]`` lists the members of batch ``it`` that lie in the rank's block [c0, c1) of fixed cells
    (``column_block``), in batch order, as local column indices; ``pos[it]`` holds their positions in the batch. The rest
    of the row is padding: the null column ``c1 - c0`` in ``local`` and -1 in ``pos``. ``w`` is the largest number of
    members any iteration puts in the block (at least 1, so that every launch has a column), so every iteration of the
    rank runs the same E-step launch shape."""
    from .distributed import column_block

    c0, c1 = column_block(n_fixed, rank, world)
    inside = (sched >= c0) & (sched < c1)
    width = max(1, int(inside.sum(axis=1).max()))
    local = np.full((sched.shape[0], width), c1 - c0, dtype=np.int32)
    pos = np.full((sched.shape[0], width), -1, dtype=np.int32)
    for it in range(sched.shape[0]):
        members = np.flatnonzero(inside[it])
        local[it, : members.size] = sched[it, members] - c0
        pos[it, : members.size] = members
    return local, pos


# Coordinates of the null column that pads an SVI shard's iterations to one width (shard_svi_schedule). It lies so far from
# every moving cell that build_col_lists_kernel culls it from every row block, and on the opposite side from the pad rows
# of XAHat (+1e18), which would sit at distance 0 from a null column placed at +1e18. Its cost row is zero as well, so
# even without culling every weight it takes part in is an exact zero.
_NULL_COLUMN_COORD = -1e18


def resolve_device(device) -> torch.device:
    """Reference semantics: "cpu" or a GPU index string (utils.py:35-66). Here every value maps to a CUDA device —
    there is no CPU path; ``CUDA_VISIBLE_DEVICES`` is NOT mutated (the reference does, utils.py:51)."""
    _capi.require_cuda()
    if isinstance(device, torch.device):
        return device
    if device is None or device == "cpu" or device == "cuda":
        return torch.device("cuda", torch.cuda.current_device())
    if isinstance(device, int):
        return torch.device("cuda", device)
    s = str(device)
    if s.startswith("cuda:"):
        return torch.device(s)
    return torch.device("cuda", int(s))


class GeneCostBuilder:
    """Device pipeline for ``calc_distance`` + ``calc_probability`` of one representation layer (utils.py:866-985).

    The contraction is a wgmma / TMA kernel with a 3xTF32 error-compensated split (fp32-accurate).
    """

    def __init__(self, lib, dev):
        self.lib, self.dev = lib, dev

    def prepare(self, X: torch.Tensor, metric: str, fixed: bool, centre: Optional[torch.Tensor] = None):
        """Row pre-pass. Returns (operand [n, Gp] fp32 zero-padded to 32 features, rowterm [n] or None).

        KL, fixed side: ``centre`` (the mean normalised moving profile, length G) centres every log-row so the contraction
        stays near zero (see kl_prepare_rows_kernel); the centring term comes back as the row term."""
        n, G = X.shape
        Gp = _round_up(G, 32)
        st = _capi.current_stream_ptr()
        if metric == "kl":
            out = torch.empty((n, Gp), dtype=torch.float32, device=self.dev)
            want_rt = (not fixed) or (centre is not None)
            rt = torch.empty((n,), dtype=torch.float32, device=self.dev) if want_rt else None
            check(self.lib.spb_kl_prepare_rows(ptr(X), n, G, X.stride(0), ptr(out), Gp, ptr(rt), 1 if fixed else 0,
                                               ptr(centre), st), "spb_kl_prepare_rows")
            return out, rt
        if metric in ("cos", "cosine"):
            out = torch.empty((n, Gp), dtype=torch.float32, device=self.dev)
            check(self.lib.spb_rows_normalize(ptr(X), n, G, X.stride(0), ptr(out), Gp, st), "spb_rows_normalize")
            return out, None
        # euclidean family: raw values (padded) + squared norms
        if Gp == G and X.is_contiguous():
            out = X
        else:
            out = torch.zeros((n, Gp), dtype=torch.float32, device=self.dev)
            out[:, :G] = X
        rt = torch.empty((n,), dtype=torch.float32, device=self.dev)
        check(self.lib.spb_rows_sqnorm(ptr(out), n, G, Gp, ptr(rt), st), "spb_rows_sqnorm")
        return out, rt

    def prepare_pair(self, A: torch.Tensor, B: torch.Tensor, metric: str):
        """Operands + row terms of (moving A, fixed B) for ``metric``. Returns (opA, rtA, opB, rtB, G_effective).

        ``sym_kl`` = (KL(a||b) + KL(b||a)) / 2 (utils.py:922-932) is ONE contraction over 2G features:
        [Xn | log X - d_i] . [log Y - c_j | Yn], with both log blocks centred (c_j by the mean moving profile, d_i by the
        mean fixed profile) and e = ((sum Xn log X - d_i) + (sum Yn log Y - c_j) - dot) / 2."""
        G = A.shape[1]
        if metric != "sym_kl":
            opA, rtA = self.prepare(A, metric, fixed=False)
            opB, rtB = self.prepare(B, metric, fixed=True, centre=self.centre_of(opA, G) if metric == "kl" else None)
            return opA, rtA, opB, rtB, G
        Xn, ta = self.prepare(A, "kl", fixed=False)              # Xn, sum Xn (log Xn + log G)
        Yn, tb = self.prepare(B, "kl", fixed=False)
        LY, cj = self.prepare(B, "kl", fixed=True, centre=self.centre_of(Xn, G))   # log Y + log G - c_j
        LX, di = self.prepare(A, "kl", fixed=True, centre=self.centre_of(Yn, G))   # log X + log G - d_i
        Gp = Xn.shape[1]
        opA = torch.cat([Xn, LX], dim=1).contiguous()
        opB = torch.cat([LY, Yn], dim=1).contiguous()
        return opA, (ta - di).contiguous(), opB, (tb - cj).contiguous(), 2 * Gp

    @staticmethod
    def centre_of(opA: torch.Tensor, G: int) -> torch.Tensor:
        """Mean normalised moving profile (fp32, length G) used to centre the fixed side of the KL contraction."""
        return opA[:, :G].mean(dim=0, dtype=torch.float64).float().contiguous()

    def _split(self, op: torch.Tensor):
        hi, lo = torch.empty_like(op), torch.empty_like(op)
        check(self.lib.spb_split_tf32(ptr(op), ptr(hi), ptr(lo), op.numel(), _capi.current_stream_ptr()), "spb_split_tf32")
        return hi, lo

    def cost(self, opA, rtA, opB, rtB, NA, NB, G, metric, prob_type, prob_param, accumulate, GT, ldx):
        ahi, alo = self._split(opA)
        bhi, blo = self._split(opB)
        self.cost_split(ahi, alo, rtA, bhi, blo, rtB, NA, NB, G, metric, prob_type, prob_param, accumulate, GT, ldx)
        self._keep = (ahi, alo, bhi, blo)  # stay alive until the stream has consumed them

    def split_pair(self, opA, rtA, opB, rtB, G):
        """Operands of ``prepare_pair`` as the tf32 hi / lo pairs ``cost_split`` takes (split once, kept for a streamed run)."""
        ahi, alo = self._split(opA)
        bhi, blo = self._split(opB)
        return dict(ahi=ahi, alo=alo, rtA=rtA, bhi=bhi, blo=blo, rtB=rtB, G=G)

    def cost_split(self, ahi, alo, rtA, bhi, blo, rtB, NA, NB, G, metric, prob_type, prob_param, accumulate, GT, ldx):
        """GT[j][i] (op)= prob(metric(A_i, B_j)) for the NB rows of the fixed-side operands ``bhi`` / ``blo`` / ``rtB``
        (all fixed cells, a row range of them or the gathered columns of an iteration chunk)."""
        pp = float(prob_param) if prob_param is not None else 1.0
        check(
            self.lib.spb_gene_cost_tc(
                ptr(ahi), ptr(alo), ahi.stride(0), ptr(rtA), ptr(bhi), ptr(blo), bhi.stride(0), ptr(rtB), NA, NB, G,
                _METRIC_CODE[metric], _PROB_CODE[prob_type], pp, 1 if accumulate else 0, ptr(GT), ldx,
                _capi.current_stream_ptr(),
            ),
            "spb_gene_cost_tc",
        )


class Morpho_pairwise:
    """Align a moving slice ``sampleA`` onto a fixed slice ``sampleB`` (same constructor as morpho_class.py:110-167).

    Extra keywords (not in the reference): ``materialize_P`` — when False ``run()`` skips building the dense
    N_A x N_B posterior (40 GB at 100k x 100k) and returns None; every other output is unaffected; ``"auto"`` builds it
    unless the cost matrix is streamed (the default of ``morpho_align``).
    ``compute_mapping`` — ``self.mapping`` (an ``ArgmaxPi``) receives the row / column maxima of the final posterior from a
    fused kernel, for ``get_optimal_mapping_relationship`` / ``mapping_aligned_coords`` without a dense P.
    ``spatial_sort`` / ``cull_zero_tiles`` — the moving cells are processed in k-d order (``kd_order``) so that each row block
    (SPB_ROW_TILE = 512 cells) and each of its four 128-cell quarters is spatially compact, and the (quarter, fixed cell) pairs
    of rows whose every pair underflows to exactly 0 in fp32 are neither read nor computed; results are bit-identical to the
    dense sweep in the same row order (all outputs are returned in the caller's row order).
    ``column_shard`` — set by ``morpho_align_pair_sharded`` and ``morpho_align_column_sharded``: one pair's fixed cells
    split over several GPUs. A shard runs
    the full EM or SVI (each rank runs its members of every batch, padded with a null column), with ``return_mapping``,
    guidance, ``sparse_calculation_mode`` and ``compute_mapping``; ``K_NB``, ``P`` (sparse COO) and ``mapping`` are gathered
    into the unsharded column order on every rank. A dense ``materialize_P=True`` is refused (NotImplementedError).
    Cost matrix: resident ([N_B][roundup(N_A, 512)] fp32, built once) whenever the pair fits the device's free memory,
    otherwise streamed — recomputed every iteration in column chunks that fit (``cost_plan`` records which, the chunk width
    and count; ``verbose`` prints it). This is chosen from the input size and the device alone, and lets one GPU align pairs
    above ~135k cells per slice (80 GB). A streamed pair supports full EM and SVI, every metric, multi-layer products, guidance,
    ``kernel_type="geodist"``, any K, ``sparse_calculation_mode``, ``return_mapping`` and ``iter_key_added``; it refuses
    (NotImplementedError) dense ``materialize_P=True``, ``compute_mapping`` and ``column_shard``. With one chunk (default SVI)
    its results are bit-identical to the resident run.
    ``transfer_B`` / ``transfer_A`` — carry cell features through the final posterior without forming it: ``P_FB = P @
    F_B`` ([N_A, F], the caller's row order of ``sampleA``) and ``PT_FA = P^T @ F_A`` ([n_cols, F], P's column order, that
    of ``K_NB``), un-normalised float32, ``None`` when not requested. Each is a float array in the slice's row order
    ([N_B, F] for ``transfer_B``, [N_A, F] for ``transfer_A``), an ``.obsm`` key, or an ``.obs`` key one-hot encoded in
    category order (``transfer_categories = {"A": [...], "B": [...]}``). The posterior is the one ``run()`` returns as P:
    that of the last E-step (sparse mode: the kept entries w >= tau_j). Under ``SVI_mode`` a transfer requires
    ``return_mapping=True``, whose closing E-step covers every fixed cell. Resident, streamed and column-sharded pairs.
    Accepted but without effect (memory work-arounds whose results are identical): ``use_chunk``, ``chunk_capacity``,
    ``pre_compute_dist``. ``sparse_calculation_mode`` keeps the top ``sparse_top_k`` posterior entries of every column by an
    exact on-device radix select (P comes back as ``scipy.sparse.coo_matrix``).
    """

    def __init__(
        self,
        sampleA,
        sampleB,
        rep_layer: Union[str, List[str]] = "X",
        rep_field: Union[str, List[str]] = "layer",
        genes=None,
        spatial_key: str = "spatial",
        key_added: str = "align_spatial",
        iter_key_added: Optional[str] = None,
        save_concrete_iter: bool = False,
        vecfld_key_added: Optional[str] = None,
        dissimilarity: Union[str, List[str]] = "kl",
        probability_type: Union[str, List[str]] = "gauss",
        probability_parameters=None,
        label_transfer_dict=None,
        use_hvg: bool = True,
        nn_init: bool = True,
        init_transform: bool = True,
        allow_flip: bool = False,
        init_layer: str = "X",
        init_field: str = "layer",
        nn_init_top_K: int = 10,
        nn_init_weight: float = 1.0,
        max_iter: int = 200,
        nonrigid_start_iter: int = 80,
        SVI_mode: bool = True,
        batch_size: Optional[int] = None,
        pre_compute_dist: bool = True,
        sparse_calculation_mode: bool = False,
        sparse_top_k: int = 1024,
        lambdaVF: Union[int, float] = 1e2,
        beta: Union[int, float] = 0.01,
        K: Union[int, float] = 15,
        kernel_type: str = "euc",
        graph=None,
        graph_knn: int = 10,
        sigma2_init_scale: Optional[Union[int, float]] = 0.1,
        sigma2_end: Optional[Union[int, float]] = None,
        gamma_a: float = 1.0,
        gamma_b: float = 1.0,
        kappa: Union[float, np.ndarray] = 1.0,
        partial_robust_level: float = 10,
        normalize_c: bool = True,
        normalize_g: bool = False,
        separate_mean: bool = True,
        separate_scale: bool = False,
        dtype: str = "float32",
        device: str = "cpu",
        verbose: bool = True,
        guidance_pair=None,
        guidance_effect=False,
        guidance_weight: float = 1.0,
        use_chunk: bool = False,
        chunk_capacity: float = 1.0,
        return_mapping: bool = False,
        update_R: bool = True,
        materialize_P: bool = True,
        compute_mapping: bool = False,
        spatial_sort: bool = True,
        cull_zero_tiles: bool = True,
        column_shard=None,
        transfer_B=None,
        transfer_A=None,
    ) -> None:
        self.verbose = verbose
        self.sampleA, self.sampleB = sampleA, sampleB
        self.rep_layer, self.rep_field, self.genes = rep_layer, rep_field, genes
        self.spatial_key, self.key_added = spatial_key, key_added
        self.iter_key_added, self.save_concrete_iter = iter_key_added, save_concrete_iter
        self.vecfld_key_added = vecfld_key_added
        self.dissimilarity, self.probability_type = dissimilarity, probability_type
        self.probability_parameters = probability_parameters
        self.label_transfer_dict = label_transfer_dict
        self.use_hvg, self.nn_init, self.init_transform = use_hvg, nn_init, init_transform
        self.nn_init_top_K, self.max_iter, self.allow_flip = nn_init_top_K, max_iter, allow_flip
        self.init_layer, self.init_field = init_layer, init_field
        self.SVI_mode, self.batch_size, self.pre_compute_dist = SVI_mode, batch_size, pre_compute_dist
        self.sparse_calculation_mode, self.sparse_top_k = sparse_calculation_mode, sparse_top_k
        self.beta, self.lambdaVF, self.K = beta, lambdaVF, int(K)
        self.kernel_type, self.kernel_bandwidth = kernel_type, beta
        self.graph, self.graph_knn = graph, graph_knn
        self.sigma2_init_scale, self.sigma2_end = sigma2_init_scale, sigma2_end
        self.partial_robust_level = partial_robust_level
        self.normalize_c, self.normalize_g = normalize_c, normalize_g
        self.separate_mean, self.separate_scale = separate_mean, separate_scale
        self.dtype, self.device = dtype, device
        self.guidance_pair, self.guidance_effect, self.guidance_weight = guidance_pair, guidance_effect, guidance_weight
        self.use_chunk, self.chunk_capacity = use_chunk, chunk_capacity
        self.nn_init_weight = nn_init_weight
        self.gamma_a, self.gamma_b, self.kappa = gamma_a, gamma_b, kappa
        self.nonrigid_start_iter = nonrigid_start_iter
        self.return_mapping, self.update_R = return_mapping, update_R
        self.materialize_P = materialize_P
        self.compute_mapping = compute_mapping
        self.spatial_sort, self.cull_zero_tiles = spatial_sort, cull_zero_tiles
        # iterations per captured graph: light iterations (SVI batches, small pairs) are bound by the host's graph launches
        # on a slow host, so several identical iterations ride in one graph; 0 = choose from the pairs per iteration
        self.graph_unroll = 0
        # column-sharded pair: (rank, world, mode) — this process holds the fixed cells [NB * rank / world, NB * (rank + 1) /
        # world) of ONE pair; see alignment/distributed.py:morpho_align_pair_sharded
        self.column_shard = column_shard
        from .distributed import Collectives

        self._shard_comm = Collectives()

        self._np_dtype = np.float32 if dtype == "float32" else np.float64
        self._check()
        self._check_transfer(transfer_B, transfer_A)
        self._lib = _capi.load_library()
        self._dev = resolve_device(device)
        with torch.cuda.device(self._dev):
            self._align_preprocess()
            self._construct_kernel()

    # ------------------------------------------------------------------------------------------------------------------
    # validation (morpho_class.py:316-440)
    # ------------------------------------------------------------------------------------------------------------------
    def _check(self):
        if self.rep_layer is None:
            raise ValueError(
                "No representation input is detected, which may not produce meaningful result. Please check the rep_layer and rep_field."
            )
        if self.rep_field is None:
            self.rep_field = "layer"
        if isinstance(self.rep_layer, str):
            self.rep_layer = [self.rep_layer]
        if isinstance(self.rep_field, str):
            self.rep_field = [self.rep_field] * len(self.rep_layer)
        if not U.check_rep_layer([self.sampleA, self.sampleB], self.rep_layer, self.rep_field):
            raise ValueError("The specified representation is not found in the attribute of the AnnData objects.")
        self.obs_key = U.check_obs(self.rep_layer, self.rep_field)
        if self.spatial_key not in self.sampleA.obsm:
            raise KeyError(f"Spatial key '{self.spatial_key}' not found in sampleA AnnData object.")
        if self.spatial_key not in self.sampleB.obsm:
            raise KeyError(f"Spatial key '{self.spatial_key}' not found in sampleB AnnData object.")
        if self.obs_key is not None and self.label_transfer_dict is not None:
            catA = self.sampleA.obs[self.obs_key].cat.categories.tolist()
            catB = self.sampleB.obs[self.obs_key].cat.categories.tolist()
            U.check_label_transfer_dict(catA, catB, self.label_transfer_dict)
        if self.dissimilarity is None:
            self.dissimilarity = "kl"
        if isinstance(self.dissimilarity, str):
            self.dissimilarity = [self.dissimilarity] * len(self.rep_layer)
        valid = ["kl", "sym_kl", "euc", "euclidean", "square_euc", "square_euclidean", "cos", "cosine", "label"]
        self.dissimilarity = [d.lower() for d in self.dissimilarity]
        for d in self.dissimilarity:
            if d not in valid:
                raise ValueError(f"Invalid `metric` value: {d}. Available `metrics` are: " f"{', '.join(valid)}.")
        if self.probability_type is None:
            self.probability_type = "gauss"
        if isinstance(self.probability_type, str):
            self.probability_type = [self.probability_type] * len(self.rep_layer)
        validp = ["gauss", "gaussian", "cos", "cosine", "prob"]
        self.probability_type = [p.lower() for p in self.probability_type]
        for p in self.probability_type:
            if p not in validp:
                raise ValueError(f"Invalid `metric` value: {p}. Available `metrics` are: " f"{', '.join(validp)}.")
        for i, f in enumerate(self.rep_field):
            if f == "obs":
                self.dissimilarity[i] = "label"
                self.probability_type[i] = "prob"
        if self.probability_parameters is None:
            self.probability_parameters = [None] * len(self.rep_layer)
        elif not isinstance(self.probability_parameters, (list, tuple)):
            self.probability_parameters = [self.probability_parameters] * len(self.rep_layer)
        self.probability_parameters = list(self.probability_parameters)
        if self.nn_init:
            if not U.check_rep_layer([self.sampleA, self.sampleB], [self.init_layer], [self.init_field]):
                raise ValueError("The specified representation is not found in the attribute of the AnnData objects.")
        if self.guidance_effect:
            valid_g = ["nonrigid", "rigid", "both"]
            if self.guidance_effect not in valid_g:
                raise ValueError(
                    f"Invalid `guidance_effect` value: {self.guidance_effect}. Available `guidance_effect` values are: "
                    f"{', '.join(valid_g)}."
                )
        # ---- features of the reference that this round does not cover: fail loudly, never silently differ ----
        if self.sparse_calculation_mode:
            self.pre_compute_dist = False  # morpho_class.py:439-440 (no effect here: residency follows the pair's size)
            if int(self.sparse_top_k) < 1:
                raise ValueError("sparse_top_k must be a positive integer.")
        if self.kernel_type not in ("euc", "geodist"):
            raise NotImplementedError(f"Kernel type '{self.kernel_type}' is not implemented.")
        if self.dtype != "float32":
            # the reference honours dtype="float64" end to end (morpho_class.py:165, utils.py:35-66); the device kernels of
            # this package compute in float32 (with fp64 reductions), so a float64 request is refused rather than served
            # with narrower arithmetic
            raise NotImplementedError(
                f"dtype={self.dtype!r} is not implemented in spateo_release_b200: the device path computes in float32 "
                "(fp64 reductions / solves); use dtype='float32'."
            )

    def _check_transfer(self, transfer_B, transfer_A):
        """Posterior-transfer features of both slices (``resolve_transfer``); under SVI only with ``return_mapping``."""
        self.P_FB = self.PT_FA = None
        self.transfer_categories = {"A": None, "B": None}
        self._FB_host = self._FA_host = None
        if transfer_B is None and transfer_A is None:
            return
        if self.SVI_mode and not self.return_mapping:
            raise ValueError("transfer_B / transfer_A under SVI_mode=True need return_mapping=True: the last SVI posterior "
                             "covers one batch of fixed cells, the closing E-step of return_mapping covers all of them")
        nA, nB = self.sampleA.obsm[self.spatial_key].shape[0], self.sampleB.obsm[self.spatial_key].shape[0]
        if transfer_B is not None:
            self._FB_host, self.transfer_categories["B"] = resolve_transfer(self.sampleB, transfer_B, nB, "transfer_B")
        if transfer_A is not None:
            self._FA_host, self.transfer_categories["A"] = resolve_transfer(self.sampleA, transfer_A, nA, "transfer_A")

    @property
    def _transfer_on(self) -> bool:
        return self._FB_host is not None or self._FA_host is not None

    def _transfer_dims(self) -> Optional[tuple]:
        """Feature counts (F_B, F_A) of the requested transfer (0 = that side not requested), None without one."""
        if not self._transfer_on:
            return None
        return tuple(0 if f is None else f.shape[1] for f in (self._FB_host, self._FA_host))

    # ------------------------------------------------------------------------------------------------------------------
    # preprocessing (morpho_class.py:443-558)
    # ------------------------------------------------------------------------------------------------------------------
    def _align_preprocess(self):
        dt = self._np_dtype
        if self.use_hvg and ("highly_variable" in self.sampleA.var.columns) and ("highly_variable" in self.sampleB.var.columns):
            gl = [
                self.sampleA.var.index[self.sampleA.var.highly_variable],
                self.sampleB.var.index[self.sampleB.var.highly_variable],
            ]
        else:
            gl = [self.sampleA.var.index, self.sampleB.var.index]
        common = U.filter_common_genes(*gl, verbose=self.verbose)
        self.genes = common if self.genes is None else U.intersect_lsts(common, list(self.genes))

        self.exp_layers_A = [U.get_rep(self.sampleA, r, f, self.genes, dt) for r, f in zip(self.rep_layer, self.rep_field)]
        self.exp_layers_B = [U.get_rep(self.sampleB, r, f, self.genes, dt) for r, f in zip(self.rep_layer, self.rep_field)]
        if self.obs_key is not None:
            self.label_transfer = U.check_label_transfer(self.sampleA, self.sampleB, self.obs_key, self.label_transfer_dict)
        else:
            self.label_transfer = None

        self.coordsA = U.check_spatial_coords(self.sampleA, self.spatial_key).astype(dt)
        self.coordsB = U.check_spatial_coords(self.sampleB, self.spatial_key).astype(dt)
        assert self.coordsA.shape[1] == self.coordsB.shape[1], "Spatial coordinate dimensions are different, please check again."
        self.NA, self.NB, self.D = self.coordsA.shape[0], self.coordsB.shape[0], self.coordsA.shape[1]
        if self.normalize_c:
            self.coordsA, self.coordsB, self.normalize_scales, self.normalize_means = U.normalize_coords(
                self.coordsA, self.coordsB, self.separate_mean, self.separate_scale
            )
        if self.normalize_g:
            self._normalize_exps()
        # guidance pairs [X_BI on the fixed slice, X_AI on the moving slice] (morpho_class.py:551-587)
        if (self.guidance_pair is not None) and (self.guidance_effect != False) and (self.guidance_weight > 0):  # noqa: E712
            if not isinstance(self.guidance_pair, list) or len(self.guidance_pair) != 2:
                raise ValueError("guidance_pair must be a list with two elements: [X_BI, X_AI].")
            self.X_BI = np.asarray(self.guidance_pair[0]).astype(dt)
            self.X_AI = np.asarray(self.guidance_pair[1]).astype(dt)
            if self.normalize_c:
                self.X_AI = (self.X_AI - self.normalize_means[0]) / self.normalize_scales[0]
                self.X_BI = (self.X_BI - self.normalize_means[1]) / self.normalize_scales[1]
            self.guidance = True
        else:
            self.guidance = False

    def _normalize_exps(self):
        """morpho_class.py:657-680: shared RMS scale for 'layer' representations whose metric is not KL."""
        for i, (f, d) in enumerate(zip(self.rep_field, self.dissimilarity)):
            if f == "layer" and d != "kl":
                sc = 0.0
                for e in (self.exp_layers_A[i], self.exp_layers_B[i]):
                    sc += np.sqrt(np.sum(e.astype(np.float64) ** 2) / e.shape[0])
                sc /= 2
                self.exp_layers_A[i] = (self.exp_layers_A[i] / sc).astype(self._np_dtype)
                self.exp_layers_B[i] = (self.exp_layers_B[i] / sc).astype(self._np_dtype)

    # ------------------------------------------------------------------------------------------------------------------
    # inducing points + kernel (morpho_class.py:825-875)
    # ------------------------------------------------------------------------------------------------------------------
    def _construct_kernel(self, inducing_idx: Optional[np.ndarray] = None):
        """Inducing points (drawn from the global ``np.random`` stream, or the moving cells ``inducing_idx`` when given) and
        the kernel matrices built from them."""
        if inducing_idx is None:
            uniq, uniq_idx = np.unique(self.coordsA, return_index=True, axis=0)
            if uniq.shape[0] > self.K:
                pick = np.random.choice(uniq.shape[0], self.K, replace=False)
            else:
                pick = np.arange(uniq.shape[0])
            inducing_idx = uniq_idx[pick]
        self.inducing_variables_idx = np.asarray(inducing_idx)
        self.inducing_variables = self.coordsA[self.inducing_variables_idx, :]
        self.K = self.inducing_variables.shape[0]
        z = self.inducing_variables.astype(np.float64)
        d2 = ((z[:, None, :] - z[None, :, :]) ** 2).sum(-1)
        self.GammaSparse = np.exp(-self.kernel_bandwidth * d2).astype(np.float32)
        if self.guidance and self.guidance_effect in ("nonrigid", "both"):
            xa = self.X_AI.astype(np.float64)
            self.U_I = np.exp(-self.kernel_bandwidth * ((xa[:, None, :] - z[None, :, :]) ** 2).sum(-1))  # [N_I, K] fp64
        else:
            self.U_I = None
        # U^T on the device from the pre-initialisation coordinates (the reference builds U before the coarse init)
        self.ldx = _round_up(self.NA, _capi.ROW_TILE)
        dev = self._dev
        if self.kernel_type == "geodist":
            self._construct_geodesic_kernel()
            return
        x_soa = torch.zeros((3, self.ldx), dtype=torch.float32, device=dev)
        x_soa[: self.D, : self.NA] = torch.from_numpy(np.ascontiguousarray(self.coordsA.T, dtype=np.float32)).to(dev)
        zt = torch.zeros((self.K, 3), dtype=torch.float32, device=dev)
        zt[:, : self.D] = torch.from_numpy(self.inducing_variables.astype(np.float32)).to(dev)
        self._UT = torch.empty((self.K, self.ldx), dtype=torch.float32, device=dev)
        check(
            self._lib.spb_rbf_kernel_T(ptr(x_soa), self.NA, self.ldx, ptr(zt), self.K, float(self.kernel_bandwidth),
                                       ptr(self._UT), _capi.current_stream_ptr()),
            "spb_rbf_kernel_T",
        )

    def _construct_geodesic_kernel(self):
        """``kernel_type="geodist"`` (morpho_class.py:865-871, utils.py:1161-1217): U = exp(-beta d_g^2) with d_g the
        shortest-path distance on the k-nearest-neighbour graph of the moving cells, from every cell to the K inducing
        cells; unreachable pairs get d_g = 1e5 like the reference. One-off host work (scipy's Dijkstra on the sparse graph
        instead of the reference's dense N x N adjacency + networkx loop), the kernel matrix then lives on the device."""
        import scipy.sparse as sp
        from scipy.sparse.csgraph import dijkstra

        N = self.NA
        if self.graph is None:
            from sklearn.neighbors import kneighbors_graph

            adj = kneighbors_graph(self.coordsA, self.graph_knn, mode="distance", include_self=False)
        elif sp.issparse(self.graph):
            adj = sp.csr_matrix(self.graph)
        else:  # a networkx graph, as the reference accepts
            import networkx

            adj = networkx.to_scipy_sparse_array(self.graph, nodelist=list(range(N)), weight="weight", format="csr")
        adj = sp.csr_matrix(adj.maximum(adj.T))  # networkx.Graph is undirected: an edge exists if either end lists it
        dist = dijkstra(adj, directed=False, indices=np.asarray(self.inducing_variables_idx, dtype=np.int64))  # [K, N]
        dist = np.where(np.isfinite(dist), dist, 1e5)
        UT64 = np.exp(-float(self.kernel_bandwidth) * dist**2)  # [K, N] float64 like the reference's
        self.GammaSparse = np.ascontiguousarray(UT64[:, self.inducing_variables_idx].T, dtype=np.float32)
        self.U_I = None  # guidance points are not nodes of the graph (morpho_class.py:871)
        self._UT = torch.zeros((self.K, self.ldx), dtype=torch.float32, device=self._dev)
        self._UT[:, :N] = torch.from_numpy(np.ascontiguousarray(UT64, dtype=np.float32)).to(self._dev)

    @property
    def U(self) -> np.ndarray:
        """[N_A, K] kernel matrix as the reference exposes it."""
        u = self._UT[:, : self.NA].T.contiguous().cpu().numpy().astype(self._np_dtype)
        return self._unsorted(u) if getattr(self, "_UT_is_sorted", False) else u

    # ------------------------------------------------------------------------------------------------------------------
    # device-side expression distances for small helper problems (coarse init, beta^2 init)
    # ------------------------------------------------------------------------------------------------------------------
    def _raw_cost_T(self, XA_host, XB_host, metric):
        """E^T[j][i] = metric(A_i, B_j) as a device tensor [nB, ldx_s] (columns beyond nA are padding).
        Inputs: host arrays or device tensors (the device voxel means are passed straight through)."""
        dev = self._dev
        gc = GeneCostBuilder(self._lib, dev)

        def up(x):
            if torch.is_tensor(x):
                return x.to(device=dev, dtype=torch.float32).contiguous()
            t = torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32))
            _count_h2d(t)
            return t.to(dev)

        A, B = up(XA_host), up(XB_host)
        opA, rtA, opB, rtB, G = gc.prepare_pair(A, B, metric)
        nA, nB = A.shape[0], B.shape[0]
        lds = _round_up(nA, 256)
        ET = torch.empty((nB, lds), dtype=torch.float32, device=dev)
        gc.cost(opA, rtA, opB, rtB, nA, nB, G, metric, "prob", None, False, ET, lds)
        return ET, nA

    # ------------------------------------------------------------------------------------------------------------------
    # coarse rigid alignment (morpho_class.py:898-1041): voxelise, mutual top-K by expression, robust Procrustes
    # ------------------------------------------------------------------------------------------------------------------
    def _coarse_rigid_alignment(self, n_sampling: int = 20000):
        top_K = self.nn_init_top_K
        ia = np.random.choice(self.NA, n_sampling, replace=False) if self.NA > n_sampling else np.arange(self.NA)
        ib = np.random.choice(self.NB, n_sampling, replace=False) if self.NB > n_sampling else np.arange(self.NB)
        cA, cB = self.coordsA[ia, :], self.coordsB[ib, :]
        N, M, D = cA.shape[0], cB.shape[0], cA.shape[1]
        import time as _time

        _t = _time.perf_counter()
        XA = self._device_rows(self.init_layer, self.init_field, "A", ia)
        XB = self._device_rows(self.init_layer, self.init_field, "B", ib)
        if XA is None or XB is None:  # an initialisation layer that is not part of the alignment: host extraction
            XA = U.get_rep(self.sampleA[ia], self.init_layer, self.init_field, self.genes, self._np_dtype)
            XB = U.get_rep(self.sampleB[ib], self.init_layer, self.init_field, self.genes, self._np_dtype)
        # the first use of the representations uploads them (staged H2D of both expression matrices) — the one upload of a run
        self._timing["coarse.upload_and_gather_s"] = _time.perf_counter() - _t
        _t = _time.perf_counter()
        cA, XA = self._voxel_data_device(cA, XA, voxel_num=max(min(int(N / 20), 1000), 100))
        cB, XB = self._voxel_data_device(cB, XB, voxel_num=max(min(int(M / 20), 1000), 100))
        self._timing["coarse.voxel_data_s"] = _time.perf_counter() - _t
        _t = _time.perf_counter()
        metric = "kl" if self.init_field == "layer" else "euc"
        ET, nA = self._raw_cost_T(XA, XB, metric)  # [nB, lds]: ET[b, a] = dist(voxel a of A, voxel b of B)
        ET = ET[:, :nA]
        nB = ET.shape[0]
        while True:
            try:
                if top_K > nA - 1 or top_K > nB - 1:  # np.argpartition(kth=top_K) needs kth < size
                    raise ValueError(f"kth(={top_K}) out of bounds")
                # for every voxel b of B: the top_K voxels a of A (reference: argpartition over axis 0 of [nA, nB])
                d1, a_idx = torch.topk(ET, top_K, dim=1, largest=False)
                NN1 = np.stack([np.repeat(np.arange(nB), top_K), a_idx.reshape(-1).cpu().numpy()], axis=1)
                dist1 = d1.reshape(-1).cpu().numpy()
                # for every voxel a of A: the top_K voxels b of B
                d2, b_idx = torch.topk(ET, top_K, dim=0, largest=False)
                NN2 = np.stack([b_idx.T.reshape(-1).cpu().numpy(), np.repeat(np.arange(nA), top_K)], axis=1)
                dist2 = d2.T.reshape(-1).cpu().numpy()
                break
            except Exception as e:
                top_K -= 1
                if top_K == 0:
                    raise RuntimeError("Failed to perform coarse rigid alignment after reducing top_K.") from e
        NN = np.vstack((NN1, NN2))
        distance = np.r_[dist1, dist2].astype(np.float64)
        train_x, train_y = cA[NN[:, 1], :], cB[NN[:, 0], :]
        self._timing["coarse.expression_knn_s"] = _time.perf_counter() - _t
        _t = _time.perf_counter()
        P, R, t, sigma2, gamma = self._inlier_from_NN_device(train_x, train_y, distance)
        self._timing["coarse.inlier_from_NN_s"] = _time.perf_counter() - _t
        self._timing["coarse.n_pairs"] = int(train_x.shape[0])
        if self.allow_flip:
            Rf = np.eye(D)
            Rf[-1, -1] = -1
            P2, R2, t2, s2, g2 = self._inlier_from_NN_device(train_x @ Rf, train_y, distance)
            if g2 > gamma:
                P, R, t, sigma2 = P2, R2 @ Rf, t2, s2
        thr = min(P[np.argsort(-P[:, 0])[20], 0], 0.5)
        keep = np.where(P[:, 0] > thr)[0]
        dt = self._np_dtype
        self.inlier_A = train_x[keep, :].astype(dt)
        self.inlier_B = train_y[keep, :].astype(dt)
        self.inlier_P = P[keep, :].astype(dt)
        self.init_R = R.astype(dt)
        self.init_t = np.asarray(t).astype(dt)
        if self.init_transform:
            self.inlier_A = self.inlier_A @ self.init_R.T + self.init_t
            self.coordsA = self.coordsA @ self.init_R.T + self.init_t

    def _voxel_data_device(self, coords: np.ndarray, gene_exp: np.ndarray, voxel_size=None, voxel_num: int = 10000):
        """``voxel_data`` (utils.py:1283-1336) on the device: returns (voxel coordinates [n_used, D] numpy, voxel mean
        expression [n_used, G] float64 DEVICE tensor). The grid axes come from the same ``np.arange`` calls as the
        reference (host, tiny); membership uses the reference's test in the coordinates' dtype (csrc/voxel.cu)."""
        dev, lib = self._dev, self._lib
        N, D = coords.shape
        if coords.dtype not in (np.float32, np.float64):
            coords = coords.astype(np.float64)
        lo, hi = np.min(coords, axis=0), np.max(coords, axis=0)
        if voxel_size is None:
            voxel_size = np.sqrt(np.prod(hi - lo)) / (np.sqrt(N) / 5)
        steps = (hi - lo) / int(np.sqrt(voxel_num))
        # np.arange on float32 scalars returns float64, so the reference's `coords - voxel_coord` is evaluated in float64
        axes = [np.ascontiguousarray(np.arange(a, b, st_), dtype=np.float64) for a, b, st_ in zip(lo, hi, steps)]
        grid = np.stack(np.meshgrid(*[np.arange(a, b, st_) for a, b, st_ in zip(lo, hi, steps)]), axis=-1).reshape(-1, D)
        radius = float(voxel_size / 2)
        is_f64 = 1
        cd = torch.from_numpy(np.ascontiguousarray(coords, dtype=np.float64)).to(dev)
        _count_h2d(cd)
        axd = [torch.from_numpy(a).to(dev) for a in axes]
        while len(axd) < 3:
            axd.append(axd[0])
        lo3 = np.zeros(3); lo3[:D] = lo.astype(np.float64)
        st3 = np.ones(3); st3[:D] = np.maximum(steps.astype(np.float64), 1e-300)
        n = [len(a) for a in axes] + [1] * (3 - D)
        counts = torch.zeros((grid.shape[0],), dtype=torch.int32, device=dev)
        stp = _capi.current_stream_ptr()
        geom = (ptr(cd), is_f64, N, D, ptr(axd[0]), n[0], ptr(axd[1]), n[1], ptr(axd[2]), n[2], radius, ptr(lo3), ptr(st3))
        check(lib.spb_voxel_count(*geom, ptr(counts), stp), "spb_voxel_count")
        used = counts > 0
        new_id = (torch.cumsum(used.to(torch.int32), 0) - 1).to(torch.int32)
        n_used = int(used.sum().item())
        if torch.is_tensor(gene_exp):
            ex = gene_exp.to(device=dev, dtype=torch.float32).contiguous()
        else:
            ex = torch.from_numpy(np.ascontiguousarray(gene_exp, dtype=np.float32)).to(dev)
            _count_h2d(ex)
        G = ex.shape[1]
        means = torch.zeros((n_used, G), dtype=torch.float64, device=dev)
        check(lib.spb_voxel_accumulate(*geom, ptr(counts), ptr(new_id), ptr(ex), G, G, ptr(means), G, stp),
              "spb_voxel_accumulate")
        return grid[used.cpu().numpy(), :], means

    def _inlier_from_NN_device(self, train_x: np.ndarray, train_y: np.ndarray, distance: np.ndarray):
        """``inlier_from_NN`` (utils.py:1220-1280) on the device: returns (P [N,1], R [D,D], t [D], sigma2, gamma)."""
        dev, lib = self._dev, self._lib
        N, D = train_x.shape
        x64 = np.zeros((N, 3)); x64[:, :D] = train_x
        y64 = np.zeros((N, 3)); y64[:, :D] = train_y
        dist = np.maximum(0, np.asarray(distance, dtype=np.float64).reshape(-1))
        dist = dist / (np.max(dist) / (np.log(10) * 2))
        area = float(np.maximum(np.prod(train_x.max(0) - train_x.min(0)), np.prod(train_y.max(0) - train_y.min(0))))
        sigma2_init = float(np.sum((train_x.astype(np.float64) - train_y.astype(np.float64)) ** 2) / (D * N))
        w0 = np.exp(-dist)
        xd, yd, dd = (torch.from_numpy(a).to(dev) for a in (x64, y64, dist))
        Pd = torch.from_numpy(w0).to(dev)
        resid = torch.empty((N,), dtype=torch.float64, device=dev)
        state = torch.zeros((128,), dtype=torch.float64, device=dev)
        out = torch.zeros((16,), dtype=torch.float64, device=dev)
        check(
            lib.spb_inlier_from_nn(ptr(xd), ptr(yd), ptr(dd), N, D, area, float(dist.min()), sigma2_init, float(w0.sum()),
                                   ptr(Pd), ptr(resid), ptr(state), ptr(out), _capi.current_stream_ptr()),
            "spb_inlier_from_nn",
        )
        o = out.cpu().numpy()
        R = o[:9].reshape(3, 3)[:D, :D].copy()
        return Pd.cpu().numpy()[:, None], R, o[9 : 9 + D].copy(), float(o[12]), float(o[13])

    # ------------------------------------------------------------------------------------------------------------------
    # variational initialisation (morpho_class.py:683-820; utils.py:1339-1354)
    # ------------------------------------------------------------------------------------------------------------------
    def _init_guess_sigma2(self, subsample: int = 20000) -> float:
        NA, NB, D = self.NA, self.NB, self.D
        sa = np.random.choice(NA, subsample, replace=False) if NA > subsample else np.arange(NA)
        sb = np.random.choice(NB, subsample, replace=False) if NB > subsample else np.arange(NB)
        xa = torch.from_numpy(self.coordsA[sa].astype(np.float64)).to(self._dev)
        xb = torch.from_numpy(self.coordsB[sb].astype(np.float64)).to(self._dev)
        total = torch.zeros((), dtype=torch.float64, device=self._dev)
        for c in range(0, xa.shape[0], 4096):
            d2 = torch.cdist(xa[c : c + 4096], xb) ** 2
            total += (d2 * d2).sum()  # the reference squares the already squared distance (utils.py:1352)
        return float(total.item()) / (D * sa.shape[0] * sa.shape[0])

    def _init_probability_parameters(self, subsample: int = 20000):
        for i, (eA, eB, d_s, p_t, p_p) in enumerate(
            zip(self.exp_layers_A, self.exp_layers_B, self.dissimilarity, self.probability_type, self.probability_parameters)
        ):
            if p_p is not None or p_t.lower() not in ("gauss", "gaussian"):
                continue
            sa = np.random.choice(self.NA, subsample, replace=False) if self.NA > subsample else np.arange(self.NA)
            sb = np.random.choice(self.NB, subsample, replace=False) if self.NB > subsample else np.arange(self.NB)
            if d_s == "label":
                ET, nA = self._raw_cost_T(eA[sa], eB[sb], d_s)
            else:  # gather the sub-samples on the device from the resident copies
                dA, dB = self._to_device_pinned(eA), self._to_device_pinned(eB)
                to_dev = lambda ix: torch.from_numpy(np.ascontiguousarray(ix, dtype=np.int64)).to(self._dev)
                ET, nA = self._raw_cost_T(dA if sa.shape[0] == self.NA else dA.index_select(0, to_dev(sa)),
                                          dB if sb.shape[0] == self.NB else dB.index_select(0, to_dev(sb)), d_s)
            mn = ET[:, :nA].min(dim=0).values  # min over fixed cells for every moving cell (utils: nx.min(exp_dist, 1))
            srt = torch.sort(mn).values
            val = float(srt[int(sa.shape[0] * 0.05)].item()) / 5
            self.probability_parameters[i] = np.maximum(np.asarray(val, dtype=self._np_dtype), np.asarray(0.01, dtype=self._np_dtype))
            del ET

    def _initialize_variational_variables(self):
        dt = self._np_dtype
        self.sigma2 = np.asarray(self.sigma2_init_scale * self._init_guess_sigma2(), dtype=dt)
        self._sigma2_init = float(self.sigma2)
        self._init_probability_parameters()
        self.sigma2_variance = 1.0
        self.sigma2_variance_end = float(self.partial_robust_level)
        self.sigma2_variance_decress = float(np.power(np.asarray(self.sigma2_variance_end / self.sigma2_variance, dtype=dt), 1 / 100))
        if isinstance(self.kappa, float):
            self.kappa = np.ones((self.NA,), dtype=dt) * self.kappa
        elif isinstance(self.kappa, np.ndarray):
            self.kappa = self.kappa.astype(dt)
        else:
            raise ValueError("kappa should be a float or a numpy array.")
        self.gamma = np.asarray(0.5, dtype=dt)
        self.samples_s = float(
            np.maximum(
                np.prod(self.coordsA.max(axis=0) - self.coordsA.min(axis=0)),
                np.prod(self.coordsB.max(axis=0) - self.coordsB.min(axis=0)),
            )
        )
        self.outlier_s = self.samples_s * self.NA
        self.nonrigid_flag = False
        if self.SVI_mode:
            if self.batch_size is None:
                self.batch_size = min(max(int(self.NB / 10), 1000), self.NB)
            else:
                self.batch_size = min(self.batch_size, self.NB)
            self.batch_perm = np.random.permutation(self.NB)

    # ------------------------------------------------------------------------------------------------------------------
    # device state
    # ------------------------------------------------------------------------------------------------------------------
    def _set_row_order(self):
        """Processing order of the moving cells (after the coarse initialisation moved them)."""
        if self.spatial_sort and self.NA > _capi.ROW_TILE:
            self._perm = kd_order(self.coordsA, _capi.ROW_TILE, _capi.ROW_TILE // 4)
            self._perm_dev = torch.from_numpy(self._perm).to(self._dev)
        else:
            self._perm, self._perm_dev = None, None

    def _sorted(self, host_rows: np.ndarray) -> np.ndarray:
        return host_rows if self._perm is None else host_rows[self._perm]

    def _unsorted(self, sorted_rows: np.ndarray) -> np.ndarray:
        if self._perm is None:
            return sorted_rows
        out = np.empty_like(sorted_rows)
        out[self._perm] = sorted_rows
        return out

    def _build_gene_cost(self):
        """GT[j][i] = prod_layers prob(metric(A_i, B_j)) (morpho_class.py:265-268 + utils.py:1080-1081). Resident: every
        row is written once, from one layer's operands at a time. Streamed: the operands of every layer are kept for the
        run, and every iteration refills one [width][ldx] chunk column chunk by column chunk (``_chunk_cost``)."""
        dev = self._dev
        self._set_row_order()
        c0, c1 = self._col_range()
        nb_loc = c1 - c0
        self._plan_cost(nb_loc)
        self._gc = GeneCostBuilder(self._lib, dev)
        specs = list(zip(self.exp_layers_A, self.exp_layers_B, self.dissimilarity, self.probability_type,
                         self.probability_parameters))
        if self.cost_plan.streamed:
            width = self.cost_plan.width
            self._layers = [self._cost_layer(c0, c1, *spec) for spec in specs]
            if self.SVI_mode:  # an SVI chunk's fixed-side operands, gathered from its columns every iteration
                for L in self._layers:
                    L["g"] = {f: torch.empty((width,) + t.shape[1:], dtype=t.dtype, device=dev) for f, t in L["B"].items()}
            self._GT = torch.empty((width, self.ldx), dtype=torch.float32, device=dev)
            self.cost_events = None  # a list: (start, end) CUDA events around the cost of every chunk are appended to it
        else:
            # an SVI shard pads its iterations to one width with the null column nb_loc: an all-zero cost row
            self._null_column = self.column_shard is not None and self.SVI_mode
            self._GT = torch.empty((nb_loc + int(self._null_column), self.ldx), dtype=torch.float32, device=dev)
            if self._null_column:
                self._GT[nb_loc:].zero_()
            for k, spec in enumerate(specs):
                self._write_cost(k, self._cost_layer(c0, c1, *spec), 0, nb_loc)
        self.__dict__.pop("_dev_rep", None)  # the resident copies of the representations are no longer needed

    def _cost_layer(self, c0: int, c1: int, eA, eB, d_s, p_t, p_p) -> dict:
        """Device operands of one layer against this process's fixed cells [c0, c1): the label indices, or the tf32 hi / lo
        operands of ``GeneCostBuilder.split_pair``. ``B`` holds the fixed side, whose row j is fixed cell c0 + j."""
        dev = self._dev
        if d_s == "label":
            return dict(metric=d_s,
                        la=torch.from_numpy(np.ascontiguousarray(self._sorted(eA), dtype=np.int32)).to(dev),
                        LT=torch.from_numpy(np.ascontiguousarray(self.label_transfer, dtype=np.float32)).to(dev),
                        B=dict(lb=torch.from_numpy(np.ascontiguousarray(eB[c0:c1], dtype=np.int32)).to(dev)))
        A = self._to_device_pinned(eA)
        if self._perm is not None:
            A = A.index_select(0, self._perm_dev)  # moving cells in processing order
        B = self._to_device_pinned(eB) if self.column_shard is None else staged_to_device(eB[c0:c1], dev)
        L = self._gc.split_pair(*self._gc.prepare_pair(A, B, d_s))
        fixed = {f: L.pop(f) for f in ("bhi", "blo", "rtB")}
        L.update(metric=d_s, p_t=p_t, p_p=p_p, B={f: t for f, t in fixed.items() if t is not None})
        return L

    def _write_cost(self, k: int, L: dict, c0: int, c1: int, idx: Optional[torch.Tensor] = None):
        """Cost rows of layer ``k`` (operands ``L`` of ``_cost_layer``) into ``_GT``: row j from the fixed-side row c0 + j,
        or, given ``idx`` (an SVI chunk's columns), from row idx[j], gathered first. Layer 0 writes, later layers multiply."""
        n = c1 - c0
        if idx is None:
            B = {f: t[c0:c1] for f, t in L["B"].items()}
        else:
            B = L["g"]
            for f, t in L["B"].items():
                self._gather(t, idx, n, B[f])
        if L["metric"] == "label":
            check(self._lib.spb_label_cost(ptr(L["la"]), ptr(B["lb"]), ptr(L["LT"]), L["LT"].shape[1], self.NA, n, int(k > 0),
                                           ptr(self._GT), self.ldx, _capi.current_stream_ptr()), "spb_label_cost")
        else:
            self._gc.cost_split(L["ahi"], L["alo"], L["rtA"], B["bhi"], B["blo"], B.get("rtB"), self.NA, n, L["G"],
                                L["metric"], L["p_t"], L["p_p"], k > 0, self._GT, self.ldx)

    def _cost_features(self) -> int:
        """Features of the expression operands of all layers together (sym_kl contracts over both of its halves)."""
        return sum(0 if d == "label" else (2 * _round_up(e.shape[1], 32) if d == "sym_kl" else e.shape[1])
                   for e, d in zip(self.exp_layers_A, self.dissimilarity))

    def _plan_cost(self, nb_loc: int):
        """Resident or streamed cost matrix, from the pair's size and the memory the device has (``plan_cost``)."""
        cols = min(self.batch_size, nb_loc) if self.SVI_mode else nb_loc
        n_sms = torch.cuda.get_device_properties(self._dev).multi_processor_count
        plan = plan_cost(self.NA, nb_loc, self._cost_features(), cols, _device_budget(self._dev), n_sms,
                         transfer=self._transfer_dims())
        if isinstance(self.materialize_P, str) and self.materialize_P == "auto":  # the public drivers' default
            self.materialize_P = not plan.streamed
        if plan.streamed:
            why = None
            if self.column_shard is not None:
                why = "column_shard: a column-sharded pair keeps its block of the cost matrix resident"
            elif self.compute_mapping:
                why = "compute_mapping: the posterior maxima are read from the resident cost matrix after the run"
            elif self.materialize_P and not self.sparse_calculation_mode:
                why = "materialize_P=True: a dense P is as large as the cost matrix that does not fit"
            if why is not None:
                raise NotImplementedError(
                    f"the cost matrix of this pair ({plan.need} bytes streamed, {plan.budget} available) does not fit the "
                    f"device and is streamed in column chunks, which does not support {why}")
        self.cost_plan = plan
        if self.verbose:
            if plan.streamed:
                print(f"|-----> Cost matrix streamed: {plan.n_chunks} chunk(s) of {plan.width} columns per iteration "
                      f"({plan.need / 2**30:.1f} GiB of {plan.budget / 2**30:.1f} GiB).")
            else:
                print(f"|-----> Cost matrix resident ({plan.need / 2**30:.1f} GiB of {plan.budget / 2**30:.1f} GiB).")

    @property
    def _streamed(self) -> bool:
        plan = getattr(self, "cost_plan", None)
        return plan is not None and plan.streamed

    def _gather(self, src: torch.Tensor, idx: torch.Tensor, n: int, dst: torch.Tensor):
        """dst[:n] = src[idx[:n]] (rows of 4-byte words) on the device."""
        width = src.shape[1] if src.dim() == 2 else 1
        ld_src = src.stride(0) if src.dim() == 2 else 1
        ld_dst = dst.stride(0) if dst.dim() == 2 else 1
        check(self._lib.spb_gather_rows(ptr(src), ld_src, width, ptr(idx), n, ptr(dst), ld_dst, _capi.current_stream_ptr()),
              "spb_gather_rows")

    def _chunk_cost(self, c0: int, c1: int, idx: Optional[torch.Tensor]):
        """Cost rows of one column chunk into ``_GT`` (row j = column c0 + j of the iteration): the fixed cells [c0, c1)
        when ``idx`` is None, else the fixed cells ``idx`` (this iteration's row of the chunk's SVI schedule), whose
        operands are gathered first."""
        ev = self.cost_events
        if ev is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
        for k, L in enumerate(self._layers):
            self._write_cost(k, L, c0, c1, idx)
        if ev is not None:
            e1.record()
            ev.append((e0, e1))

    def _col_range(self):
        """Fixed cells (columns of P) held by this process: all of them, or this rank's block of a column-sharded pair."""
        from .distributed import column_block

        if self.column_shard is None:
            return 0, self.NB
        return column_block(self.NB, int(self.column_shard[0]), int(self.column_shard[1]))

    def _to_device_pinned(self, host_array: np.ndarray) -> torch.Tensor:
        """Device copy of one dense representation, uploaded ONCE per preparation (the coarse initialisation, the beta^2
        initialisation and the cost matrix all read it): straight from pinned memory when ``pin_inputs`` staged it,
        otherwise through the reusable pinned staging buffers."""
        key = id(host_array)
        dcache = self.__dict__.setdefault("_dev_rep", {})
        if key in dcache:
            return dcache[key]
        cache = self.__dict__.setdefault("_pinned", {})
        self._h2d_bytes = getattr(self, "_h2d_bytes", 0) + host_array.size * 4
        if key in cache:
            _count_h2d(cache[key])
            t = cache[key].to(self._dev, non_blocking=True)
        else:
            t = staged_to_device(host_array, self._dev)
        dcache[key] = t
        return t

    def _device_rows(self, layer: str, field: str, side: str, idx: np.ndarray):
        """Rows ``idx`` of a dense representation as a device tensor, gathered on the device when the representation is
        one of the alignment's own layers (the usual case: init_layer == rep_layer); None when it is not."""
        for r, f, eA, eB in zip(self.rep_layer, self.rep_field, self.exp_layers_A, self.exp_layers_B):
            if r == layer and f == field and f != "obs":
                full = self._to_device_pinned(eA if side == "A" else eB)
                if idx.shape[0] == full.shape[0] and np.array_equal(idx, np.arange(full.shape[0])):
                    return full
                return full.index_select(0, torch.from_numpy(np.ascontiguousarray(idx, dtype=np.int64)).to(self._dev))
        return None

    def pin_inputs(self):
        """Stage the dense representations in pinned host memory ahead of time (part of preprocessing)."""
        for e in list(self.exp_layers_A) + list(self.exp_layers_B):
            if e.dtype.kind == "f":
                key = id(e)
                cache = self.__dict__.setdefault("_pinned", {})
                if key not in cache:
                    t = torch.from_numpy(np.ascontiguousarray(e, dtype=np.float32))
                    cache[key] = t if t.is_pinned() else t.pin_memory()

    @staticmethod
    def _choose_segments(nrb: int, nbb: int, n_sms: int, max_cols: int = 4096) -> int:
        """Column segments so that CTAs ~ a multiple of the resident CTA slots (n_sms x 2048 / ROW_TILE) and a segment is at most ``max_cols`` columns
        (short CTAs keep the tail of the last wave small once culling has shortened the column lists)."""
        max_seg = max(1, nbb // _capi.COL_STAGE)
        slots = n_sms * (2048 // _capi.ROW_TILE)  # resident CTAs of the sweeps
        seg = 1
        for waves in range(1, 256):
            seg = max(1, min(max_seg, (slots * waves) // max(nrb, 1)))
            if (nbb + seg - 1) // seg <= max_cols or seg == max_seg:
                break
        return seg

    def _allocate_state(self):
        dev, D, NA, K, ldx = self._dev, self.D, self.NA, self.K, self.ldx
        f32, f64 = torch.float32, torch.float64
        c0, c1 = self._col_range()
        NB = c1 - c0  # columns held by this process (all of them unless the pair is column-sharded)
        if self.column_shard is not None and self.materialize_P and not self.sparse_calculation_mode:
            raise NotImplementedError("materialize_P=True (dense) on a column-sharded pair: the N_A x N_B posterior does not fit "
                                      "one host; use sparse_calculation_mode=True or compute_mapping=True")
        sched = svi_schedule(self.batch_perm, self.max_iter, self.batch_size) if self.SVI_mode else None
        self._shard_pos = None
        self.__dict__.pop("_shard_pos_cache", None)
        if self.SVI_mode and self.column_shard is not None:
            # this rank's columns of every batch, padded to one width with the null column NB (_build_gene_cost)
            sched_local, self._shard_pos = shard_svi_schedule(sched, self.NB, int(self.column_shard[0]),
                                                              int(self.column_shard[1]))
        nbb = self.batch_size if self.SVI_mode else NB
        if self._shard_pos is not None:
            nbb = sched_local.shape[1]
        nbb_alloc = NB if (self.return_mapping and self.SVI_mode) else nbb
        self._NBb = nbb
        nrb = ldx // _capi.ROW_TILE
        # per-column buffers hold every column of an E-step, or one column chunk of it when the cost matrix is streamed
        width = self.cost_plan.width if self._streamed else nbb_alloc
        self._nbb_pad = _round_up(width, 8) + 8
        s = {}
        s["xa"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["xa"][:D, :NA] = torch.from_numpy(np.ascontiguousarray(self._sorted(self.coordsA).T, dtype=np.float32)).to(dev)
        s["xb4"] = torch.zeros((NB + int(self._shard_pos is not None), 4), dtype=f32, device=dev)
        s["xb4"][:NB, :D] = torch.from_numpy(self.coordsB[c0:c1].astype(np.float32)).to(dev)
        if self._shard_pos is not None:
            s["xb4"][NB, :3] = _NULL_COLUMN_COORD
        s["Gamma"] = torch.from_numpy(np.ascontiguousarray(self.GammaSparse, dtype=np.float32)).to(dev)
        s["kappa"] = torch.ones((ldx,), dtype=f32, device=dev)
        s["kappa"][:NA] = torch.from_numpy(self._sorted(self.kappa).astype(np.float32)).to(dev)
        if self._perm is not None and not getattr(self, "_UT_is_sorted", False):
            ut = torch.zeros_like(self._UT)
            ut[:, :NA] = self._UT[:, :NA].index_select(1, self._perm_dev)
            self._UT, self._UT_is_sorted = ut, True
        s["alpha"] = torch.ones((ldx,), dtype=f32, device=dev)
        s["SigmaDiag"] = torch.zeros((ldx,), dtype=f32, device=dev)
        s["lm"] = torch.zeros((ldx,), dtype=f32, device=dev)
        s["mm"] = torch.zeros((ldx,), dtype=f32, device=dev)
        s["VnA"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["RnA"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["XAHat"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["XAHat"][:, NA:] = 1e18  # pad rows sit infinitely far from every fixed cell
        for k in ("K_NA", "K_NA_spatial", "K_NA_sigma2"):
            s[k] = torch.zeros((ldx,), dtype=f32, device=dev)
        s["PXB"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["PXB_term"] = torch.zeros((3, ldx), dtype=f32, device=dev)
        s["K_NB"] = torch.zeros((_round_up(nbb_alloc, 8) + 8,), dtype=f32, device=dev)
        s["colgeom"] = torch.zeros((self._nbb_pad, 8), dtype=f32, device=dev)
        s["colconst"] = torch.zeros((self._nbb_pad, _capi.CONST["SPB_COLCONST_FLOATS"]), dtype=f32, device=dev)
        s["colpart"] = torch.zeros((nrb, 4, self._nbb_pad), dtype=f32, device=dev)
        s["keepmask"] = torch.zeros((nrb, (self._nbb_pad + 31) // 32), dtype=torch.int32, device=dev)
        s["livemask"] = torch.zeros_like(s["keepmask"])
        s["keepoff"] = torch.zeros((nrb, (self._nbb_pad + 31) // 32, 2), dtype=torch.int32, device=dev)
        n_sms = torch.cuda.get_device_properties(dev).multi_processor_count
        seg = self._choose_segments(nrb, min(nbb, width), n_sms)  # column segments of both sweeps
        seg_alloc = max(seg, self._choose_segments(nrb, width, n_sms))
        s["rowpart"] = torch.zeros((seg_alloc, 8, ldx), dtype=f32, device=dev)
        s["bbox"] = torch.zeros((nrb, 4, 8), dtype=f32, device=dev)
        s["collist"] = torch.zeros((nrb, self._nbb_pad), dtype=torch.int32, device=dev)
        s["colquarters"] = torch.zeros((nrb, self._nbb_pad), dtype=torch.uint8, device=dev)
        s["colspatial"] = torch.zeros((nrb, self._nbb_pad), dtype=torch.uint8, device=dev)
        s["colcount"] = torch.zeros((nrb,), dtype=torch.int32, device=dev)
        s["colsplit"] = torch.zeros((nrb,), dtype=torch.int32, device=dev)
        if self.sparse_calculation_mode:
            s["colmask"] = torch.zeros((self._nbb_pad, _capi.CONST["SPB_COLMASK_WORDS"]), dtype=torch.int32, device=dev)
        s["UtWU"] = torch.zeros((K, K), dtype=f64, device=dev)
        s["UtPXB"] = torch.zeros((K, 3), dtype=f64, device=dev)
        s["SigmaInv"] = torch.zeros((K, K), dtype=f64, device=dev)
        s["Sigma"] = torch.zeros((K, K), dtype=f64, device=dev)
        s["Coff"] = torch.zeros((K, 3), dtype=f64, device=dev)
        s["moments"] = torch.zeros((32,), dtype=f64, device=dev)
        s["trace_buf"] = torch.zeros((max(self.max_iter, 1), _capi.TRACE_STRIDE), dtype=f64, device=dev)
        s["optimal"] = torch.zeros((12,), dtype=f64, device=dev)
        if self.SVI_mode:
            self.batch_idx = sched[self.max_iter - 1].astype(np.int64) if self.max_iter > 0 else None
            s["batch_idx"] = torch.from_numpy(sched if self._shard_pos is None else sched_local).to(dev)
            if self._streamed:
                s["chunk_sched"] = [torch.from_numpy(q).to(dev) for q in svi_chunk_schedules(sched, self.cost_plan.chunks)]
        else:
            s["batch_idx"] = None
        if self._streamed:  # fp64 row statistics, summed over the column chunks of an E-step (spb_row_fold)
            s["rowstat"] = torch.zeros((2 * 8 * ldx,), dtype=f64, device=dev)
        # scalars
        sc = SpbScalars()
        sc.sigma2 = float(self._sigma2_init)
        sc.sigma2_variance = 1.0
        sc.gamma = 0.5
        sc.iter = -1  # device-side iteration counter: graph replays advance it (spb_em_iteration_ex)
        for q in range(9):
            sc.R[q] = 1.0 if q in (0, 4, 8) else 0.0
        host_sc = np.frombuffer(bytes(sc), dtype=np.uint8).copy()
        s["sc"] = torch.from_numpy(host_sc).to(dev)
        self._state = s
        self._P_captured = False  # set by _capture_begin: this state's final posterior has been captured
        self.__dict__.pop("_graphs", None)  # captured iteration graphs hold the old state's pointers
        # params
        p = SpbEmParams()
        p.NA, p.NB, p.NBb, p.D, p.K, p.ldx = NA, NB, nbb, D, K, ldx
        # the whole iteration's column count: all fixed cells, or the SVI batch, of which this shard sees its part
        p.NB_total = 0 if self.column_shard is None else (self.batch_size if self.SVI_mode else self.NB)
        # block partials + tickets of the ordered (reproducible) grid reductions
        n_red = max(592 * 29, ((NA + 255) // 256) * 4, 320 * K * (K + 3) if K <= 32 else 0) + 64
        s["red_scratch"] = torch.zeros((n_red,), dtype=f64, device=dev)
        s["red_counter"] = torch.zeros((8,), dtype=torch.int32, device=dev)
        p.red_scratch, p.red_scratch_doubles, p.red_counter = s["red_scratch"].data_ptr(), n_red, s["red_counter"].data_ptr()
        p.shard_rank = p.shard_world = 0
        p.rowstat = p.peer_rowstat = p.shard_flags = p.peer_flags = None
        if self.column_shard is not None:
            self._setup_column_shard(p, s)
        if self._streamed:
            p.rowstat = s["rowstat"].data_ptr()
        p.svi, p.nn_init, p.update_R = int(self.SVI_mode), int(self.nn_init), int(self.update_R)
        p.nonrigid_start_iter = int(self.nonrigid_start_iter)
        p.seg1, p.seg2, p.nbb_pad, p.trace = seg, seg, self._nbb_pad, 1
        p.cull = int(bool(self.cull_zero_tiles))
        p.sparse_k = int(self.sparse_top_k) if self.sparse_calculation_mode else 0
        p.lambdaVF, p.gamma_a, p.gamma_b = float(self.lambdaVF), float(self.gamma_a), float(self.gamma_b)
        p.samples_s = float(self.samples_s)
        p.pinv_eps = self._pinv_eps()
        p.nn_init_weight = float(self.nn_init_weight)
        p.sigma2_variance_decress = float(self.sigma2_variance_decress)
        p.sigma2_variance_end = float(self.sigma2_variance_end)
        if self.nn_init:
            Pn = self.inlier_P.astype(np.float64)[:, 0]
            a = np.zeros((Pn.shape[0], 3))
            b = np.zeros((Pn.shape[0], 3))
            a[:, :D] = self.inlier_A.astype(np.float64)
            b[:, :D] = self.inlier_B.astype(np.float64)
            p.inl_SP = float(Pn.sum())
            Sa, Sb = Pn @ a, Pn @ b
            Mab = (a * Pn[:, None]).T @ b
            for d in range(3):
                p.inl_Sa[d], p.inl_Sb[d] = float(Sa[d]), float(Sb[d])
            for q in range(9):
                p.inl_Mab[q] = float(Mab.reshape(-1)[q])
        else:
            p.inl_SP = 1.0
        if self.guidance:
            NI = self.X_AI.shape[0]
            pad = lambda a: np.pad(np.asarray(a, dtype=np.float64), ((0, 0), (0, 3 - a.shape[1])))
            s["g_XA"] = torch.from_numpy(pad(self.X_AI)).to(dev)
            s["g_XB"] = torch.from_numpy(pad(self.X_BI)).to(dev)
            s["g_VA"] = torch.zeros((NI, 3), dtype=f64, device=dev)
            s["g_RA"] = torch.zeros((NI, 3), dtype=f64, device=dev)
            UI = self.U_I if self.U_I is not None else np.zeros((NI, K))
            s["g_UI"] = torch.from_numpy(np.ascontiguousarray(UI, dtype=np.float64)).to(dev)
            s["g_G1"] = torch.from_numpy(np.ascontiguousarray(UI.T @ UI, dtype=np.float64)).to(dev)
            p.g_on, p.g_NI = 1, NI
            p.g_nonrigid = int(self.guidance_effect in ("nonrigid", "both"))
            p.g_rigid = int(self.guidance_effect in ("rigid", "both"))
            p.g_weight = float(self.guidance_weight)
            p.g_meanXB, p.g_meanXA = float(self.X_BI.astype(np.float64).mean()), float(self.X_AI.astype(np.float64).mean())
            for name in ("g_XA", "g_XB", "g_VA", "g_RA", "g_UI", "g_G1"):
                setattr(p, name, s[name].data_ptr())
        p.GT, p.UT = ptr(self._GT).value, ptr(self._UT).value
        for name in ("xa", "xb4", "Gamma", "kappa", "batch_idx", "alpha", "SigmaDiag", "lm", "mm", "VnA", "RnA", "XAHat",
                     "K_NA", "K_NA_spatial", "K_NA_sigma2", "PXB", "PXB_term", "K_NB", "colgeom", "colconst", "colpart", "keepmask",
                     "livemask", "keepoff", "rowpart", "bbox", "collist", "colquarters", "colspatial", "colcount", "colsplit", "UtWU", "UtPXB", "SigmaInv", "Sigma", "Coff", "moments", "sc",
                     "trace_buf"):
            t = s[name]
            setattr(p, name, None if t is None else t.data_ptr())
        # eigenbasis of the previous non-rigid solve (warm start of the in-library Jacobi); [0] = K once valid
        s["jacobi_ws"] = torch.zeros((1 + K * K,), dtype=f64, device=dev) if K <= _capi.MAX_K_FUSED else None
        p.jacobi_ws = None if s["jacobi_ws"] is None else s["jacobi_ws"].data_ptr()
        p.colmask = s["colmask"].data_ptr() if "colmask" in s else None
        # K^T P K contraction: wgmma (3xTF32) above 32 inducing points, exact fp64 SIMT kernel for small K
        if K > 32:
            if "UT_hi" not in self.__dict__.setdefault("_gram", {}) or self._gram["UT_hi"].shape != self._UT.shape:
                hi, lo = torch.empty_like(self._UT), torch.empty_like(self._UT)
                mean = torch.empty((K,), dtype=f32, device=dev)
                check(self._lib.spb_gram_center(ptr(self._UT), ldx, NA, K, ptr(mean), ptr(hi), ptr(lo), _capi.current_stream_ptr()),
                      "spb_gram_center")
                need = C.c_int64(0)
                check(self._lib.spb_gram_tc_scratch_floats(K, 3, NA, C.byref(need)), "spb_gram_tc_scratch_floats")
                self._gram = dict(
                    UT_hi=hi, UT_lo=lo, mean=mean,
                    GB_hi=torch.zeros((K + 4, ldx), dtype=f32, device=dev), GB_lo=torch.zeros((K + 4, ldx), dtype=f32, device=dev),
                    scratch=torch.empty((need.value,), dtype=f32, device=dev), sums=torch.zeros((4,), dtype=f64, device=dev),
                )
            g = self._gram
            p.UT_hi, p.UT_lo, p.UT_mean = g["UT_hi"].data_ptr(), g["UT_lo"].data_ptr(), g["mean"].data_ptr()
            p.GB_hi, p.GB_lo, p.gram_sums = g["GB_hi"].data_ptr(), g["GB_lo"].data_ptr(), g["sums"].data_ptr()
            p.gram_scratch, p.gram_scratch_floats = g["scratch"].data_ptr(), g["scratch"].numel()
        else:
            p.UT_hi = p.UT_lo = p.UT_mean = p.GB_hi = p.GB_lo = p.gram_scratch = p.gram_sums = None
            p.gram_scratch_floats = 0
        self._params = p
        if self._transfer_on:
            self._allocate_transfer(s, NB, nrb)

    def _allocate_transfer(self, s, nb_loc: int, nrb: int):
        """Device buffers of the posterior transfer: F_B [nb_loc + 1][ldf] (this process's fixed cells, then the zero row of
        an SVI shard's null column; ldf = F rounded up to the panel width, so every panel row is 64-byte aligned), F_A
        [roundup(F, panel)][ldx] in processing order, the fp64 P @ F_B accumulator [ldf][ldx], and the partials of the two
        kernels: [segments][panel][ldx] (P @ F_B) and [row blocks][panel][nbb_pad] by list position (P^T @ F_A)."""
        W, dev, ldx, f32 = _capi.CONST["SPB_TRANSFER_PANEL"], self._dev, self.ldx, torch.float32
        if self._FB_host is not None:
            c0, c1 = self._col_range()
            F = self._FB_host.shape[1]
            fb = torch.zeros((nb_loc + 1, _round_up(F, W)), dtype=f32, device=dev)
            fb[:nb_loc, :F] = torch.from_numpy(self._FB_host[c0:c1]).to(dev)
            s["xfer_FB"] = fb
            s["xfer_PFB"] = torch.zeros((fb.shape[1], ldx), dtype=torch.float64, device=dev)
            s["xfer_rowpart"] = torch.zeros((s["rowpart"].shape[0], W, ldx), dtype=f32, device=dev)
        if self._FA_host is not None:
            F = self._FA_host.shape[1]
            fa = torch.zeros((_round_up(F, W), ldx), dtype=f32, device=dev)
            fa[:F, : self.NA] = torch.from_numpy(np.ascontiguousarray(self._sorted(self._FA_host).T)).to(dev)
            s["xfer_FA"] = fa
            s["xfer_colpart"] = torch.zeros((nrb, W, self._nbb_pad), dtype=f32, device=dev)

    def _transfer_begin(self):
        """Output of P^T @ F_A for the columns of the E-step about to be captured (P @ F_B accumulates in xfer_PFB)."""
        if self._FA_host is not None:
            self._xfer_PTFA = torch.zeros((self._NBb, self._FA_host.shape[1]), dtype=torch.float32, device=self._dev)

    def _transfer_capture(self, q: SpbEmParams, it: int, st, c0: int = 0):
        """P @ F_B and P^T @ F_A of the E-step that ``q`` describes, while its lists and column constants are live: the
        whole E-step, or its column chunk [c0, c0 + q.NBb) (P @ F_B is added in chunk order through ``q.fold_add``)."""
        lib, s = self._lib, self._state
        if self._FB_host is not None:
            fb = s["xfer_FB"]
            # the F_B rows follow xb4: a full-EM chunk's columns are fixed cells c0.., an SVI chunk's schedule is global
            base = fb.data_ptr() + (0 if q.svi else c0) * fb.shape[1] * 4
            check(lib.spb_posterior_transfer_rows(C.byref(q), it, C.c_void_p(base), fb.shape[1], self._FB_host.shape[1],
                                                  ptr(s["xfer_rowpart"]), ptr(s["xfer_PFB"]), st),
                  "spb_posterior_transfer_rows")
        if self._FA_host is not None:
            F = self._FA_host.shape[1]
            out = self._xfer_PTFA[c0:]
            check(lib.spb_posterior_transfer_cols(C.byref(q), it, ptr(s["xfer_FA"]), F, ptr(s["xfer_colpart"]), ptr(out), F,
                                                  st), "spb_posterior_transfer_cols")

    def _transfer_results(self, n_cols: int):
        """``P_FB`` (caller's row order) and ``PT_FA`` (P's column order) of the captured posterior, float32 like the other
        outputs. A column-sharded pair sums the ranks' P @ F_B in fp64 in rank order and gathers P^T @ F_A by column."""
        s = self._state
        if self._FB_host is not None:
            acc = s["xfer_PFB"]
            if self.column_shard is not None:  # the collective, whatever sums the row statistics
                self._shard_comm.sum_(self, acc)
            pfb = acc[: self._FB_host.shape[1], : self.NA].T.contiguous().to(torch.float32)
            _count_d2h(pfb)
            self.P_FB = self._unsorted(pfb.cpu().numpy())
        if self._FA_host is not None:
            t = self._xfer_PTFA
            self.PT_FA = self._shard_columns(t, n_cols) if self.column_shard is not None else t.cpu().numpy()
            self._xfer_PTFA = None

    def _setup_column_shard(self, p, s):
        """Buffers of the column-sharded pair: fp64 row statistics of this rank's columns (double-buffered) + epoch flags.
        ``mode`` "p2p" (default when available): the buffer is symmetric memory, every rank maps every peer's copy and the
        row-finalize kernel sums them straight over NVLink; "nccl": plain buffer + ``all_reduce`` (the baseline)."""
        import torch.distributed as dist

        rank, world = int(self.column_shard[0]), int(self.column_shard[1])
        mode = self.column_shard[2] if len(self.column_shard) > 2 else "auto"
        dev, ldx = self._dev, self.ldx
        n_stat = 2 * 8 * ldx
        p.shard_rank, p.shard_world = rank, world
        self._shard_epoch = 0
        self._shard_mode = "nccl"
        buf = None
        if mode in ("auto", "p2p") and world > 1:
            try:
                import torch.distributed._symmetric_memory as symm

                buf = symm.empty((n_stat + 64,), dtype=torch.float64, device=dev)
                buf.zero_()
                try:
                    hdl = symm.rendezvous(buf, dist.group.WORLD.group_name)
                except Exception:
                    hdl = symm.rendezvous(buf, dist.group.WORLD)
                ptrs = [int(q) for q in hdl.buffer_ptrs]
                s["shard_hdl"] = hdl
                s["peer_rowstat"] = torch.tensor(ptrs, dtype=torch.int64, device=dev)
                s["peer_flags"] = torch.tensor([q + n_stat * 8 for q in ptrs], dtype=torch.int64, device=dev)
                p.peer_rowstat, p.peer_flags = s["peer_rowstat"].data_ptr(), s["peer_flags"].data_ptr()
                self._shard_mode = "p2p"
                hdl.barrier()
            except Exception as e:  # no symmetric memory on this system: fall back to the collective
                if mode == "p2p":
                    raise
                buf = None
                self._shard_fallback_reason = repr(e)
        if buf is None:
            buf = torch.zeros((n_stat + 64,), dtype=torch.float64, device=dev)
        s["rowstat"] = buf
        p.rowstat = buf.data_ptr()
        p.shard_flags = buf.data_ptr() + n_stat * 8

    def _shard_fold(self, st) -> torch.Tensor:
        """Column-sharded pair: fold this rank's row partials of the E-step into the fp64 row statistics; returns the view
        that the ranks sum."""
        parity = self._shard_epoch & 1
        self._shard_epoch += 1
        check(self._lib.spb_row_fold(C.byref(self._params), parity, st), "spb_row_fold")
        return self._state["rowstat"][parity * 8 * self.ldx : (parity + 1) * 8 * self.ldx]

    def _shard_sum(self, view: torch.Tensor, st):
        """Sum the view of ``_shard_fold`` over the ranks, in place. ``p2p``: one kernel reads the peers' views over NVLink
        in rank order and also finishes the row statistics."""
        if self._shard_mode == "p2p":
            check(self._lib.spb_row_stats_p2p(C.byref(self._params), (self._shard_epoch - 1) & 1, self._shard_epoch, st),
                  "spb_row_stats_p2p")
            return
        self._shard_comm.sum_(self, view)

    def _shard_finish_rows(self, st):
        """Finish the row statistics from the view of ``_shard_fold`` once ``_shard_sum`` made it the sum over the ranks
        (``p2p``: already finished by ``_shard_sum``)."""
        if self._shard_mode == "p2p":
            return
        check(self._lib.spb_row_stats_finalize(C.byref(self._params), (self._shard_epoch - 1) & 1, st),
              "spb_row_stats_finalize")

    def _shard_row_statistics(self, st):
        """Row statistics of a column-sharded pair: local fold, sum over the ranks, finish (replaces spb_row_finalize)."""
        self._shard_sum(self._shard_fold(st), st)
        self._shard_finish_rows(st)

    def _shard_positions(self) -> list:
        """Output column of every E-step column of every rank, in rank order (-1: null column): batch positions for an SVI
        E-step, fixed cells for a full one."""
        from .distributed import column_block

        world, svi = int(self.column_shard[1]), bool(self._params.svi)
        cache = self.__dict__.setdefault("_shard_pos_cache", {})
        if svi not in cache:
            if svi:
                sched = svi_schedule(self.batch_perm, self.max_iter, self.batch_size)
                it = max(self.max_iter - 1, 0)
                cache[svi] = [shard_svi_schedule(sched, self.NB, r, world)[1][it] for r in range(world)]
            else:
                cache[svi] = [np.arange(*column_block(self.NB, r, world), dtype=np.int32) for r in range(world)]
        return cache[svi]

    def _shard_columns(self, t: torch.Tensor, n_out: int, fill=0) -> np.ndarray:
        """Per-column rows ``t`` [NBb, ...] of every rank's last E-step, assembled on the host in the unsharded column order
        ([n_out, ...]; null columns dropped). Without a process group only this rank's columns are returned."""
        from .distributed import assemble_columns

        parts = [q.cpu().numpy() for q in self._shard_comm.gather(self, t)]
        pos = self._shard_positions()
        if len(parts) == 1 and len(pos) > 1:  # no collective: this rank's own columns
            mine = pos[int(self.column_shard[0])]
            return parts[0][: mine.shape[0]][mine >= 0]
        return assemble_columns(parts, pos, n_out, fill)

    def _pinv_eps(self) -> float:
        """Machine epsilon behind scipy.linalg.pinv's default cutoff in the reference (utils.py:1435): float32 for the
        Euclidean kernel; the geodesic kernel matrix is float64 there (con_K_graph, utils.py:1208-1217), which promotes
        SigmaInv and makes the cutoff K * eps(float64)."""
        return 2.220446049250313e-16 if self.kernel_type == "geodist" else 1.1920928955078125e-07

    def _read_scalars(self) -> SpbScalars:
        raw = self._state["sc"].cpu().numpy().tobytes()
        return SpbScalars.from_buffer_copy(raw)

    # ------------------------------------------------------------------------------------------------------------------
    # the EM loop
    # ------------------------------------------------------------------------------------------------------------------
    def _nonrigid_solve_large_K(self, st):
        """K > SPB_MAX_K_FUSED: eigen pseudo-inverse through cuSOLVER (torch.linalg.eigh, fp64), same cutoff rule as
        scipy.linalg.pinv on the reference's fp32 matrix (utils.py:1435). Everything stays on the device: the kept
        eigen-directions are sorted first and handed to the row kernel as a factor of Sigma, with their count in device memory."""
        lib, p, s = self._lib, self._params, self._state
        check(lib.spb_nonrigid_blend(C.byref(p), st), "spb_nonrigid_blend")
        A = s["SigmaInv"]
        A = 0.5 * (A + A.T)
        ev, V = torch.linalg.eigh(A)
        ev, V = ev.flip(0), V.flip(1)  # descending: directions above the cutoff come first
        cutoff = ev.abs().max() * self.K * self._pinv_eps()
        keep = ev.abs() > cutoff
        inv = torch.where(keep, 1.0 / ev, torch.zeros_like(ev))
        VS = V * inv
        s["Sigma"].copy_(VS @ V.T)
        rhs = s["UtPXB"]
        g_nonrigid = self.guidance and self.guidance_effect in ("nonrigid", "both")
        if g_nonrigid:  # morpho_class.py:1286-1288, 1294-1295 (the SigmaInv part is added by spb_nonrigid_blend)
            sc = s["sc"][:80].view(torch.float64)  # sigma2 = [0], Sp = [3] (spb_scalars layout)
            cg = sc[0] * float(self.guidance_weight) * sc[3] / self.X_AI.shape[0]
            rhs = rhs + cg * (s["g_UI"].T @ (s["g_XB"] - s["g_RA"]))
        s["Coff"].copy_(VS @ (V.T @ rhs))
        if g_nonrigid:
            s["g_VA"].copy_(s["g_UI"] @ s["Coff"])
        # factor of Sigma for the row kernel: G = V sqrt(|inv|) sign-safe (kept eigenvalues of the PSD matrix are positive)
        G = s.setdefault("sigma_factor", torch.zeros((self.K, self.K), dtype=torch.float64, device=self._dev))
        G.copy_(V * torch.sqrt(inv.clamp_min(0.0)))
        rank = s.setdefault("sigma_rank", torch.zeros((1,), dtype=torch.int32, device=self._dev))
        rank.copy_((keep & (ev > 0)).sum().to(torch.int32).reshape(1))

    def _fusable(self, it: int) -> bool:
        """Iteration ``it`` can run as the fused single call and be replayed from a CUDA graph: a resident, unsharded pair,
        outside the non-rigid phase of K > SPB_MAX_K_FUSED (eigen solve through cuSOLVER)."""
        large_K = it > self.nonrigid_start_iter and self.K > _capi.MAX_K_FUSED
        return not (large_K or self.column_shard is not None or self._streamed)

    def _iteration(self, it: int, st, capture_P: bool = False, sweep_events: Optional[list] = None):
        """One EM iteration (morpho_class.py:280-294). The fused C entry point is used unless the iteration has to be
        split: it is not ``_fusable``, it records ``sweep_events``, or it captures the posterior of THIS E-step
        (``capture_P``), which must be read before the M-step moves the cells."""
        if self._fusable(it) and not capture_P and sweep_events is None:
            check(self._lib.spb_em_iteration(C.byref(self._params), it, st), "spb_em_iteration")
            return
        if self.column_shard is not None:
            view = self._shard_iteration_local(it, st, capture_P, sweep_events)
            self._shard_sum(view, st)
            self._shard_iteration_finish(it, st)
            return
        self._estep_only(it, st, sweep_events, on_chunk=self._capture_begin() if capture_P else None)
        self._mstep(it, st)

    def _shard_iteration_local(self, it: int, st, capture_P: bool = False,
                               sweep_events: Optional[list] = None) -> torch.Tensor:
        """First half of a column-sharded iteration: the E-step of this rank's columns (and the posterior capture of the
        last iteration) up to the fold of its row statistics. Returns the fp64 view that ``_shard_sum`` sums over the ranks
        before ``_shard_iteration_finish`` (``_iteration`` runs the three in this order)."""
        self._estep_local(it, st, sweep_events, on_chunk=self._capture_begin() if capture_P else None)
        return self._shard_fold(st)

    def _shard_iteration_finish(self, it: int, st):
        """Second half of a column-sharded iteration, once ``_shard_sum`` made the view of ``_shard_iteration_local`` the sum
        over the ranks: finish the row statistics, then the replicated M-step."""
        self._shard_finish_rows(st)
        self._mstep(it, st)

    def _mstep(self, it: int, st):
        """The M-step of one iteration (split path of ``_iteration``)."""
        lib, p = self._lib, self._params
        nonrigid = it > self.nonrigid_start_iter
        large_K = nonrigid and self.K > _capi.MAX_K_FUSED
        check(lib.spb_update_gamma_alpha(C.byref(p), st), "spb_update_gamma_alpha")
        if nonrigid:
            check(lib.spb_nonrigid_accumulate(C.byref(p), st), "spb_nonrigid_accumulate")
            if large_K:
                self._nonrigid_solve_large_K(st)
                check(lib.spb_field_apply_lowrank(C.byref(p), ptr(self._state["sigma_factor"]), self.K,
                                                  ptr(self._state["sigma_rank"]), st), "spb_field_apply_lowrank")
            else:
                check(lib.spb_nonrigid_solve(C.byref(p), st), "spb_nonrigid_solve")
                check(lib.spb_field_apply(C.byref(p), st), "spb_field_apply")
        check(lib.spb_rigid_moments(C.byref(p), st), "spb_rigid_moments")
        check(lib.spb_rigid_solve(C.byref(p), it, st), "spb_rigid_solve")
        check(lib.spb_row_update(C.byref(p), st), "spb_row_update")

    def _capture_begin(self):
        """Outputs of the posterior capture of the E-step about to run (``_NBb`` columns): P @ F_B / P^T @ F_A, the argmax
        keys, and the dense P or, in sparse_calculation_mode, its COO entries (top-k rows and values per column), as the
        options ask. Returns ``_capture_chunk``, the ``on_chunk`` hook of ``_estep_only`` that fills them."""
        dev, n = self._dev, self._NBb
        if self._transfer_on:
            self._transfer_begin()
        if self.compute_mapping:  # row / column maxima of the same posterior, straight from the cost matrix
            self._rowbest = torch.zeros((self.NA,), dtype=torch.int64, device=dev)
            self._colbest = torch.zeros((n,), dtype=torch.int64, device=dev)
            self._colmap = None
            if self.column_shard is not None:  # row keys carry the unsharded column index; null columns are skipped
                self._colmap = torch.from_numpy(self._shard_positions()[int(self.column_shard[0])]).to(dev)
        if self.materialize_P and self.sparse_calculation_mode:
            k = int(self.sparse_top_k)
            self._P_rows = torch.zeros((n, k), dtype=torch.int32, device=dev)
            self._P_vals = torch.zeros((n, k), dtype=torch.float32, device=dev)
        elif self.materialize_P:
            self._P_dev = torch.empty((self.NA, n), dtype=torch.float32, device=dev)
        self._P_captured = True
        return self._capture_chunk

    def _capture_chunk(self, q: SpbEmParams, it: int, c0: int, c1: int, st=None):
        """The posterior of the E-step columns [c0, c1) that ``q`` describes, while their lists and column constants are
        live, launched on ``st`` (default: the current stream, on which ``on_chunk`` runs). The argmax keys and the dense P
        are only captured from a whole E-step: a streamed pair, the only one whose E-step comes in several chunks, refuses
        both (``_plan_cost``)."""
        lib = self._lib
        st = _capi.current_stream_ptr() if st is None else st
        if self._transfer_on:
            self._transfer_capture(q, it, st, c0)
        if self.compute_mapping:
            check(lib.spb_posterior_argmax_mapped(C.byref(q), it, ptr(self._colmap), ptr(self._rowbest), ptr(self._colbest),
                                                  st), "spb_posterior_argmax_mapped")
        if self.materialize_P and self.sparse_calculation_mode:
            check(lib.spb_sparse_P_emit(C.byref(q), it, ptr(self._P_rows[c0:c1]), ptr(self._P_vals[c0:c1]), st),
                  "spb_sparse_P_emit")
        elif self.materialize_P:
            check(lib.spb_materialize_P(C.byref(q), it, ptr(self._P_dev), self._NBb, st), "spb_materialize_P")

    def _capture_P(self, it: int, st):
        """Capture the posterior of the whole E-step that has just run (``_capture_begin`` + ``_capture_chunk``)."""
        self._capture_begin()(self._params, it, 0, self._NBb, st)

    def _sparse_P_to_coo(self, dt, P_rows: Optional[torch.Tensor] = None, P_vals: Optional[torch.Tensor] = None):
        """scipy COO in the reference's layout (utils.py:1385-1392,1506-1510) from the [n_cols][sparse_top_k] entries of
        ``spb_sparse_P_emit`` (default: this solver's last capture): per column the k entries in descending order, columns
        concatenated."""
        import scipy.sparse as sp

        P_rows = self._P_rows if P_rows is None else P_rows
        P_vals = self._P_vals if P_vals is None else P_vals

        k = min(int(self.sparse_top_k), self.NA)
        n_cols = P_rows.shape[0]
        vals, order = torch.sort(P_vals[:, :k], dim=1, descending=True, stable=True)
        rows = torch.gather(P_rows[:, :k].long(), 1, order).cpu().numpy()
        if self._perm is not None:
            rows = self._perm[rows]
        col = np.repeat(np.arange(n_cols), k)
        return sp.coo_matrix((vals.cpu().numpy().astype(dt).reshape(-1), (rows.reshape(-1), col)), shape=(self.NA, n_cols))

    def _estep_only(self, it: int, st, sweep_events: Optional[list] = None, on_chunk=None):
        """One E-step + its row statistics, which the M-step and the closing similarity read (``_estep_local``)."""
        lib, p = self._lib, self._params
        self._estep_local(it, st, sweep_events, on_chunk)
        if self._streamed:
            check(lib.spb_row_stats_finalize(C.byref(p), 0, st), "spb_row_stats_finalize")
        elif self.column_shard is not None:
            self._shard_row_statistics(st)
        else:
            check(lib.spb_row_finalize(C.byref(p), st), "spb_row_finalize")

    def _estep_local(self, it: int, st, sweep_events: Optional[list] = None, on_chunk=None):
        """The E-step of this process's columns up to its row partials (sweep 2). A streamed cost matrix is recomputed
        chunk by chunk: per chunk the cost rows, then the sweeps, whose row partials are folded into the fp64 row statistics
        in chunk order (reproducible). ``on_chunk(params, it, c0, c1)`` runs after every sweep 2, while its cost rows and
        column constants are live: once with ``_params`` over all columns, or once per chunk [c0, c1) of a streamed E-step.
        ``sweep_events`` receives the events of ``_estep_sweeps`` (not recorded for a streamed E-step)."""
        lib, p, s = self._lib, self._params, self._state
        check(lib.spb_iter_begin(C.byref(p), it, st), "spb_iter_begin")
        if not self._streamed:
            self._estep_sweeps(p, it, st, sweep_events)
            if on_chunk is not None:
                on_chunk(p, it, 0, p.NBb)
            return
        cols, width = p.NBb, self.cost_plan.width
        for k, c0 in enumerate(range(0, cols, width)):
            c1 = min(cols, c0 + width)
            q = self._chunk_params(k, c0, c1)
            q.fold_add = int(k > 0)
            self._chunk_cost(c0, c1, s["chunk_sched"][k][it] if p.svi else None)
            if c1 - c0 < width:  # ragged chunk: the pad column record after the last column is zero, as in a full one
                s["colgeom"][c1 - c0:].zero_()
                s["colconst"][c1 - c0:].zero_()
            self._estep_sweeps(q, it, st)
            if on_chunk is not None:
                on_chunk(q, it, c0, c1)
            check(lib.spb_row_fold(C.byref(q), 0, st), "spb_row_fold")

    def _estep_sweeps(self, q: SpbEmParams, it: int, st, sweep_events: Optional[list] = None):
        """The E-step launches of the columns ``q`` describes, from the column gather to sweep 2. ``sweep_events``: a list
        that receives (start, after sweep 1, before sweep 2, end) CUDA events."""
        lib, qp = self._lib, C.byref(q)
        check(lib.spb_gather_cols(qp, it, st), "spb_gather_cols")
        check(lib.spb_estep_col_lists(qp, st), "spb_estep_col_lists")
        if sweep_events is not None:
            e0, e1, e2, e3 = (torch.cuda.Event(enable_timing=True) for _ in range(4))
            e0.record()
        check(lib.spb_estep_sweep1(qp, it, st), "spb_estep_sweep1")
        if sweep_events is not None:
            e1.record()
        check(lib.spb_col_finalize(qp, st), "spb_col_finalize")
        if self.sparse_calculation_mode:
            check(lib.spb_estep_col_select(qp, it, st), "spb_estep_col_select")
        if sweep_events is not None:
            e2.record()
        check(lib.spb_estep_sweep2(qp, it, st), "spb_estep_sweep2")
        if sweep_events is not None:
            e3.record()
            sweep_events.append((e0, e1, e2, e3))

    def _chunk_params(self, k: int, c0: int, c1: int) -> SpbEmParams:
        """Parameters of one column chunk [c0, c1) of the E-step that ``_params`` describes: its columns are fixed cells
        [c0, c1) (full EM, or the full posterior of return_mapping) or positions [c0, c1) of the SVI batch, whose schedule
        is the chunk's own slice; the cost chunk holds them by position, the column sums land in K_NB[c0:c1]."""
        p, s = self._params, self._state
        q = SpbEmParams.from_buffer_copy(p)
        q.NBb, q.NB_total, q.gt_by_position = c1 - c0, p.NBb, 1
        q.GT = self._GT.data_ptr()
        q.K_NB = s["K_NB"].data_ptr() + 4 * c0
        if p.svi:
            q.batch_idx = s["chunk_sched"][k].data_ptr()
        else:
            q.batch_idx = None
            q.xb4 = s["xb4"].data_ptr() + 16 * c0
        return q

    def prepare_host(self):
        """Coarse rigid initialisation + variational initialisation (host numpy with small device helpers); consumes
        the global ``np.random`` stream in the reference's order (morpho_class.py:258-261)."""
        import time as _time

        self._timing = {}
        with torch.cuda.device(self._dev):
            t0 = _time.perf_counter()
            if self.nn_init:
                self._coarse_rigid_alignment()
            # (stream-level waits: a second pair may be running its EM on another stream of this device)
            torch.cuda.current_stream().synchronize()
            self._timing["coarse_rigid_alignment_s"] = _time.perf_counter() - t0
            t0 = _time.perf_counter()
            self._initialize_variational_variables()
            torch.cuda.current_stream().synchronize()
            self._timing["variational_init_s"] = _time.perf_counter() - t0
        self._host_ready = True

    def prepare_device(self):
        """Host -> device copies of the inputs, expression-cost matrix, EM state (morpho_class.py:265-268)."""
        if not getattr(self, "_host_ready", False):
            self.prepare_host()
        with torch.cuda.device(self._dev):
            self._build_gene_cost()
            self._allocate_state()
            check(self._lib.spb_row_update(C.byref(self._params), _capi.current_stream_ptr()), "spb_row_update")
        self._prepared = True

    def prepare(self):
        """Everything ``run`` does before the loop: coarse init, variational init, cost matrix, device state."""
        self.prepare_host()
        self.prepare_device()

    def reset_state(self):
        """Rewind the EM state to iteration 0 (benchmark repetitions); the cost matrix stays resident."""
        with torch.cuda.device(self._dev):
            self._allocate_state()
            check(self._lib.spb_row_update(C.byref(self._params), _capi.current_stream_ptr()), "spb_row_update")

    def run_em(self, n_iter: Optional[int] = None, start: int = 0, sweep_events: Optional[list] = None):
        """Enqueue EM iterations [start, start + n_iter) on the current stream (no host synchronisation).

        Runs of iterations of the same phase (rigid-only up to ``nonrigid_start_iter``, with the non-rigid solve after) are
        replayed from ONE captured CUDA graph of the iteration's launch sequence (the iteration index — SVI batch, step
        size, trace row — is a device counter). Iterations that need host involvement
        (history recording, per-sweep events, the posterior capture of the last iteration, K > SPB_MAX_K_FUSED in the
        non-rigid phase) take the plain path.

        ``sweep_events``: optional list that receives (start, mid, end) CUDA events recorded around the two E-step sweep
        kernels of every iteration on the launching stream (bench.py's live roofline measurement)."""
        n_iter = self.max_iter - start if n_iter is None else n_iter
        with torch.cuda.device(self._dev):
            st = _capi.current_stream_ptr()
            hist = self._state.get("hist")
            it, end = start, start + n_iter
            while it < end:
                last = it == self.max_iter - 1
                want_P = self._captures_posterior and last and not (self.return_mapping and self.SVI_mode)
                nonrigid = it > self.nonrigid_start_iter
                if not (hist is not None or sweep_events is not None or want_P or not self._fusable(it)):
                    # iterations [it, stop) share the phase and need nothing from the host
                    stop = min(end, self.nonrigid_start_iter + 1) if not nonrigid else end
                    if self._captures_posterior and stop == self.max_iter and not (self.return_mapping and self.SVI_mode):
                        stop -= 1  # the last iteration captures the posterior: plain path
                    if stop - it >= 3:
                        self._iteration(it, st)  # explicit index: also the warm-up launch of every kernel of the phase
                        if not nonrigid and end > self.nonrigid_start_iter + 4 and self.K <= _capi.MAX_K_FUSED:
                            # capture the graph of the later non-rigid phase now as well: a capture synchronises the
                            # device, and doing it here keeps the host free to enqueue the whole run without stopping
                            check(self._lib.spb_nonrigid_warm(), "spb_nonrigid_warm")
                            self._iteration_graph(True)
                            if self._graph_unroll() > 1 and end - self.nonrigid_start_iter - 2 >= 2 * self._graph_unroll():
                                self._iteration_graph(True, self._graph_unroll())
                        n_rep = stop - it - 1
                        unroll = self._graph_unroll()
                        replayed = 0
                        if unroll > 1 and n_rep >= 2 * unroll:
                            graph_u, n_kernels_u = self._iteration_graph(nonrigid, unroll)
                            for _ in range(n_rep // unroll):
                                graph_u.replay()
                            replayed += n_kernels_u * (n_rep // unroll)
                            n_rep -= (n_rep // unroll) * unroll
                        graph, n_kernels = self._iteration_graph(nonrigid)
                        for _ in range(n_rep):
                            graph.replay()
                        # kernels launched through graph replays are not seen by the library's launch counter
                        self.graph_replayed_launches = getattr(self, "graph_replayed_launches", 0) + replayed + n_kernels * n_rep
                        it = stop
                        continue
                if hist is not None:
                    hist[it].copy_(self._state["XAHat"])
                    self._state["hist_sigma2"][it].copy_(self._state["sc"][:8].view(torch.float64)[0])
                self._iteration(it, st, capture_P=want_P, sweep_events=sweep_events)
                it += 1

    @property
    def _captures_posterior(self) -> bool:
        """The posterior of the final E-step has a consumer: dense / sparse P, the mapping or the transfer."""
        return bool(self.materialize_P or self.compute_mapping or self._transfer_on)

    def _graph_unroll(self) -> int:
        """Iterations per captured graph: 8 when an iteration touches fewer than 2e9 cell pairs (about 2 ms of device time:
        the default SVI batch of the 100k pair, or any small pair), where one graph launch per iteration can make a slow
        host the bottleneck; 1 for the heavy full-EM iterations."""
        u = getattr(self, "graph_unroll", 0)
        if u > 0:
            return u
        cols = self.batch_size if self.SVI_mode else self.NB
        return 8 if float(self.NA) * float(cols) < 2e9 else 1

    def _iteration_graph(self, nonrigid: bool, unroll: int = 1):
        """CUDA graph of ``unroll`` consecutive EM iterations of the given phase (captured once per device state; the
        iteration index is a device counter, so the copies are identical launch sequences)."""
        graphs = self.__dict__.setdefault("_graphs", {})
        key = (bool(nonrigid), int(unroll))
        if key not in graphs:
            g = torch.cuda.CUDAGraph()
            n0 = self._lib.spb_launch_count()
            with torch.cuda.graph(g):
                for _ in range(unroll):
                    check(self._lib.spb_em_iteration_ex(C.byref(self._params), -1, 1 if nonrigid else 0,
                                                        _capi.current_stream_ptr()), "spb_em_iteration_ex(capture)")
            graphs[key] = (g, int(self._lib.spb_launch_count() - n0))
        return graphs[key]

    @torch.no_grad()
    def run(self):
        """morpho_class.py:242-313. Returns P [N_A, N_B | batch] (numpy) or None when ``materialize_P=False``."""
        if not getattr(self, "_prepared", False):
            self.prepare_device()
        with torch.cuda.device(self._dev):
            if self.iter_key_added is not None:
                self._state["hist"] = torch.empty((max(self.max_iter, 1), 3, self.ldx), dtype=torch.float32, device=self._dev)
                self._state["hist_sigma2"] = torch.zeros((max(self.max_iter, 1),), dtype=torch.float64, device=self._dev)
            self.run_em()
            self._finish()
        return self.P

    # ------------------------------------------------------------------------------------------------------------------
    # closing similarity + output wrapping (morpho_class.py:296-313, 1437-1528)
    # ------------------------------------------------------------------------------------------------------------------
    def _finish(self):
        lib, p, s = self._lib, self._params, self._state
        st = _capi.current_stream_ptr()
        dt = self._np_dtype
        D, NA = self.D, self.NA
        last_iter = max(self.max_iter - 1, 0)
        if self.sigma2_end is not None:
            sc = self._read_scalars()
            sc.sigma2 = float(self.sigma2_end)
            s["sc"].copy_(torch.from_numpy(np.frombuffer(bytes(sc), dtype=np.uint8).copy()))
            check(lib.spb_row_update(C.byref(p), st), "spb_row_update")
        full_mapping = self.return_mapping and self.SVI_mode
        # the closing E-step (max_iter == 0, or the full posterior of return_mapping) is the one whose posterior is captured
        capture = self._captures_posterior
        if self.max_iter == 0:
            self._estep_only(0, st, on_chunk=self._capture_begin() if capture and not full_mapping else None)
            check(lib.spb_rigid_moments(C.byref(p), st), "spb_rigid_moments")
        if full_mapping:
            # full (non-SVI) posterior with the final parameters (morpho_class.py:300-302)
            self.SVI_mode = False
            nb = self._col_range()[1] - self._col_range()[0]  # a shard's closing E-step covers its whole block
            p.svi, p.NBb = 0, nb
            if self.column_shard is not None:
                p.NB_total = self.NB
            if not self._streamed:  # streamed: the column segments stay those of the chunk width
                p.seg1 = p.seg2 = self._choose_segments(self.ldx // _capi.ROW_TILE, nb,
                                                        torch.cuda.get_device_properties(self._dev).multi_processor_count)
            self._NBb = nb
            self._estep_only(last_iter, st, on_chunk=self._capture_begin() if capture else None)
            # scalar Sp's must become the un-averaged sums (morpho_class.py:1183-1185)
            sc = self._read_scalars()
            sc.Sp_spatial, sc.Sp_sigma2, sc.Sp = sc.sums[0], sc.sums[1], sc.sums[2]
            s["sc"].copy_(torch.from_numpy(np.frombuffer(bytes(sc), dtype=np.uint8).copy()))
            s["moments"].zero_()
            check(lib.spb_rigid_moments(C.byref(p), st), "spb_rigid_moments")
        check(lib.spb_optimal_rigid(C.byref(p), ptr(s["optimal"]), st), "spb_optimal_rigid")
        opt = s["optimal"].cpu().numpy()
        sc = self._read_scalars()
        R3 = np.array(list(sc.R), dtype=np.float64).reshape(3, 3)
        self.R = R3[:D, :D].astype(dt)
        self.t = np.array(list(sc.t), dtype=np.float64)[None, :D].astype(dt)
        self.optimal_R = opt[:9].reshape(3, 3)[:D, :D].astype(dt)
        self.optimal_t = opt[9 : 9 + D].astype(dt)
        self.sigma2 = np.asarray(sc.sigma2, dtype=dt)
        self.gamma = np.asarray(sc.gamma, dtype=dt)
        self.sigma2_variance = np.asarray(sc.sigma2_variance, dtype=dt)
        self.Sp, self.Sp_spatial, self.Sp_sigma2 = sc.Sp, sc.Sp_spatial, sc.Sp_sigma2
        self.nonrigid_flag = self.max_iter - 1 > self.nonrigid_start_iter

        def rows(name):  # [3, ldx] SoA (processing order) -> [NA, D] in the caller's row order
            t = s[name][:D, :NA].T.contiguous()
            _count_d2h(t)
            return self._unsorted(t.cpu().numpy().astype(dt))

        def vec(name):
            _count_d2h(s[name][:NA])
            return self._unsorted(s[name][:NA].cpu().numpy().astype(dt))

        self.XAHat, self.RnA, self.VnA = rows("XAHat"), rows("RnA"), rows("VnA")
        self.optimal_RnA = (self.coordsA.astype(np.float64) @ self.optimal_R.astype(np.float64).T + self.optimal_t).astype(dt)
        self.K_NA = vec("K_NA")
        # the unsharded column count of the last E-step: the SVI batch or all fixed cells
        n_cols = self.batch_size if self._params.svi else self.NB
        if self.column_shard is None:
            self.K_NB = s["K_NB"][: self._NBb].cpu().numpy().astype(dt)
        else:  # every rank holds the column sums of its own columns: gathered into the unsharded order
            self.K_NB = self._shard_columns(s["K_NB"][: self._NBb], n_cols).astype(dt)
        self.K_NA_spatial = vec("K_NA_spatial")
        self.K_NA_sigma2 = vec("K_NA_sigma2")
        self.alpha = vec("alpha")
        self.SigmaDiag = vec("SigmaDiag")
        if self.nonrigid_flag:
            self.Coff = s["Coff"][:, :D].cpu().numpy().astype(dt)
            self.SigmaInv = s["SigmaInv"].cpu().numpy().astype(dt)
        else:
            self.Coff = np.zeros(self.K, dtype=dt)  # the reference's initial value (morpho_class.py:733)
        self.trace = s["trace_buf"].cpu().numpy()
        if capture and not self._P_captured:  # run_em stopped before the last iteration: the E-step that ran last
            self._capture_P(last_iter, st)
        if self._transfer_on:
            self._transfer_results(n_cols)
        if self.compute_mapping:
            from .mapping import ArgmaxPi

            rowbest, colbest = self._rowbest.cpu().numpy(), self._colbest.cpu().numpy()
            if self.column_shard is not None:  # row keys: the largest over the ranks; column keys: gathered
                self._shard_comm.max_(self, self._rowbest)
                rowbest = self._rowbest.cpu().numpy()
                colbest = self._shard_columns(self._colbest, n_cols)
            ra, rv = ArgmaxPi.decode(rowbest.view(np.uint64))
            ca, cv = ArgmaxPi.decode(colbest.view(np.uint64))
            if self._perm is not None:  # device rows are in processing order
                ra, rv, ca = self._unsorted(ra), self._unsorted(rv), self._perm[ca]
            self.mapping = ArgmaxPi((NA, colbest.shape[0]), ra, rv.astype(dt), ca, cv.astype(dt))
            self._rowbest = self._colbest = self._colmap = None
        if self.materialize_P:
            if self.sparse_calculation_mode:
                rows, vals = self._P_rows, self._P_vals
                if self.column_shard is not None:  # every rank emitted the entries of its own columns
                    rows = torch.from_numpy(self._shard_columns(rows, n_cols))
                    vals = torch.from_numpy(self._shard_columns(vals, n_cols))
                self.P = self._sparse_P_to_coo(dt, rows, vals)
                self._P_rows = self._P_vals = None
            else:
                _count_d2h(self._P_dev)
                self.P = self._unsorted(self._P_dev.cpu().numpy().astype(dt))
        else:
            self.P = None
        self._P_dev, self._P_captured = None, False
        if self.iter_key_added is not None:
            hist_d = s["hist"][:, :D, :NA].permute(0, 2, 1).contiguous()
            _count_d2h(hist_d)
            hist = hist_d.cpu().numpy().astype(dt)
            del hist_d
            if self._perm is not None:
                un = np.empty_like(hist)
                un[:, self._perm, :] = hist
                hist = un
            sig = s["hist_sigma2"].cpu().numpy()
            self.iter_added = {self.key_added: {}, "sigma2": {}}
            for it in range(self.max_iter):
                xa = hist[it]
                if self.normalize_c:
                    xa = xa * self.normalize_scales[1] + self.normalize_means[1]
                self.iter_added[self.key_added][it] = xa
                self.iter_added["sigma2"][it] = np.asarray(sig[it], dtype=dt)
        self._wrap_output()

    def _wrap_output(self):
        if self.normalize_c:
            sc1, m1 = self.normalize_scales[1], self.normalize_means[1]
            self.XAHat = self.XAHat * sc1 + m1
            self.RnA = self.RnA * sc1 + m1
            self.optimal_RnA = self.optimal_RnA * sc1 + m1
        if self.vecfld_key_added is not None:
            norm_dict = {
                "mean_transformed": self.normalize_means[0],
                "mean_fixed": self.normalize_means[1],
                "scale": self.normalize_scales[0],
                "scale_transformed": self.normalize_scales[0],
                "scale_fixed": self.normalize_scales[1],
            } if self.normalize_c else None
            self.vecfld = {
                "R": self.R,
                "t": self.t,
                "optimal_R": self.optimal_R,
                "optimal_t": self.optimal_t,
                "init_R": self.init_R if self.nn_init else np.eye(self.D),
                "init_t": self.init_t if self.nn_init else np.zeros(self.D),
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
                "kernel_type": self.kernel_type,
            }

    # ------------------------------------------------------------------------------------------------------------------
    # test / debugging access to the device state
    # ------------------------------------------------------------------------------------------------------------------
    def device_vector(self, name: str) -> np.ndarray:
        t = self._state[name]
        return t.cpu().numpy()
