"""Multi-GPU chain alignment: independent slice pairs shard one per GPU, ONE all-gather of the per-pair rigid
transforms, then the serial prefix composition of the reference's ``morpho_align_apply_transformation``
(spateo/alignment/morpho_alignment.py:181-217 for the independent pairs, :300-303 for the composition).

One process per GPU (``torchrun``); the data path has no collective — the pairs are independent problems — and the only
exchange is ``[R(2x2) | t(2)]`` per pair (48 bytes), which is what BASELINE.json calls the global rigid-consensus step.

Two more layouts split the work of ONE pair over the ranks instead: ``morpho_align_pair_sharded`` (one pair, its fixed
cells column-sharded) and ``morpho_align_column_sharded`` (``morpho_align``'s serial chain, every pair column-sharded).
"""

from __future__ import annotations

import contextlib
import gc
import threading
from typing import Callable, List, Optional

import numpy as np
import torch
import torch.distributed as dist

from .morpho_alignment import (_seed_keys, _store_pair, _store_transfer, _transfer_keys, _working_copy,
                               compose_transformations, pair_transformation)
from .utils import empty_cache


def shard_pairs(n_pairs: int, rank: int, world: int) -> List[int]:
    """Pair p (fixed = slice p, moving = slice p+1) runs on rank p mod world."""
    return [p for p in range(n_pairs) if p % world == rank]


def gather_transformations(local: dict, n_pairs: int, device=None) -> List[dict]:
    """``local`` maps pair index -> {"Rotation", "Translation"}; returns the full ordered list on every rank using a
    single ``all_gather`` of fixed-size per-rank slabs (NCCL on GPUs, gloo on CPU)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    per_rank = (n_pairs + world - 1) // world
    if dist.is_initialized() and dist.get_backend() == "nccl":
        from .morpho_class import resolve_device  # GPU-index strings ("0") / None -> torch.device("cuda", i)

        device = resolve_device(device)
    slab = torch.zeros((per_rank, 8), dtype=torch.float64, device=device)  # [pair index + 1, R00 R01 R10 R11, t0 t1, pad]
    for slot, p in enumerate(shard_pairs(n_pairs, rank, world)):
        tr = local[p]
        slab[slot, 0] = p + 1
        slab[slot, 1:5] = torch.as_tensor(np.asarray(tr["Rotation"], dtype=np.float64).reshape(-1)[:4])
        slab[slot, 5:7] = torch.as_tensor(np.asarray(tr["Translation"], dtype=np.float64).reshape(-1)[:2])
    if world > 1:
        out = torch.zeros((world, per_rank, 8), dtype=torch.float64, device=device)
        dist.all_gather_into_tensor(out.view(world * per_rank, 8), slab)
    else:
        out = slab[None]
    rows = out.reshape(-1, 8).cpu().numpy()
    result = [None] * n_pairs
    for r in rows:
        if r[0] > 0:
            result[int(round(r[0])) - 1] = {"Rotation": r[1:5].reshape(2, 2).copy(), "Translation": r[5:7].copy()}
    assert all(t is not None for t in result), "a pair transformation is missing after the all-gather"
    return result


def morpho_align_chain_sharded(
    models: List,
    spatial_key: str = "spatial",
    key_added: str = "align_spatial",
    pair_fn: Optional[Callable] = None,
    device=None,
    **pairwise_kwargs,
):
    """Sharded equivalent of ``morpho_align_transformation`` + ``morpho_align_apply_transformation`` (rigid, 2-D, raw
    coordinates — NOT bitwise ``morpho_align``, whose pairs are serially dependent; SURVEY.md §8(e)). For ``morpho_align``'s
    semantics over several GPUs see ``morpho_align_column_sharded``.

    Every rank receives the whole list of slices (or at least the ones it touches), aligns its pairs, joins the single
    all-gather, composes the chain and writes ``obsm[key_added]`` of every slice it holds. Returns
    ``(models, transformations)``.
    """
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    n_pairs = len(models) - 1
    pair_fn = pair_transformation if pair_fn is None else pair_fn
    local = {}
    for p in shard_pairs(n_pairs, rank, world):
        kw = dict(pairwise_kwargs)
        if device is not None and pair_fn is pair_transformation:
            kw.setdefault("device", device)
        local[p] = pair_fn(models[p], models[p + 1], spatial_key=spatial_key, **kw)
    transformation = gather_transformations(local, n_pairs, device=device if dist.is_initialized() and dist.get_backend() == "nccl" else None)
    models[0].obsm[key_added] = np.asarray(models[0].obsm[spatial_key]).copy()
    for i, (R, t) in enumerate(compose_transformations(transformation)):
        m = models[i + 1]
        m.obsm[key_added] = np.asarray(m.obsm[spatial_key]).copy()[:, :2] @ R.T + t
    return models, transformation


def transfer_device_bytes(n_moving: int, n_fixed: int, transfer: tuple, width: int, n_sms: int = 132) -> int:
    """Device memory of a posterior transfer with (F_B, F_A) features (0 = side not requested) when the E-step's column
    buffers are ``width`` columns wide: F_B [n_fixed + 1][ldf] and the fp64 P @ F_B accumulator [ldf][ldx] (ldf = F_B
    rounded up to the panel), the sweep-2 segment partials of one panel, F_A [roundup(F_A, panel)][ldx], the list-position
    partials of one panel [row blocks][panel][width] and the fp32 P^T @ F_A of every column."""
    from .. import _capi
    from .morpho_class import Morpho_pairwise

    W = _capi.CONST["SPB_TRANSFER_PANEL"]
    ldx = -(-n_moving // _capi.ROW_TILE) * _capi.ROW_TILE
    nrb = ldx // _capi.ROW_TILE
    f_b, f_a = transfer
    total = 0
    if f_b:
        ldf = -(-f_b // W) * W
        total += 4 * (n_fixed + 1) * ldf + 8 * ldf * ldx + 4 * Morpho_pairwise._choose_segments(nrb, width, n_sms) * W * ldx
    if f_a:
        pad = -(-width // 8) * 8 + 8
        total += 4 * (-(-f_a // W) * W) * ldx + 4 * nrb * W * pad + 4 * n_fixed * f_a
    return total


def pair_device_bytes(n_moving: int, n_fixed: int, n_genes: int, chunk_cols: Optional[int] = None, n_sms: int = 132,
                      transfer: Optional[tuple] = None, cols: Optional[int] = None) -> int:
    """Device memory one prepared pair needs, dominated by its fp32 cost matrix [n_fixed][roundup(n_moving, 512)]; the
    expression operands of the cost precompute (two sides, value + tf32 hi / lo, genes padded to 32) and 1 GiB for the
    per-cell state are added on top.

    ``chunk_cols``: the footprint of a streamed pair instead, whose cost matrix is recomputed every iteration in chunks of
    that many columns. The resident matrix is replaced by one [chunk_cols][ldx] cost chunk and every per-column buffer of
    the E-step at that width: column partials, keep masks, work lists, quarter masks, column records, the row partials
    of the sweep's column segments (``n_sms`` sets their count) and the gathered fixed-side operands of an SVI chunk.

    ``transfer``: (F_B, F_A) feature counts of a posterior transfer, whose buffers (``transfer_device_bytes``) are added at
    the chunk width, or at ``cols`` (the columns of one E-step, default ``n_fixed``) for a resident pair."""
    from .. import _capi

    ldx = -(-n_moving // _capi.ROW_TILE) * _capi.ROW_TILE
    gp = -(-n_genes // 32) * 32
    operands = 4 * 3 * (n_moving + n_fixed) * gp + (1 << 30)
    if transfer is not None:
        width = chunk_cols if chunk_cols is not None else (n_fixed if cols is None else cols)
        operands += transfer_device_bytes(n_moving, n_fixed, transfer, width, n_sms)
    if chunk_cols is None:
        return 4 * n_fixed * ldx + operands
    from .morpho_class import Morpho_pairwise

    nrb = ldx // _capi.ROW_TILE
    pad = -(-chunk_cols // 8) * 8 + 8
    per_col = (
        4 * ldx                                  # cost chunk
        + nrb * (4 * 4 + 4 + 2) + nrb // 2 + 1   # colpart [nrb][4], collist, colquarters, colspatial; per 32 columns:
                                                 # keepmask and livemask bits, the two list offsets (keepoff)
        + 4 + 8 * 4 + _capi.CONST["SPB_COLCONST_FLOATS"] * 4 + _capi.CONST["SPB_COLMASK_WORDS"] * 4  # K_NB, colgeom, colconst, colmask
        + 2 * 4 * gp + 2 * 4                     # gathered tf32 hi / lo operands, row term, label
    )
    seg = Morpho_pairwise._choose_segments(nrb, chunk_cols, n_sms)
    return pad * per_col + 4 * 8 * ldx * seg + operands


def _room_for_next_pair(dev, need: int) -> bool:
    """True when ``need`` bytes are free on ``dev`` (``morpho_class._device_budget``)."""
    from .morpho_class import _device_budget

    return _device_budget(dev) >= need


def align_chain_pipelined(
    get_slice: Callable[[int], object],
    n_slices: int,
    spatial_key: str = "spatial",
    key_added: str = "align_spatial",
    device=None,
    stats: Optional[dict] = None,
    **pairwise_kwargs,
):
    """Chain alignment of ``n_slices`` serial sections on this rank's GPU, software-pipelined (BASELINE configs[2]).

    Same result as ``morpho_align_chain_sharded`` (independent pairs on raw coordinates, morpho_alignment.py:181-217; ONE
    all-gather of the per-pair 2-D similarities; serial prefix composition, :300-303) but a rank that owns several pairs
    overlaps them: the EM of pair p is only *enqueued* on the main stream (CUDA-graph replays, no host waits), and while it
    runs the host prepares pair p + world on a second stream — constructor, coarse initialisation, the staged host-to-device
    copy of its two expression matrices and its cost matrix — so that the next EM starts as soon as the current one ends.

    The next pair is prepared early only when the device has room for its cost matrix beside the current pair's
    (``pair_device_bytes``); otherwise the current pair is finished and freed first. Two 125k-cell cost matrices (63 GB each)
    do not fit one 80 GB GPU, so such chains run one pair at a time.

    ``get_slice(k)`` returns slice k (AnnData-like, host arrays); only the slices of this rank's pairs are requested, and
    only they receive ``obsm[key_added]``. Returns ``(placed, transformations)`` with ``placed`` = {slice index: slice}.
    ``stats`` (optional dict) receives per-pair timings.
    """
    import time

    from .morpho_class import Morpho_pairwise, resolve_device
    from .utils import solve_RT_by_correspondence

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    dev = resolve_device(device)
    n_pairs = n_slices - 1
    mine = shard_pairs(n_pairs, rank, world)
    pairwise_kwargs.setdefault("materialize_P", False)
    cache = {}

    def slice_(k):
        if k not in cache:
            cache[k] = get_slice(k)
        return cache[k]

    def make(p):  # fixed = slice p, moving = slice p + 1
        s = Morpho_pairwise(sampleA=slice_(p + 1), sampleB=slice_(p), spatial_key=spatial_key, device=dev, **pairwise_kwargs)
        s.prepare()
        return s

    def room_for(p):  # can pair p be prepared while the current pair still holds its buffers?
        na, nb = slice_(p + 1).shape[0], slice_(p).shape[0]
        return _room_for_next_pair(dev, pair_device_bytes(na, nb, slice_(p).shape[1]))

    local = {}
    t_pairs = []
    from .. import _capi

    launches0, replayed = _capi.load_library().spb_launch_count(), 0
    with torch.cuda.device(dev):
        main, side = torch.cuda.current_stream(), torch.cuda.Stream()
        nxt = make(mine[0]) if mine else None
        for i, p in enumerate(mine):
            t0 = time.perf_counter()
            cur = nxt
            cur.run_em()  # enqueued only: the host is free while the device iterates
            nxt = None
            if i + 1 < len(mine) and room_for(mine[i + 1]):
                with torch.cuda.stream(side):
                    nxt = make(mine[i + 1])
            cur._finish()  # device -> host of the pair's results (waits for its EM)
            R, t = solve_RT_by_correspondence(cur.optimal_RnA[:, :2], np.asarray(slice_(p + 1).obsm[spatial_key])[:, :2])
            local[p] = {"Rotation": R, "Translation": t}
            replayed += getattr(cur, "graph_replayed_launches", 0)
            del cur
            main.wait_stream(side)
            if i + 1 < len(mine) and nxt is None:  # no room beside the current pair: prepare the next one in its place
                gc.collect()  # the solver's buffers and captured graphs go back to the allocator before the next allocation
                nxt = make(mine[i + 1])
            t_pairs.append(time.perf_counter() - t0)
    transformation = gather_transformations(local, n_pairs, device=dev if dist.is_initialized() and dist.get_backend() == "nccl" else None)
    placed = {}
    composed = [(np.diag((1.0, 1.0)), np.zeros((2,)))] + compose_transformations(transformation)
    for k in sorted(cache):
        R, t = composed[k]
        sl = cache[k]
        raw = np.asarray(sl.obsm[spatial_key]).copy()
        sl.obsm[key_added] = raw if k == 0 else raw[:, :2] @ R.T + t
        placed[k] = sl
    if stats is not None:
        stats.update(pairs=list(mine), seconds_per_pair=t_pairs,
                     kernel_launches=int(_capi.load_library().spb_launch_count() - launches0 + replayed))
    return placed, transformation


def column_block(n_cols: int, rank: int, world: int):
    """Fixed cells [begin, end) of rank ``rank`` when one pair's columns are split over ``world`` GPUs."""
    return (n_cols * rank) // world, (n_cols * (rank + 1)) // world


class Collectives:
    """The exchanges of a column-sharded pair's ranks, on ``torch.distributed``: in place sum and element-wise maximum, the
    gather of every rank's per-column rows in rank order, and the broadcast of rank 0's host objects. Without a process
    group of several ranks the sum and the maximum leave ``t`` as it is, the gather returns this rank's own rows and the
    broadcast returns ``obj``. ``m`` is the calling solver; tests that run several shards in one process substitute an
    object with the same methods that tells the shards apart by it."""

    @staticmethod
    def _several_ranks() -> bool:
        return dist.is_initialized() and dist.get_world_size() > 1

    def sum_(self, m, t: torch.Tensor):
        if self._several_ranks():
            dist.all_reduce(t)

    def max_(self, m, t: torch.Tensor):
        if self._several_ranks():
            dist.all_reduce(t, op=dist.ReduceOp.MAX)

    def gather(self, m, t: torch.Tensor) -> List[torch.Tensor]:
        return all_gather_rows(t) if self._several_ranks() else [t]

    def broadcast(self, m, obj):
        """Rank 0's ``obj`` (any picklable object; the other ranks pass None) on every rank."""
        if not self._several_ranks():
            return obj
        box = [obj]
        dist.broadcast_object_list(box, src=0)
        return box[0]


def assemble_columns(parts: List[np.ndarray], positions: List[np.ndarray], n_out: int, fill=0) -> np.ndarray:
    """Per-column rows of a column-sharded E-step in the unsharded column order: row ``k`` of rank r's ``parts[r]`` goes to
    output column ``positions[r][k]``; positions of -1 (null columns) and rows beyond ``len(positions[r])`` (padding of
    the gather) are dropped. Returns [n_out, ...]; columns no rank holds keep ``fill``."""
    out = np.full((n_out,) + parts[0].shape[1:], fill, dtype=parts[0].dtype)
    for part, pos in zip(parts, positions):
        pos = np.asarray(pos)
        keep = pos >= 0
        out[pos[keep]] = part[: pos.shape[0]][keep]
    return out


def all_gather_rows(t: torch.Tensor) -> List[torch.Tensor]:
    """Every rank's ``t`` ([n_r, ...], n_r may differ between ranks), in rank order: one ``all_gather`` of slabs padded to
    the largest n_r (the caller knows which rows are real; ``assemble_columns`` drops the padding)."""
    world = dist.get_world_size()
    n = torch.tensor([t.shape[0]], dtype=torch.int64, device=t.device)
    sizes = [torch.zeros_like(n) for _ in range(world)]
    dist.all_gather(sizes, n)
    width = int(max(int(q.item()) for q in sizes))
    slab = torch.zeros((width,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    slab[: t.shape[0]] = t
    parts = [torch.zeros_like(slab) for _ in range(world)]
    dist.all_gather(parts, slab)
    return [q[: int(m.item())] for q, m in zip(parts, sizes)]


_HOST_INIT_FIELDS = ("coordsA", "init_R", "init_t", "inlier_A", "inlier_B", "inlier_P", "sigma2", "_sigma2_init",
                     "probability_parameters", "samples_s", "outlier_s", "sigma2_variance_decress", "batch_perm")


def morpho_align_pair_sharded(fixed, moving, mode: str = "auto", device=None, **pairwise_kwargs):
    """ONE slice pair over all ranks of the process group (SURVEY.md 8(e), "single huge pair across GPUs").

    Every rank holds the whole moving slice (rows of P) and a block of the fixed slice's cells (columns of P): its block of
    the expression-probability matrix (N_A x N_B / world), sweep 1 and the column constants are local, and the only exchange is
    the sum of the per-row statistics of sweep 2 — [K_NA_spatial, K_NA_sigma2, sum P d, K_NA, P @ XB] = 7 fp64 per moving cell,
    5.6 MB at 100k cells — once per iteration. ``mode="p2p"`` (default when symmetric memory is available): that sum is done
    INSIDE the row-finalize kernel by reading the peers' partial vectors over NVLink in rank order (bit-identical replicas, no
    separate collective); ``mode="nccl"``: ``all_reduce`` + a finishing kernel (the baseline). The M-step runs replicated.

    Rank 0's inducing points and host initialisation (coarse rigid alignment, sigma2 / beta2 guesses, the SVI batch
    permutation) are broadcast so the replicas start from the same bits whatever the ranks' NumPy random state; rank 0
    draws them from the global ``np.random`` stream as ``Morpho_pairwise`` does, and every rank's stream ends where rank
    0's does. Returns the solver (same result attributes as ``Morpho_pairwise``; identical on every rank).

    Runs the full EM unless the caller passes ``SVI_mode=True`` (earlier versions replaced an explicit ``SVI_mode=True``
    with the full EM without saying so). Under SVI every rank runs the members of each batch that fall in its block,
    padded to one width per rank with a null column (``shard_svi_schedule``). Also supported: ``return_mapping``,
    ``guidance_pair``, ``sparse_calculation_mode`` with ``materialize_P=True`` (one ``scipy.sparse.coo_matrix``, gathered
    from the ranks' columns, on every rank) and ``compute_mapping``. ``K_NB``, ``P`` and ``mapping`` come back in the
    unsharded column order. A dense ``materialize_P=True`` raises NotImplementedError, as does a pair whose block of the
    cost matrix does not fit its GPU. ``transfer_B`` / ``transfer_A`` take keys only, as in ``morpho_align``; after
    ``run()`` every rank holds the whole ``P_FB`` and ``PT_FA``."""
    _transfer_keys(pairwise_kwargs)

    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    kw = dict(pairwise_kwargs)
    kw.setdefault("materialize_P", False)
    kw.setdefault("SVI_mode", False)
    return _shard_solver(fixed, moving, rank, world, mode, device, Collectives(), **kw)


# One lock per process around every shard's draws from the global NumPy stream: shards run by the threads of one process
# (the tests emulate ranks that way) share that stream.
_NP_STREAM = threading.Lock()


@contextlib.contextmanager
def _draws_of(rank: int):
    """A shard's draws from the global ``np.random`` stream. Rank 0's are the unsharded solver's; another rank's are
    replaced by rank 0's (broadcast), so it leaves the stream as it found it."""
    with _NP_STREAM:
        state = np.random.get_state() if rank else None
        try:
            yield
        finally:
            if state is not None:
                np.random.set_state(state)


def _shard_solver(fixed, moving, rank: int, world: int, exchange: str, device, comm, **kw):
    """Shard ``rank`` of ``world`` of the pair, prepared for ``run()``, with ``comm`` (a ``Collectives``) for every
    exchange: rank 0's inducing points and host initialisation broadcast to the others, whose NumPy stream then continues
    from where rank 0's stands."""
    from .morpho_class import Morpho_pairwise

    with _draws_of(rank):
        solver = Morpho_pairwise(sampleA=moving, sampleB=fixed, device=device, column_shard=(rank, world, exchange), **kw)
    solver._shard_comm = comm
    if world > 1:  # rank 0's inducing points, so that every rank builds the same kernel matrices (U, Gamma, guidance U_I)
        idx = comm.broadcast(solver, solver.inducing_variables_idx if rank == 0 else None)
        if not np.array_equal(idx, solver.inducing_variables_idx):
            with torch.cuda.device(solver._dev):
                solver._construct_kernel(idx)
    with _draws_of(rank):
        solver.prepare_host()
        stream = np.random.get_state() if rank == 0 else None
    if world > 1:
        init = ({k: getattr(solver, k) for k in _HOST_INIT_FIELDS if hasattr(solver, k)}, stream) if rank == 0 else None
        fields, stream = comm.broadcast(solver, init)
        for k, v in fields.items():
            setattr(solver, k, v)
        if rank:
            with _NP_STREAM:
                np.random.set_state(stream)
    solver.prepare_device()
    return solver


def sharded_chain_pair(fixed, moving, pair: int, rank: int, world: int, comm, mode: str = "SN-S",
                       exchange: str = "auto", device=None, **solver_kwargs):
    """Pair ``pair`` of ``morpho_align_column_sharded`` on one rank: ``moving`` aligned onto ``fixed`` with this rank's
    block of the fixed cells, every exchange through ``comm`` (a ``Collectives``), and the outputs written onto the two
    slices as ``morpho_align`` writes them. ``solver_kwargs`` go to ``Morpho_pairwise`` (``spatial_key``, ``key_added``,
    ``iter_key_added`` and ``vecfld_key_added`` among them). Returns the pair's entry of ``pis``: ``P.T``, or None when the
    posterior is not materialised. The pair's device state (cost-matrix block, solver state, row-statistics buffer and its
    symmetric-memory handle) is released before returning, so a chain holds one pair's at a time."""
    try:
        solver = _shard_solver(fixed, moving, rank, world, exchange, device, comm, **solver_kwargs)
    except NotImplementedError as e:
        if "column_shard" not in str(e):  # the refusal of a block that would have to be streamed (Morpho_pairwise._plan_cost)
            raise
        raise NotImplementedError(
            f"pair {pair} (slice {pair + 1} onto slice {pair}), rank {rank} of {world}: {e}. More ranks would make each "
            "rank's block of the cost matrix smaller, and resident") from e
    P = solver.run()
    _store_pair(moving, solver, solver.key_added, mode, solver.iter_key_added, solver.vecfld_key_added)
    _store_transfer(fixed, moving, solver, *_transfer_keys(solver_kwargs))
    # The last exchange of run() (the gather of K_NB) has completed on every rank, and with it every peer's reads of this
    # rank's symmetric buffer, so the buffer can go.
    del solver
    gc.collect()
    empty_cache()
    return None if P is None else P.T


def morpho_align_column_sharded(
    models: List, rep_layer="X", rep_field="layer", genes=None, spatial_key: str = "spatial",
    key_added: str = "align_spatial", iter_key_added: Optional[str] = "iter_spatial",
    vecfld_key_added: str = "VecFld_morpho", mode: str = "SN-S", dissimilarity="kl", max_iter: int = 200,
    dtype: str = "float32", device=None, verbose: bool = True, exchange: str = "auto", **kwargs,
):
    """``morpho_align`` with every slice pair column-sharded over the ranks of the process group (one process per GPU,
    ``torchrun``; without a process group it runs on one GPU). Same signature, defaults, pairs, order and ``.obsm`` /
    ``.uns`` keys as ``morpho_align``: pair i aligns slice i+1 onto slice i's aligned coordinates (``key_added``), SN-S /
    SN-N, 2-D or 3-D, the non-rigid field stored per slice; inputs are not mutated. Returns ``(align_models, pis)``.

    Every pair runs through ``morpho_align_pair_sharded``'s solver: each rank holds 1/W of the pair's cost matrix, so pairs
    stay resident on their GPUs up to about sqrt(W) times the slice size one GPU holds. ``exchange``: how the ranks sum the
    per-row statistics ("auto", "p2p" or "nccl", the ``mode`` of ``morpho_align_pair_sharded``).

    ``np.random.seed(s)`` on rank 0 before the call gives rank 0 the draws ``morpho_align`` makes after the same seed,
    pair by pair (inducing points, coarse initialisation, SVI batch permutation); the other ranks use rank 0's, and every
    rank's stream ends where rank 0's does. Every rank returns the same slices.

    Defaults that differ from ``morpho_align_pair_sharded``'s: ``SVI_mode=True`` (the reference's) and
    ``materialize_P=False``. ``pis[i]`` is the gathered ``scipy.sparse.coo_matrix`` ``P.T`` with
    ``sparse_calculation_mode=True, materialize_P=True``, otherwise None; a dense ``materialize_P`` raises
    NotImplementedError, as does a pair whose block of the cost matrix does not fit its GPU (a sharded block is not
    streamed). ``transfer_B`` / ``transfer_A``: keys only, as in ``morpho_align``."""
    kwargs.setdefault("SVI_mode", True)
    kwargs.setdefault("materialize_P", False)
    if kwargs["materialize_P"] and not kwargs.get("sparse_calculation_mode", False):
        raise NotImplementedError("materialize_P (dense) on column-sharded pairs: the N_A x N_B posterior does not fit "
                                  "one GPU; pass sparse_calculation_mode=True for the sparse posterior")
    _transfer_keys(kwargs)
    world = dist.get_world_size() if dist.is_initialized() else 1
    rank = dist.get_rank() if dist.is_initialized() else 0
    comm = Collectives()
    aligned = [_working_copy(m) for m in models]
    _seed_keys(aligned, spatial_key, key_added)
    pis = []
    for i, (fixed, moving) in enumerate(zip(aligned[:-1], aligned[1:])):
        pis.append(sharded_chain_pair(
            fixed, moving, i, rank, world, comm, mode=mode, exchange=exchange, device=device, rep_layer=rep_layer,
            rep_field=rep_field, dissimilarity=dissimilarity, genes=genes, spatial_key=key_added, key_added=key_added,
            iter_key_added=iter_key_added, vecfld_key_added=vecfld_key_added, max_iter=max_iter, dtype=dtype,
            verbose=verbose and rank == 0, **kwargs,
        ))
    return aligned, pis
