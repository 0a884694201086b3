"""Pair layouts in the GPU tests: a streamed cost matrix forced by the memory budget, and a column-sharded pair emulated
by W solver objects of one process, stepped in lock-step."""

import threading
from concurrent.futures import ThreadPoolExecutor

import numpy as np


def force_width(monkeypatch, n_moving, n_fixed, features, width):
    """Budget that fits a streamed run of ``width``-column chunks, and nothing wider."""
    import torch

    from spateo_release_b200.alignment import morpho_class as mc
    from spateo_release_b200.alignment.distributed import pair_device_bytes

    n_sms = torch.cuda.get_device_properties(0).multi_processor_count
    budget = pair_device_bytes(n_moving, n_fixed, features, chunk_cols=width, n_sms=n_sms)
    assert budget < pair_device_bytes(n_moving, n_fixed, features)
    monkeypatch.setattr(mc, "_device_budget", lambda dev: budget)


def three_chunks(cols):
    """A width that splits ``cols`` columns into three chunks, the last one shorter."""
    w = -(-cols // 3)
    w = -(-w // 8) * 8
    assert cols - 2 * w < w
    return w


class LockStep:
    """Collectives of W shards of one process, each driven by its own thread: sums in rank order, like the peer-memory
    kernel, so every replica gets the same bits."""

    def __init__(self, world):
        self.bar = threading.Barrier(world, timeout=600)
        self.slot = [None] * world

    def _exchange(self, m, t):
        self.slot[int(m.column_shard[0])] = t.clone()
        self.bar.wait()
        out = list(self.slot)
        self.bar.wait()
        return out

    def sum_(self, m, view):
        parts = self._exchange(m, view)
        total = parts[0].clone()
        for v in parts[1:]:
            total += v
        view.copy_(total)

    def max_(self, m, keys):
        keys.copy_(__import__("torch").stack(self._exchange(m, keys)).max(dim=0).values)

    def gather(self, m, t):
        return self._exchange(m, t)


def sharded_solvers(A, B, world, **kw):
    """The unsharded solver of moving ``B`` onto fixed ``A`` and W column shards of it, all with the same host
    initialisation (the driver broadcasts rank 0's). Returns (ref, shards), device state prepared on the shards only."""
    import spateo_release_b200 as st
    from spateo_release_b200.alignment.distributed import _HOST_INIT_FIELDS

    np.random.seed(0)
    ref = st.align.Morpho_pairwise(sampleA=B, sampleB=A, **kw)
    ref.prepare_host()  # consumes the random stream (SVI batch permutation) before the shards reseed it
    shards = []
    for r in range(world):
        np.random.seed(0)
        m = st.align.Morpho_pairwise(sampleA=B, sampleB=A, column_shard=(r, world, "nccl"), **kw)
        m.prepare_host()
        shards.append(m)
    for m in shards[1:]:
        for k in _HOST_INIT_FIELDS:
            if hasattr(shards[0], k):
                setattr(m, k, getattr(shards[0], k))
    for m in shards:
        m.prepare_device()
    return ref, shards


def stream():
    import ctypes as C

    import torch

    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def lockstep_iterations(shards, iters):
    """The shards' iterations through the solver's two halves of a sharded iteration, with the cross-rank sum of the row
    statistics done here in rank order; the last iteration captures the posterior as ``run_em`` does."""
    import torch

    st, m0 = stream(), shards[0]
    for it in iters:
        want_P = m0._captures_posterior and it == m0.max_iter - 1 and not (m0.return_mapping and m0.SVI_mode)
        views = [m._shard_iteration_local(it, st, capture_P=want_P) for m in shards]
        total = torch.zeros_like(views[0])
        for v in views:  # rank order
            total += v
        for v in views:
            v.copy_(total)
        for m in shards:
            m._shard_iteration_finish(it, st)


def finish_all(shards):
    """The closing ``_finish`` of every shard, one thread each, exchanging through a ``LockStep``."""
    comm = LockStep(len(shards))
    for m in shards:
        m._shard_comm = comm
    with ThreadPoolExecutor(len(shards)) as ex:
        for f in [ex.submit(m._finish) for m in shards]:
            f.result()


def run_sharded(shards):
    lockstep_iterations(shards, range(shards[0].max_iter))
    finish_all(shards)
