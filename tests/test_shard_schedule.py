"""CPU: the host side of a column-sharded SVI pair — every rank's padded share of the batch schedule, the assembly of the
ranks' per-column outputs into the unsharded column order, and the collectives that carry them (gloo, world size 2)."""

import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from spateo_release_b200.alignment.distributed import Collectives, all_gather_rows, assemble_columns, column_block
from spateo_release_b200.alignment.morpho_class import shard_svi_schedule, svi_schedule


@pytest.mark.parametrize("world", [1, 2, 3, 7])
@pytest.mark.parametrize("nb,batch", [(500, 50), (500, 500), (97, 13), (40, 1)])
def test_shard_schedule_partitions_every_batch(world, nb, batch):
    rng = np.random.default_rng(nb * 31 + batch + world)
    max_iter = 23
    sched = svi_schedule(rng.permutation(nb), max_iter, batch)
    shares = [shard_svi_schedule(sched, nb, r, world) for r in range(world)]
    for r, (local, pos) in enumerate(shares):
        c0, c1 = column_block(nb, r, world)
        assert local.shape == pos.shape and local.shape[0] == max_iter and local.dtype == pos.dtype == np.int32
        counts = ((sched >= c0) & (sched < c1)).sum(axis=1)
        assert local.shape[1] == max(1, counts.max())  # the narrowest width that holds every iteration
        real = pos >= 0
        assert np.array_equal(real.sum(axis=1), counts)
        assert (local[~real] == c1 - c0).all()  # the padding is the null column
        for it in range(max_iter):
            p = pos[it][real[it]]
            assert np.array_equal(p, np.sort(p)) and np.all(real[it][: p.size])  # batch order, padding at the end
            assert np.array_equal(local[it][real[it]] + c0, sched[it][p])  # the member at that position, in the block
            assert ((local[it][real[it]] >= 0) & (local[it][real[it]] < c1 - c0)).all()
    for it in range(max_iter):  # the ranks' members together are the batch, each member once
        p = np.concatenate([pos[it][pos[it] >= 0] for _, pos in shares])
        assert np.array_equal(np.sort(p), np.arange(batch))


def test_shard_schedule_block_without_members():
    sched = np.array([[0, 1, 2], [3, 4, 5]], dtype=np.int32)  # rank 1 of 2 owns cells 3..5: none in iteration 0
    local, pos = shard_svi_schedule(sched, 6, 1, 2)
    assert local.tolist() == [[3, 3, 3], [0, 1, 2]] and pos.tolist() == [[-1, -1, -1], [0, 1, 2]]
    local, pos = shard_svi_schedule(np.array([[0, 1]], dtype=np.int32), 6, 1, 2)  # never a member: one null column
    assert local.tolist() == [[3]] and pos.tolist() == [[-1]]


def test_assemble_columns_drops_null_and_gather_padding():
    parts = [np.array([[1, 1], [2, 2], [9, 9]]), np.array([[3, 3], [7, 7], [8, 8]])]
    positions = [np.array([2, 0]), np.array([1, -1])]  # rank 0's third row is gather padding, rank 1's second is null
    out = assemble_columns(parts, positions, 4, fill=-5)
    assert out.tolist() == [[2, 2], [3, 3], [1, 1], [-5, -5]]
    keys = [np.array([5, 1, 0], dtype=np.int64), np.array([2, 2, 7], dtype=np.int64)]
    assert assemble_columns(keys, [np.array([0, 1, 2]), np.array([3, 4, 5])], 6).tolist() == [5, 1, 0, 2, 2, 7]


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    # the solver's own collectives of a column-sharded pair (they touch no device state and ignore the solver)
    comm = Collectives()
    rows = torch.arange(3 + 2 * rank, dtype=torch.int32).reshape(-1, 1) * 10 + rank  # 3 and 5 rows
    parts = [p.numpy() for p in comm.gather(None, rows)]
    # argmax keys: (float bits of p) << 32 | (0xffffffff - column); the row keys are merged with a MAX all_reduce
    vals = np.array([[0.5, 0.25, 0.0], [0.125, 0.75, 0.0]], dtype=np.float32)[rank]
    cols = np.array([[0, 1, 2], [3, 4, 5]], dtype=np.int64)[rank]
    keys = torch.from_numpy((vals.view(np.uint32).astype(np.int64) << 32) | (0xFFFFFFFF - cols))
    comm.max_(None, keys)
    view = torch.tensor([1.0, 2.0 ** -40, -3.0], dtype=torch.float64) * (rank + 1)  # row statistics of this rank
    comm.sum_(None, view)
    q.put((rank, parts, keys.numpy(), view.numpy(), [p.numpy() for p in all_gather_rows(rows[:1])]))
    dist.destroy_process_group()


def test_gather_and_key_merge_world2():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    results = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    want0, want1 = np.arange(3).reshape(-1, 1) * 10, np.arange(5).reshape(-1, 1) * 10 + 1
    for rank, parts, keys, view, firsts in results:
        assert len(parts) == 2 and np.array_equal(parts[0], want0) and np.array_equal(parts[1], want1)
        assert [f.tolist() for f in firsts] == [[[0]], [[1]]]
        assert view.tolist() == [3.0, 3 * 2.0 ** -40, -9.0]
        val = (keys.astype(np.uint64) >> np.uint64(32)).astype(np.uint32).view(np.float32)
        col = 0xFFFFFFFF - (keys & 0xFFFFFFFF)
        assert val.tolist() == [0.5, 0.75, 0.0] and col.tolist() == [0, 4, 2]  # ties at 0: the lowest column
