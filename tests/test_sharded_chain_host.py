"""Host logic of ``morpho_align_column_sharded`` that needs no GPU: the refusal of a dense posterior, the broadcast of
``Collectives`` without a process group, and the shards' use of the global NumPy stream."""

import threading

import numpy as np
import pytest


def test_dense_posterior_refused_up_front():
    import spateo_release_b200 as st

    for P in (True, "auto"):
        with pytest.raises(NotImplementedError, match="sparse_calculation_mode=True"):
            st.align.morpho_align_column_sharded([object(), object()], materialize_P=P)


def test_transfer_takes_keys_only():
    import spateo_release_b200 as st

    with pytest.raises(ValueError, match="ambiguous"):
        st.align.morpho_align_column_sharded([object(), object()], transfer_B=np.ones((3, 1)))


def test_broadcast_without_process_group_returns_the_object():
    from spateo_release_b200.alignment.distributed import Collectives

    obj = {"a": np.arange(3)}
    assert Collectives().broadcast(None, obj) is obj


def test_draws_of_other_ranks_leave_the_stream():
    from spateo_release_b200.alignment.distributed import _draws_of

    np.random.seed(0)
    want = np.random.permutation(50)
    np.random.seed(0)
    with _draws_of(2):
        other = np.random.permutation(50)
    with _draws_of(0):
        got = np.random.permutation(50)
    assert np.array_equal(other, want) and np.array_equal(got, want)


def test_rank0_draws_are_the_serial_ones_while_other_threads_draw():
    """Shards emulated by threads of one process share the stream: rank 0's draws must be those of the unsharded solver
    however the other ranks' draws interleave with them, and the stream must end where rank 0 left it."""
    from spateo_release_b200.alignment.distributed import _draws_of

    np.random.seed(7)
    want = [np.random.permutation(1000) for _ in range(20)]
    end = np.random.get_state()
    np.random.seed(7)
    got, start = [], threading.Barrier(3)

    def rank(r):
        start.wait()
        for _ in range(20):
            with _draws_of(r):
                x = np.random.permutation(1000)
            if r == 0:
                got.append(x)

    threads = [threading.Thread(target=rank, args=(r,)) for r in range(3)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert all(np.array_equal(a, b) for a, b in zip(got, want)) and len(got) == 20
    assert all(np.array_equal(a, b) for a, b in zip(np.random.get_state(), end))
