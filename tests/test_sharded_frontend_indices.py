"""The index rule of the collective front end (sharded.frontend_chunks / frontend_indices): what the GPU tests of
tests/test_gpu_frontend_peer.py build their sequential oracle order from.  CPU only."""
import numpy as np
import pytest

from ct_mapreduce_b200 import sharded


@pytest.mark.parametrize("ns,E", [([0], 7), ([5, 0], 4), ([40, 3, 17], 5), ([1000, 1], 64), ([8, 8], 8), ([9, 8, 0, 30], 3)])
def test_indices_unique_increasing_and_span(ns, E):
    chunks = [sharded.frontend_chunks(np.ones(n, np.uint16), E) for n in ns]
    for n, c in zip(ns, chunks):
        assert sum(c) == n and all(0 < s <= E for s in c) and all(s == E for s in c[:-1])
    idx, span = sharded.frontend_indices(chunks, E, next_index=1000)
    world, rounds = len(ns), max(1, max(len(c) for c in chunks))
    assert span == rounds * world * E
    assert [a.size for a in idx] == ns
    # increasing in (round, rank, position): the sorted order of all indices is that lexicographic order
    key = [(k, r, j) for r, c in enumerate(chunks) for k, s in enumerate(c) for j in range(s)]
    flat = np.concatenate(idx)
    assert np.unique(flat).size == flat.size
    assert [key[i] for i in np.argsort(flat, kind="stable")] == sorted(key)
    assert flat.size == 0 or (flat.min() >= 1000 and flat.max() < 1000 + span)


def test_tiles_chunks_are_whole_tiles_within_the_budget():
    widths = [256, 256, 100, 256, 3, 256]
    assert sharded.frontend_chunks(widths, 600) == [512, 359, 256]
    assert sharded.frontend_chunks(widths, 256) == [256, 256, 100, 256, 3, 256]
    assert sharded.frontend_chunks([], 256) == []


@pytest.mark.parametrize("ns,E", [([300, 300], 100), ([250, 120, 0], 50), ([7], 7)])
def test_agrees_with_host_batch_order(ns, E):
    """With the front end's entry budget equal to the host pipeline's stage size, a collective front-end call orders its
    entries as the collective ctmr_process_batch does (sharded.host_batch_order)."""
    chunks = [sharded.frontend_chunks(np.ones(n), E) for n in ns]
    idx, _ = sharded.frontend_indices(chunks, E)
    order = [(r, j) for r, lo, hi in sharded.host_batch_order(ns, E) for j in range(lo, hi)]
    flat = [(r, j) for r, a in enumerate(idx) for j in range(a.size)]
    by_index = sorted(flat, key=lambda rj: int(idx[rj[0]][rj[1]]))
    assert by_index == order
