"""not-gpu: the reduce tests' restatement of the kernel's launch geometry (tests/reduce_geometry.py), checked
against a thread-by-thread walk of the kernel's three loops."""
import numpy as np
import pytest

from reduce_geometry import PACKET, THREADS, reduce_geometry

T = 64 * 1024


def _walk(n, es, addr, loads, cap):
    """Run the loops of map_reduce_kernel for every (CTA, thread) of the launch, vectorised over threads.
    Returns (values added by each thread, packet indices read, element indices read)."""
    grid = reduce_geometry(n, es, addr, loads, cap).grid
    block = np.repeat(np.arange(grid, dtype=np.int64), THREADS)
    tid = np.tile(np.arange(THREADS, dtype=np.int64), grid)
    stride = grid * THREADS
    n_vec = (n * es) // PACKET if addr % PACKET == 0 else 0
    tile_packets = loads * THREADS
    n_tiles = n_vec // tile_packets
    count = np.zeros(grid * THREADS, dtype=np.int64)
    packets, elems = [], []
    t = block.copy()                                   # for (t = blockIdx.x; t < n_tiles; t += gridDim.x)
    while (live := t < n_tiles).any():
        v = t[live] * tile_packets + tid[live]
        for j in range(loads):
            packets.append(v + j * THREADS)
        count[live] += loads * (PACKET // es)
        t += grid
    v = n_tiles * tile_packets + block * THREADS + tid  # remainder packets
    while (live := v < n_vec).any():
        packets.append(v[live])
        count[live] += PACKET // es
        v += stride
    e = (n_vec * PACKET) // es + block * THREADS + tid  # element tail
    while (live := e < n).any():
        elems.append(e[live])
        count[live] += 1
        e += stride
    cat = lambda xs: np.concatenate(xs) if xs else np.zeros(0, dtype=np.int64)  # noqa: E731
    return count, cat(packets), cat(elems), n_vec


def _cases():
    out = []
    for es in (2, 4, 8):
        for nbytes in (0, es, 32 - es, 32, 32 + es, T - 32, T - es, T, T + es, T + 32, 2 * T, 7 * T + 3 * 32 + es,
                       5 * T + 3 * 32 * 256 + 7 * es):
            for addr in (0, es, 32 - es):
                out.append((nbytes // es, es, addr, 8, 4))
        # LOADS 4 and the 1024-CTA cap, with more tiles than CTAs so the tile loop strides
        out.append(((1025 * T // 2 + 3 * 32 * 256 + 7 * es) // es, es, 0, 4, 1))
        out.append(((2048 * T + 32 + es) // es, es, 0, 8, 1))
        out.append(((33 * T // 2) // es, es, es, 4, 1))
    return out


@pytest.mark.parametrize("n,es,addr,loads,cap", _cases())
def test_reduce_geometry_matches_thread_walk(n, es, addr, loads, cap):
    g = reduce_geometry(n, es, addr, loads, cap)
    count, packets, elems, n_vec = _walk(n, es, addr, loads, cap)
    # the walk reads every packet and every tail element exactly once
    assert g.n_vec == n_vec
    assert np.array_equal(np.sort(packets), np.arange(n_vec))
    assert np.array_equal(np.sort(elems), np.arange(n_vec * PACKET // es, n))
    assert g.tail == len(elems) and g.n_tiles * loads * THREADS + g.rem == n_vec
    assert int(count.sum()) == n
    # m bounds the busiest thread, and is reached whenever only one of the three loops runs
    assert g.m >= int(count.max())
    if (g.n_tiles > 0) + (g.rem > 0) + (g.tail > 0) <= 1:
        assert g.m == int(count.max())


def test_reduce_geometry_grid():
    assert reduce_geometry(0, 4).grid == 1
    assert reduce_geometry(T // 4 + 1, 4).grid == 2
    assert reduce_geometry(4096 * T // 4, 4).grid == 4096
    assert reduce_geometry(4097 * T // 4, 4).grid == 4096
    assert reduce_geometry(4097 * T // 4, 4, cap=1).grid == 1024
    assert reduce_geometry(4096 * T // 4, 4, loads=4).grid == 4096          # 8192 tiles of 32 KiB
    assert reduce_geometry(T // 4, 4, loads=4).grid == 2
    g = reduce_geometry(4097 * T // 4 + 3 * 8 * 256 + 7, 4)
    assert (g.n_tiles, g.rem, g.tail, g.m) == (4097, 3 * 256, 7, 2 * 64 + 8 + 1)
    g = reduce_geometry(1000, 2, addr=2)
    assert (g.n_vec, g.tail, g.m) == (0, 1000, 4)
