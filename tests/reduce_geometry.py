"""The launch geometry of `map_reduce_kernel` (csrc/ktb_reduce.cu), restated for the reduce tests.

`launch_reduce_typed` sizes the grid as one tile of LOADS x 256 x 32 bytes per CTA, capped at
min(4096, 1024 * ktb_set_tuning key 6). Inside the kernel each thread adds, in this order:
  1. whole tiles, grid-strided by CTA: LOADS 32-byte packets per thread and tile;
  2. the remainder packets past the last whole tile, one per thread, grid-strided;
  3. the element tail past the last packet, one element per thread, grid-strided.
A start address that is not 32-byte aligned has no packets: everything is element tail.
"""
from dataclasses import dataclass

THREADS = 256
PACKET = 32
MAX_GRID = 4096


def _cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Geometry:
    tile: int      # bytes per tile
    grid: int      # CTAs launched
    n_vec: int     # 32-byte packets
    n_tiles: int   # whole tiles
    rem: int       # remainder packets after the whole tiles
    tail: int      # elements after the last packet
    m: int         # most mapped values any one thread adds (an upper bound: the three loops' maxima summed)


def reduce_geometry(n, es, addr=0, loads=8, cap=4):
    """Geometry of one `ktb_map_reduce_sum` launch over n elements of es bytes starting at byte address addr.
    loads is ktb_set_tuning key 13 (8 or 4), cap is key 6 (the grid cap in units of 1024 CTAs; <= 0 means 4096)."""
    loads = 4 if loads == 4 else 8
    tile = loads * THREADS * PACKET
    tiles = _cdiv(n * es, tile)
    grid_cap = min(MAX_GRID, cap * 1024) if cap > 0 else MAX_GRID
    grid = min(max(tiles, 1), grid_cap)
    n_vec = (n * es) // PACKET if addr % PACKET == 0 else 0
    tile_packets = loads * THREADS
    n_tiles = n_vec // tile_packets
    rem = n_vec - n_tiles * tile_packets
    tail = n - n_vec * PACKET // es
    per_packet = PACKET // es
    m = (_cdiv(n_tiles, grid) * loads * per_packet + _cdiv(rem, THREADS * grid) * per_packet
         + _cdiv(tail, THREADS * grid))
    return Geometry(tile, grid, n_vec, n_tiles, rem, tail, m)
