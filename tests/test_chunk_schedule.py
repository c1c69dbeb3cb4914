"""Chunk table of the dynamically scheduled tensor-core GLM kernel (host code of csrc/glm_tc.cu, no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from pytensor_federated_b200.ops import native

TILE = 128


def chunk_table(n_rows, sm_count=132, multiple=2, max_chunk=32, min_chunk=4):
    lib = native.load()
    rows = (C.c_longlong * len(n_rows))(*n_rows)
    cap = 1 << 20
    out = (C.c_int * (3 * cap))()
    n = lib.b200_glm_tc_chunk_table(rows, len(n_rows), sm_count, multiple, max_chunk, min_chunk, out, cap)
    assert 0 < n <= cap
    return np.frombuffer(out, dtype=np.int32, count=3 * n).reshape(n, 3).copy()


@pytest.mark.parametrize("n_rows", [[10_000_000], [10_000_000] * 8, [4096 + 37, 4096], [1], [128 * 3, 128 * 5 + 1, 77]])
def test_every_tile_is_covered_exactly_once_by_even_chunks(n_rows):
    table = chunk_table(n_rows)
    next_tile = [0] * len(n_rows)
    for seg, first, n in table:
        assert n % 2 == 0 and 2 <= n <= 32                      # the two epilogue groups alternate tiles: even sizes
        assert first == next_tile[seg]                          # consecutive within a segment, segments in order
        tiles = -(-n_rows[seg] // TILE)
        real = min(n, tiles - first)
        assert real >= n - 1 and real >= 1                      # at most one empty tile, at the end of an odd segment
        next_tile[seg] += real
    assert next_tile == [-(-r // TILE) for r in n_rows]
    assert list(table[:, 0]) == sorted(table[:, 0])


def test_chunks_shrink_towards_the_end_of_the_work():
    table = chunk_table([10_000_000] * 8)
    sizes = table[:, 2]
    assert sizes[0] == 32 and sizes[len(sizes) // 2] == 32
    assert sizes[-1] <= 6
    # the tail that keeps 132 SMs busy after the last big chunk is handed out is made of small chunks
    tail = sizes[-300:]
    assert tail.max() <= 8 and (np.diff(sizes[-2000:].astype(int)) <= 2).all()
    # far more chunks than SMs, but not so many that claiming them matters (one atomic per chunk)
    assert 132 * 20 < len(sizes) < 132 * 300


def test_small_problems_still_spread_over_the_sms():
    table = chunk_table([100_000])            # 782 tiles
    assert len(table) >= 132
    tiny = chunk_table([9000])                # 71 tiles
    assert (tiny[:, 2] == 2).all() and len(tiny) == 36


@pytest.mark.parametrize("n_rows", [[10_000_000] * 8, [128 * 7 + 1, 128 * 3, 50]])
def test_fp8_kernel_chunks_hold_whole_rotations_of_its_three_epilogue_groups(n_rows):
    table = chunk_table(n_rows, multiple=3, max_chunk=30, min_chunk=6)
    next_tile = [0] * len(n_rows)
    for seg, first, n in table:
        assert n % 3 == 0 and 3 <= n <= 30 and first == next_tile[seg]
        tiles = -(-n_rows[seg] // TILE)
        real = min(n, tiles - first)
        assert real >= n - 2 and real >= 1              # at most two empty tiles, at the end of a segment
        next_tile[seg] += real
    assert next_tile == [-(-r // TILE) for r in n_rows]
