"""CPU: the host side of the grouped evaluation (several checkpoints side by side in one device call).

- pack_groups: how BatchedAgent.evaluate_policies splits K checkpoints x n clips into calls of at most E envs and 64 groups;
- group_core.h's row-tile schedule of the grouped GEMM, through its host build: every (row, group) in exactly one tile, no tile
  reaching into another group's rows, a bounded tile count, bad group layouts refused;
- the C ABI's argument checks that run before any device call."""
import ctypes as C
import itertools
import math

import numpy as np
import pytest

from tests.emu import group_emu
from uhc_b200.agent import MAX_EVAL_GROUPS, pack_groups


@pytest.mark.parametrize("K,n,E", [(1, 1, 1), (1, 10, 4096), (4, 16, 4096), (32, 128, 4096), (32, 512, 4096), (16, 512, 4096),
                                   (3, 10, 4), (2, 7, 7), (5, 3, 8), (300, 16, 4096), (64, 1, 64), (65, 1, 64), (7, 4096, 4096), (2, 5000, 4096)])
def test_pack_groups_covers_every_pair_once(K, n, E):
    calls = pack_groups(K, n, E)
    seen = []
    for call in calls:
        assert 1 <= len(call) <= MAX_EVAL_GROUPS
        assert sum(c1 - c0 for _, c0, c1 in call) <= E
        ks = [k for k, _, _ in call]
        assert len(set(ks)) == len(ks), "a checkpoint appears twice in one call"
        for k, c0, c1 in call:
            assert 0 <= c0 < c1 <= n
            seen.extend((k, c) for c in range(c0, c1))
    assert seen == [(k, c) for k in range(K) for c in range(n)], "every (checkpoint, clip) once, checkpoint-major"
    # calls are full except the last: as few as E envs and the group cap allow
    for call in calls[:-1]:
        assert sum(c1 - c0 for _, c0, c1 in call) == E or len(call) == MAX_EVAL_GROUPS
    groups = sum(len(c) for c in calls)
    assert len(calls) <= math.ceil(K * n / E) + math.ceil(groups / MAX_EVAL_GROUPS)
    if n <= E and K <= MAX_EVAL_GROUPS and K * n <= E:
        assert len(calls) == 1 and [c for c in calls[0]] == [(k, 0, n) for k in range(K)]


def test_pack_groups_group_cap():
    calls = pack_groups(100, 2, 4096)
    assert [len(c) for c in calls] == [64, 36]
    assert pack_groups(4, 3, 5, max_groups=2) == [[(0, 0, 3), (1, 0, 2)], [(1, 2, 3), (2, 0, 3)], [(3, 0, 3)]]


def _check_plan(row0, rows, M):
    rc, tiles = group_emu.group_tiles(row0, rows, M)
    assert rc == 0
    owner = np.full(M, -1)
    for g, r0, n in zip(itertools.count(), row0, rows):
        owner[r0:r0 + n] = g
    cover = np.zeros(M, np.int64)
    for t, (g, first, end) in enumerate(tiles):
        assert end == row0[g] + rows[g] and row0[g] <= first < end
        assert (first - row0[g]) % 128 == 0
        stored = np.arange(first, min(first + 128, end))       # the rows the tile writes
        assert (owner[stored] == g).all(), "a tile writes rows of another group"
        cover[stored] += 1
        if t > 0:
            assert tiles[t - 1][0] <= g, "tiles are in group order"
    assert (cover[owner >= 0] == 1).all(), "every row of every group in exactly one tile"
    assert (cover[owner < 0] == 0).all(), "rows outside the groups are never written"
    assert len(tiles) == sum((n + 127) // 128 for n in rows)
    assert len(tiles) <= math.ceil(sum(rows) / 128) + len(rows) - 1
    return tiles


@pytest.mark.parametrize("sizes", [[1], [63], [64], [127], [128], [129], [300], [1, 63, 64, 127, 128, 129, 300],
                                   [64] * 64, [1] * 64, [4096], [2048, 1024, 512, 256, 128, 64, 32, 16, 8, 4, 2, 1, 1]])
def test_tile_plan_contiguous_groups(sizes):
    row0 = np.concatenate([[0], np.cumsum(sizes)[:-1]]).astype(int)
    _check_plan(row0, sizes, int(sum(sizes)) + 17)


def test_tile_plan_with_gaps_and_random_layouts():
    rng = np.random.default_rng(0)
    for _ in range(300):
        G = int(rng.integers(1, 65))
        rows = rng.integers(1, 300, G)
        gaps = rng.integers(0, 3, G) * rng.integers(0, 200, G)
        row0 = np.cumsum(np.concatenate([[gaps[0]], rows[:-1] + gaps[1:]]))
        _check_plan(row0.astype(int), rows.astype(int), int(row0[-1] + rows[-1] + rng.integers(0, 100)))


@pytest.mark.parametrize("row0,rows,M", [([], [], 10), ([0] * 65, [1] * 65, 100), ([0], [0], 10), ([0, 5], [6, 3], 20), ([5, 0], [3, 3], 20),
                                         ([0], [11], 10), ([-1], [3], 10), ([0, 3], [3, -1], 10)])
def test_tile_plan_refuses_bad_layouts(row0, rows, M):
    rc, _ = group_emu.group_tiles(row0, rows, M)
    assert rc == -2


def _lib():
    from uhc_b200 import build
    return C.CDLL(build.build())


def test_grouped_gemm_argument_checks_before_any_device_call():
    L = _lib()
    L.uhc_tc_last_error.restype = C.c_char_p
    ip = lambda a: (C.c_int * len(a))(*a)
    W = (C.c_void_p * 2)(16, 32)
    f = L.uhc_linear_forward_tc_grouped
    x, y = C.c_void_p(64), C.c_void_p(128)
    args = lambda G=2, r0=(0, 100), rs=(100, 50), Wp=W, Kp=704, N=2048, M=4096, ldy=2048, yb=y, yf=None: \
        f(C.c_int(G), ip(r0), ip(rs), x, Wp, None, yb, yf, C.c_int(M), C.c_int(N), C.c_int(Kp), C.c_int(ldy), C.c_int(1), None)
    for bad in (dict(G=0), dict(G=65), dict(r0=(0, 50)), dict(rs=(100, 0)), dict(r0=(0, 4050)), dict(Kp=700), dict(N=0), dict(M=0), dict(ldy=2044),
                dict(ldy=1024), dict(yb=None), dict(Wp=(C.c_void_p * 2)(16, None)), dict(Wp=None)):
        assert args(**bad) == -2, bad
        assert L.uhc_tc_last_error().startswith(b"uhc_linear_forward_tc_grouped")


def test_eval_run_groups_null_engine_is_refused():
    L = _lib()
    L.uhc_eval_last_error.restype = C.c_char_p
    for fn in (L.uhc_eval_run_groups, L.uhc_eval_run_groups_mcp):
        n = (C.c_int * 1)(1)
        rc = fn(None, C.c_int(1), n, n, None, None, C.c_float(5.0), C.c_int(1), C.c_int(32), None, None, None, None)
        assert rc == -2 and b"null" in L.uhc_eval_last_error()
