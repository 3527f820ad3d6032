"""CPU: the global curriculum's payload (uhc_curriculum_stage / uhc_curriculum_update_gathered, rules in uhc_b200/csrc/curriculum_core.h)
compiled for the host, and the Python update path's encoding of it in the value gradient's tail (nn.pack_stats_tail / unpack_stats_tail)
over a real gloo all-reduce of two processes.

The claim under test: each rank writes only its own slot of a zeroed [world][T][E][3] fp32 array, so an fp32 sum over the ranks, in any
order, returns every rank's log bit for bit, and the rings one curriculum builds from it equal the rings it builds from the concatenated logs."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.emu import curriculum_emu as CE
from tests.emu import curriculum_global_emu as E

BIG = 1 << 24


def _log(rs, T, Ed, C, max_start, p_end=0.6, hot=None):
    clip = np.where(rs.uniform(size=(T, Ed)) < p_end, rs.randint(0, C, (T, Ed)), -1).astype(np.int32)
    if hot is not None:
        clip[(clip >= 0) & (rs.uniform(size=(T, Ed)) < 0.5)] = hot
    pct = np.where(rs.uniform(size=(T, Ed)) < 0.4, 1.0, rs.uniform(size=(T, Ed))).astype(np.float32)
    pct[rs.uniform(size=(T, Ed)) < 0.05] = 0.0
    start = rs.randint(max(0, max_start - 1000), max_start + 1, (T, Ed)).astype(np.int32)
    start[clip < 0] = -1                                        # the step kernel's "never recorded" start of an env with no ended episode
    return clip, pct, start


def _staged(logs, W):
    """every rank's slots array: zeros except its own slot"""
    T, Ed = logs[0][0].shape
    out = []
    for r in range(W):
        s = np.zeros((W, T * Ed, 3), np.float32)
        s[r] = E.stage(*logs[r])
        out.append(s.reshape(-1))
    return out


def _sums(slots, rs):
    """fp32 sums of the ranks' arrays in several association orders: rank order, reversed, a random order, a pairwise tree"""
    W = len(slots)
    orders = [list(range(W)), list(range(W))[::-1], list(rs.permutation(W))]
    out = []
    for o in orders:
        acc = slots[o[0]].copy()
        for r in o[1:]:
            acc = (acc + slots[r]).astype(np.float32)
        out.append(acc)
    level = [s.copy() for s in slots]
    while len(level) > 1:
        level = [(level[i] + level[i + 1]).astype(np.float32) if i + 1 < len(level) else level[i] for i in range(0, len(level), 2)]
    out.append(level[0])
    return out


@pytest.mark.parametrize("W", [2, 3, 8])
@pytest.mark.parametrize("C, max_start", [(7, 300), (BIG, BIG - 1)])
def test_stage_sum_unpack_is_exact(W, C, max_start):
    """clip indices and starts up to 2^24 - 1, percents in [0, 1], empty entries: the unpacked sum is the concatenated logs (rank-major, then
    step-major, then env-minor), bit for bit, whatever order the sum takes; empty entries come back as (-1, 0, 0)"""
    rs = np.random.RandomState(W * 31 + C % 97)
    T, Ed = 5, 37
    logs = [_log(rs, T, Ed, C, max_start) for _ in range(W)]
    cat = [np.concatenate([l[k].reshape(-1) for l in logs]) for k in range(3)]
    valid = cat[0] >= 0
    if C == BIG:
        assert cat[0].max() > BIG - 1000 or (cat[0] > BIG // 2).any()
        assert cat[2][valid].max() > BIG - 1000
    for s in _sums(_staged(logs, W), rs):
        c, p, st = E.unpack(s)
        assert np.array_equal(c, np.where(valid, cat[0], -1))
        assert np.array_equal(p.view(np.int32), np.where(valid, cat[1], 0.0).astype(np.float32).view(np.int32))
        assert np.array_equal(st, np.where(valid, cat[2], 0))


@pytest.mark.parametrize("W", [2, 4])
def test_gathered_rings_equal_one_curriculum_fed_every_log(W):
    """the rings and weights from the unpacked sum equal those of one curriculum fed the concatenated logs, over three rollouts; one clip ends
    more than max_freq times across the ranks in each rollout"""
    rs = np.random.RandomState(5 + W)
    C, M, T, Ed = 11, 20, 6, 24
    a, b = CE.Rings(C, M), CE.Rings(C, M)
    for it in range(3):
        logs = [_log(rs, T, Ed, C, 300, hot=3) for _ in range(W)]
        cat = [np.concatenate([l[k].reshape(-1) for l in logs]) for k in range(3)]
        assert (cat[0] == 3).sum() > M
        a.append(*cat)
        b.append(*E.unpack(_sums(_staged(logs, W), rs)[2]))
        assert np.array_equal(a.meta, b.meta) and np.array_equal(a.pct.view(np.int32), b.pct.view(np.int32)) and np.array_equal(a.start, b.start), it
        wa, ca = a.weights(0.2, 0.5)
        wb, cb = b.weights(0.2, 0.5)
        assert np.array_equal(wa, wb) and np.array_equal(ca, cb)


def test_exactness_bound():
    """the stage refuses (uhc_curriculum_stage returns -2) above 2^24 clips or 2^24 frames: the first integer fp32 cannot hold is 2^24 + 1"""
    assert E.stage_exact(BIG, BIG) and E.stage_exact(1, 1)
    assert not E.stage_exact(BIG + 1, 10) and not E.stage_exact(10, BIG + 1)
    assert int(np.float32(BIG - 1)) == BIG - 1 and int(np.float32(BIG + 1)) != BIG + 1


# ---- the Python update path's tail over gloo
def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _tail_worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from uhc_b200 import nn
    try:
        D, T, Ed, C = 5, 3, 16, BIG
        rs = np.random.RandomState(40 + rank)
        logs = [_log(np.random.RandomState(40 + r), T, Ed, C, BIG - 1) for r in range(world)]   # every rank can rebuild the others' logs
        d = torch.tensor(rs.normal(0.0, 100.0, 4 + 1 + 2 * D))
        slots = np.zeros((world, T * Ed, 3), np.float32)
        slots[rank] = E.stage(*logs[rank])
        extra = torch.from_numpy(slots.reshape(-1))
        tail = torch.full((nn.stats_tail_floats(D) + extra.numel() + 7,), 3.0)       # stale contents beyond the payload must not leak in
        nn.pack_stats_tail(tail, d, extra)
        plain = torch.zeros(nn.stats_tail_floats(D))
        nn.pack_stats_tail(plain, d)
        ok_layout = bool(torch.equal(tail[:plain.numel()], plain) and torch.equal(plain, nn.split_double(d).reshape(-1)) and (tail[-7:] == 0).all())
        try:
            nn.pack_stats_tail(torch.zeros(plain.numel() + extra.numel() - 1), d, extra)
            ok_refuse = False
        except ValueError:
            ok_refuse = True
        nn.GradComm(world).start(tail)                                        # gloo: synchronous all-reduce(sum)
        g, ex = nn.unpack_stats_tail(tail, d.numel(), extra.numel())
        c, p, s = E.unpack(ex.numpy())
        cat = [np.concatenate([l[k].reshape(-1) for l in logs]) for k in range(3)]
        valid = cat[0] >= 0
        ok_payload = (np.array_equal(c, np.where(valid, cat[0], -1)) and np.array_equal(p, np.where(valid, cat[1], 0.0)) and np.array_equal(s, np.where(valid, cat[2], 0)))
        gathered = [None] * world
        dist.all_gather_object(gathered, d.tolist())
        ref = np.sum(np.array(gathered), axis=0)
        ok_stats = bool(np.allclose(g.numpy(), ref, rtol=0, atol=2.0 ** -28))
        out.put((rank, ok_layout, ok_refuse, bool(ok_payload), ok_stats, None))
    except BaseException as e:
        out.put((rank, False, False, False, False, repr(e)))
    dist.destroy_process_group()


def test_python_path_tail_encode_decode_world2():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_tail_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = sorted(q.get(timeout=120) for _ in ps)
    [p.join(30) for p in ps]
    assert all(r[1] and r[2] and r[3] and r[4] for r in res), res
