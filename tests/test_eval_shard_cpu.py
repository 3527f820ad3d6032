"""CPU: the evaluation's split of clips over the ranks (uhc_b200.agent.assign_clips) and, over a two-process gloo group, the helpers that
exchange every rank's results and eval outcomes (uhc/agents/agent_copycat.py exchange, merge_results, merge_outcomes, gather_to_root)."""
import os
import socket
import types

import numpy as np
import pytest
import torch.multiprocessing as mp

from uhc_b200.agent import assign_clips, call_env_steps, shard_clips


def _lens(n, seed):
    return np.random.RandomState(seed).randint(2, 400, n)


@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("n,E", [(37, 4), (101, 7), (9, 2), (64, 3)])
def test_assignment_partitions_and_balances(world, n, E):
    if n % world == 0:
        n += 1                                   # a clip count the ranks do not divide
    assert E < -(-n // world) or world == 8      # E below a rank's share (for world 8 at the smallest n the share is 2)
    lens = _lens(n, n * 31 + world)
    calls = assign_clips(lens, world, E)
    assert len(calls) == world
    for r in range(world):
        assert [c.tolist() for c in shard_clips(lens, world, r, E)] == [c.tolist() for c in calls[r]]
    every = np.concatenate([c for rank in calls for c in rank])
    assert sorted(every.tolist()) == list(range(n))                       # a partition: every clip on exactly one rank, once
    assert all(1 <= len(c) <= E and c.dtype == np.int32 for rank in calls for c in rank)
    steps = [sum(call_env_steps(lens[c]) for c in rank) for rank in calls]
    total = sum(call_env_steps(lens[c]) for rank in calls for c in rank)
    largest = max(call_env_steps(lens[c]) for rank in calls for c in rank)
    assert max(steps) <= total / world + largest
    if world == 1:                               # today's contiguous chunks
        assert [c.tolist() for c in calls[0]] == [list(range(c0, min(n, c0 + E))) for c0 in range(0, n, E)]
    else:                                        # calls of consecutive clips in descending length
        b = min(E, -(-n // world))
        order = np.argsort(-lens, kind="stable")
        blocks = sorted((c.tolist() for rank in calls for c in rank), key=lambda c: order.tolist().index(c[0]))
        assert [x for c in blocks for x in c] == order.tolist() and all(len(c) == b for c in blocks[:-1])


def test_assignment_edge_cases():
    assert assign_clips(np.zeros(0, np.int64), 3, 4) == [[], [], []]
    assert [c.tolist() for c in assign_clips([5, 9], 3, 4)[0]] == [[1]]            # more ranks than clips: the last rank has none
    assert assign_clips([5, 9], 3, 4)[2] == []
    assert call_env_steps([]) == 0 and call_env_steps([3, 10, 4]) == 27


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from uhc.agents.agent_copycat import AgentCopycat, exchange, gather_to_root, merge_outcomes, merge_results
        keys = [f"clip{c:02d}" for c in range(7)]
        mine = [6, 2, 3] if rank == 0 else [5, 0, 1, 4]           # each rank's clips in the order of its calls, not in clip order
        res = {keys[c]: {"mpjpe": np.full(c + 1, 0.1 * c), "succ": np.array([c % 2 == 0]), "pred": np.full((c + 2, 3), float(c))} for c in mine}
        outcomes = [(c, 10 + c % 3, 0.25 * c) for c in mine]    # (table clip, training clip, outcome): clips 0 / 3 / 6 share training clip 10
        parts = exchange(lambda: ({k: {m: v for m, v in d.items() if m != "pred"} for k, d in res.items()}, outcomes))
        merged = merge_results([p[0] for p in parts], keys)
        pend = merge_outcomes([p[1] for p in parts])
        stub = types.SimpleNamespace(curriculum_on_device=False, max_freq=2, data_loader=types.SimpleNamespace(data_keys=[f"t{i}" for i in range(13)]),
                                     freq_dict={f"t{i}": [] for i in range(13)})
        AgentCopycat._apply_outcomes(stub, pend)
        pushed = []
        dev = types.SimpleNamespace(curriculum_on_device=True, agent=types.SimpleNamespace(curriculum_push=lambda c, p, s: pushed.append((c, p, s))))
        AgentCopycat._apply_outcomes(dev, pend)
        full = gather_to_root(res, max_bytes=64)                    # one clip per piece at this bound
        try:
            exchange(lambda: 1 / (rank - 1))                        # rank 1 raises: both ranks must raise, neither may wait
            failed = None
        except RuntimeError as e:
            failed = str(e)
        q.put((rank, list(merged), {k: (v["mpjpe"].tolist(), bool(v["succ"][0])) for k, v in merged.items()}, all("pred" not in v for v in merged.values()),
               pend, stub.freq_dict, pushed, sorted(full), {k: v["pred"].tolist() for k, v in full.items()}, failed))
    except Exception as e:       # reported, so a failure shows the error and does not leave the parent waiting
        q.put((rank, repr(e)))
    finally:
        dist.destroy_process_group()


def test_exchange_helpers_gloo():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    try:
        out = dict((r[0], r) for r in (q.get(timeout=180) for _ in ps))
    finally:
        for p in ps:
            p.join(30)
            if p.is_alive():
                p.terminate()
                p.join()
    assert all(len(out[r]) > 2 for r in (0, 1)), out
    keys = [f"clip{c:02d}" for c in range(7)]
    for r in (0, 1):
        _, order, vals, stripped, pend, fd, pushed, full_keys, full_pred, failed = out[r]
        assert order == keys                                                    # clip-key order, whatever each rank's call order
        assert vals == {keys[c]: ([0.1 * c] * (c + 1), c % 2 == 0) for c in range(7)}
        assert stripped
        assert pend == [(c, 10 + c % 3, 0.25 * c) for c in range(7)]            # clip-index order
        # applied in clip order: training clip 10 gets clips 0, 3, 6 in that order, kept to max_freq = 2
        assert fd["t10"] == [[0.75, 0], [1.5, 0]] and fd["t11"] == [[0.25, 0], [1.0, 0]] and fd["t12"] == [[0.5, 0], [1.25, 0]]
        assert pushed == [([10 + c % 3 for c in range(7)], [0.25 * c for c in range(7)], [0] * 7)]
        assert failed is not None and "rank 1" in failed and "ZeroDivisionError" in failed
    assert out[0][7] == keys and out[0][8] == {keys[c]: [[float(c)] * 3] * (c + 2) for c in range(7)}      # rank 0 holds every trajectory
    assert out[1][7] == sorted(keys[c] for c in (5, 0, 1, 4))                                           # rank 1 only its own


def test_clip_betas_of_an_empty_shard():
    """render_motion(body="mesh") with has_shape on a rank that gets no clips (a loader with fewer clips than ranks) passes [0][10] betas"""
    from uhc.agents.agent_copycat import clip_betas
    shapes = [np.arange(17, dtype=np.float64) + 100 * c for c in range(2)]
    for clips in (np.concatenate([np.zeros(0, np.int32)] + shard_clips([30, 40], 3, r, 4)) for r in range(3)):
        b = clip_betas(shapes, clips)
        assert b.shape == (len(clips), 10) and b.dtype == np.float64
        assert np.array_equal(b, np.stack([shapes[c][:10] for c in clips]) if len(clips) else np.zeros((0, 10)))
    assert len(shard_clips([30, 40], 3, 2, 4)) == 0
