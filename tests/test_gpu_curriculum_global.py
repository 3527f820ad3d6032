"""GPU: the global curriculum (BatchedAgent(curriculum_global=True), uhc_curriculum_stage / uhc_curriculum_update_gathered, uhc_ppo_update_ex)
on one GPU: W ranks are W BatchedAgents with their own engines and rank seeds, joined by the in-process all-reduce of tests/loopback_comm.py.

After every update each rank must hold the same rings and CDF, bit for bit, as one curriculum fed every rank's episode log through
uhc_curriculum_push in rank-major, step-major, env-minor order; and the payload must not move a bit of the update itself (parameters, Adam
moments, running_state, losses against ranks without the flag, on the same buffers).  The update itself is not bitwise reproducible from one
run to the next (its split-K weight gradients and bias gradients are fp32 atomic sums), so parameters, Adam moments and losses are held to the
criterion tests/test_gpu_ppo_multirank.py holds two update paths to; what does not go through those sums is compared bit for bit: running_state,
the step counters, and the collective's length, which puts the payload past the gradients and the statistics.  The fp32 exactness bound of
the payload (more than 2^24 clips or frames) is checked by tests/test_emu_curriculum_global.py: no test engine can load a table that large."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests.loopback_comm import LoopbackGradComm, LoopbackGroup

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")
LENS = [30, 45, 60, 33]
M, T, E = 8, 12, 64


def _clips():
    z = np.load(os.path.join(G, "expert_sway.npz"))
    ex = {k: z[k] for k in z.files}
    so = np.concatenate([ex["beta"][0], [ex["gender"][0]]])
    n = len(ex["qpos"])

    def clip(L):
        idx = np.arange(L) % n
        return {k: (np.asarray(v)[idx] if np.ndim(v) > 0 and len(v) == n else v) for k, v in ex.items()}
    return [clip(L) for L in LENS], [so] * len(LENS)


def _agent(rank, W, path="c", flag=True, cur=True):
    """rank `rank` of W; path "c": uhc_ppo_update_ex, "py": the Python-orchestrated tensor-core update"""
    from uhc_b200.agent import BatchedAgent
    clips, shapes = _clips()
    ag = BatchedAgent(E, clips, shapes, policy_hsize=(64,), value_hsize=(64,), seed=3, t_min=2, t_max=8, rank=rank, world=W, curriculum_global=flag,
                      c_update=path == "c", num_optim_epoch=2)
    if cur:
        ag.curriculum_enable(M, 0.2, 0.5, 0.0, -1)
    return ag


def _join(ags, path):
    """the ranks' collective: the loopback group in place of ncclAllReduce (C path) or of torch.distributed (Python path)"""
    from uhc_b200 import nn
    g = LoopbackGroup(len(ags))
    for r, ag in enumerate(ags):
        if path == "c":
            ag._nccl = g.comm(r)
            ag._ctrainer = nn.CPpoTrainer(ag.policy, ag.value, ag.opt_p, ag.opt_v, T * E, E, ag.dev, all_reduce=g.fn)
        else:
            ag.comm = LoopbackGradComm(g, r)
    return g


def _rings(ag):
    ln, p, s = ag.curriculum_get()
    return ln, p.view(np.int32), s, ag.engine.clip_cdf().view(np.int32)


def _same_rings(a, b):
    return all(np.array_equal(x, y) for x, y in zip(a, b))


def _log(buf):
    return [getattr(buf, k)[:T].cpu().numpy().reshape(-1) for k in ("ep_clip", "ep_pct", "ep_start")]


def _push(ref, logs):
    """the reference: one curriculum fed every rank's log, rank-major, then step-major, then env-minor (only ended episodes)"""
    c, p, s = (np.concatenate([l[k] for l in logs]) for k in range(3))
    sel = c >= 0
    ref.engine.curriculum_push(c[sel], p[sel], s[sel])
    return np.bincount(c[sel], minlength=len(LENS))


def _state(ag):
    return [t.clone() for t in (ag.policy.flat, ag.value.flat, ag.opt_p.mflat, ag.opt_p.vflat, ag.opt_v.mflat, ag.opt_v.vflat, ag.running_state.stats)]


def _close_update(on, off, first, lr_p=5e-5, lr_v=3e-4, tag=""):
    """flag on against flag off after the same updates from the same first parameters: the parameter changes agree as
    test_gpu_ppo_multirank's sharded / unsharded paths must (mean |difference| / mean |change| < 0.02), the Adam moments to 1e-2 relative"""
    for i, lr in ((0, lr_p), (1, lr_v)):
        d1, d2 = on[i] - first[i], off[i] - first[i]
        assert d1.abs().max().item() > 0.1 * lr, (tag, i)
        rel = (d1 - d2).abs().mean().item() / d1.abs().mean().item()
        assert rel < 0.02, (tag, i, rel)
    for i in range(2, 6):
        rel = ((on[i] - off[i]).norm() / on[i].norm().clamp(min=1e-30)).item()
        assert rel < 1e-2, (tag, i, rel)


def _iteration(ags, bufs, group, offs=None, off_group=None, fill=None, first=None):
    """sample on every rank, then every rank's update_params at once; offs: ranks without the flag that update on the same buffers from the
    same running_state.  fill(r, buf): rewrites rank r's episode log before it is staged again.  Returns the ranks' logs and update logs."""
    W = len(ags)
    for r, ag in enumerate(ags):
        ag.sample(T, bufs[r])
        if fill is not None:
            fill(r, bufs[r])
            ag.engine.curriculum_stage(bufs[r], T, r, W, ag._cur_slots)
    torch.cuda.synchronize()
    logs = [_log(b) for b in bufs]
    z = [ag.running_state.stats.clone() for ag in ags]
    out = group.run(lambda r: ags[r].update_params(bufs[r]))
    if offs is not None:
        for r, ag in enumerate(offs):
            ag.running_state.stats.copy_(z[r])
        out_off = off_group.run(lambda r: offs[r].update_params(bufs[r]))
        for r in range(W):
            on, off = _state(ags[r]), _state(offs[r])
            _close_update(on, off, first, tag=r)
            assert torch.equal(on[6], off[6]), r                       # running_state: the statistics planes are exact
            for k in ("surr_loss", "value_loss"):
                # the surrogate loss is a small mean of terms of either sign: measured 5.2e-6 apart at 1.6e-3 on an H100 80GB HBM3 (700 W)
                assert abs(out[r][k] - out_off[r][k]) <= 1e-2 * abs(out_off[r][k]) + 1e-4, (r, k, out[r][k], out_off[r][k])
            assert ags[r].opt_p.step_n == offs[r].opt_p.step_n and ags[r].opt_v.step_n == offs[r].opt_v.step_n
    return logs, out


@pytest.mark.parametrize("path", ["c", "py"])
@pytest.mark.parametrize("W", [2, 3, 4])
def test_ranks_hold_one_curriculum(W, path):
    """three iterations, then one whose log has an ended episode in every entry (the payload full): after each, every rank's rings and CDF
    are the same bits and equal one curriculum fed the concatenated logs, with a clip ending more than max_freq times in the iteration;
    parameters, Adam moments and losses agree with ranks without the flag and running_state is the same bits; the payload is W T E 3 floats
    behind the statistics, in the first collective only"""
    from uhc_b200 import nn
    from uhc_b200.agent import RolloutBuffer
    ags = [_agent(r, W, path) for r in range(W)]
    offs = [_agent(r, W, path, flag=False, cur=False) for r in range(W)]
    ref = _agent(0, 1, flag=False)
    g, g_off = _join(ags, path), _join(offs, path)
    bufs = [RolloutBuffer(T, E, ags[0].dev, ags[0].act_dim, ags[0].obs_dim) for _ in range(W)]
    gen = torch.Generator().manual_seed(11 + W)
    first = _state(ags[0])
    for r in range(W):
        assert all(torch.equal(x, y) for x, y in zip(_state(ags[r])[:6], first[:6])) and all(torch.equal(x, y) for x, y in zip(_state(offs[r])[:6], first[:6]))

    def fill(r, buf):
        buf.ep_clip.copy_(torch.randint(0, len(LENS), (T, E), generator=gen, dtype=torch.int32))
        buf.ep_pct.copy_(torch.where(torch.rand(T, E, generator=gen) < 0.4, torch.ones(T, E), torch.rand(T, E, generator=gen)))
        buf.ep_start.copy_(torch.randint(0, min(LENS), (T, E), generator=gen, dtype=torch.int32))
    for it in range(4):
        logs, _ = _iteration(ags, bufs, g, offs, g_off, fill if it == 3 else None, first)
        counts = _push(ref, logs)
        assert counts.max() > M, (it, counts)
        if it == 3:
            assert counts.sum() == W * T * E
            assert bool((ags[0]._cur_sum.view(-1, 3)[:, 0] >= 0).all())
        rr = _rings(ref)
        for r, ag in enumerate(ags):
            assert _same_rings(_rings(ag), rr), (it, r)
        assert ags[0].value.grad_tail == nn.stats_tail_floats(ags[0].obs_dim) + W * T * E * 3
        assert offs[0].value.grad_tail == nn.stats_tail_floats(offs[0].obs_dim)
        for r in range(W):
            for parts in ((ags[r], W * T * E * 3), (offs[r], 0)):
                n = parts[0].value.nflat + nn.stats_tail_floats(parts[0].obs_dim) + parts[1]
                log = g.log[r] if parts[0] is ags[r] else g_off.log[r]
                assert log[0][0] == n and all(c != n for c, _ in log[1:]), (it, r)      # only the first collective carries tail and payload
                log.clear()
    if path == "c" and W == 3:
        # eval outcomes keep their route: every rank evaluates the same clips with the same weights and running_state and pushes the same outcomes
        outs = []
        for ag in ags:
            ag.engine.set_cfg(auto_reset=0)
            res = ag.evaluate(list(range(len(LENS))), fail_safe=False)
            ag.engine.set_cfg(auto_reset=1)
            outs.append([1.0 if not d["fail_any"] else min(d["last_t"] / (LENS[c] - 1), 0.999) for c, d in enumerate(res)])
        assert all(o == outs[0] for o in outs), outs
        for ag in ags + [ref]:
            ag.curriculum_push(list(range(len(LENS))), outs[0], [0] * len(LENS))
        rr = _rings(ref)
        for r, ag in enumerate(ags):
            assert _same_rings(_rings(ag), rr), ("eval", r)
        _iteration(ags, bufs, g)                            # and training goes on from the re-seeded envs
        for ag in ags[1:]:
            assert _same_rings(_rings(ag), _rings(ags[0]))


def test_world_one_is_the_device_curriculum():
    """at world 1 the flag is the device curriculum: three rollouts give the same bits (buffers, rings, CDF), and an update stages nothing
    and leaves the rings alone (the update is compared only once: it is not bitwise reproducible, see the module docstring)"""
    from uhc_b200.agent import RolloutBuffer
    a, b = _agent(0, 1, flag=True, cur=False), _agent(0, 1, flag=False, cur=False)
    b.curriculum_enable()
    assert a.engine.cur_cfg == b.engine.cur_cfg
    for it in range(3):
        bufs = []
        for ag in (a, b):
            buf = RolloutBuffer(T, E, ag.dev, ag.act_dim, ag.obs_dim)
            ag.sample(T, buf)
            bufs.append(buf)
        for k in ("states", "actions", "rewards", "masks", "ep_clip", "ep_pct", "ep_start"):
            assert torch.equal(getattr(bufs[0], k), getattr(bufs[1], k)), (it, k)
        assert _same_rings(_rings(a), _rings(b)), it
        assert (bufs[0].ep_clip >= 0).any()
    assert a._cur_staged is None and getattr(a, "_cur_slots", None) is None
    rings = _rings(a)
    a.update_params(bufs[0])
    assert _same_rings(_rings(a), rings)
    assert a.value.grad_tail == b.value.grad_tail


@pytest.mark.parametrize("path", ["c", "py"])
def test_failed_collective_leaves_the_rings(path):
    """a collective that fails (the loopback's barrier broken: ERR_BARRIER on every rank) fails every rank's update; rings, CDF and
    parameters stay as they were, and the next iteration merges normally"""
    from uhc_b200.agent import RolloutBuffer
    W = 2
    ags = [_agent(r, W, path) for r in range(W)]
    ref = _agent(0, 1, flag=False)
    g = _join(ags, path)
    bufs = [RolloutBuffer(T, E, ags[0].dev, ags[0].act_dim, ags[0].obs_dim) for _ in range(W)]
    logs, _ = _iteration(ags, bufs, g)
    _push(ref, logs)
    before = [(_rings(ag), _state(ag)) for ag in ags]
    for r, ag in enumerate(ags):
        ag.sample(T, bufs[r])
    torch.cuda.synchronize()
    g.abort()
    with pytest.raises(AssertionError, match="failed"):
        g.run(lambda r: ags[r].update_params(bufs[r]))
    torch.cuda.synchronize()
    for ag, (rings, st) in zip(ags, before):
        assert _same_rings(_rings(ag), rings)
        for x, y in zip(_state(ag)[:6], st[:6]):
            assert torch.equal(x, y)
    assert all(ag._cur_staged is None for ag in ags)
    g._b1.reset(); g._b2.reset(); g.errors.clear()
    logs, _ = _iteration(ags, bufs, g)
    _push(ref, logs)
    rr = _rings(ref)
    for ag in ags:
        assert _same_rings(_rings(ag), rr)


def _trainer_pair(W, k=dict(D=657, A=105, hs=(64,), T=4, E=32)):
    from uhc_b200 import nn
    pol = nn.MLPNet(k["D"], k["hs"], k["A"], "gelu", device="cuda", head_name="action_mean", seed=41)
    val = nn.MLPNet(k["D"], k["hs"], 1, "gelu", device="cuda", head_name="value_head", seed=42)
    return pol, val, nn.Adam(pol.params(), 5e-5, net=pol), nn.Adam(val.params(), 3e-4, net=val)


def _batch(r, k=dict(D=657, A=105, T=4, E=32)):
    g = torch.Generator().manual_seed(500 + r)
    T_, E_, D, A = k["T"], k["E"], k["D"], k["A"]
    d = lambda x: x.contiguous().cuda()
    return dict(states=d(torch.randn(T_ * E_, D, generator=g).clamp(-5, 5)), last=d(torch.randn(E_, D, generator=g).clamp(-5, 5)),
                actions=d(0.1 * torch.randn(T_ * E_, A, generator=g)), rewards=d(torch.rand(T_, E_, generator=g)), masks=d((torch.rand(T_, E_, generator=g) > 0.1).float()),
                exps=d(torch.ones(T_ * E_)), log_std=d(torch.linspace(-2.5, -1.5, A)), T=T_, E=E_)


def _raw_update(tr, b, losses, zf, zs, comm, W, extra=None):
    """uhc_ppo_update itself (extra None) or uhc_ppo_update_ex (extra = (in, out, n)), returns the return code"""
    from uhc_b200 import nn
    cfg = nn.UhcPpoCfg(0.95, 0.95, 0.2, 40.0, 1, 2)
    sp, sv, done = C.c_int(tr.opt_p.step_n), C.c_int(tr.opt_v.step_n), C.c_int(0)
    p = nn._p
    args = [tr.h, p(b["states"]), p(b["last"]), p(b["actions"]), p(b["rewards"]), p(b["masks"]), p(b["exps"]), p(b["log_std"]), C.c_int(b["T"]), C.c_int(b["E"]),
            C.byref(cfg), C.byref(sp), C.byref(sv), C.byref(done), p(zf), p(zs), comm, C.c_int(W), p(losses)]
    st = nn._stream(b["states"])
    if extra is None:
        rc = tr.L.uhc_ppo_update(*args, st)
    else:
        rc = tr.L.uhc_ppo_update_ex(*args, p(extra[0]), p(extra[1]), C.c_long(extra[2]), st)
    if rc == 0:
        tr.opt_p.step_n, tr.opt_v.step_n = sp.value, sv.value
    return rc


def test_update_ex_equals_update_and_refuses_bad_payloads():
    """uhc_ppo_update_ex with n_extra = 0, and with a payload, agrees with uhc_ppo_update at world 1 and 2 (loopback; the statistics bit for bit)
    and makes the same collectives, the first one longer by the payload, whose sum it returns; a tail too small, a negative n_extra and missing
    buffers return -2 with a message"""
    from uhc_b200 import nn
    from uhc_b200.engine import load_library
    D = 657
    for W in (1, 2):
        runs = {}
        for mode in ("plain", "ex0", "payload"):
            g = LoopbackGroup(W)
            reps = [_trainer_pair(W) for _ in range(W)]
            n = 1000 + 3 * W
            if mode == "payload":
                for rep in reps:
                    rep[1].ensure_grad_tail(nn.stats_tail_floats(D) + n)
            trs = [nn.CPpoTrainer(*rep, 128, 32, torch.device("cuda"), all_reduce=g.fn) for rep in reps]
            zf = [torch.zeros(1 + 2 * D, device="cuda", dtype=torch.float64) for _ in range(W)]
            zs = [torch.zeros_like(z) for z in zf]
            losses = [torch.zeros(2, device="cuda") for _ in range(W)]
            ins = [torch.arange(n, device="cuda", dtype=torch.float32) * (r + 1) - 7.5 for r in range(W)]
            outs = [torch.full((n,), float("nan"), device="cuda") for _ in range(W)]

            def rank(r):
                ex = None if mode == "plain" else (ins[r], outs[r], 0 if mode == "ex0" else n)
                assert _raw_update(trs[r], _batch(r), losses[r], zf[r], zs[r], g.comm(r) if W > 1 else None, W, ex) == 0
            g.run(rank)
            torch.cuda.synchronize()
            runs[mode] = [[t.clone() for t in (p.flat, v.flat, op.mflat, op.vflat, ov.mflat, ov.vflat, zf[r])] for r, (p, v, op, ov) in enumerate(reps)]
            runs[mode + "_log"] = [list(l) for l in g.log]
            if mode == "payload":
                want = sum(ins)
                for o in outs:
                    assert torch.equal(o, want)
            for t in trs:
                t.close()
        first = [t.clone() for t in (_trainer_pair(W)[0].flat, _trainer_pair(W)[1].flat)] + [None] * 4
        for mode in ("ex0", "payload"):
            for a, b in zip(runs["plain"], runs[mode]):
                _close_update(b, a, first, tag=(W, mode))
                assert torch.equal(a[6], b[6]), (W, mode)
        if W > 1:
            nv = reps[0][1].nflat + nn.stats_tail_floats(D)
            assert runs["plain_log"] == runs["ex0_log"] and runs["plain_log"][0][0] == (nv, 4 * nv)
            assert runs["payload_log"][0][0] == (nv + n, 4 * (nv + n)) and runs["payload_log"][0][1:] == runs["plain_log"][0][1:]
    # refusals: checked before any collective, so a single rank of a world-2 job returns at once
    L = load_library()
    g = LoopbackGroup(2)
    rep = _trainer_pair(2)
    tr = nn.CPpoTrainer(*rep, 128, 32, torch.device("cuda"), all_reduce=g.fn)
    zf = torch.zeros(1 + 2 * D, device="cuda", dtype=torch.float64)
    buf = torch.zeros(64, device="cuda")
    tail = rep[1].grad_tail - nn.stats_tail_floats(D)
    for ex, msg in (((buf, buf, tail + 1), "gradient tail holds"), ((buf, buf, -1), "n_extra"), ((None, buf, 4), "n_extra"), ((buf, None, 4), "n_extra")):
        assert _raw_update(tr, _batch(0), torch.zeros(2, device="cuda"), zf, torch.zeros_like(zf), g.comm(0), 2, ex) == -2, msg
        assert msg in L.uhc_last_error().decode(), (msg, L.uhc_last_error())
    assert tr.opt_p.step_n == 0 and g.log[0] == []
    tr.close()


def test_stage_and_merge_refuse_bad_shapes():
    from uhc_b200.agent import RolloutBuffer, UhcRolloutBuf
    from uhc_b200.engine import load_library
    L = load_library()
    ag = _agent(0, 2)
    h = ag.engine.h
    buf = RolloutBuffer(T, E, ag.dev, ag.act_dim, ag.obs_dim)
    b = UhcRolloutBuf(); b.ep_clip, b.ep_pct, b.ep_start, b.T_cap = buf.ep_clip.data_ptr(), buf.ep_pct.data_ptr(), buf.ep_start.data_ptr(), T
    slots = torch.zeros(2 * T * E * 3, device="cuda")
    sp = C.c_void_p(slots.data_ptr())
    for args in ((T, 2, 2, sp), (T, -1, 2, sp), (T, 0, 0, sp), (T + 1, 0, 2, sp), (0, 0, 2, sp), (T, 0, 2, C.c_void_p(None))):
        assert L.uhc_curriculum_stage(h, C.byref(b), C.c_int(args[0]), C.c_int(args[1]), C.c_int(args[2]), args[3], None) == -2, args
        assert L.uhc_last_error().decode().startswith("uhc_curriculum_stage:")
    b2 = UhcRolloutBuf(); b2.ep_clip, b2.ep_pct, b2.T_cap = b.ep_clip, b.ep_pct, T
    assert L.uhc_curriculum_stage(h, C.byref(b2), C.c_int(T), C.c_int(0), C.c_int(2), sp, None) == -2          # no ep_start
    for args in ((T, 0, sp), (0, 2, sp), (T, 2, C.c_void_p(None))):
        assert L.uhc_curriculum_update_gathered(h, args[2], C.c_int(args[0]), C.c_int(args[1]), None) == -2, args
        assert L.uhc_last_error().decode().startswith("uhc_curriculum_update_gathered:")
    with pytest.raises(ValueError, match="world \\* T \\* E \\* 3"):
        ag.engine.curriculum_stage(buf, T, 0, 2, slots[:-3])
    with pytest.raises(ValueError, match="world \\* T \\* E \\* 3"):
        ag.engine.curriculum_update_gathered(slots[:-3], T, 2)
    ag.curriculum_enable(0)
    assert L.uhc_curriculum_stage(h, C.byref(b), C.c_int(T), C.c_int(0), C.c_int(2), sp, None) == -2        # not enabled
    assert "not enabled" in L.uhc_last_error().decode()
    # a rank that samples twice without an update would lose a log: refused before the rollout
    ag.curriculum_enable(M)
    ag.sample(T, buf)
    with pytest.raises(RuntimeError, match="update_params"):
        ag.sample(T, buf)
