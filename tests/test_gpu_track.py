"""GPU: the batched physics tracker (include/uhc_track.h, uhc_b200/tracker.py).

- rows streamed frame by frame, through rebases and masked pushes, are the rows uhc_load_motions builds for the same clips, bit for bit;
- the observation pass from the stored state is k_env_step's own observation of that state, bit for bit;
- a clip replayed through the tracker (reset(f0, f1), step(), step(f2), ...) is uhc_eval_run over the same clip: the recorded qpos / xpos,
  the fail flags and the rewards, bit for bit, up to the first failure (after a fail_safe re-seat the tracker observes the re-seated state,
  as HumanoidKinEnv.get_cc_obs does, while the evaluation feeds the policy the observation of the failed state, as eval_policy does);
- an env without row cur_t + 1 is flagged and counted, never stepped; graphs are not replayed across table / cfg changes;
- arguments the stream cannot serve are rejected and leave the engine usable;
- a closed loop of 4096 envs whose targets depend on the simulated state runs 300 steps without a host synchronise inside the call."""
import ctypes as C
import time

import numpy as np
import pytest

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Gimbal lock")]

TRACK_KW = dict(trail_steps=1, body_diff_thresh=0.2)


def _torch():
    import torch
    return torch


def _policy(kind="gauss", seed=1, obs_dim=657, act_dim=105):
    from uhc_b200 import nn
    if kind == "mcp":
        net = nn.MCPNet(obs_dim, (64, 32), act_dim, "gelu", num_primitive=3, composer_dim=(32,), seed=seed)
        return net, nn.mcp_struct(net)
    net = nn.MLPNet(obs_dim, (64, 32), act_dim, "gelu", head_name="action_mean", seed=seed)
    return net, nn.mlp_struct(net)


def _zfilter(D, seed=0):
    from uhc_b200 import nn
    rng = np.random.default_rng(seed)
    z = nn.ZFilter(D)
    z.load(100, rng.normal(0, 0.1, D), 1.0 + rng.uniform(0, 0.5, D))
    return z


class Run:
    """policy + ZFilter + output buffers of one engine's tracker"""

    def __init__(self, eng, kind="gauss", fail_safe=True, seed=1):
        t = _torch()
        self.eng, self.fail_safe = eng, fail_safe
        self.net, self.pol = _policy(kind, seed, eng.obs_dim, eng.act_dim)
        self.zf = _zfilter(eng.obs_dim, seed)
        self.log_std = t.full((eng.act_dim,), -2.3, device="cuda")
        self.state = t.zeros(eng.E, 223, device="cuda", dtype=t.float32 if eng.precision == 32 else t.float64)
        self.rew = t.zeros(eng.E, device="cuda")
        self.fail = t.zeros(eng.E, device="cuda", dtype=t.int32)

    def step(self, nxt=None, mask=None):
        self.eng.track_step(nxt, mask, self.pol, self.log_std, self.zf.stats, self.zf.clip, self.fail_safe, self.state, self.rew, self.fail)
        return self.state, self.rew, self.fail


def _clips(rng, lens, kind):
    from uhc_b200 import motion_lib as ML
    if kind == "qpos":
        return [{"qpos": ML.synthetic_clip(T, rng)["qpos"]} for T in lens]
    return [{"pose_aa": rng.normal(0, 0.25, (T, 72)), "trans": np.cumsum(rng.normal(0, 0.01, (T, 3)), 0) + [0, 0, 0.92]} for T in lens]


def _rows(eng, c, first, n):
    """rows first .. first + n - 1 of clip c as the engine holds them (uhc_get_clip_frames), all 576 columns"""
    out = np.zeros((n, 576))
    assert eng.lib.uhc_get_clip_frames(eng.h, c, first, n, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
    return out


def _raw(ms, c):
    a = int(np.concatenate([[0], np.cumsum(ms.lens)])[c])
    return ms.rows[a:a + ms.lens[c]]


# ---- 1. rows
@pytest.mark.parametrize("precision", [32, 64])
@pytest.mark.parametrize("kind", ["qpos", "smpl"])
def test_streamed_rows_equal_loaded_rows(precision, kind):
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    from uhc_b200.model import HumanoidModel
    rng = np.random.default_rng(3)
    E, H = 5, 4
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    fk = np.array([0, 1, 1, 0, 1], np.int32)
    ms = ML.MotionSet(_clips(rng, [23, 17, 30, 12, 26], kind))
    eng = Engine(E, model=variants[0], precision=precision, variants=variants, **TRACK_KW)
    eng.load_motions(ms, fk_models=fk)
    want = [_rows(eng, c, 0, int(ms.lens[c])) for c in range(E)]
    run = Run(eng)
    eng.track_begin(H, kind, ms.pose_dim, fk_models=fk)
    raw = [_raw(ms, c) for c in range(E)]
    eng.track_reset(np.arange(E), t.tensor(np.stack([r[:2] for r in raw]), device="cuda"))
    run.step()
    pushed = np.ones(E, int)                  # last frame index pushed per env
    mrng = np.random.default_rng(5)
    for it in range(60):
        mask = (mrng.uniform(size=E) < 0.7).astype(np.int32)
        mask[pushed + 1 >= ms.lens] = 0
        nxt = np.stack([raw[c][min(pushed[c] + 1, ms.lens[c] - 1)] for c in range(E)])
        run.step(t.tensor(nxt, device="cuda"), t.tensor(mask, device="cuda"))
        pushed += mask
        st = eng.track_state()
        assert (st["dropped"] == 0).all()
        for c in range(E):
            n = int(st["rows"][c])
            got = _rows(eng, c, 0, n)
            assert np.array_equal(got, want[c][pushed[c] + 1 - n:pushed[c] + 1]), (c, it)
            assert st["cur_t"][c] == n - 1 and st["steps"][c] == pushed[c]
    assert (pushed + 1 > H).sum() >= 3 and len(set(pushed.tolist())) > 2      # rebased windows, streams at different phases
    eng.close()


# ---- 2. observation pass
@pytest.mark.parametrize("precision,obs_v", [(64, 2), (32, 2), (64, 6), (32, 6), (64, 1)])
def test_observation_pass_equals_step_observation(precision, obs_v):
    t = _torch()
    from tests import step_corpus as S
    from uhc_b200.engine import Engine
    s = S.setup("base")
    cases = S.corpus("base")[0]
    E = len(cases)
    qpos = s.clips[0]["qpos"]
    eng = Engine(E, model=s.models[0], precision=precision, obs_v=obs_v, **TRACK_KW)
    eng.track_begin(8, "qpos")
    st = np.array([c["start"] for c in cases])
    fr = lambda k: qpos[np.minimum(st + k, len(qpos) - 1)]
    f01 = np.stack([fr(0), fr(1)], 1)
    q = t.tensor(np.stack([c["qpos"] for c in cases]), dtype=t.float32, device="cuda")
    v = t.tensor(np.stack([c["qvel"] for c in cases]), dtype=t.float32, device="cuda")
    eng.track_reset(np.arange(E), t.tensor(f01, device="cuda"), q, v)
    obs0 = eng.reset(np.arange(E), clip=np.arange(E), start=0, length=8, qpos=q.cpu().numpy(), qvel=v.cpu().numpy()).clone()   # the same reset, with its obs
    assert t.equal(eng.track_obs(), obs0)
    eng.track_push(t.tensor(fr(2), device="cuda"))
    act = t.tensor(np.stack([c["action"] for c in cases]), dtype=t.float32, device="cuda")
    obs1 = eng.step(act)[0].clone()
    got = eng.track_obs()
    d = (got - obs1).abs().max().item()
    print(f"fp{precision} obs v{obs_v}: max |tracker obs - step obs| = {d:.3e} over {E} corpus states")
    assert t.equal(got, obs1)
    assert set(c["regime"] for c in cases) == set(S.REGIMES)
    eng.close()


# ---- 3. replay equals evaluation
@pytest.mark.parametrize("precision,kind,fail_safe,H", [(64, "gauss", True, 4), (64, "gauss", False, 64), (64, "mcp", True, 5), (32, "gauss", True, 3),
                                                        (32, "mcp", False, 6)])
def test_replay_equals_evaluation(precision, kind, fail_safe, H):
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(8)
    E, n = 6, 4
    ms = ML.MotionSet(_clips(rng, [31, 24, 40, 18], "qpos"))
    eng = Engine(E, precision=precision, **TRACK_KW)
    eng.load_motions(ms)
    run = Run(eng, kind, fail_safe)
    ev = eng.eval_run(np.arange(n), run.pol, run.log_std, run.zf.stats, run.zf.clip, fail_safe, window=7, record_states=True)
    eng.track_begin(H, "qpos")
    raw = [_raw(ms, c) for c in range(n)]
    eng.track_reset(np.arange(n), t.tensor(np.stack([r[:2] for r in raw]), device="cuda"))
    T = int(ms.lens.max())
    qs, xs, rs, fs, reseated = [], [], [], [], []
    for s in range(T - 1):
        nxt = None
        if s > 0:
            nxt = np.zeros((E, 76))
            for c in range(n):
                nxt[c] = raw[c][min(s + 1, ms.lens[c] - 1)]
            nxt = t.tensor(nxt, device="cuda")
        state, rew, fail = run.step(nxt)
        st = state.double().cpu().numpy()
        qs.append(st[:n, :76]); xs.append(st[:n, 151:]); rs.append(rew.cpu().numpy()[:n].copy()); fs.append(fail.cpu().numpy()[:n].copy())
        if fail_safe and fs[-1].any():
            reseated.append((s, eng.get_states(np.arange(n))["qpos"].copy()))
    qs, xs, rs, fs = map(np.stack, (qs, xs, rs, fs))
    compared = failed = same_steps = 0
    for c in range(n):
        L = int(ms.lens[c]) - 1                                        # steps whose target row exists in the clip
        f_idx = np.flatnonzero(fs[:L, c])
        k = min(L, f_idx[0] + 1 if len(f_idx) else L, int(ev["nframes"][c]))
        assert np.array_equal(qs[:k, c], ev["states"][c, :k, :76]) and np.array_equal(xs[:k, c], ev["states"][c, :k, 76:]), c
        if ev["nframes"][c] == k:                 # the evaluation recorded exactly these steps (it stopped at a failure, or at the longest clip's end)
            acc = 0.0
            for r in rs[:k, c]:
                acc += float(r)
            assert acc == ev["reward_sum"][c] and bool(ev["fail_any"][c]) == bool(fs[:k, c].any()), c
            same_steps += 1
        if len(f_idx) and f_idx[0] < k:
            assert ev["fail_any"][c], c
        compared += k
        failed += bool(len(f_idx))
    assert compared >= n * 10 and failed >= 1 and (same_steps >= 1 or fail_safe)
    for s, q in reseated:                          # a re-seat puts the env on row cur_t (its target of that step) rounded to fp32
        for c in np.flatnonzero(fs[s]):
            if s + 1 < ms.lens[c]:
                assert np.array_equal(q[c], raw[c][s + 1].astype(np.float32).astype(np.float64)), (s, c)
    eng.close()


# ---- 4. missing or stale rows, graph invalidation
def test_missing_rows_are_flagged_never_stepped():
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(2)
    E, H = 4, 4
    ms = ML.MotionSet(_clips(rng, [40] * E, "qpos"))
    raw = [_raw(ms, c) for c in range(E)]
    eng = Engine(E, **TRACK_KW)
    run = Run(eng, fail_safe=False)
    eng.track_begin(H, "qpos")
    f01 = t.tensor(np.stack([r[:2] for r in raw]), device="cuda")
    eng.track_reset(np.arange(E), f01)
    frames = lambda k: t.tensor(np.stack([r[k] for r in raw]), device="cuda")
    run.step()
    skipped0 = eng.counters["invalid_env_steps"]
    q0 = eng.get_states()["qpos"].copy()
    _, rew, fail = run.step(frames(2), t.tensor([1, 0, 1, 1], dtype=t.int32, device="cuda"))     # env 1 gets no frame
    q1 = eng.get_states()["qpos"].copy()
    assert fail[1].item() == 1 and rew[1].item() == 0.0 and np.array_equal(q1[1], q0[1]) and not np.array_equal(q1[0], q0[0])
    assert eng.counters["invalid_env_steps"] == skipped0 + 1
    assert list(eng.track_state()["steps"]) == [2, 1, 2, 2]
    _, _, fail = run.step()                                                                     # no frame: every env is one row short
    assert (fail.cpu().numpy() == 1).all() and eng.counters["invalid_env_steps"] == skipped0 + 1 + E
    assert np.array_equal(eng.get_states()["qpos"], q1)
    for k in range(3, 30):                                                                      # rebases: old rows remain behind the window
        run.step(frames(k), t.tensor([0, 1, 1, 1], dtype=t.int32, device="cuda"))
    eng.track_reset([2], f01[2:3].contiguous())                                                # env 2 starts over: rows 2.. are stale
    run.step()
    q2 = eng.get_states()["qpos"].copy()
    _, _, fail = run.step()
    assert fail[2].item() == 1 and np.array_equal(eng.get_states()["qpos"][2], q2[2])
    assert eng.track_state()["steps"][2] == 1
    eng.close()


def test_graphs_follow_cfg_and_table_changes():
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(4)
    E = 8
    ms = ML.MotionSet(_clips(rng, [12] * E, "qpos"))
    raw = [_raw(ms, c) for c in range(E)]
    eng = Engine(E, **dict(TRACK_KW, body_diff_thresh=10.0))
    run = Run(eng)

    def episode():
        eng.track_reset(np.arange(E), t.tensor(np.stack([r[:2] for r in raw]), device="cuda"))
        fails = [run.step()[2].cpu().numpy().copy()]
        for k in range(2, 12):
            fails.append(run.step(t.tensor(np.stack([r[k] for r in raw]), device="cuda"))[2].cpu().numpy().copy())
        return np.array(fails)
    eng.track_begin(6, "qpos")
    assert episode().sum() == 0
    eng.set_cfg(**dict(TRACK_KW, body_diff_thresh=1e-6))      # every step fails under this threshold: a stale graph would not see it
    assert (episode() == 1).all()
    eng.load_clips([{k: v for k, v in ML.qpos_fk(raw[0]).items()}])
    with pytest.raises(ValueError, match="tracking ended"):
        run.step()
    eng.set_cfg(**dict(TRACK_KW, body_diff_thresh=10.0))
    eng.track_begin(6, "qpos")
    assert episode().sum() == 0
    eng.close()


# ---- 5. bad arguments
def test_bad_arguments_leave_the_engine_usable():
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(6)
    E = 4
    ms = ML.MotionSet(_clips(rng, [20] * E, "qpos"))
    for bad in (dict(obs_v=3), dict(term_body="root"), dict(term_body="Head"), dict(auto_reset=1), dict(reactive_v=1), dict(trail_steps=0),
                dict(env_episode_len=3)):
        eng = Engine(E, **dict(TRACK_KW, **bad))
        eng.load_motions(ms)
        before = eng.clip_frames(1)["qpos"]
        with pytest.raises(ValueError):
            eng.track_begin(4, "qpos")
        assert np.array_equal(eng.clip_frames(1)["qpos"], before) and eng.clip_len.tolist() == [20] * E, bad
        eng.close()
    eng = Engine(E, **TRACK_KW)
    eng.load_motions(ms)
    for args in ((2, "qpos"), (4, "smpl", 75), (4, "qpos", 72)):
        with pytest.raises(ValueError):
            eng.track_begin(*args)
    with pytest.raises(ValueError):
        eng.track_begin(4, "qpos", fk_models=[0, 0, 1, 0])           # one shape variant only
    run = Run(eng)
    with pytest.raises(ValueError, match="not tracking"):
        run.step()
    eng.track_begin(4, "qpos")
    raw = [_raw(ms, c) for c in range(E)]
    f01 = t.tensor(np.stack([r[:2] for r in raw]), device="cuda")
    L, h = eng.lib, eng.h
    chk = lambda rc: rc == -2
    ids = (C.c_int * 5)(0, 1, 2, 3, 4)
    assert chk(L.uhc_track_reset(h, 0, ids, C.c_void_p(f01.data_ptr()), None, None, None))
    assert chk(L.uhc_track_reset(h, E + 1, ids, C.c_void_p(f01.data_ptr()), None, None, None))
    assert chk(L.uhc_track_reset(h, 2, (C.c_int * 2)(0, E), C.c_void_p(f01.data_ptr()), None, None, None))
    assert chk(L.uhc_track_reset(h, 2, ids, None, None, None, None))
    p = lambda x: C.c_void_p(x.data_ptr())
    for nul in range(6):
        a = [p(run.log_std), p(run.zf.stats), p(run.state), p(run.rew), p(run.fail)]
        pol = C.byref(run.pol)
        if nul == 5:
            pol = None
        else:
            a[nul] = None
        assert chk(L.uhc_track_step(h, None, None, pol, a[0], a[1], C.c_float(5.0), 1, a[2], a[3], a[4], None)), nul
    _, bad_pol = _policy("gauss", 1, 600, 105)
    assert chk(L.uhc_track_step(h, None, None, C.byref(bad_pol), p(run.log_std), p(run.zf.stats), C.c_float(5.0), 1, p(run.state), p(run.rew), p(run.fail), None))
    assert chk(L.uhc_track_push(h, None, None, None)) and chk(L.uhc_track_obs(h, None, None))
    eng.track_reset(np.arange(E), f01)                                  # still usable
    run.step()
    _, _, fail = run.step(t.tensor(np.stack([r[2] for r in raw]), device="cuda"))
    assert list(eng.track_state()["steps"]) == [2] * E
    eng.close()


# ---- 6. closed loop
def test_closed_loop_4096_envs_no_host_sync():
    t = _torch()
    from uhc_b200 import motion_lib as ML
    from uhc_b200.agent import BatchedAgent
    rng = np.random.default_rng(9)
    E, T = 4096, 300
    clips = [ML.synthetic_clip(T + 2, rng) for _ in range(8)]
    agent = BatchedAgent(E, clips, policy_hsize=(64, 32), value_hsize=(64, 32), auto_reset=False, **TRACK_KW)
    trk = agent.tracker(window=8, kind="qpos", fail_safe=True)
    ref = t.tensor(np.stack([clips[e % 8]["qpos"] for e in range(E)]), device="cuda")          # [E][T + 2][76]
    trk.reset(ref[:, 0], ref[:, 1])
    state, _, _ = trk.step()
    t.cuda.synchronize()
    slow = []
    for k in range(1, T):
        # the kinematic rule: expert frame k + 1, shifted by the root's current drift from expert frame k
        nxt = ref[:, k + 1].clone()
        nxt[:, :2] += state[:, :2].double() - ref[:, k, :2]
        if k == T // 2:
            t.cuda._sleep(200_000_000)                     # the device is busy for a while: a synchronising call would wait for it
            t0 = time.perf_counter()
            state, _, fail = trk.step(nxt)
            dt = time.perf_counter() - t0
            t.cuda.synchronize()
            t1 = time.perf_counter() - t0
            slow.append((dt, t1))
        else:
            state, _, fail = trk.step(nxt)
    t.cuda.synchronize()
    steps = trk.steps()
    assert (steps == T).all(), np.unique(steps)
    dt, t1 = slow[0]
    print(f"track_step returned after {dt * 1e3:.2f} ms while the device was busy for {t1 * 1e3:.1f} ms")
    assert dt < 0.25 * t1
    assert t.isfinite(state).all()
    agent.engine.close()
