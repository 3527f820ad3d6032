"""GPU: several checkpoints side by side in one device evaluation (uhc_eval_run_groups, BatchedAgent.evaluate_policies,
AgentCopycat.eval_checkpoints).  The criterion is exact: every group's results must be bit-identical to a separate uhc_eval_run of its
policy on its clips, and the grouped GEMM's rows bit-identical to uhc_linear_forward_tc run per group."""
import ctypes as C
import os
import pickle

import joblib
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ACTS = {"none": 0, "gelu": 1, "tanh": 2, "relu": 3, "sigmoid": 4}


# ---------------------------------------------------------------- 1. the grouped GEMM against uhc_linear_forward_tc per group
def _gemm_case(sizes, K, N, act, out, gap=0, seed=0):
    import torch
    from uhc_b200 import nn
    L = nn._lib()
    L.uhc_tc_last_error.restype = C.c_char_p
    g = torch.Generator(device="cuda").manual_seed(seed)
    G = len(sizes)
    row0 = np.concatenate([[0], np.cumsum(np.asarray(sizes) + gap)[:-1]]).astype(np.int32) + gap
    M = int(row0[-1] + sizes[-1] + gap + 5)
    Kp, ldy = (K + 63) // 64 * 64, (N + 63) // 64 * 64
    bf = torch.bfloat16
    x = torch.zeros(M, Kp, device="cuda", dtype=bf)
    x[:, :K] = (torch.randn(M, K, device="cuda", generator=g) * 2).to(bf)
    W = [torch.zeros(N, Kp, device="cuda", dtype=bf) for _ in range(G)]
    for w in W:
        w[:, :K] = (torch.randn(N, K, device="cuda", generator=g) / np.sqrt(K)).to(bf)
    b = [torch.randn(N, device="cuda", generator=g) * 0.3 for _ in range(G)]
    sentinel_bf, sentinel_f = torch.full((M, ldy), 7.0, device="cuda", dtype=bf), torch.full((M, N), 7.0, device="cuda")
    yb, yf = sentinel_bf.clone(), sentinel_f.clone()
    Wp = (C.c_void_p * G)(*[w.data_ptr() for w in W])
    bp = (C.c_void_p * G)(*[t.data_ptr() for t in b])
    ip = lambda a: np.ascontiguousarray(a, np.int32).ctypes.data_as(C.POINTER(C.c_int))
    rc = L.uhc_linear_forward_tc_grouped(C.c_int(G), ip(row0), ip(sizes), C.c_void_p(x.data_ptr()), Wp, bp,
                                         C.c_void_p(yb.data_ptr() if out == "bf16" else None), C.c_void_p(yf.data_ptr() if out == "f32" else None),
                                         C.c_int(M), C.c_int(N), C.c_int(Kp), C.c_int(ldy if out == "bf16" else 0), C.c_int(act), None)
    assert rc == 0, L.uhc_tc_last_error()
    inside = torch.zeros(M, dtype=torch.bool, device="cuda")
    for k in range(G):
        r0, n = int(row0[k]), int(sizes[k])
        inside[r0:r0 + n] = True
        rb, rf = torch.zeros(n, ldy, device="cuda", dtype=bf), torch.zeros(n, N, device="cuda")
        assert L.uhc_linear_forward_tc(C.c_void_p(x[r0:].data_ptr()), C.c_void_p(W[k].data_ptr()), C.c_void_p(b[k].data_ptr()),
                                       C.c_void_p(rb.data_ptr() if out == "bf16" else None), C.c_void_p(rf.data_ptr() if out == "f32" else None),
                                       C.c_int(n), C.c_int(N), C.c_int(Kp), C.c_int(ldy if out == "bf16" else 0), C.c_int(act), None) == 0
        if out == "bf16":
            assert torch.equal(yb[r0:r0 + n].view(torch.int16), rb.view(torch.int16)), f"group {k} ({n} rows) differs"
        else:
            assert torch.equal(yf[r0:r0 + n].view(torch.int32), rf.view(torch.int32)), f"group {k} ({n} rows) differs"
    ys, sen = (yb, sentinel_bf) if out == "bf16" else (yf, sentinel_f)
    assert torch.equal(ys[~inside], sen[~inside]), "rows outside every group were written"


@pytest.mark.parametrize("sizes", [[1], [63], [64], [127], [128], [129], [300], [300, 1], [1, 63, 64, 127, 128, 129, 300],
                                   [64] * 64, [2048, 1024, 512, 256, 128, 64, 32, 16, 8, 4, 2, 1, 1]])
def test_grouped_gemm_group_sizes(sizes):
    _gemm_case(sizes, 657, 1024, ACTS["gelu"], "bf16")
    _gemm_case(sizes, 512, 105, ACTS["none"], "f32")


@pytest.mark.parametrize("act", list(ACTS))
@pytest.mark.parametrize("out", ["bf16", "f32"])
def test_grouped_gemm_activations_and_small_widths(act, out):
    _gemm_case([5, 130, 1, 40, 200, 64, 7], 37, 50, ACTS[act], out, seed=1)
    _gemm_case([129, 3], 200, 300, ACTS[act], out, gap=9, seed=2)       # gaps between the groups stay untouched


def test_grouped_gemm_production_net():
    dims = [657, 2048, 1024, 512, 105]
    for i in range(4):
        last = i == 3
        _gemm_case([1, 63, 64, 127, 128, 129, 300, 3284], dims[i], dims[i + 1], ACTS["none" if last else "gelu"], "f32" if last else "bf16", seed=10 + i)


# ---------------------------------------------------------------- 2. uhc_eval_run_groups against one uhc_eval_run per group
def _clips(n, seed, lo=12, hi=40):
    from uhc_b200.motion_lib import synthetic_clip
    rng = np.random.default_rng(seed)
    return [synthetic_clip(int(rng.integers(lo, hi)), rng) for _ in range(n)]


def _engine(E, nclips=7, precision=32, tables="host", seed=0, **cfg):
    from uhc_b200.engine import Engine
    from uhc_b200.motion_lib import MotionSet
    eng = Engine(E, precision=precision, body_diff_thresh=cfg.pop("body_diff_thresh", 0.2), **cfg)
    clips = _clips(nclips, seed)
    if tables == "device":
        eng.load_motions(MotionSet([{"qpos": c["qpos"]} for c in clips]), [np.zeros(17)] * nclips)
    else:
        eng.load_clips(clips, [np.zeros(17)] * nclips)
    return eng


def _policy(kind, seed, hsize=(128, 64), htype="gelu", D=657, A=105):
    from uhc_b200 import nn
    if kind == "gauss":
        net = nn.MLPNet(D, hsize, A, htype, head_name="action_mean", seed=seed)
        return net, nn.mlp_struct(net)
    net = nn.MCPNet(D, hsize, A, htype, num_primitive=kind, composer_dim=(64, 32), seed=seed)
    return net, nn.mcp_struct(net)


def _zstats(seed, D=657, const_cols=()):
    import torch
    rng = np.random.default_rng(seed)
    n = 50.0 + seed
    mean = rng.normal(0, 0.3, D)
    S = rng.uniform(0.05, 2.0, D) * (n - 1)
    for c in const_cols:
        S[c] = 0.0
    return torch.as_tensor(np.concatenate([[n], mean, S]), device="cuda", dtype=torch.float64)


def _same(a, b, what=""):
    assert np.array_equal(a["nframes"], b["nframes"]), what
    assert np.array_equal(a["last_t"], b["last_t"]) and np.array_equal(a["fail_any"], b["fail_any"]), what
    assert np.array_equal(a["reward_sum"], b["reward_sum"]), what
    for i, k in enumerate(a["nframes"]):
        assert np.array_equal(a["frames"][i, :k], b["frames"][i, :k]), what
        if a["states"] is not None or b["states"] is not None:
            assert np.array_equal(a["states"][i, :k], b["states"][i, :k]), what


def _check_groups(eng, groups, fail_safe, window, record_states=True, log_std=None):
    import torch
    log_std = torch.full((eng.act_dim,), -2.3, device="cuda") if log_std is None else log_std
    got = eng.eval_run_groups(groups, 5.0, fail_safe, window, record_states)
    assert len(got) == len(groups)
    for k, ((clips, pol, zs), r) in enumerate(zip(groups, got)):
        ref = eng.eval_run(clips, pol, log_std, zs, 5.0, fail_safe, window, record_states)
        _same(r, ref, f"group {k}")
    return got


@pytest.mark.parametrize("fail_safe", [True, False])
@pytest.mark.parametrize("kind", ["gauss", 1, 3, 8])
def test_groups_equal_separate_runs(fail_safe, kind):
    E = 16
    eng = _engine(E)
    pols = [_policy(kind, s) for s in range(4)]
    zs = [_zstats(s, const_cols=(640, 641, 650) if s % 2 else ()) for s in range(4)]
    # uneven groups, one of a single env, groups sharing clips and with disjoint clips, sum n < E
    groups = [([0, 1, 2, 3, 4], pols[0][1], zs[0]), ([5], pols[1][1], zs[1]), ([0, 1, 6], pols[2][1], zs[2]), ([6, 5, 4, 3], pols[3][1], zs[3])]
    got = _check_groups(eng, groups, fail_safe, 7)
    assert any(r["fail_any"].any() for r in got), "no failure: the fail / fail_safe path was not exercised"
    # sum n = E, the same policy object in two groups
    groups = [([0, 1, 2, 3, 4, 5, 6], pols[0][1], zs[0]), ([6, 6, 6], pols[1][1], zs[1]), ([1, 2, 3, 4, 5, 0], pols[0][1], zs[2])]
    _check_groups(eng, groups, fail_safe, 7)
    eng.close()


@pytest.mark.parametrize("precision,tables", [(64, "host"), (32, "device"), (64, "device")])
def test_groups_precisions_and_tables(precision, tables):
    eng = _engine(8, precision=precision, tables=tables, nclips=5)
    pols = [_policy("gauss", s) for s in range(3)]
    groups = [([0, 1, 2], pols[0][1], _zstats(0)), ([3], pols[1][1], _zstats(1, const_cols=(3,))), ([4, 0, 2], pols[2][1], _zstats(2))]
    _check_groups(eng, groups, True, 5)
    eng.close()


@pytest.mark.parametrize("window", [1, 7, 500])
def test_groups_windows(window):
    eng = _engine(12, nclips=5)
    pols = [_policy("gauss", s) for s in range(3)]
    groups = [([0, 1], pols[0][1], _zstats(0)), ([2, 3, 4, 0], pols[1][1], _zstats(1)), ([4], pols[2][1], _zstats(2))]
    _check_groups(eng, groups, True, window, record_states=window == 7)
    eng.close()


# ---------------------------------------------------------------- 3. isolation from the other entry points and graph invalidation
def test_isolation_and_recapture():
    import torch
    from uhc_b200 import nn
    from uhc_b200.agent import BatchedAgent
    E = 12
    ag = BatchedAgent(E, _clips(6, 3, 60, 90), [np.zeros(17)] * 6, policy_hsize=(128, 64), value_hsize=(64,), seed=3, noise_rate=0.5)
    eng = ag.engine
    buf_rows = 3

    def rollout_once():
        ag.running_state.stats.copy_(z0)
        ag.global_step = 0
        ag._ro_step = None
        ag.obs = eng.reset(np.arange(E), np.arange(E) % 6, np.arange(E) % 3, None)
        from uhc_b200.agent import RolloutBuffer
        buf = RolloutBuffer(buf_rows, E, ag.dev, ag.act_dim, ag.obs_dim)
        ag.rollout(buf, buf_rows)
        torch.cuda.synchronize()
        return [getattr(buf, k).clone() for k in ("states", "actions", "rewards", "masks", "logp")]

    z0 = _zstats(7)
    ls = ag.log_std
    pol_c = nn.mlp_struct(ag.policy)
    ro1 = rollout_once()
    eng.set_cfg(auto_reset=0)
    ev1 = eng.eval_run([0, 1, 2], pol_c, ls, z0, 5.0, True, 7, True)
    pols = [_policy("gauss", s) for s in range(3)]
    groups = [([0, 1, 2, 3], pols[0][1], _zstats(0)), ([4, 5], pols[1][1], _zstats(1)), ([1], pols[2][1], _zstats(2))]
    first = _check_groups(eng, groups, True, 7)
    _same(eng.eval_run([0, 1, 2], pol_c, ls, z0, 5.0, True, 7, True), ev1, "uhc_eval_run after a grouped call")
    eng.set_cfg(auto_reset=1)
    ro2 = rollout_once()
    assert all(torch.equal(a, b) for a, b in zip(ro1, ro2)), "uhc_rollout changed after a grouped call"
    eng.set_cfg(auto_reset=0)
    # a cfg change re-captures
    eng.set_cfg(body_diff_thresh=10.0)
    after_cfg = _check_groups(eng, groups, True, 7)
    assert any(not np.array_equal(a["fail_any"], b["fail_any"]) or not np.array_equal(a["last_t"], b["last_t"]) for a, b in zip(first, after_cfg))
    eng.set_cfg(body_diff_thresh=0.2)
    # weights changed in place are read anew (the bf16 copies keep their addresses)
    net = pols[1][0]
    net.W[0].mul_(1.5)
    net._prep_bf16()
    changed = _check_groups(eng, groups, True, 7)
    assert not np.array_equal(changed[1]["frames"][0, :3], first[1]["frames"][0, :3])
    # another checkpoint set (order swapped) re-captures
    swapped = [(groups[0][0], groups[2][1], groups[2][2]), (groups[1][0], groups[0][1], groups[0][2]), (groups[2][0], groups[1][1], groups[1][2])]
    _check_groups(eng, swapped, True, 7)
    # a table swap re-captures
    eng.load_clips(_clips(6, 11), [np.zeros(17)] * 6)
    _check_groups(eng, groups, True, 7)
    eng.close()


# ---------------------------------------------------------------- 4. bad arguments
def test_bad_arguments_leave_the_engine_usable():
    import torch
    E = 8
    eng = _engine(E, nclips=4)
    p0, p1 = _policy("gauss", 0), _policy("gauss", 1)
    z0, z1 = _zstats(0), _zstats(1)
    good = [([0, 1], p0[1], z0), ([2, 3, 0], p1[1], z1)]
    ref = eng.eval_run_groups(good, 5.0, True, 4)
    wide, relu, m3, m8 = _policy("gauss", 2, hsize=(64, 64)), _policy("gauss", 2, htype="relu"), _policy(3, 4), _policy(8, 5)
    narrow = _policy("gauss", 2, D=600)
    bad_kp = _policy("gauss", 6)[1]
    bad_kp.kp[1] = 192
    bads = [[], [([0], p0[1], z0)] * 65, [([0, 1], p0[1], z0), ([], p1[1], z1)], [([0, 1, 2, 3, 0], p0[1], z0), ([0, 1, 2, 3], p1[1], z1)],
            [([0, 4], p0[1], z0)], [([-1], p0[1], z0)], [([0], p0[1], z0), ([1], wide[1], z1)], [([0], p0[1], z0), ([1], relu[1], z1)],
            [([0], p0[1], z0), ([1], bad_kp, z1)], [([0], m3[1], z0), ([1], m8[1], z1)], [([0], narrow[1], z0)]]
    for groups in bads:
        with pytest.raises(ValueError):
            eng.eval_run_groups(groups, 5.0, True, 4)
        for a, b in zip(eng.eval_run_groups(good, 5.0, True, 4), ref):
            _same(a, b, "after a refused call")
    with pytest.raises(ValueError):
        eng.eval_run_groups(good, 5.0, True, 0)
    # null policy array and null statistics pointer, through the C ABI directly
    L = eng.lib
    fr = torch.empty(5, 40, 6, dtype=torch.float64, pin_memory=True)
    from uhc_b200.engine import UhcEvalClip
    from uhc_b200.nn import UhcMlp
    rec = (UhcEvalClip * 5)()
    sizes, clips = (C.c_int * 2)(2, 3), (C.c_int * 5)(0, 1, 2, 3, 0)
    pols = (UhcMlp * 2)(p0[1], p1[1])
    for pol, zs in ((None, (C.c_void_p * 2)(z0.data_ptr(), z1.data_ptr())), (pols, (C.c_void_p * 2)(z0.data_ptr(), None)), (pols, None)):
        assert L.uhc_eval_run_groups(eng.h, C.c_int(2), sizes, clips, pol, zs, C.c_float(5.0), C.c_int(1), C.c_int(4), C.c_void_p(fr.data_ptr()), rec,
                                     None, eng._stream()) == -2
        for a, b in zip(eng.eval_run_groups(good, 5.0, True, 4), ref):
            _same(a, b, "after a refused call")
    eng.close()


# ---------------------------------------------------------------- 5. BatchedAgent.evaluate_policies and AgentCopycat.eval_checkpoints
def _state(agent):
    import torch
    return [agent.policy.flat.clone(), agent.log_std.clone(), agent.running_state.stats.clone()], torch


@pytest.mark.parametrize("actor", ["gauss", "mcp"])
def test_evaluate_policies_equals_per_checkpoint_evaluate(actor):
    from uhc_b200.agent import BatchedAgent
    E = 8
    kw = dict(policy_hsize=(128, 64), value_hsize=(64,), auto_reset=False, body_diff_thresh=0.2)
    if actor == "mcp":
        kw.update(actor_type="mcp", num_primitive=3, composer_dim=(64, 32), auto_reset=True)
    ag = BatchedAgent(E, _clips(7, 5), [np.zeros(17)] * 7, seed=5, **kw)
    ag.engine.set_cfg(auto_reset=0)
    cps = []
    for s in range(3):                     # K * n = 21 > E: several calls, groups split across calls
        ag.policy.flat.mul_(1.0 + 0.1 * s)
        ag.policy.invalidate_bf16()
        ag.running_state.load_sums(40 + s, np.random.default_rng(s).normal(0, 0.2, ag.obs_dim), np.full(ag.obs_dim, 30.0 + s))
        cps.append(ag.state_dicts())
    ag.log_std.fill_(-1.7)
    before, torch = _state(ag)
    clips = np.array([0, 1, 2, 3, 4, 5, 6], np.int32)
    got = ag.evaluate_policies(cps, clips, True, window=7, record_states=True)
    after, _ = _state(ag)
    assert all(torch.equal(a, b) for a, b in zip(before, after)), "evaluate_policies touched the agent's weights / log_std / running_state"
    for k, cp in enumerate(cps):
        ag.load_state_dicts(cp)
        want = ag.evaluate(clips, True, window=7, record_states=True)
        assert len(got[k]) == len(want)
        for a, b in zip(got[k], want):
            assert a.keys() == b.keys() and a["last_t"] == b["last_t"] and a["fail_any"] == b["fail_any"] and a["reward_sum"] == b["reward_sum"]
            assert np.array_equal(a["frames"], b["frames"]) and np.array_equal(a["states"], b["states"])
    ag.engine.close()


@pytest.mark.parametrize("device_curriculum", [False, True])
def test_eval_checkpoints_equals_load_checkpoint_and_eval_policy(tmp_path, monkeypatch, device_curriculum):
    import torch
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, num_envs=8, nclips=6, test_clips=4)
    if device_curriculum:
        agent.curriculum_on_device = True
        agent._enable_device_curriculum()
    ag = agent.agent
    agent.sample(256)                       # some training outcomes in the curriculum
    epochs = []
    for s in range(3):
        ag.policy.flat.mul_(1.0 + 0.05 * s)
        ag.policy.invalidate_bf16()
        ag.running_state.stats[0] += 10.0
        agent.save_checkpoint(2 * s)
        epochs.append(2 * s + 1)
    cfg.cfg_dict["eval_on_device"] = True
    before = [ag.policy.flat.clone(), ag.log_std.clone(), ag.running_state.stats.clone()]
    freq0 = pickle.dumps(agent.get_freq_dict())
    lens0, cdf0 = ag.engine.clip_len.copy(), ag.engine.clip_cdf()
    got = agent.eval_checkpoints(epochs, dump=True)
    dumps = {(e, ld.name): joblib.load(os.path.join(cfg.output_dir, f"{e}_{ld.name}_coverage_full.pkl")) for e in epochs for ld in agent.test_data_loaders}
    assert all(torch.equal(a, b) for a, b in zip(before, [ag.policy.flat, ag.log_std, ag.running_state.stats]))
    assert pickle.dumps(agent.get_freq_dict()) == freq0, "eval_checkpoints fed outcomes to the curriculum"
    assert np.array_equal(ag.engine.clip_len, lens0) and np.array_equal(ag.engine.clip_cdf(), cdf0), "the training table / sampler was not restored"
    assert (ag.engine.cur_cfg is not None) == device_curriculum
    for e in epochs:
        agent.load_checkpoint(e)
        want = agent.eval_policy(e, dump=True)
        assert got[e] == want, e
        for ld in agent.test_data_loaders:
            h, g = joblib.load(os.path.join(cfg.output_dir, f"{e}_{ld.name}_coverage_full.pkl")), dumps[(e, ld.name)]
            assert list(h) == list(g)
            for key in h:
                assert set(h[key]) == set(g[key])
                for m in h[key]:
                    assert np.array_equal(np.asarray(h[key][m]), np.asarray(g[key][m])), (key, m)
    ag.engine.close()
