"""GPU: the failure-weighted curriculum on the device (uhc_curriculum_*, include/uhc_rollout.h) against the host rules it replaces --
AgentCopycat._update_freq_dict with start frames, failure_weights + upload_clip_cdf, and the reference's precision-mode and
fit_single_key draws (tests/golden/precision_hist.npz, recorded from the unmodified reference)."""
import os
import pickle
import types

import numpy as np
import pytest
from scipy import stats

from tests.helpers import write_synthetic_pkl

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(__file__), "golden")


def _expert(name):
    z = np.load(os.path.join(G, f"expert_{name}.npz"))
    ex = {k: z[k] for k in z.files}
    return ex, np.concatenate([ex["beta"][0], [ex["gender"][0]]])


def _clip(ex, L):
    """an expert table of L frames (the clip's frames repeated): the sampler only reads the lengths"""
    idx = np.arange(L) % len(ex["qpos"])
    n = len(ex["qpos"])
    return {k: (np.asarray(v)[idx] if np.ndim(v) > 0 and len(v) == n else v) for k, v in ex.items()}


def _agent(E, lens, t_min, t_max, seed=3, **kw):
    from uhc_b200.agent import BatchedAgent
    sway, so = _expert("sway")
    return BatchedAgent(E, [_clip(sway, int(L)) for L in lens], [so] * len(lens), policy_hsize=(64,), value_hsize=(64,), seed=seed, t_min=t_min, t_max=t_max, **kw)


def _host_update(fd, buf, T, M=50):
    clip, pct, start = (getattr(buf, k)[:T].cpu().numpy().reshape(-1) for k in ("ep_clip", "ep_pct", "ep_start"))
    for c, p, s in zip(clip, pct, start):
        if c >= 0:
            fd[int(c)].append([float(p), int(s)])
    return [h[-M:] for h in fd]


def _upload_cdf(w):
    out, acc = np.zeros(len(w), np.float32), 0.0
    for i, x in enumerate(w):
        acc += float(x)
        out[i] = acc
    return out


def _ulps(a, b):
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max())


@pytest.mark.parametrize("nclips", [7, 3334])
def test_history_and_cdf_match_host_freq_dict(nclips):
    """many episode ends per rollout (short slices; with 7 clips some clip ends > 50 times in one rollout, with 3334 the weight kernel runs
    several clips per thread and the pairwise sum recurses): the rings hold the host freq_dict entry for entry, also after a batch of eval
    outcomes pushed in one call, and the CDF is upload_clip_cdf(failure_weights(history)) to 1 fp32 ulp (device exp against glibc's)"""
    import torch
    from uhc_b200.agent import RolloutBuffer, failure_weights
    lens = [30, 45, 60, 33, 90, 41, 52] if nclips == 7 else list(np.random.RandomState(4).randint(12, 30, nclips))
    ag = _agent(1024, lens, t_min=2, t_max=6)
    ag.curriculum_enable(50, 0.2, 0.5, 0.0, -1)
    fd = [[] for _ in lens]
    worst = 0

    def check(tag):
        nonlocal worst
        ln, p, s = ag.curriculum_get()
        for c in range(len(lens)):
            assert ln[c] == len(fd[c]) and [[float(p[c, j]), int(s[c, j])] for j in range(ln[c])] == fd[c], (tag, c)
        ref = _upload_cdf(failure_weights([[r[0] for r in h] for h in fd], 0.2, 0.5))
        worst = max(worst, _ulps(ag.engine.clip_cdf(), ref))

    for it in range(4):
        T = 8
        buf = RolloutBuffer(T, ag.E, ag.dev, ag.act_dim, ag.obs_dim)
        ag.sample(T, buf)
        torch.cuda.synchronize()
        fd = _host_update([list(h) for h in fd], buf, T)
        ends = buf.ep_clip[:T].cpu().numpy()
        if nclips == 7:
            assert np.bincount(ends[ends >= 0], minlength=len(lens)).max() > 50
        check(it)
    rs = np.random.RandomState(1)                     # eval outcomes: one push of many, one clip more than max_freq times
    clips = np.concatenate([rs.randint(0, nclips, 3 * nclips), np.full(70, 1)]).astype(np.int32)
    outs = np.where(rs.uniform(size=len(clips)) < 0.5, 1.0, 0.999).astype(np.float32)
    ag.curriculum_push(clips, outs, np.zeros(len(clips), np.int32))
    for c, o in zip(clips, outs):
        fd[c].append([float(o), 0])
    fd = [h[-50:] for h in fd]
    check("push")
    print("clips", nclips, "worst CDF difference (fp32 ulps):", worst)
    assert worst <= 1


def _golden_draws(freq, fit_clip, n_rounds, E=2048):
    z = np.load(os.path.join(G, "precision_hist.npz"))
    lens, t_min, t_max = z["lens"], int(z["t_min"]), int(z["t_max"])
    ag = _agent(E, lens, t_min=t_min, t_max=t_max)
    ag.curriculum_enable(50, 0.2, 0.5, freq, fit_clip)
    ag.curriculum_set(z["nent"], z["pct"], z["start"])
    clips, starts, slens = [], [], []
    for _ in range(n_rounds):
        ag.engine.curriculum_reseed()
        st = ag.engine.get_states()
        clips.append(st["clip"].copy()); starts.append(st["start"].copy()); slens.append(st["len"].copy())
    clip, start, slen = np.concatenate(clips), np.concatenate(starts), np.concatenate(slens)
    assert (slen == np.minimum(t_max, lens[clip] - start)).all()
    return z, clip, start


def _same_law(a, b):
    m = (a + b) > 0
    return stats.chi2_contingency(np.stack([a[m], b[m]])).pvalue


def test_precision_reseeds_match_reference():
    """>= 10 k in-kernel re-seeds with prec_freq = sampling_freq = 0.5 against sample_seq(precision_mode=True) of the reference"""
    z, clip, start = _golden_draws(0.5, -1, 8)
    assert len(clip) >= 10000
    p = _same_law(np.bincount(clip, minlength=len(z["lens"])), z["seq.clip_hist"])
    assert p > 1e-4, p
    for c in range(len(z["lens"])):
        p = _same_law(np.bincount(start[clip == c], minlength=z["seq.start_hist"].shape[1]), z["seq.start_hist"][c])
        assert p > 1e-4, (c, p)


@pytest.mark.parametrize("k", [0, 1])
def test_fit_clip_reseeds_follow_get_sample_from_key(k):
    z = np.load(os.path.join(G, "precision_hist.npz"))
    c = int(z["fit_keys"][k])
    z, clip, start = _golden_draws(0.75, c, 6)
    assert (clip == c).all()
    p = _same_law(np.bincount(start, minlength=len(z[f"key{c}.start_hist"])), z[f"key{c}.start_hist"])
    assert p > 1e-4, p


def _rollout_outputs(ag, T=12):
    import torch
    from uhc_b200.agent import RolloutBuffer
    ag.reset_envs()
    out = []
    for _ in range(2):
        buf = RolloutBuffer(T, ag.E, ag.dev, ag.act_dim, ag.obs_dim)
        ag.sample(T, buf)
        torch.cuda.synchronize()
        out.append({k: getattr(buf, k).clone() for k in ("states", "actions", "rewards", "masks", "ep_clip", "ep_pct", "ep_start")})
    return out


def test_curriculum_off_is_bit_identical():
    """an engine that ran rollouts with the curriculum (precision starts, a fit clip), then reloaded the same table (env records and episode
    counters reset) and disabled it, rolls out bit for bit like an engine that never enabled it -- start log included"""
    import torch
    from uhc_b200.agent import RolloutBuffer
    lens = [30, 45, 60, 33]
    sway, so = _expert("sway")
    ref_ag = _agent(256, lens, 2, 8)
    ag = _agent(256, lens, 2, 8)
    z0 = ag.running_state.stats.clone()
    ag.curriculum_enable(50, 0.2, 0.5, 0.5, 1)
    buf = RolloutBuffer(12, ag.E, ag.dev, ag.act_dim, ag.obs_dim)
    for _ in range(2):
        ag.sample(12, buf)
    torch.cuda.synchronize()
    assert (buf.ep_start >= 0).any() and (buf.ep_clip[buf.ep_clip >= 0] == 1).all()
    ag.engine.load_clips([_clip(sway, int(L)) for L in lens], [so] * len(lens))     # same clip count: the curriculum stays on
    assert ag.engine.cur_cfg is not None
    ag.curriculum_enable(0)
    ag.running_state.stats.copy_(z0)
    ag.global_step = 0
    ref, off = _rollout_outputs(ref_ag), _rollout_outputs(ag)
    for a, b in zip(ref, off):
        for k in a:
            assert torch.equal(a[k], b[k]), k
    assert (ref[0]["ep_clip"] >= 0).any()
    assert (ref[0]["ep_start"] == -1).all()         # the start log is written by the curriculum's step kernel only


def test_bad_arguments_return_minus_2():
    import ctypes as C
    from uhc_b200.agent import RolloutBuffer, UhcRolloutBuf
    ag = _agent(64, [30, 40], 2, 8)
    L, h = ag.engine.lib, ag.engine.h
    dbl = C.c_double
    for args in ((-1, 0.2, 0.5, 0.0, -1), (5000, 0.2, 0.5, 0.0, -1), (50, 0.0, 0.5, 0.0, -1), (50, float("nan"), 0.5, 0.0, -1), (50, 0.2, 1.5, 0.0, -1),
                 (50, 0.2, 0.5, -0.1, -1), (50, 0.2, 0.5, 0.0, 2), (50, 0.2, 0.5, 0.0, -2)):
        assert L.uhc_curriculum_enable(h, C.c_int(args[0]), dbl(args[1]), dbl(args[2]), dbl(args[3]), C.c_int(args[4])) == -2, args
    buf = RolloutBuffer(2, 64, ag.dev, ag.act_dim, ag.obs_dim)
    b = UhcRolloutBuf(); b.ep_clip, b.ep_pct, b.ep_start, b.T_cap = buf.ep_clip.data_ptr(), buf.ep_pct.data_ptr(), buf.ep_start.data_ptr(), 2
    z = np.zeros(2, np.int32); f = np.zeros(2, np.float32)
    ip = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    assert L.uhc_curriculum_update(h, C.byref(b), 2, None) == -2                  # not enabled
    assert L.uhc_curriculum_push(h, 1, ip(z), fp(f), ip(z)) == -2
    assert L.uhc_curriculum_get(h, ip(z), fp(f), ip(z)) == -2
    ag.curriculum_enable(2, 0.2, 0.5, 0.0, -1)
    assert L.uhc_set_clip_weights(h, 2, fp(np.ones(2, np.float32))) == -2          # the curriculum owns the CDF
    assert L.uhc_curriculum_update(h, C.byref(b), 3, None) == -2                  # T > T_cap
    assert L.uhc_curriculum_update(h, C.byref(b), 0, None) == -2
    b2 = UhcRolloutBuf(); b2.ep_clip, b2.ep_pct, b2.T_cap = b.ep_clip, b.ep_pct, 2
    assert L.uhc_curriculum_update(h, C.byref(b2), 2, None) == -2                 # no ep_start
    assert L.uhc_curriculum_push(h, 1, ip(np.array([2], np.int32)), fp(f), ip(z)) == -2
    assert L.uhc_curriculum_push(h, 1, ip(z), fp(f), ip(np.array([-1], np.int32))) == -2
    assert L.uhc_curriculum_push(h, 1, ip(z), fp(np.array([np.nan], np.float32)), ip(z)) == -2
    assert L.uhc_curriculum_set(h, ip(np.array([3, 0], np.int32)), fp(np.zeros(4, np.float32)), ip(np.zeros(4, np.int32))) == -2
    # the engine is still usable: a push lands, and a table of another clip count turns the curriculum off
    ag.engine.curriculum_push([1, 1, 1], [0.5, 1.0, 0.25], [3, 4, 5])
    ln, p, s = ag.curriculum_get()
    assert ln.tolist() == [0, 2] and p[1].tolist() == [1.0, 0.25] and s[1].tolist() == [4, 5]
    sway, so = _expert("sway")
    ag.engine.load_clips([_clip(sway, 30)] * 3, [so] * 3)
    assert ag.engine.cur_cfg is None
    assert L.uhc_curriculum_get(h, ip(np.zeros(3, np.int32)), fp(np.zeros(6, np.float32)), ip(np.zeros(6, np.int32))) == -2
    ag.obs = ag.engine.reset()
    ag.sample(2)


# ---- the drop-in AgentCopycat: eval_seq and scripts/fit_uhc.py's loop
def _cfg(tmp_path, monkeypatch, **extra):
    import yaml
    monkeypatch.chdir(tmp_path)
    from uhc.utils.config_utils.copycat_config import Config
    base = yaml.safe_load(open(os.path.join(os.path.dirname(__file__), "..", "config", "uhc_b200_default.yml")))
    base.update(policy_hsize=[128, 64], value_hsize=[128, 64], min_batch_size=1024, num_optim_epoch=2, num_envs=64, save_n_epochs=2, num_epoch=1)
    base["data_specs"]["file_path"] = write_synthetic_pkl(str(tmp_path / "sample_data" / "clips.pkl"), nclips=4)
    base["data_specs"]["t_max"] = 40
    base["data_specs"]["t_min"] = 5
    base["body_diff_thresh_test"] = 0.2
    base.update(extra)
    cfg = Config(cfg_id="cur_test", create_dirs=True, cfg_dict=base)
    cfg.update(types.SimpleNamespace(cfg="cur_test", render=False, test=False, num_threads=30, gpu_index=0, epoch=0, show_noise=False,
                                     resume=None, no_log=True, debug=False, full_eval=False))
    return cfg


@pytest.mark.parametrize("fail_safe", [False, True])
def test_eval_seq_equals_eval_policy_entry(tmp_path, monkeypatch, fail_safe):
    import torch
    import joblib
    from uhc.agents.agent_copycat import AgentCopycat
    from uhc_b200.metrics import compute_metrics
    cfg = _cfg(tmp_path, monkeypatch, eval_on_device=True, fail_safe=fail_safe, curriculum_on_device=True)
    agent = AgentCopycat(cfg, torch.float64, torch.device("cuda", 0))
    agent.eval_policy(0, dump=True)
    full = joblib.load(os.path.join(cfg.output_dir, f"0_{agent.data_loader.name}_coverage_full.pkl"))
    for key in agent.data_loader.data_keys:
        r = agent.eval_seq(key, agent.data_loader)
        ref = full[key]
        assert set(ref) <= set(r) and {"gt", "pred", "gt_jpos", "pred_jpos", "reward", "percent", "fail_safe", "succ"} <= set(r)
        for k in ref:
            np.testing.assert_array_equal(np.asarray(r[k]), np.asarray(ref[k]), err_msg=k)
        assert len(r["pred"]) == len(r["gt"]) == len(r["pred_jpos"]) == len(r["gt_jpos"]) and r["pred"].shape[1] == 76
        # the trajectory arrays are the ones the metrics were taken on: compute_metrics over them gives the device metrics (the host-built
        # expert frames are fp64 here, the engine's fp32: the same bound as the drop-in evaluation tests, relative with a 1 mm floor)
        ex = agent.data_loader.experts[agent.data_loader.data_keys.index(key)]
        tt = np.minimum(np.arange(1, len(r["gt"]) + 1), ex["len"] - 1)
        np.testing.assert_array_equal(r["gt"], np.asarray(ex["qpos"])[tt])
        if len(r["pred"]) >= 3:
            hm = compute_metrics({"pred": r["pred"], "gt": r["gt"], "pred_jpos": r["pred_jpos"], "gt_jpos": r["gt_jpos"], "percent": 1.0, "fail_safe": False})
            for k in ("root_dist", "mpjpe_g", "mpjpe", "pa_mpjpe", "vel_dist", "accel_dist"):
                assert (np.abs(hm[k] - r[k]) / np.maximum(np.abs(hm[k]), 1.0)).max() < 3e-4, k


def test_fit_uhc_loop(tmp_path, monkeypatch):
    """scripts/fit_uhc.py's statements against the drop-in: precision_mode, load_curr, eval_seq, fit_single_key + optimize_policy(save_model=False),
    save_curr, save_singles; the pickles and freq_dict.pt load back"""
    import torch
    import joblib
    from uhc.agents.agent_copycat import AgentCopycat
    cfg = _cfg(tmp_path, monkeypatch, eval_on_device=True)
    agent = AgentCopycat(cfg, torch.float64, torch.device("cuda", 0))
    agent.precision_mode = True
    assert agent.curriculum_on_device
    os.makedirs(f"{cfg.model_dir}_singles", exist_ok=True)
    agent.save_curr()
    agent.load_curr()
    keys = agent.data_loader.data_keys
    for epoch, take_key in enumerate(keys[:2]):
        res = agent.eval_seq(take_key, agent.data_loader)
        agent.fit_single_key = take_key
        agent.optimize_policy(epoch, save_model=False)
        ln, _, _ = agent.agent.curriculum_get()
        st = agent.agent.engine.get_states()
        assert (st["clip"] == keys.index(take_key)).all()                  # every re-seed landed on the fitted clip
        agent.save_curr()
        agent.save_singles(epoch, take_key)
        assert "succ" in res
    for k in keys[:2]:
        cp = pickle.load(open(f"{cfg.model_dir}_singles/{k}.p", "rb"))
        assert set(cp) == {"policy_dict", "value_dict", "running_state"}
    cp = pickle.load(open(f"{cfg.model_dir}/iter_best.p", "rb"))
    assert set(cp) == {"policy_dict", "value_dict", "running_state"}
    agent.save_checkpoint(0)
    fd = joblib.load(os.path.join(cfg.result_dir, "freq_dict.pt"))
    assert set(fd) == set(keys) and sum(len(v) for v in fd.values()) > 0
    assert all(len(r) == 2 for v in fd.values() for r in v)
    agent2 = AgentCopycat(cfg, torch.float64, torch.device("cuda", 0), checkpoint_epoch=1)
    agent2.precision_mode = True
    assert agent2.get_freq_dict() == fd
