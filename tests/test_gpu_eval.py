"""GPU: the device evaluation (uhc_eval_run, BatchedAgent.evaluate, eval_on_device: true) against the host loop of
AgentCopycat.eval_policy, which stays the default and is the reference here.

Both paths run on the same agent, weights and clips.  The simulated trajectories must be bit-identical (the host loop's recorded qpos /
xpos, captured where it hands them to compute_metrics, against the device path's optional state record), and so must last_t, fail_any,
percent, succ and the reward sums.  The per-frame metrics must agree with compute_metrics on the same states and the same expert frames
to METRIC_RTOL."""
import functools
import os
import types

import joblib
import numpy as np
import pytest

from tests.helpers import write_synthetic_pkl

pytestmark = pytest.mark.gpu

# device metrics against compute_metrics on identical inputs: worst 1.23e-14 relative over every test below, measured on an
# H100 80GB HBM3 at 700 W and at 400 W power limits (printed by each test)
METRIC_RTOL = 1e-9
# the host loop reads the expert frames of host-built tables in fp64, the fp32 engine (and so the device path) holds them rounded to
# fp32: the drop-in metrics then differ by that rounding, most on accel_dist, whose second differences amplify it (half an fp32 ulp of a
# coordinate below 4 m is 2.4e-7 m, so at most ~1e-3 mm).  Worst measured, relative with a 1 mm floor, same card and power limit:
# 8.4e-6 in these tests, 8.0e-5 over scripts/eval_time.py's 4096 clips of 150-300 frames (400 W).  The bound is 3x the larger
DROPIN_RTOL = 3e-4
KEYS = ("root_dist", "mpjpe_g", "mpjpe", "pa_mpjpe", "vel_dist", "accel_dist")
_WORST = {"metric": 0.0}


def _pkl_with_short_clips(path, nclips, seed, short):
    write_synthetic_pkl(path, nclips=nclips, seed=seed)
    if short:
        d = joblib.load(path)
        for key, T in zip(sorted(d)[:len(short)], short):
            for f in ("pose_aa", "pose_6d", "trans"):
                d[key][f] = d[key][f][:T]
        joblib.dump(d, path)
    return path


def _cfg(tmp_path, cfg_file, tables, num_envs, nclips, test_clips, short, fail_safe):
    import yaml
    from uhc.utils.config_utils.copycat_config import Config
    base = yaml.safe_load(open(os.path.join(os.path.dirname(__file__), "..", "config", cfg_file)))
    base.update(policy_hsize=[128, 64], value_hsize=[128, 64], min_batch_size=1024, num_optim_epoch=2, num_envs=num_envs, save_n_epochs=2, num_epoch=1)
    base["data_specs"]["file_path"] = _pkl_with_short_clips(str(tmp_path / "sample_data" / "clips.pkl"), nclips, 0, short)
    if test_clips:
        base["data_specs"]["test_file_path"] = _pkl_with_short_clips(str(tmp_path / "sample_data" / "test_clips.pkl"), test_clips, 1, ())
    base["data_specs"]["t_max"] = 40
    base["data_specs"]["t_min"] = 1
    base["data_specs"]["expert_tables"] = tables
    base["fail_safe"] = fail_safe
    base["body_diff_thresh_test"] = 0.2        # an untrained policy drifts past this within a few dozen frames: failures are exercised
    cid = f"eval_{tables}_{num_envs}"
    cfg = Config(cfg_id=cid, create_dirs=True, cfg_dict=base)
    cfg.update(types.SimpleNamespace(cfg=cid, render=False, test=False, num_threads=30, gpu_index=0, epoch=0, show_noise=False,
                                     resume=None, no_log=True, debug=False, full_eval=False))
    return cfg


def _agent(tmp_path, monkeypatch, cfg_file="uhc_b200_default.yml", tables="host", num_envs=8, nclips=10, test_clips=4, short=(), fail_safe=True,
           precision=32):
    import torch
    import uhc.agents.agent_copycat as ac
    from uhc_b200.agent import BatchedAgent
    monkeypatch.chdir(tmp_path)
    if precision != 32:
        monkeypatch.setattr(ac, "BatchedAgent", functools.partial(BatchedAgent, precision=precision))
    cfg = _cfg(tmp_path, cfg_file, tables, num_envs, nclips, test_clips, short, fail_safe)
    np.random.seed(cfg.seed); torch.manual_seed(cfg.seed)
    return ac.AgentCopycat(cfg, torch.float64, torch.device("cuda", 0), training=True, checkpoint_epoch=0), cfg


def _compare(tmp_path, monkeypatch, window=7, record_states=True, **kw):
    agent, cfg = _agent(tmp_path, monkeypatch, **kw)
    out = _pair(monkeypatch, agent, cfg, window, record_states, kw.get("tables", "host"), kw.get("precision", 32))
    agent.agent.engine.close()
    return out


def _pair(monkeypatch, agent, cfg, window, record_states, tables, precision, epoch=0):
    """eval_policy with the host loop, then with eval_on_device, on the same agent; compares everything both record.  Without
    record_states the device path runs its production graph (no state record): its metrics are then compared with compute_metrics on
    the host loop's trajectories, which agree to METRIC_RTOL only if the trajectories are the same"""
    from uhc_b200 import metrics
    loaders = agent.test_data_loaders
    cfg.cfg_dict["eval_on_device"] = False

    host_in = []                                  # what the host loop hands to compute_metrics, per clip with >= 3 frames, in clip order
    real = metrics.compute_metrics
    monkeypatch.setattr(metrics, "compute_metrics", lambda r: (host_in.append(r), real(r))[1])
    freq0 = {k: list(v) for k, v in agent.freq_dict.items()}
    host = agent.eval_policy(epoch=epoch, dump=True)
    host_pkl = {ld.name: joblib.load(os.path.join(cfg.output_dir, f"{epoch}_{ld.name}_coverage_full.pkl")) for ld in loaders}
    monkeypatch.setattr(metrics, "compute_metrics", real)

    dev_out = []
    evaluate = agent.agent.evaluate

    def recording(clips, fail_safe, **kw):
        out = evaluate(clips, fail_safe, window=window, record_states=record_states)
        dev_out.extend(out)
        return out
    monkeypatch.setattr(agent.agent, "evaluate", recording)
    agent.freq_dict = freq0
    cfg.cfg_dict["eval_on_device"] = True
    dev = agent.eval_policy(epoch=epoch + 1, dump=True)
    dev_pkl = {ld.name: joblib.load(os.path.join(cfg.output_dir, f"{epoch + 1}_{ld.name}_coverage_full.pkl")) for ld in loaders}
    monkeypatch.setattr(agent.agent, "evaluate", evaluate)

    # every clip of every loader, in evaluation order
    assert len(dev_out) == sum(ld.get_len() for ld in loaders)
    long_clips = [d for d in dev_out if len(d["frames"]) >= 3]
    assert len(long_clips) == len(host_in)
    worst = 0.0
    for d, r in zip(long_clips, host_in):
        if record_states:
            st = d["states"]
            assert np.array_equal(st[:, :76], r["pred"]) and np.array_equal(st[:, 76:], r["pred_jpos"]), "trajectories differ"
        gt, gtj = r["gt"], r["gt_jpos"]
        if precision == 32 and tables == "host":          # the device reads the engine's fp32 table
            gt, gtj = gt.astype(np.float32).astype(np.float64), gtj.astype(np.float32).astype(np.float64)
        want = real(dict(r, gt=gt, gt_jpos=gtj))
        got = metrics.metrics_from_frames(d["frames"], r["percent"], r["fail_safe"])
        for k in KEYS:
            assert got[k].shape == want[k].shape
            worst = max(worst, float((np.abs(got[k] - want[k]) / np.maximum(np.abs(want[k]), 1e-9)).max()))
    _WORST["metric"] = max(_WORST["metric"], worst)
    print(f"device vs compute_metrics on the same states: worst relative metric difference {worst:.2e} (all tests so far {_WORST['metric']:.2e})")
    assert worst <= METRIC_RTOL

    dropin = 0.0
    for name in host_pkl:
        h, g = host_pkl[name], dev_pkl[name]
        assert list(h) == list(g)
        for key in h:
            assert set(h[key]) == set(g[key]), key
            assert np.array_equal(h[key]["succ"], g[key]["succ"]) and h[key]["percent"] == g[key]["percent"] and h[key]["reward"] == g[key]["reward"]
            for m in KEYS:
                if m in h[key]:
                    a, b = np.asarray(h[key][m]), np.asarray(g[key][m])
                    assert a.shape == b.shape, (key, m)
                    dropin = max(dropin, float((np.abs(a - b) / np.maximum(np.abs(a), 1.0)).max()) if a.size else 0.0)
    for rh, rd in zip(host, dev):
        for name in rh:
            for k, v in rh[name].items():
                dropin = max(dropin, abs(v - rd[name][k]) / max(abs(v), 1.0))
    print(f"drop-in (host loop vs eval_on_device): worst relative difference {dropin:.2e}")
    assert dropin <= (DROPIN_RTOL if precision == 32 and tables == "host" else METRIC_RTOL)
    return dev_out


@pytest.mark.parametrize("fail_safe", [True, False])
def test_default_config_fail_safe(tmp_path, monkeypatch, fail_safe):
    out = _compare(tmp_path, monkeypatch, fail_safe=fail_safe)
    assert any(d["fail_any"] for d in out), "no failure: the fail / fail_safe path was not exercised"
    if not fail_safe:
        assert all(len(d["frames"]) <= d["last_t"] for d in out if d["fail_any"])


@pytest.mark.parametrize("cfg_file", ["uhc_b200_explicit.yml", "uhc_b200_implicit.yml"])
def test_explicit_and_mcp_actors(tmp_path, monkeypatch, cfg_file):
    _compare(tmp_path, monkeypatch, cfg_file=cfg_file, window=5)


@pytest.mark.parametrize("window", [1, 500])
def test_windows(tmp_path, monkeypatch, window):
    _compare(tmp_path, monkeypatch, window=window, nclips=5, test_clips=0)


def test_short_clips_and_idle_envs(tmp_path, monkeypatch):
    out = _compare(tmp_path, monkeypatch, num_envs=16, nclips=6, test_clips=0, short=(2, 3))
    assert sorted(len(d["frames"]) for d in out)[:2] == [1, 2]


def test_device_tables(tmp_path, monkeypatch):
    _compare(tmp_path, monkeypatch, tables="device")


def test_production_graph_without_state_record(tmp_path, monkeypatch):
    _compare(tmp_path, monkeypatch, record_states=False)


def test_repeated_evaluation_across_table_swaps_and_cfg_changes(tmp_path, monkeypatch):
    """each eval_policy loads the test loader's table and reloads the training one, and the second round runs under another cfg: the
    device path must recapture instead of replaying graphs that hold the old tables or the old cfg"""
    agent, cfg = _agent(tmp_path, monkeypatch, nclips=6, test_clips=3, num_envs=8)
    out1 = _pair(monkeypatch, agent, cfg, 7, False, "host", 32, epoch=0)
    cfg.cfg_dict["body_diff_thresh_test"] = 10.0          # nothing fails under this threshold
    out2 = _pair(monkeypatch, agent, cfg, 7, False, "host", 32, epoch=2)
    assert [d["last_t"] for d in out1] != [d["last_t"] for d in out2] or [d["fail_any"] for d in out1] != [d["fail_any"] for d in out2], \
        "the cfg change did not change the roll-outs: the test would not see a stale cfg"
    cfg.cfg_dict["body_diff_thresh_test"] = 0.2
    _pair(monkeypatch, agent, cfg, 7, False, "host", 32, epoch=4)
    agent.agent.engine.close()


def test_fp64_engine(tmp_path, monkeypatch):
    _compare(tmp_path, monkeypatch, precision=64, nclips=4, test_clips=0, num_envs=4)


def test_bad_arguments_leave_the_engine_usable():
    import torch
    from uhc_b200 import nn
    from uhc_b200.engine import Engine
    from uhc_b200.motion_lib import synthetic_clip
    E = 4
    eng = Engine(E)
    with pytest.raises(ValueError):        # no table loaded
        eng.eval_run([0], nn.mlp_struct(nn.MLPNet(657, (64,), 105, "gelu", head_name="action_mean", seed=1)), torch.zeros(105, device="cuda"),
                     torch.zeros(1 + 2 * 657, device="cuda", dtype=torch.float64))
    clips = [synthetic_clip(30, np.random.default_rng(s)) for s in range(3)]
    eng.load_clips(clips, [np.zeros(17)] * 3)
    pol = nn.MLPNet(657, (64,), 105, "gelu", head_name="action_mean", seed=1)
    bad = nn.MLPNet(600, (64,), 105, "gelu", head_name="action_mean", seed=1)
    ls = torch.full((105,), -2.3, device="cuda")
    zs = torch.zeros(1 + 2 * 657, device="cuda", dtype=torch.float64)
    good = lambda: eng.eval_run([0, 1, 2], nn.mlp_struct(pol), ls, zs, window=4)
    ref = good()
    for args in (dict(clips=[]), dict(clips=[0] * (E + 1)), dict(clips=[0, 3]), dict(clips=[-1]), dict(window=0), dict(policy=nn.mlp_struct(bad))):
        kw = dict(clips=[0, 1, 2], policy=nn.mlp_struct(pol), window=4)
        kw.update(args)
        with pytest.raises(ValueError):
            eng.eval_run(kw["clips"], kw["policy"], ls, zs, window=kw["window"])
        again = good()
        assert np.array_equal(again["nframes"], ref["nframes"]) and all(np.array_equal(a[:k], b[:k]) for a, b, k in zip(again["frames"], ref["frames"], ref["nframes"]))
    eng.close()
