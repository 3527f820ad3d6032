"""GPU: expert tables built on the device from raw motion (uhc_load_motions / Engine.load_motions) against the host-built tables
(uhc_b200/motion_lib.py + uhc_load_clips): the table itself in fp64 and fp32, chunking, the load_clips contract, a rollout and the
drop-in evaluation."""
import ctypes as C
import os
import types

import numpy as np
import pytest

from tests.helpers import write_synthetic_pkl
from tests.test_emu_motion import adversarial_clip, golden, host_table, smpl_clip
from uhc_b200 import motion_lib as ML
from uhc_b200.model import HumanoidModel

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Gimbal lock")]


def raw_table(eng):
    """the loaded table as the engine holds it ([frames][576], doubles), read clip by clip with uhc_get_clip_frames"""
    out = []
    for c in range(len(eng.clip_len)):
        n = int(eng.clip_len[c])
        a = np.zeros((n, 576))
        assert eng.lib.uhc_get_clip_frames(eng.h, c, 0, n, a.ctypes.data_as(C.POINTER(C.c_double))) == 0
        out.append(a)
    return np.concatenate(out)


def datasets():
    rng = np.random.default_rng(0)
    sway, kick = golden("sway"), golden("kick")
    return {
        "goldens_smpl": [{"pose_aa": g["pose_aa"], "trans": g["trans"]} for g in (sway, kick)],
        "goldens_qpos": [{"qpos": g["qpos"]} for g in (sway, kick)],
        "synthetic": [{"qpos": ML.synthetic_clip(T, rng)["qpos"]} for T in (80, 2, 45)],
        "smpl_random": [smpl_clip(T, rng, scale) for T, scale in ((60, 0.6), (3, 1.5), (50, 1.5))],
        "adversarial": [adversarial_clip()],
        "smplh": [{"pose_aa": np.concatenate([g["pose_aa"][:, :66], np.ones((len(g["pose_aa"]), 90))], 1), "trans": g["trans"]} for g in (sway, kick)],
    }


@pytest.mark.parametrize("name", list(datasets()))
def test_fp64_table_matches_host_table(name):
    from uhc_b200.engine import Engine
    clips = datasets()[name]
    eng = Engine(2, precision=64)
    eng.load_motions(ML.MotionSet(clips))
    d = np.abs(raw_table(eng) - host_table(clips))
    assert d.max() <= 1e-12, "column %d differs by %g" % (np.argmax(d.max(0)), d.max())
    eng.close()


def fp32_compare(got, host):
    """values of the fp32 table that are not the host table's value rounded to fp32, and the largest difference in fp32 ulps.  The device
    fp64 values agree with the host's to 1e-12 (test_fp64_table_matches_host_table), not bit for bit: CUDA's sin / atan2 / hypot round the
    last bit differently from glibc's.  So a value is held to one fp32 ulp plus that 1e-12; it matters only where an fp32 ulp is finer
    than 1e-12, e.g. the pitch 2 atan2(h, h) - pi/2 of an unrotated joint, exactly 0 on the host and +-2e-16 on the device."""
    want = host.astype(np.float32)
    g = got.astype(np.float32)
    assert (g.astype(np.float64) == got).all()
    d = np.abs(g.astype(np.float64) - want)
    assert (d <= np.spacing(np.abs(want)) + 1e-12).all()
    return int((g != want).sum()), float((d / np.spacing(np.abs(want))).max())


@pytest.mark.parametrize("name", list(datasets()))
def test_fp32_table_within_one_ulp_of_host_table(name):
    from uhc_b200.engine import Engine
    clips = datasets()[name]
    eng = Engine(2)
    eng.load_motions(ML.MotionSet(clips))
    got = raw_table(eng)
    host = host_table(clips)
    nbad, worst = fp32_compare(got, host)
    print(f"{name}: {nbad} of {got.size} fp32 values not bit-identical to the host table, worst {worst:.0f} ulp")
    if name == "goldens_qpos":
        assert nbad == 0
    # the host table through uhc_load_clips reads back as the same fp32 values
    eng.load_clips([ML.make_expert(c["pose_aa"], c["trans"]) if "pose_aa" in c else ML.qpos_fk(c["qpos"]) for c in clips])
    assert (raw_table(eng) == host.astype(np.float32)).all()
    eng.close()


@pytest.mark.parametrize("precision", [32, 64])
def test_chunked_load_matches_single_chunk(precision):
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(4)
    lens = (5, 3, 19, 2, 7, 30, 4, 6)                      # chunks of at most 7 frames: one chunk per clip or two, and clips longer than a chunk
    clips = [smpl_clip(T, rng) for T in lens]
    ms = ML.MotionSet(clips)
    eng = Engine(2, precision=precision)
    eng.load_motions(ms)
    one = raw_table(eng)
    eng.load_motions(ms, chunk_frames=7)
    assert (raw_table(eng) == one).all()
    eng.load_motions(ms, chunk_frames=1)
    assert (raw_table(eng) == one).all()
    host = host_table(clips)
    if precision == 64:
        assert np.abs(one - host).max() <= 1e-12
    else:
        fp32_compare(one, host)
    t = eng.load_motions_time
    assert t["kernel_ms"] > 0 and t["copy_ms"] > 0
    assert list(eng.clip_len) == list(lens)
    ex = eng.clip_frames(2, 4, 6)                         # a slice: qpos_fk field names and shapes
    assert ex["qpos"].shape == (6, 76) and ex["wbquat"].shape == (6, 96) and ex["com"].shape == (6, 3) and ex["len"] == 6
    assert (ex["qpos"] == one[sum(lens[:2]) + 4:sum(lens[:2]) + 10, :76]).all()
    eng.close()


def test_contract_parity_with_load_clips():
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(2)
    clips = [{"qpos": ML.synthetic_clip(T, rng)["qpos"]} for T in (40, 25, 60)]
    ms = ML.MotionSet(clips)
    E = 4
    hm0 = HumanoidModel()
    eng = Engine(E, hm0, t_max=20, auto_reset=0, variants=[hm0, HumanoidModel(scale=np.full(24, 1.05))])
    eng.load_motions(ms)
    eng.reset()
    import torch
    a = torch.zeros(E, eng.act_dim, device="cuda")
    eng.step(a)
    before = eng.counters["invalid_env_steps"]
    eng.load_motions(ms)                                  # stale records: skipped, flagged and counted
    _, _, _, fail, end, _ = eng.step(a)
    torch.cuda.synchronize()
    assert eng.counters["invalid_env_steps"] == before + E and (fail.cpu().numpy() == 1).all() and (end.cpu().numpy() == 1).all()
    eng.set_clip_weights([1.0, 0.0, 2.0])
    eng.set_clip_weights(None)
    with pytest.raises(RuntimeError):
        eng.set_clip_weights([1.0, 1.0])                  # one weight per clip of the new table
    eng.load_motions(ms, clip_models=[1, 0, 1])
    with pytest.raises(RuntimeError):
        eng.load_motions(ms, clip_models=[0, 2, 0])       # variant out of range
    # bad arguments: an error code and text, the previous table stays loaded and usable
    eng.load_motions(ms)
    table = raw_table(eng)
    L = eng.lib
    lens = np.ascontiguousarray(ms.lens, np.int32)
    rows = ms.rows.ctypes.data_as(C.POINTER(C.c_double))
    shp = np.zeros((3, 17)).ctypes.data_as(C.POINTER(C.c_double))
    ip = lambda x: np.ascontiguousarray(x, np.int32).ctypes.data_as(C.POINTER(C.c_int))
    short = np.array([40, 1, 60], np.int32)
    bad = [(3, ip(lens), 2, 76, rows, shp, None, 0), (3, ip(lens), 1, 72, rows, shp, None, 0), (3, ip(lens), 0, 76, rows, shp, None, 0),
           (3, ip(lens), 1, 76, rows, shp, ip([0, 2, 0]), 0), (3, ip(lens), 1, 76, rows, shp, ip([0, -1, 0]), 0), (3, ip(lens), 1, 76, None, shp, None, 0),
           (3, ip(lens), 1, 76, rows, None, None, 0), (0, ip(lens), 1, 76, rows, shp, None, 0), (3, ip(short), 1, 76, rows, shp, None, 0),
           (3, ip(lens), 1, 76, rows, shp, None, -1)]
    for n, ln, kind, pd, r, s, fk, ch in bad:
        rc = L.uhc_load_motions(eng.h, n, ln, kind, pd, r, s, fk, ch)
        assert rc == -2 and L.uhc_last_error().startswith(b"uhc_load_motions"), (kind, pd)
    assert (raw_table(eng) == table).all()
    out = np.zeros((5, 576))
    for c, first, n in ((3, 0, 1), (-1, 0, 1), (0, 38, 3), (0, -1, 2)):
        assert L.uhc_get_clip_frames(eng.h, c, first, n, out.ctypes.data_as(C.POINTER(C.c_double))) == -2
    eng.reset(clip=[0, 1, 2, 0])
    eng.step(a)
    torch.cuda.synchronize()
    eng.close()


def _pair(E, clips, shapes, clip_models, fk_models, models, precision=32, **cfg):
    from uhc_b200.engine import Engine
    host = Engine(E, models[0], precision=precision, variants=models, **cfg)
    host.load_clips([ML.qpos_fk(c["qpos"], models[m]) for c, m in zip(clips, fk_models)], shapes, clip_models)
    dev = Engine(E, models[0], precision=precision, variants=models, **cfg)
    dev.load_motions(ML.MotionSet(clips), shapes, clip_models, fk_models)
    return host, dev


def test_rollout_from_device_table_is_bit_identical():
    import torch
    rng = np.random.default_rng(9)
    models = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    z = golden("sway")
    clips = [{"qpos": z["qpos"]}, {"qpos": golden("kick")["qpos"]}]
    shapes = [np.concatenate([z["beta"][0], [z["gender"][0]]])] * 2
    E = 64
    host, dev = _pair(E, clips, shapes, [0, 1], [0, 1], models, auto_reset=1, t_min=5, t_max=40)
    assert (raw_table(host) == raw_table(dev)).all(), "the two tables differ: the rollouts cannot be compared"
    ids = np.arange(E, dtype=np.int32)
    for eng in (host, dev):
        eng.reset(ids, ids % 2, ids % 20, None)
    acts = torch.tensor(np.random.default_rng(1).normal(0, 0.1, (40, E, host.act_dim)), dtype=torch.float32, device="cuda")
    ends = 0
    for t in range(40):
        if t == 20:
            for eng in (host, dev):
                eng.set_clip_weights([0.2, 0.8])
        outs = [[x.cpu().numpy().copy() for x in eng.step(acts[t].contiguous())] for eng in (host, dev)]
        for a, b, name in zip(outs[0], outs[1], ("obs", "reward", "cinfo", "fail", "end", "percent")):
            assert np.array_equal(a, b), f"step {t}: {name} differs"
        ends += int(outs[0][4].sum())
    assert ends > 0, "no episode ended: auto_reset was not exercised"
    sh, sd = host.get_states(), dev.get_states()
    assert all(np.array_equal(sh[k], sd[k]) for k in sh)
    host.close(); dev.close()


def _dropin_cfg(tmp_path, tables):
    import yaml
    from uhc.utils.config_utils.copycat_config import Config
    base = yaml.safe_load(open(os.path.join(os.path.dirname(__file__), "..", "config", "uhc_b200_default.yml")))
    base.update(policy_hsize=[128, 64], value_hsize=[128, 64], min_batch_size=1024, num_optim_epoch=2, num_envs=8, save_n_epochs=2, num_epoch=1)
    base["data_specs"]["file_path"] = write_synthetic_pkl(str(tmp_path / "sample_data" / "clips.pkl"), nclips=10)
    base["data_specs"]["test_file_path"] = write_synthetic_pkl(str(tmp_path / "sample_data" / "test_clips.pkl"), nclips=4, seed=1)
    base["data_specs"]["t_max"] = 40
    base["data_specs"]["expert_tables"] = tables
    cfg = Config(cfg_id=f"motion_{tables}", create_dirs=True, cfg_dict=base)
    cfg.update(types.SimpleNamespace(cfg=f"motion_{tables}", render=False, test=False, num_threads=30, gpu_index=0, epoch=0, show_noise=False,
                                     resume=None, no_log=True, debug=False, full_eval=False))
    return cfg


def test_dropin_eval_with_device_tables(tmp_path, monkeypatch):
    import joblib
    import torch
    from uhc.agents import agent_dict
    monkeypatch.chdir(tmp_path)
    res, per_clip = {}, {}
    for tables in ("host", "device"):
        cfg = _dropin_cfg(tmp_path, tables)
        np.random.seed(cfg.seed)
        torch.manual_seed(cfg.seed)
        agent = agent_dict[cfg.agent_name](cfg, torch.float64, torch.device("cuda", 0), training=True, checkpoint_epoch=0)
        assert hasattr(agent.data_loader, "experts") == (tables == "host") and hasattr(agent.data_loader, "motions") == (tables == "device")
        res[tables] = agent.eval_policy(epoch=0, dump=True)
        per_clip[tables] = {ld.name: joblib.load(os.path.join(cfg.output_dir, f"0_{ld.name}_coverage_full.pkl")) for ld in agent.test_data_loaders}
        agent.agent.engine.close()
    worst = 0.0
    for rh, rd in zip(res["host"], res["device"]):
        for name in rh:
            mh, md = rh[name], rd[name]
            assert mh["num_coverage"] == md["num_coverage"] and mh["all_coverage"] == md["all_coverage"]
            for k, v in mh.items():
                worst = max(worst, abs(v - md[k]) / max(abs(v), 1e-12))
    for name, clips_h in per_clip["host"].items():
        clips_d = per_clip["device"][name]
        assert set(clips_h) == set(clips_d)
        for key in clips_h:
            for m, v in clips_h[key].items():
                a, b = np.asarray(v, dtype=np.float64), np.asarray(clips_d[key][m], dtype=np.float64)
                assert a.shape == b.shape, (key, m)
                worst = max(worst, float((np.abs(a - b) / np.maximum(np.abs(a), 1e-12)).max()) if a.size else 0.0)
    print(f"drop-in eval, device vs host expert tables: worst relative metric difference {worst:.2e}")
    assert worst <= 1e-5
