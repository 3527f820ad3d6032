"""GPU: the floor measurements -- uhc_floor_qpos and uhc_motion_floor against the host emulation of the same code, the evaluation's floor
rows (uhc_eval_run*_ex with floor_host) against the standalone kernel and the plain evaluation, MotionSet.fix_height end to end, and
Tracker.floor."""
import ctypes as C

import numpy as np
import pytest

from tests.emu import floor_emu as emu
from tests.test_gpu_eval_groups import _policy, _same, _zstats
from tests.test_gpu_export import _variant_engine

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Gimbal lock")]
# The reduction (vertex transform, sums, butterfly) is the emulation's arithmetic operation for operation, but the pose pass before it takes
# sin / cos of the joint angles, which CUDA may round differently from the host's libm in the last bit (the 1e-12-class bound
# tests/test_gpu_motion_lib.py documents): so the device rows are held to a bound, not to the emulation's bits.
TOL_M, TOL_MM = 1e-12, 1e-9


def _close(got, want):
    assert np.abs(got[:, 0] - want[:, 0]).max() <= TOL_M
    assert np.abs(got[:, 1:4] - want[:, 1:4]).max() <= TOL_MM
    assert np.array_equal(got[:, 4], want[:, 4])


def _poses(n, seed, pitch=76):
    rng = np.random.default_rng(seed)
    rows = rng.normal(size=(n, pitch))
    rows[:, :3] = rng.normal(0, 0.2, (n, 3)) + [0, 0, 0.5]
    rows[:, 3:7] /= np.linalg.norm(rows[:, 3:7], axis=1, keepdims=True)
    rows[:, 7:76] = rng.normal(0, 0.5, (n, 69))
    rows[1::2, :76] = rows[0::2, :76] + rng.normal(0, 0.01, (n // 2, 76))     # consecutive frames close enough to share floor vertices
    return rows


@pytest.mark.parametrize("precision", [32, 64])
@pytest.mark.parametrize("pitch", [76, 148, 223])
def test_standalone_against_the_emulation(precision, pitch):
    import torch
    eng, variants, _ = _variant_engine()
    n = 64
    q = torch.tensor(_poses(n, pitch, pitch), device="cuda").to(torch.float32 if precision == 32 else torch.float64)
    q_in = q.double().cpu().numpy()                      # what the kernel reads (fp32 inputs: the rounded values)
    var, first = np.arange(n) // 2 % 2, (np.arange(n) % 8 == 0).astype(np.int32)
    got = eng.floor_qpos(q, variants=var, first=first).cpu().numpy()
    _close(got, emu.floor_qpos(q_in, variants, var, first))
    assert (got[:, 1] > 0).any() and (got[:, 2] > 0).any() and (got[first == 1, 2] == 0).all()
    _close(eng.floor_qpos(q).cpu().numpy(), emu.floor_qpos(q_in, variants))
    eng.close()


def test_bad_arguments_leave_the_engine_usable():
    import torch
    from uhc_b200.engine import Engine, UhcEvalClip, UhcEvalOut, load_library
    eng, _, _ = _variant_engine()
    L = eng.lib
    q = torch.tensor(_poses(4, 0), device="cuda")
    out = torch.zeros(4, 5, device="cuda", dtype=torch.float64)
    P = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)

    def call(n=4, prec=64, pitch=76, var=None, qq=q, oo=out, e=eng.h):
        return L.uhc_floor_qpos(e, P(qq), C.c_int(prec), C.c_long(n), C.c_long(pitch), P(var), None, P(oo), None)
    err = lambda: load_library().uhc_last_error().decode()
    assert call() == -2 and "uhc_floor_init" in err()                                    # no hulls yet
    _, pol = _policy("gauss", 0)
    zs, ls = _zstats(0), torch.full((eng.act_dim,), -2.3, device="cuda")
    fr, fl = torch.empty(2, 100, 6, dtype=torch.float64, pin_memory=True), torch.empty(2, 100, 5, dtype=torch.float64, pin_memory=True)
    rec = (UhcEvalClip * 2)()
    o = Engine._eval_out(fr, rec, None, None, fl)
    clips = np.zeros(2, np.int32)
    args = (eng.h, C.c_int(2), clips.ctypes.data_as(C.POINTER(C.c_int)), C.byref(pol), P(ls), P(zs), C.c_float(5.0), C.c_int(1), C.c_int(4), C.byref(o), None)
    assert L.uhc_eval_run_ex(*args) == -2 and "uhc_floor_init" in err()
    eng._floor_init()
    bad_v = torch.tensor([0, 1, 2, 0], device="cuda", dtype=torch.int32)
    for kw, word in ((dict(n=-1), "n < 0"), (dict(prec=16), "precision"), (dict(pitch=75), "qpos_pitch"), (dict(qq=None), "null pointer"),
                     (dict(oo=None), "null pointer"), (dict(var=bad_v), "variant"), (dict(e=None), "null engine")):
        assert call(**kw) == -2 and word in err(), kw
    assert call(n=0, qq=None, oo=None) == 0
    s223 = torch.zeros(eng.E, 223, device="cuda")
    assert L.uhc_track_floor(eng.h, P(s223), P(out), None) == -2 and "not tracking" in err()
    with pytest.raises(ValueError, match="floor_qpos"):
        eng.floor_qpos(np.zeros((3, 75)))
    assert call() == 0 and L.uhc_eval_run_ex(*args) == 0
    torch.cuda.synchronize()
    _close(out.cpu().numpy(), emu.floor_qpos(q.cpu().numpy()))
    lens = np.array([3, 2], np.int32)
    rows = np.zeros((5, 76))
    ml = lambda n=2, kind=1, dim=76, chunk=0, oo=out: L.uhc_motion_floor(eng.h, C.c_int(n), lens.ctypes.data_as(C.POINTER(C.c_int)), C.c_int(kind), C.c_int(dim),
                                                                         rows.ctypes.data_as(C.POINTER(C.c_double)), None, C.c_int(chunk), P(oo), None)
    for kw in (dict(n=0), dict(kind=2), dict(dim=72), dict(kind=0, dim=76), dict(chunk=-1), dict(oo=None)):
        assert ml(**kw) == -2, kw
    eng.close()


def _check_floor(eng, r, clips, models):
    import torch
    for i, k in enumerate(r["nframes"]):
        st = torch.tensor(r["states"][i, :k], device="cuda")                           # [k][148]: one clip, read in place at pitch 148
        v = None if models is None else np.full(k, models[clips[i]])
        assert np.array_equal(r["floor"][i, :k], eng.floor_qpos(st, variants=v).cpu().numpy()), i
        assert k == 0 or r["floor"][i, 0, 2] == 0


@pytest.mark.parametrize("fail_safe", [True, False])
@pytest.mark.parametrize("precision", [32, 64])
def test_eval_floor_rows(fail_safe, precision):
    import torch
    eng, _, models = _variant_engine(E=8, precision=precision)
    _, pol = _policy("gauss", 1)
    zs, ls = _zstats(1), torch.full((eng.act_dim,), -2.3, device="cuda")
    clips = [0, 1, 2, 3, 4, 5]
    plain = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True)
    count = eng.eval_graph_count
    again = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True)            # floor NULL: the cached graph, no second entry
    assert eng.eval_graph_count == count
    fl = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True, True)       # its window buffer is new: graphs holding the old scratch go
    _same(eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True), plain)
    assert eng.eval_graph_count == 2                                                   # one graph with the floor rows, one without, side by side
    fl2 = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True, True)
    eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True)
    assert eng.eval_graph_count == 2 and all(np.array_equal(fl2["floor"][i, :k], fl["floor"][i, :k]) for i, k in enumerate(fl["nframes"]))
    _same(fl, plain)
    _same(again, plain)
    for k in ("pose_aa", "trans"):
        assert np.array_equal(fl[k], plain[k])
    _check_floor(eng, fl, clips, models)
    eng._floor_ready = False                                                           # the hulls uploaded again: the graph that holds the freed
    eng._floor_init()                                                                  # copy is keyed on it and is not replayed
    fl3 = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, 7, True, True, True)
    _same(fl3, plain)
    _check_floor(eng, fl3, clips, models)
    assert all(np.array_equal(fl3["floor"][i, :k], fl["floor"][i, :k]) for i, k in enumerate(fl["nframes"]))
    assert fl["fail_any"].any(), "no failure: the fail / fail_safe path was not exercised"
    one = eng.eval_run([5, 2], pol, ls, zs, 5.0, fail_safe, 1, True, False, True)      # window 1: the previous frame crosses every replay
    _check_floor(eng, one, [5, 2], models)
    eng.close()


@pytest.mark.parametrize("fail_safe", [True, False])
def test_eval_floor_rows_groups(fail_safe):
    eng, _, models = _variant_engine(E=12)
    pols = [_policy("gauss", s)[1] for s in range(2)]
    groups = [([0, 1, 2], pols[0], _zstats(0)), ([4, 5, 0, 1], pols[1], _zstats(1))]
    got = eng.eval_run_groups(groups, 5.0, fail_safe, 5, True, False, True)
    plain = eng.eval_run_groups(groups, 5.0, fail_safe, 5, True)
    for (clips, _, _), g, p in zip(groups, got, plain):
        _same(g, p)
        _check_floor(eng, g, clips, models)
    eng.close()


def test_motion_floor_and_height_fix_end_to_end():
    from uhc_b200.engine import Engine
    from uhc_b200.model import HumanoidModel
    from uhc_b200.motion_lib import MotionSet
    from tests.test_emu_floor import golden
    rng = np.random.default_rng(8)
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24)), HumanoidModel(scale=rng.uniform(0.9, 1.15, 24))]
    eng = Engine(4, model=variants[0], variants=variants)
    sets = [(MotionSet([{"qpos": golden(t)} for t in ("sway", "kick")]), None)]
    pose = rng.normal(0, 0.2, (7, 40, 72))
    pose[:, :, 0] += np.pi / 2
    sets.append((MotionSet([{"pose_aa": p[:T], "trans": rng.normal(0, 0.1, (T, 3)) + [0, 0, 0.95]} for p, T in zip(pose, (40, 1, 17, 40, 3, 25, 9))]),
                 np.arange(7) % 3))
    for ms, fk in sets:
        want, wfeet = emu.EmuFloor(variants).motion_floor(ms, fk)
        for chunk in (0, 30):                                                       # several chunks, both staging buffers reused
            rows, feet = eng.motion_floor(ms, fk, chunk)
            _close(rows.cpu().numpy(), want)
            assert np.abs(feet.cpu().numpy() - wfeet).max() <= TOL_M
    ms, fk = sets[1]
    audit = ms.floor_audit(eng, fk)
    fixed = ms.fix_height(audit, "first_frame")
    assert np.abs(fixed.floor_audit(eng, fk)["dz_first"]).max() < 1e-12
    keep = fixed.lens >= 2
    fixed = fixed.drop(~keep)
    eng.load_motions(fixed, fk_models=fk[keep], clip_models=fk[keep])
    q0 = np.stack([eng.clip_frames(c, 0, 1)["qpos"][0] for c in range(len(fixed))])  # the table's first frames stand on the floor
    assert np.abs(eng.floor_qpos(q0, variants=fk[keep], first=np.ones(len(q0))).cpu().numpy()[:, 0]).max() < 1e-6
    eng.close()


def test_tracker_floor():
    import torch
    from tests.test_gpu_track import TRACK_KW
    from uhc_b200 import motion_lib as ML
    from uhc_b200.agent import BatchedAgent
    rng = np.random.default_rng(9)
    E = 4
    clips = [ML.synthetic_clip(8, rng) for _ in range(E)]
    agent = BatchedAgent(E, clips, policy_hsize=(64, 32), value_hsize=(64, 32), auto_reset=False, **TRACK_KW)
    trk = agent.tracker(window=8, kind="qpos", fail_safe=True)
    ref = torch.tensor(np.stack([c["qpos"] for c in clips]), device="cuda")
    trk.reset(ref[:, 0], ref[:, 1])
    state, _, _ = trk.step()
    for k in range(1, 4):
        state, _, _ = trk.step(ref[:, k + 1])
    got = trk.floor().cpu().numpy()
    rows = state.double().cpu().numpy()                                              # [E][223]
    want = agent.engine.floor_qpos(torch.tensor(rows, device="cuda"), first=np.ones(E)).cpu().numpy()   # the fp64 copy at pitch 223
    assert np.array_equal(got, want) and (got[:, 2] == 0).all()
    _close(got, emu.floor_qpos(rows, first=np.ones(E)))
    agent.engine.close()


def test_training_after_drop_implausible_drops_a_clip(tmp_path, monkeypatch):
    """data_specs.fix_height + drop_implausible through AgentCopycat: a clip that starts too high is dropped before the agent's clip table and
    clip sampler are built, a rollout and an update train on what is left, and eval_policy reports the floor metrics on both evaluation paths"""
    import joblib
    import torch
    from tests.test_gpu_dropin import _cfg
    from uhc.agents import agent_dict
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                    # as the reference's scripts run
    try:
        cfg = _cfg(tmp_path, monkeypatch)
        path = cfg.data_specs["file_path"]
        data = joblib.load(path)
        keys = list(data)
        data[keys[1]]["trans"][:, 2] += 0.5                   # starts half a metre up: fix_height_smpl's "Starting too high"
        joblib.dump(data, path)
        cfg.data_specs.update(expert_tables="device", fix_height="first_frame", drop_implausible=True)
        cfg.cfg_dict.update(eval_floor_metrics=True, eval_on_device=True)
        agent = agent_dict[cfg.agent_name](cfg, torch.float64, torch.device("cuda", index=0), training=True, checkpoint_epoch=0)
        left = [keys[0], keys[2]]
        eng = agent.agent.engine
        assert agent.data_loader.data_keys == left and list(agent.freq_dict) == left
        assert len(eng.clip_len) == 2 and np.array_equal(agent.agent.sampler.lens, eng.clip_len)
        assert np.array_equal(eng.clip_len, [len(data[k]["pose_aa"]) for k in left])
        q0 = np.stack([eng.clip_frames(c, 0, 1)["qpos"][0] for c in range(2)])
        assert np.abs(eng.floor_qpos(q0, first=np.ones(2)).cpu().numpy()[:, 0]).max() < 1e-6          # the table's first frames stand on the floor
        info = agent.optimize_policy(0)
        assert info["log"]["num_steps"] >= cfg.min_batch_size and np.isfinite(info["log"]["avg_reward"])
        res = {}
        for on_device in (True, False):
            cfg.cfg_dict["eval_on_device"] = on_device
            res[on_device] = m = agent.eval_policy(epoch=1)[0][f"coverage_{agent.data_loader.name}"]
            assert m["all_coverage"] == 2
            for k in ("pentration", "skate", "float", "pentration_gt", "skate_gt", "float_gt"):
                assert np.isfinite(m[k]) and m[k] >= 0, k
        for k in ("pentration_gt", "skate_gt", "float_gt"):                                            # the same expert frames on both paths
            assert abs(res[True][k] - res[False][k]) <= 1e-6 * max(1.0, abs(res[True][k])), k
        eng.close()
    finally:
        torch.set_default_dtype(old)
