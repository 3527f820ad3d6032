"""GPU: the SMPL export -- uhc_qpos_to_smpl against the reference's qpos_to_smpl golden and scipy, the evaluation's export stream
(uhc_eval_run*_ex) against the standalone kernel and the plain evaluation, BatchedAgent.export_motion's chunking, and Tracker.smpl."""
import ctypes as C
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation as sRot

from tests.test_gpu_eval_groups import _policy, _same, _zstats

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Gimbal lock")]
# CUDA's atan2 / sin / cos may round the last bit differently from the host's libm (DESIGN.md 4.4), so the device export is held to a bound
TOL = 1e-12


def _golden():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "qpos_to_smpl.npz"))
    return {k: z[k] for k in z.files}


def _scipy(qpos, root_offset):
    q = np.asarray(qpos, np.float64)[:, :76]
    pose = np.zeros((len(q), 24, 3))
    pose[:, 0] = sRot.from_quat(q[:, [4, 5, 6, 3]]).as_rotvec()
    order = [0, 1, 4, 7, 10, 2, 5, 8, 11, 3, 6, 9, 12, 15, 13, 16, 18, 20, 22, 14, 17, 19, 21, 23]
    for b in range(1, 24):
        pose[:, order[b]] = sRot.from_euler("ZYX", q[:, 7 + 3 * (b - 1):10 + 3 * (b - 1)]).as_rotvec()
    return pose.reshape(len(q), 72), q[:, :3] - root_offset


def _variant_engine(E=8, precision=32, nclips=6, tables="host"):
    """an engine with two shape variants, clips alternating between them"""
    from uhc_b200.engine import Engine
    from uhc_b200.model import HumanoidModel
    from uhc_b200.motion_lib import MotionSet
    from tests.test_gpu_eval_groups import _clips
    rng = np.random.default_rng(4)
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    eng = Engine(E, model=variants[0], precision=precision, variants=variants, body_diff_thresh=0.2)
    clips = _clips(nclips, 5)
    models = np.arange(nclips, dtype=np.int32) % 2
    if tables == "device":
        eng.load_motions(MotionSet([{"qpos": c["qpos"]} for c in clips]), [np.zeros(17)] * nclips, clip_models=models)
    else:
        eng.load_clips(clips, [np.zeros(17)] * nclips, clip_models=models)
    return eng, variants, models


# ---- 1. the standalone kernel
@pytest.mark.parametrize("precision", [32, 64])
@pytest.mark.parametrize("pitch", [76, 148, 223])
def test_standalone_against_golden_and_scipy(precision, pitch):
    import torch
    eng, variants, _ = _variant_engine()
    z = _golden()
    n = len(z["qpos"])
    rows = np.random.default_rng(pitch).normal(size=(n, pitch))
    rows[:, :76] = z["qpos"]
    dt = torch.float32 if precision == 32 else torch.float64
    q = torch.tensor(rows, device="cuda").to(dt)
    q_in = q.double().cpu().numpy()                     # what the kernel reads (fp32 inputs: the rounded values)
    for v in (0, 1):
        pose, trans = eng.qpos_to_smpl(q, variants=np.full(n, v))
        pose, trans = pose.cpu().numpy(), trans.cpu().numpy()
        off = variants[v].body_f[0, :3]
        sp, st = _scipy(q_in, off)
        print(f"fp{precision} pitch {pitch} variant {v}: max |pose - scipy| = {np.abs(pose - sp).max():.3g}")
        assert np.abs(pose - sp).max() <= TOL and np.array_equal(trans, st)
        if precision == 64:
            assert np.abs(pose - z["pose"]).max() <= TOL
            if v == 0:
                assert np.array_equal(trans, z["trans"])
    mixed = np.arange(n) % 2                            # a variant per row
    _, trans = eng.qpos_to_smpl(q, variants=mixed)
    off = np.stack([m.body_f[0, :3] for m in variants])[mixed]
    assert np.array_equal(trans.cpu().numpy(), q_in[:, :3] - off)
    eng.close()


def test_bad_arguments_leave_the_engine_usable():
    import torch
    eng, _, _ = _variant_engine()
    L = eng.lib
    q = torch.zeros(4, 76, device="cuda", dtype=torch.float64)
    q[:, 3] = 1
    pose, trans = torch.zeros(4, 72, device="cuda", dtype=torch.float64), torch.zeros(4, 3, device="cuda", dtype=torch.float64)
    P = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)

    def call(n=4, prec=64, pitch=76, var=None, qq=q, pp=pose, tt=trans, e=eng.h):
        return L.uhc_qpos_to_smpl(e, P(qq), C.c_int(prec), C.c_long(n), C.c_long(pitch), P(var), P(pp), P(tt), None)
    bad_v = torch.tensor([0, 1, 2, 0], device="cuda", dtype=torch.int32)
    neg_v = torch.tensor([0, -1, 0, 0], device="cuda", dtype=torch.int32)
    for kw in (dict(n=-1), dict(prec=16), dict(prec=0), dict(pitch=75), dict(qq=None), dict(pp=None), dict(tt=None), dict(var=bad_v),
               dict(var=neg_v), dict(e=None)):
        assert call(**kw) == -2, kw
    assert call(n=0, qq=None, pp=None, tt=None) == 0
    assert L.uhc_track_smpl(eng.h, P(q), P(pose), P(trans), None) == -2                 # not in tracking mode
    e6, _, _ = _variant_engine(E=6, nclips=6)                                           # one clip per env, but no tracker
    s6 = torch.zeros(6, 223, device="cuda")
    assert L.uhc_track_smpl(e6.h, P(s6), P(pose), P(trans), None) == -2
    e6.close()
    ok = torch.tensor([0, 1, 1, 0], device="cuda", dtype=torch.int32)
    assert call(var=ok) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(pose).all() and (pose == 0).all()                             # the identity rotation
    # the evaluation entry points: a null output struct, null outputs inside it
    from uhc_b200.engine import UhcEvalClip, UhcEvalOut
    _, pol = _policy("gauss", 0)
    zs, ls = _zstats(0), torch.full((eng.act_dim,), -2.3, device="cuda")
    clips = np.zeros(2, np.int32)
    args = lambda out: (eng.h, C.c_int(2), clips.ctypes.data_as(C.POINTER(C.c_int)), C.byref(pol), P(ls), P(zs), C.c_float(5.0), C.c_int(1), C.c_int(4), out, None)
    assert L.uhc_eval_run_ex(*args(None)) == -2
    assert L.uhc_eval_run_ex(*args(C.byref(UhcEvalOut()))) == -2
    fr = torch.empty(2, 100, 6, dtype=torch.float64, pin_memory=True)
    rec = (UhcEvalClip * 2)()
    o = UhcEvalOut()
    o.frames_host, o.clips_host = fr.data_ptr(), C.addressof(rec)
    assert L.uhc_eval_run_ex(*args(C.byref(o))) == 0
    r = eng.eval_run([0, 1, 2], pol, ls, zs, 5.0, True, 4, True, True)
    assert (r["nframes"] > 0).all()
    eng.close()


# ---- 2. the export stream of the evaluation
def _check_stream(eng, clips, pol, zs, fail_safe, window, models):
    """_ex with the export against the plain evaluation (bit for bit) and its SMPL rows against uhc_qpos_to_smpl of its own state record"""
    import torch
    ls = torch.full((eng.act_dim,), -2.3, device="cuda")
    ex = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, window, True, True)
    ref = eng.eval_run(clips, pol, ls, zs, 5.0, fail_safe, window, True)
    _same(ex, ref)
    _check_smpl(eng, ex, clips, models)
    return ex


def _check_smpl(eng, r, clips, models):
    import torch
    for i, k in enumerate(r["nframes"]):
        st = torch.tensor(r["states"][i, :k], device="cuda")                          # [k][148]: qpos read in place at pitch 148
        v = None if models is None else np.full(k, models[clips[i]])
        pose, trans = eng.qpos_to_smpl(st, variants=v)
        assert np.array_equal(r["pose_aa"][i, :k], pose.cpu().numpy()), i
        assert np.array_equal(r["trans"][i, :k], trans.cpu().numpy()), i


@pytest.mark.parametrize("fail_safe", [True, False])
@pytest.mark.parametrize("kind", ["gauss", 3])
@pytest.mark.parametrize("precision,tables", [(32, "host"), (64, "host"), (32, "device")])
def test_export_stream(fail_safe, kind, precision, tables):
    eng, _, models = _variant_engine(E=8, precision=precision, tables=tables)
    _, pol = _policy(kind, 1)
    ex = _check_stream(eng, [0, 1, 2, 3, 4, 5], pol, _zstats(1), fail_safe, 7, models)
    assert ex["fail_any"].any(), "no failure: the fail / fail_safe path was not exercised"
    _check_stream(eng, [5, 2], pol, _zstats(1), fail_safe, 500, models)                # n < E, one window longer than every clip
    eng.close()


@pytest.mark.parametrize("kind", ["gauss", 3])
def test_export_stream_groups(kind):
    import torch
    eng, _, models = _variant_engine(E=12)
    pols = [_policy(kind, s)[1] for s in range(3)]
    groups = [([0, 1, 2], pols[0], _zstats(0)), ([3], pols[1], _zstats(1)), ([4, 5, 0, 1], pols[2], _zstats(2))]
    got = eng.eval_run_groups(groups, 5.0, True, 5, True, True)
    plain = eng.eval_run_groups(groups, 5.0, True, 5, True)
    ls = torch.full((eng.act_dim,), -2.3, device="cuda")
    for (clips, pol, zs), g, p in zip(groups, got, plain):
        _same(g, p)
        _check_smpl(eng, g, clips, models)
        single = eng.eval_run(clips, pol, ls, zs, 5.0, True, 5, True, True)           # each group as a call of its own
        for i, k in enumerate(g["nframes"]):
            assert np.array_equal(g["pose_aa"][i, :k], single["pose_aa"][i, :k]) and np.array_equal(g["trans"][i, :k], single["trans"][i, :k])
    eng.close()


def test_graph_cache_and_invalidation():
    import torch
    eng, _, models = _variant_engine(E=8)
    _, pol = _policy("gauss", 2)
    zs, ls = _zstats(2), torch.full((eng.act_dim,), -2.3, device="cuda")
    clips = [0, 1, 2, 3, 4]
    a = eng.eval_run(clips, pol, ls, zs, 5.0, True, 6, True)
    b = eng.eval_run(clips, pol, ls, zs, 5.0, True, 6, True, True)
    c = eng.eval_run(clips, pol, ls, zs, 5.0, True, 6, True)
    _same(a, b)
    _same(a, c)
    _check_smpl(eng, b, clips, models)
    eng.set_cfg(body_diff_thresh=1e-6)                    # every step fails: a stale export graph would not see it
    d = eng.eval_run(clips, pol, ls, zs, 5.0, False, 6, True, True)
    _same(d, eng.eval_run(clips, pol, ls, zs, 5.0, False, 6, True))
    assert (d["nframes"] == 1).all()
    _check_smpl(eng, d, clips, models)
    eng.set_cfg(body_diff_thresh=0.2)
    eng.load_clips([eng.clip_frames(k) for k in (3, 2, 1, 0, 4)], [np.zeros(17)] * 5, clip_models=[1, 1, 0, 0, 1])   # a new table
    e = eng.eval_run(clips, pol, ls, zs, 5.0, True, 6, True, True)
    _same(e, eng.eval_run(clips, pol, ls, zs, 5.0, True, 6, True))
    _check_smpl(eng, e, clips, np.array([1, 1, 0, 0, 1]))
    eng.close()


def test_large_call_4096_envs_window_500():
    """E = n = 4096, window 500, states and export: the state record passes 2^31 bytes; the last env's last rows against the kernel"""
    import torch
    from uhc_b200.engine import Engine
    from uhc_b200.motion_lib import synthetic_clip
    rng = np.random.default_rng(2)
    E = 4096
    clips = [synthetic_clip(T, rng) for T in (505, 520, 480)]
    eng = Engine(E, body_diff_thresh=10.0)
    eng.load_clips(clips, [np.zeros(17)] * 3)
    _, pol = _policy("gauss", 3)
    ls = torch.full((eng.act_dim,), -2.3, device="cuda")
    cl = np.arange(E) % 3
    cl[-1] = 1
    r = eng.eval_run(cl, pol, ls, _zstats(3), 5.0, True, 500, True, True)
    assert r["states"].nbytes > 2 ** 31
    i, k = E - 1, int(r["nframes"][-1])
    assert k > 400, k
    st = torch.tensor(r["states"][i, k - 40:k], device="cuda")
    pose, trans = eng.qpos_to_smpl(st)
    assert np.array_equal(r["pose_aa"][i, k - 40:k], pose.cpu().numpy()) and np.array_equal(r["trans"][i, k - 40:k], trans.cpu().numpy())
    assert np.isfinite(r["pose_aa"][i, :k]).all()
    eng.close()


# ---- 3. whole datasets in chunks
def test_export_motion_chunking_is_invisible():
    from uhc_b200.agent import BatchedAgent
    from tests.test_gpu_eval_groups import _clips
    clips = _clips(9, 6, 20, 90)
    # the test-mode cfg of an evaluation: with auto_reset an ended env would re-seed itself from the sampler, whose draws depend on the env
    ag = BatchedAgent(8, clips, [np.zeros(17)] * 9, policy_hsize=(128, 64), value_hsize=(64,), seed=2, body_diff_thresh=0.2, auto_reset=False)
    order = [4, 0, 8, 8, 3, 1, 7, 2, 6, 5, 0, 4, 2]
    one = ag.export_motion(order[:8], True, window=16)
    small = ag.export_motion(order[:8], True, window=16, max_bytes=40 * 223 * 8 * 3)    # a few clips per call: several chunks
    big = ag.export_motion(order, True, window=16)                                      # 13 clips > E: two calls at least
    ev = ag.evaluate(order[:8], True, window=16, record_states=True, export_smpl=True)
    for a, b, c, d in zip(one, small, big, ev):
        for k in ("pred", "pred_jpos", "pose_aa", "trans", "frames"):
            assert np.array_equal(a[k], b[k]) and np.array_equal(a[k], c[k]), k
        assert np.array_equal(a["pred"], d["states"][:, :76]) and np.array_equal(a["pose_aa"], d["pose_aa"])
        assert (a["last_t"], a["fail_any"], a["reward_sum"]) == (b["last_t"], b["fail_any"], b["reward_sum"]) == (d["last_t"], d["fail_any"], d["reward_sum"])
    lens = ag.engine.clip_len[np.asarray(order)]
    assert [len(x["pred"]) for x in big] == [len(x["frames"]) for x in big] and all(len(x["pred"]) <= L - 1 for x, L in zip(big, lens))
    ag.engine.close()


# ---- 4. the tracker
@pytest.mark.parametrize("precision", [32, 64])
def test_tracker_smpl(precision):
    import torch
    from tests.test_gpu_track import TRACK_KW, Run, _clips as _tclips
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    from uhc_b200.model import HumanoidModel
    rng = np.random.default_rng(8)
    E = 6
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    fk = np.array([0, 1, 1, 0, 1, 0], np.int32)
    ms = ML.MotionSet(_tclips(rng, [20] * E, "qpos"))
    eng = Engine(E, model=variants[0], precision=precision, variants=variants, **TRACK_KW)
    eng.load_motions(ms, fk_models=fk)
    run = Run(eng)
    eng.track_begin(6, "qpos", fk_models=fk)
    raw = [ms.rows[20 * c:20 * c + 20] for c in range(E)]
    eng.track_reset(np.arange(E), torch.tensor(np.stack([r[:2] for r in raw]), device="cuda"))
    run.step()
    for k in range(2, 8):
        run.step(torch.tensor(np.stack([r[k] for r in raw]), device="cuda"))
        pose, trans = eng.track_smpl(run.state)
        p2, t2 = eng.qpos_to_smpl(run.state, variants=fk)
        assert torch.equal(pose, p2) and torch.equal(trans, t2)
    eng.close()


def test_tracker_smpl_method():
    """Tracker.smpl() of an agent's tracker against uhc_qpos_to_smpl of its state"""
    import torch
    from tests.test_gpu_track import TRACK_KW
    from uhc_b200 import motion_lib as ML
    from uhc_b200.agent import BatchedAgent
    rng = np.random.default_rng(12)
    E = 16
    clips = [ML.synthetic_clip(30, rng) for _ in range(4)]
    agent = BatchedAgent(E, clips, policy_hsize=(64, 32), value_hsize=(64, 32), auto_reset=False, **TRACK_KW)
    trk = agent.tracker(window=8, kind="qpos", fail_safe=True)
    ref = torch.tensor(np.stack([clips[e % 4]["qpos"] for e in range(E)]), device="cuda")
    trk.reset(ref[:, 0], ref[:, 1])
    trk.step()
    for k in range(2, 6):
        trk.step(ref[:, k])
        pose, trans = trk.smpl()
        p2, t2 = agent.engine.qpos_to_smpl(trk.state)
        assert torch.equal(pose, p2) and torch.equal(trans, t2)
    trk.close()
    agent.engine.close()


# ---- 5. the drop-in layer (AgentCopycat)
TRAJ = ("gt", "pred", "gt_jpos", "pred_jpos", "pose_aa", "trans", "fail_safe")


def test_dropin_export_motion_equals_eval_seq(tmp_path, monkeypatch):
    import copy
    import joblib
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, test_clips=4)
    eng = agent.agent.engine
    freq0 = copy.deepcopy(agent.freq_dict)
    out = agent.export_motion(epoch=3, dump=True)
    assert agent.freq_dict == freq0, "export_motion fed outcomes to freq_dict"
    assert eng._cfg.auto_reset == 1, "the training cfg was not restored"
    for ld in agent.test_data_loaders:
        res = out[ld.name]
        dumped = joblib.load(os.path.join(cfg.output_dir, f"3_{ld.name}_motion.pkl"))
        assert sorted(dumped) == sorted(res) == sorted(ld.data_keys)
        for key in ld.data_keys:
            e = agent.eval_seq(key, ld)
            r = res[key]
            for k in ("pred", "gt", "pred_jpos", "gt_jpos"):
                assert np.array_equal(r[k], e[k]), (key, k)
                assert np.array_equal(dumped[key][k], e[k]), (key, k)
            assert r["percent"] == e["percent"] and r["fail_safe"] == e["fail_safe"]
            pose, trans = eng.qpos_to_smpl(r["pred"])
            assert np.array_equal(r["pose_aa"], pose.cpu().numpy()) and np.array_equal(r["trans"], trans.cpu().numpy())
    # the device curriculum: its rings stay as they were
    agent.curriculum_on_device = True
    agent._enable_device_curriculum()
    before = copy.deepcopy(agent.get_freq_dict())
    agent.export_motion(epoch=4, dump=False)
    assert agent.get_freq_dict() == before, "export_motion fed outcomes to the device curriculum"
    eng.close()


def test_eval_dump_motion_host_and_device_agree(tmp_path, monkeypatch):
    import joblib
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, test_clips=4)
    loaders = agent.test_data_loaders
    load = lambda ep: {ld.name: joblib.load(os.path.join(cfg.output_dir, f"{ep}_{ld.name}_coverage_full.pkl")) for ld in loaders}
    cfg.cfg_dict["eval_on_device"] = False
    agent.eval_policy(epoch=0, dump=True)                   # without the key: today's dump
    plain = load(0)
    cfg.cfg_dict["eval_dump_motion"] = True
    agent.eval_policy(epoch=1, dump=True)
    host = load(1)
    cfg.cfg_dict["eval_on_device"] = True
    agent.eval_policy(epoch=2, dump=True)
    dev = load(2)
    for ld in loaders:
        for key in ld.data_keys:
            assert not set(TRAJ) & set(plain[ld.name][key]), key
            assert set(host[ld.name][key]) == set(plain[ld.name][key]) | set(TRAJ) == set(dev[ld.name][key]), key
            h, d = host[ld.name][key], dev[ld.name][key]
            for k in TRAJ:
                assert np.array_equal(h[k], d[k]), (key, k)
            assert len(h["pred"]) == len(h["pose_aa"]) == len(h["trans"]) == len(h["gt"])
    agent.agent.engine.close()
