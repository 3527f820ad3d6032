"""GPU: the renderer (include/uhc_render.h) -- uhc_render_bodies against the host emulation bit for bit, the pose pass against the host FK,
uhc_render_qpos against uhc_render_bodies on its own pose table, output bounds and bad arguments, BatchedAgent.render_motion against
Engine.render, and the drop-in's mp4 files."""
import ctypes as C
import os

import numpy as np
import pytest

from tests import render_ref as RF
from tests.emu import render_emu
from tests.test_render_ref import poses

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def _qpos(n, seed=0):
    """n qpos rows: the standing / crouching / falling poses and golden frames, with seeded noise on every hinge and the root"""
    qa, qb = poses()
    base = np.concatenate([qa, qb, np.load(os.path.join(GOLDEN, "expert_kick.npz"))["qpos"]])
    rng = np.random.default_rng(seed)
    q = base[rng.integers(0, len(base), n)].copy()
    q[:, 7:] += rng.normal(0, 0.15, (n, 69))
    q[:, :2] += rng.normal(0, 0.3, (n, 2))
    return q


@pytest.fixture(scope="module")
def eng():
    from uhc_b200.engine import Engine
    from uhc_b200.model import HumanoidModel
    variants = [HumanoidModel(), HumanoidModel(scale=np.random.default_rng(11).uniform(0.9, 1.15, 24))]
    e = Engine(4, model=variants[0], variants=variants)
    yield e
    e.close()


def _pose_table(eng, n, seed, var=0):
    qa, qb = _qpos(n, seed), _qpos(n, seed + 100)
    P = np.zeros((n, 2, 24, 12), np.float32)
    P[:, 0], P[:, 1] = render_emu.pose(qa, eng.variants, var), render_emu.pose(qb, eng.variants, var)
    return P


CASES = [((1, 1), 1, 2, dict(fovy=2.0, lookat=(0.0, 0.0, 0.6), distance=3.0)),
         ((17, 9), 3, 1, dict()),
         ((17, 9), 300, 2, dict(focus=True, shift_expert=1.0)),
         ((641, 359), 3, 2, dict(focus=True, shift_expert=1.0, distance=3.5)),
         ((641, 359), 3, 1, dict(hide_im=False, azimuth=120.0, elevation=-20.0)),
         ((641, 359), 3, 2, dict(hide_expert=True, shift_expert=0.7)),
         ((1920, 1080), 1, 2, dict(shift_expert=1.0, distance=3.0))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_bodies_equal_emulation_bit_for_bit(eng, case):
    import torch
    size, n, hum, cam = CASES[case]
    var = case % 2
    P = _pose_table(eng, n, case, var)
    rgb, dep, lab = eng.render_bodies(torch.tensor(P, device="cuda"), hum, [var] * n, cam, size, depth=True, label=True)
    torch.cuda.synchronize()
    erg, edp, elb = render_emu.render_bodies(P, size, cam, hum, eng.variants, var)
    assert np.array_equal(rgb.cpu().numpy(), erg)
    assert np.array_equal(dep.cpu().numpy().view(np.uint32), edp.view(np.uint32))
    assert np.array_equal(lab.cpu().numpy(), elb)
    if size != (1, 1):
        assert (elb >= 2).any() and (elb == 1).any()


def test_pose_table_matches_host_fk(eng):
    """uhc_render_pose's fp32 table is the fp64 FK (motion_lib.qpos_fk) rounded once: equal, or one ulp apart where the fp64 value is within
    1e-12 of a rounding midpoint"""
    import torch
    q = _qpos(200, 7)
    var = np.arange(200) % 2
    got = eng.render_pose(torch.tensor(q, device="cuda"), variants=var).cpu().numpy()[:, 0]
    want = np.zeros((200, 24, 12))
    for v in (0, 1):
        want[var == v] = RF.pose_table(q[var == v], eng.variants[v])
    r = want.astype(np.float32)
    diff = got != r
    if diff.any():
        up = np.nextafter(r[diff], np.float32(np.inf)).astype(np.float64)
        dn = np.nextafter(r[diff], np.float32(-np.inf)).astype(np.float64)
        mid = np.minimum(np.abs(want[diff] - (r[diff] + up) / 2), np.abs(want[diff] - (r[diff] + dn) / 2))
        assert (mid <= 1e-12).all() and (np.abs(got[diff].astype(np.float64) - want[diff]) <= np.spacing(np.abs(r[diff]))).all()
    assert diff.mean() < 1e-3


@pytest.mark.parametrize("precision", [32, 64])
@pytest.mark.parametrize("pitch", [76, 148, 223])
def test_qpos_equals_bodies_on_its_pose_table(eng, precision, pitch):
    import torch
    dt = torch.float32 if precision == 32 else torch.float64
    n = 5
    rng = np.random.default_rng(pitch)
    wide = lambda q: np.concatenate([q, rng.normal(size=(n, pitch - 76))], 1)
    qa, qb = torch.tensor(wide(_qpos(n, 1)), dtype=dt, device="cuda"), torch.tensor(wide(_qpos(n, 2)), dtype=dt, device="cuda")
    var = np.array([1, 0, 1, 1, 0])
    for ghost, cam in ((None, dict()), (qb, dict(focus=True, shift_expert=1.0))):
        pose = eng.render_pose(qa, ghost, var)
        a = eng.render(qa, ghost, var, cam, (96, 54), depth=True, label=True)
        b = eng.render_bodies(pose, 1 if ghost is None else 2, var, cam, (96, 54), depth=True, label=True)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
        assert (a[2] >= 2).any()
        if ghost is not None:
            assert (a[2] >= 26).any()
    # rows read in place at the pitch: the same frames from a contiguous [n][76] copy
    a = eng.render(qa, qb, var, dict(), (96, 54))[0]
    b = eng.render(qa[:, :76].contiguous(), qb[:, :76].contiguous(), var, dict(), (96, 54))[0]
    assert torch.equal(a, b)


def test_outputs_stay_in_bounds(eng):
    """canary bytes around every output buffer stay untouched"""
    import torch
    W, H, n, G = 33, 17, 4, 4096
    P = torch.tensor(_pose_table(eng, n, 3), device="cuda")
    npx = n * H * W
    rgb = torch.full((npx * 3 + 2 * G,), 0xA5, dtype=torch.uint8, device="cuda")
    lab = torch.full((npx + 2 * G,), 0x5A, dtype=torch.uint8, device="cuda")
    dep = torch.full((npx + 2 * G,), -7.0, dtype=torch.float32, device="cuda")
    from uhc_b200.engine import make_camera
    cam = C.byref(make_camera(dict(shift_expert=1.0)))
    eng._render_init()
    rc = eng.lib.uhc_render_bodies(eng.h, cam, C.c_int(W), C.c_int(H), C.c_long(n), C.c_void_p(P.data_ptr()), C.c_int(2), None,
                                   C.c_void_p(rgb.data_ptr() + G), C.c_void_p(dep.data_ptr() + 4 * G), C.c_void_p(lab.data_ptr() + G), eng._stream())
    assert rc == 0
    torch.cuda.synchronize()
    for buf, fill, m in ((rgb, 0xA5, npx * 3), (lab, 0x5A, npx), (dep, -7.0, npx)):
        assert (buf[:G] == fill).all() and (buf[G + m:] == fill).all()
        assert not (buf[G:G + m] == fill).all()


def test_bad_arguments_return_minus_two_without_launching(eng):
    import torch
    from uhc_b200.engine import make_camera
    lib = eng.lib
    eng._render_init()
    P = torch.tensor(_pose_table(eng, 2, 4), device="cuda")
    q = torch.tensor(_qpos(2, 4), device="cuda")
    rgb = torch.full((2 * 8 * 8 * 3,), 7, dtype=torch.uint8, device="cuda")
    good = make_camera()
    p = lambda x: C.c_void_p(x.data_ptr())

    def bodies(cam=good, W=8, H=8, n=2, pose=P, hum=2, var=None, out=rgb):
        return lib.uhc_render_bodies(eng.h, C.byref(cam) if cam is not None else None, C.c_int(W), C.c_int(H), C.c_long(n),
                                     p(pose) if pose is not None else None, C.c_int(hum), var, p(out) if out is not None else None, None, None, eng._stream())

    def qpos(precision=64, pitch=76, n=2, ghost=None, gpitch=76):
        return lib.uhc_render_qpos(eng.h, C.byref(good), C.c_int(8), C.c_int(8), C.c_long(n), p(q), C.c_int(precision), C.c_long(pitch),
                                   ghost, C.c_long(gpitch), None, p(rgb), None, None, eng._stream())

    bad_cams = []
    for k, v in (("distance", 0.0), ("fovy", 180.0), ("fovy", 0.0), ("azimuth", float("nan")), ("shift_expert", float("inf"))):
        c = make_camera()
        setattr(c, k, v)
        bad_cams.append(c)
    rcs = [bodies(cam=None), bodies(W=0), bodies(H=16385), bodies(n=-1), bodies(hum=3), bodies(hum=0), bodies(pose=None), bodies(out=None)]
    rcs += [bodies(cam=c) for c in bad_cams]
    rcs += [qpos(precision=16), qpos(pitch=75), qpos(n=-1), qpos(ghost=p(q), gpitch=10)]
    var = torch.tensor([0, 2], dtype=torch.int32, device="cuda")
    rcs.append(bodies(var=p(var)))
    rcs.append(lib.uhc_render_pose(eng.h, C.c_long(2), p(q), C.c_int(64), C.c_long(76), None, C.c_long(76), p(var), p(P), eng._stream()))
    assert rcs == [-2] * len(rcs)
    torch.cuda.synchronize()
    assert (rgb == 7).all(), "a rejected call wrote its output"
    # uhc_render_init: a table that does not fit the engine's variants
    from uhc_b200.model import HumanoidModel
    h = HumanoidModel().render_struct(None)
    assert lib.uhc_render_init(eng.h, C.byref(h)) == -2                # one variant, the engine has two
    # without uhc_render_init: rejected
    from uhc_b200.engine import Engine
    e2 = Engine(2)
    assert e2.lib.uhc_render_bodies(e2.h, C.byref(good), 8, 8, C.c_long(2), p(P), 2, None, p(rgb), None, None, e2._stream()) == -2
    e2.close()
    assert (rgb == 7).all()
    assert bodies() == 0


def _agent_clips():
    from uhc_b200 import motion_lib as ML
    rng = np.random.default_rng(21)
    return [ML.synthetic_clip(int(T), rng) for T in (30, 45, 24, 60, 33)]


def test_render_motion_equals_engine_render_and_ignores_chunking():
    import torch
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.model import HumanoidModel
    rng = np.random.default_rng(3)
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    clips = _agent_clips()
    ag = BatchedAgent(4, clips, [np.zeros(17)] * len(clips), policy_hsize=(128, 64), value_hsize=(64,), seed=2, body_diff_thresh=0.2,
                      auto_reset=False, model=variants[0], variants=variants, clip_models=[0, 1, 1, 0, 1])
    order = [3, 0, 4, 1, 2]
    size, cam = (80, 45), dict(focus=True, shift_expert=1.0)
    a = ag.render_motion(order, True, size, cam)
    got = {}
    b = ag.render_motion(order, True, size, cam, max_bytes=3 * 80 * 45 * 3, writer=lambda i, ch: got.__setitem__(i, [c for c in ch]))
    mot = ag.export_motion(order, True)
    for i, (c, x, y, m) in enumerate(zip(order, a, b, mot)):
        nf = len(m["pred"])
        assert np.array_equal(x["pred"], m["pred"]) and x["frames"].shape == (nf, 45, 80, 3)
        assert all(len(ch) <= 3 for ch in got[i]) and np.array_equal(np.concatenate(got[i]), x["frames"])
        gt = ag.engine.clip_frames(c)["qpos"][np.minimum(np.arange(1, nf + 1), ag.engine.clip_len[c] - 1)]
        assert np.array_equal(x["gt"], gt) and np.array_equal(y["gt"], gt)
        want = ag.engine.render(m["pred"], gt, [int(ag.engine.clip_models[c])] * nf, cam, size)[0].cpu().numpy()
        assert np.array_equal(x["frames"], want)
    assert set(ag.render_times) == {"evaluation", "rendering", "copy", "writer"}
    ag.engine.close()


def test_dropin_writes_one_mp4_per_clip(tmp_path, monkeypatch):
    import copy
    import cv2
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, test_clips=4)
    eng = agent.agent.engine
    freq0 = copy.deepcopy(agent.freq_dict)
    # the loaders' clips share their keys here, and a video is named by key as the visualizer names it: one directory per loader
    out = {ld.name: agent.render_motion(epoch=7, loaders=[ld], out_dir=str(tmp_path / ld.name), size=(96, 54))[ld.name] for ld in agent.test_data_loaders}
    assert agent.freq_dict == freq0, "render_motion fed outcomes to freq_dict"
    assert eng._cfg.auto_reset == 1, "the training cfg was not restored"
    ev = agent.export_motion(epoch=0, dump=False)
    for ld in agent.test_data_loaders:
        assert sorted(out[ld.name]) == sorted(ld.data_keys)
        for key, path in out[ld.name].items():
            assert os.path.basename(path) == f"{key}_{cfg.id}_7_0.mp4"
            cap = cv2.VideoCapture(path)
            k = 0
            while True:
                ok, fr = cap.read()
                if not ok:
                    break
                assert fr.shape == (54, 96, 3)
                k += 1
            cap.release()
            assert k == len(ev[ld.name][key]["pred"])
            if ev[ld.name][key]["percent"] >= 1:                   # ran to the clip's end (fail_safe re-seats a fall): len - 1 frames
                assert k == ld.get_sample_len_from_key(key) - 1
    eng.close()
