"""CPU: the device motion library's per-frame code (uhc_b200/csrc/motion_core.h), compiled into the host emulation, against the
host motion library (uhc_b200/motion_lib.py) and against the reference's expert goldens (tests/golden/expert_*.npz)."""
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation as sRot

from tests.emu import motion_emu as emu
from uhc_b200 import motion_lib as ML
from uhc_b200.engine import pack_expert
from uhc_b200.model import HumanoidModel

TOL = 1e-12
pytestmark = pytest.mark.filterwarnings("ignore:Gimbal lock")


def host_table(clips, models=None, fk_models=None):
    """pack_expert(make_expert | qpos_fk) per clip, concatenated: the table uhc_load_clips receives today"""
    models = models or [HumanoidModel()]
    out = []
    for c, clip in enumerate(clips):
        m = models[0 if fk_models is None else fk_models[c]]
        ex = ML.qpos_fk(clip["qpos"], m) if "qpos" in clip and "pose_aa" not in clip else ML.make_expert(clip["pose_aa"], clip["trans"], m)
        out.append(pack_expert(ex))
    return np.concatenate(out)


def check(clips, models=None, fk_models=None):
    ms = ML.MotionSet(clips)
    got = emu.motion_table(ms, models, fk_models)
    want = host_table(clips, models, fk_models)
    assert got.shape == want.shape == (ms.num_frames, 576)
    d = np.abs(got - want)
    assert d.max() <= TOL, "column %d differs by %g" % (np.argmax(d.max(0)), d.max())
    return got


def golden(tag):
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"expert_{tag}.npz"))
    return {k: z[k] for k in z.files}


def smpl_clip(T, rng, scale=0.6):
    return {"pose_aa": rng.normal(0, scale, (T, 72)), "trans": rng.normal(0, 0.5, (T, 3)) + [0, 0, 0.9]}


@pytest.mark.parametrize("tag", ["sway", "kick"])
def test_goldens_smpl_and_qpos_input(tag):
    z = golden(tag)
    check([{"pose_aa": z["pose_aa"], "trans": z["trans"]}])
    check([{"qpos": z["qpos"]}])
    pose_h = np.concatenate([z["pose_aa"][:, :66], np.random.default_rng(1).normal(0, 0.3, (len(z["pose_aa"]), 90))], 1)   # SMPL-H: 156 wide
    check([{"pose_aa": pose_h, "trans": z["trans"]}])


@pytest.mark.parametrize("tag", ["sway", "kick"])
def test_goldens_against_reference(tag):
    """the emulated table against the reference's own expert table, with the tolerances of tests/test_motion_lib.py"""
    z = golden(tag)
    pose = z["pose_aa"].copy()
    pose[:, 66:] = 0
    t = emu.motion_table(ML.MotionSet([{"pose_aa": pose, "trans": z["trans"]}]))
    assert np.abs(t[:, :3] - z["qpos"][:, :3]).max() < 1e-12
    assert np.abs(t[:, 7:76] - z["qpos"][:, 7:]).max() < 3e-6
    d = np.minimum(np.abs(t[:, 3:7] - z["qpos"][:, 3:7]).max(1), np.abs(t[:, 3:7] + z["qpos"][:, 3:7]).max(1))
    assert d.max() < 1e-6
    t = emu.motion_table(ML.MotionSet([{"qpos": z["qpos"]}]))
    cols = {"qvel": (76, 151), "wbpos": (151, 223), "wbquat": (223, 319), "bquat": (319, 415), "bangvel": (415, 487), "ee_wpos": (487, 502),
            "body_com": (502, 574), "com": (502, 505)}
    for k, tol in (("qvel", 1e-8), ("wbpos", 1e-10), ("wbquat", 1e-10), ("bquat", 1e-10), ("body_com", 1e-10), ("bangvel", 1e-7),
                   ("ee_wpos", 1e-10), ("com", 1e-10)):
        a, b = cols[k]
        assert np.abs(t[:, a:b] - z[k].reshape(len(t), -1)).max() < tol, k


def test_seeded_synthetic_clips():
    rng = np.random.default_rng(7)
    check([{"qpos": ML.synthetic_clip(T, rng, kind=k)["qpos"]} for T, k in ((120, "normal"), (2, "normal"), (75, "sitting"), (33, "airborne"))])
    check([smpl_clip(T, rng) for T in (90, 2, 41)])
    check([smpl_clip(64, rng, scale=1.5)])          # large rotations: every branch of the Euler extraction


def adversarial_clip(T=12):
    """frames that take every special branch of the conversion: gimbal lock, tiny and half-turn rotation vectors, the series threshold
    of from_rotvec, a hinge angle wrapping across +-pi between frames, root quaternions with w < 0"""
    rng = np.random.default_rng(3)
    pose = rng.normal(0, 0.3, (T, 24, 3))
    for t in range(T):   # joint 1 (L_Hip): pitch within 1e-9 of +-pi/2, alternating sign and side
        s = 1 if t % 2 else -1
        pose[t, 1] = sRot.from_euler("ZYX", [0.3 + 0.05 * t, s * (np.pi / 2 - (1e-9 if t % 3 else -1e-9)), -0.2]).as_rotvec()
    pose[:, 2] = [[0, 0, 0], [1e-13, 0, 0], [0, -2e-9, 1e-9], [0.999e-3, 0, 0], [1.001e-3, 0, 0], [0, 1e-3, 0]] * (T // 6)   # ~0 and the 1e-3 threshold
    ax = np.array([0.48, -0.6, 0.64])
    for t, ang in enumerate(np.linspace(np.pi - 3e-9, np.pi + 3e-9, T)):   # joint 3 (Torso): rotation angle ~pi
        pose[t, 3] = ax * ang
    th = np.pi + np.array([-0.02, -0.01, 0.01, 0.02] * (T // 4))           # joint 4 (L_Knee): the z hinge crosses +-pi between frames
    pose[:, 4] = np.stack([np.zeros(T), np.zeros(T), th], 1)
    root_ang = np.linspace(np.pi - 0.2, np.pi + 0.4, T)                      # root: rotation angle beyond pi -> w < 0 before the sign flip
    pose[:, 0] = np.array([0.2, 0.9, -0.3]) / np.linalg.norm([0.2, 0.9, -0.3]) * root_ang[:, None]
    return {"pose_aa": pose.reshape(T, 72), "trans": rng.normal(0, 0.3, (T, 3))}


def test_adversarial_frames():
    clip = adversarial_clip()
    t = check([clip])
    eul = sRot.from_rotvec(clip["pose_aa"][:, 3:6]).as_euler("ZYX")
    assert np.abs(np.abs(eul[:, 1]) - np.pi / 2).max() < 1e-8 and (eul[:, 2] == 0).any()   # the gimbal branch was taken
    assert (sRot.from_rotvec(clip["pose_aa"][:, :3]).as_quat()[:, 3] < 0).any()             # root quaternions with w < 0
    assert (np.abs(t[:, 76:151]) == 10.0).any()                                            # the qvel clip at +-10
    pose_h = np.concatenate([clip["pose_aa"][:, :66], np.ones((len(clip["pose_aa"]), 90))], 1)
    check([{"pose_aa": pose_h, "trans": clip["trans"]}])                                  # SMPL-H: hands read as zero


def test_shape_variants_per_clip():
    rng = np.random.default_rng(11)
    base = HumanoidModel()
    models = [base, HumanoidModel(scale=rng.uniform(0.85, 1.15, 24)), HumanoidModel(scale=rng.uniform(0.9, 1.2, 24))]
    clips = [smpl_clip(30, rng) for _ in range(4)]
    check(clips, models, [2, 0, 1, 2])
    check([{"qpos": ML.synthetic_clip(25, rng)["qpos"]} for _ in range(3)], models, [1, 2, 0])


def test_motion_set_layout():
    rng = np.random.default_rng(5)
    a, b = smpl_clip(5, rng), {"pose_aa": rng.normal(0, 0.3, (4, 156)), "trans": rng.normal(0, 0.3, (4, 3))}
    ms = ML.MotionSet([a, b])
    assert (ms.kind, ms.pose_dim, list(ms.lens), ms.rows.shape) == (ML.MotionSet.SMPL, 72, [5, 4], (9, 75))
    assert (ms.rows[5:, 66:72] == 0).all() and (ms.rows[5:, 72:] == b["trans"]).all()    # mixed widths: SMPL-H hands zeroed
    check([a, b])
    ms = ML.MotionSet([{"qpos": np.zeros((3, 76))}])
    assert (ms.kind, ms.pose_dim, ms.rows.shape) == (ML.MotionSet.QPOS, 76, (3, 76))
