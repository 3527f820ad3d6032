"""CPU: the device SMPL export's per-frame code (uhc_b200/csrc/smpl_export_core.h), compiled into the host emulation, against the reference's
qpos_to_smpl (tests/golden/qpos_to_smpl.npz, tools/make_golden.py gen_qpos_to_smpl) and against the SMPL -> qpos conversion of the device motion
library (motion_core.h) that it inverts."""
import os

import numpy as np
import pytest
from scipy.spatial.transform import Rotation as sRot

from tests.emu import export_emu, motion_emu
from uhc_b200 import motion_lib as ML
from uhc_b200.model import HumanoidModel

pytestmark = pytest.mark.filterwarnings("ignore:Gimbal lock")


def golden():
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "qpos_to_smpl.npz"))
    return {k: z[k] for k in z.files}


def test_golden_root_offset_is_the_base_models():
    assert np.array_equal(golden()["root_offset"], HumanoidModel().body_f[0, :3])


def test_against_reference_golden():
    z = golden()
    pose, trans = export_emu.qpos_to_smpl(z["qpos"])
    assert np.abs(pose - z["pose"]).max() <= 1e-12
    assert np.abs(trans - z["trans"]).max() <= 1e-12


def test_golden_covers_the_branches():
    q = golden()["qpos"]
    assert (q[:, 3] < 0).any() and (np.abs(q[:, 3]) < 1e-8).any()                           # w < 0 and w ~ 0 (angle ~ pi)
    ang = 2 * np.arctan2(np.linalg.norm(q[:, 4:7], axis=1), np.abs(q[:, 3]))
    assert (ang < 1e-3).sum() >= 8                                                          # as_rotvec's small-angle series
    pitch = q[:, 8::3]
    assert (pitch == np.pi / 2).any() and (pitch == -np.pi / 2).any()
    near = np.abs(np.abs(pitch) - np.pi / 2)
    assert ((near > 0) & (near <= 1e-9)).any()


def test_pitch_and_stride():
    """rows read at a pitch wider than 76 (the evaluation's state record, the tracker's state rows) give the same result"""
    q = golden()["qpos"]
    wide = np.concatenate([q, np.random.default_rng(0).normal(size=(len(q), 223 - 76))], 1)
    a, b = export_emu.qpos_to_smpl(q), export_emu.qpos_to_smpl(wide)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


@pytest.mark.parametrize("scale", [1.0, 1.5])
def test_smpl_qpos_smpl_round_trip_every_variant(scale):
    """SMPL -> qpos (motion_core.h) -> SMPL (smpl_export_core.h) with the clip's own shape variant: the same rotations (as matrices) and trans"""
    rng = np.random.default_rng(13)
    models = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.85, 1.15, 24)), HumanoidModel(scale=rng.uniform(0.9, 1.2, 24))]
    T = 40
    clips = [{"pose_aa": rng.normal(0, 0.6 * scale, (T, 72)), "trans": rng.normal(0, 0.5, (T, 3)) + [0, 0, 0.9]} for _ in models]
    table = motion_emu.motion_table(ML.MotionSet(clips), models, list(range(len(models))))
    qpos = table[:, :76]
    variant = np.repeat(np.arange(len(models)), T)
    pose, trans = export_emu.qpos_to_smpl(qpos, models, variant)
    want = np.concatenate([c["pose_aa"] for c in clips]).reshape(-1, 3)
    d = np.abs(sRot.from_rotvec(pose.reshape(-1, 3)).as_matrix() - sRot.from_rotvec(want).as_matrix()).max()
    assert d <= 1e-12, d
    # trans: (trans + root offset) - root offset, as the reference subtracts body_pos[1]; the two roundings leave at most one ulp of the sum
    t0 = np.concatenate([c["trans"] for c in clips])
    off = np.stack([m.body_f[0, :3] for m in models])[variant]
    assert np.array_equal(trans, qpos[:, :3] - off)
    assert (np.abs(trans - t0) <= np.spacing(np.abs(t0) + np.abs(off))).all()
