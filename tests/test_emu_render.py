"""CPU: the renderer's pose pass and pixel path (uhc_b200/csrc/render_core.h), compiled into the host emulation, against the independent
fp64 ray caster of tests/render_ref.py and against the reference's FK (tests/golden/expert_*.npz)."""
import os

import numpy as np
import pytest

from tests import render_ref as RF
from tests.emu import render_emu
from tests.test_render_ref import poses
from uhc_b200.model import HumanoidModel

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


@pytest.mark.parametrize("clip", ["expert_sway", "expert_kick"])
def test_pose_pass_fk_matches_reference_golden(clip):
    z = np.load(os.path.join(GOLDEN, clip + ".npz"))
    T = len(z["qpos"])
    pose, wpos, wq = render_emu.pose(z["qpos"], fk=True)
    assert np.abs(wpos.reshape(T, 72) - z["wbpos"]).max() <= 1e-12
    gq = z["wbquat"].reshape(T, 24, 4)
    sign = np.where((wq * gq).sum(-1, keepdims=True) < 0, -1.0, 1.0)
    assert np.abs(wq * sign - gq).max() <= 1e-12
    # the fp32 rows are the fp64 rotation / position rounded once
    want = RF.pose_table(z["qpos"], HumanoidModel())
    assert np.abs(pose - want).max() <= 2 ** -23 * 2


def test_pose_pass_reads_rows_at_any_pitch_and_variant():
    qa, _ = poses()
    m1 = HumanoidModel(scale=np.random.default_rng(5).uniform(0.85, 1.2, 24))
    models = [HumanoidModel(), m1]
    wide = np.concatenate([qa, np.random.default_rng(0).normal(size=(len(qa), 223 - 76))], 1)
    a = render_emu.pose(qa, models, 1)
    assert np.array_equal(a, render_emu.pose(wide, models, 1))
    assert np.abs(a - RF.pose_table(qa, m1)).max() <= 2 ** -23 * 4
    assert not np.array_equal(a, render_emu.pose(qa, models, 0))


def compare(P, model, size, cam, humanoids, variants=None, variant=None):
    rgb, depth, label = render_emu.render_bodies(P, size, cam, humanoids, variants, variant)
    ref = RF.render(P.astype(np.float64), model, size, cam, humanoids)
    amb = ref["amb"]
    ok = ~amb
    assert amb.mean() < 1e-3 or amb.sum() <= 1, amb.mean()
    assert np.array_equal(label[ok], ref["label"][ok])
    fin = np.isfinite(ref["depth"]) & ok
    assert np.array_equal(np.isinf(depth[ok]), np.isinf(ref["depth"][ok]))
    # depth within 1e-5 relative, or, on a face seen nearly edge-on, within 1e-6 m over |cos| of the incidence angle (the conditioning of the
    # intersection: an error e in the ray's offset from the face moves the hit by e / |cos| along the ray)
    err = np.abs(depth[fin] - ref["depth"][fin])
    assert ((err <= 1e-5 * ref["depth"][fin]) | (err <= 1e-6 / ref["cos"][fin])).all()
    assert np.abs(rgb[ok].astype(int) - ref["rgb"][ok]).max(initial=0) <= 1
    return label


@pytest.mark.parametrize("size", [(1, 1), (17, 9), (320, 180)])
@pytest.mark.parametrize("ghost", [False, True])
@pytest.mark.parametrize("var", [0, 1])
def test_emulation_against_fp64_reference(size, ghost, var):
    qa, qb = poses()
    models = [HumanoidModel(), HumanoidModel(scale=np.random.default_rng(11).uniform(0.9, 1.15, 24))]
    P = np.zeros((len(qa), 2, 24, 12), np.float32)
    P[:, 0], P[:, 1] = render_emu.pose(qa, models, var), render_emu.pose(qb, models, var)
    cam = dict(distance=3.5, shift_expert=0.8 if ghost else 0.0)
    if size == (1, 1):
        cam.update(fovy=2.0, lookat=(0.0, 0.0, 0.6))                # one pixel aimed at the humanoid
    label = compare(P, models[var], size, cam, 2 if ghost else 1, models, var)
    if size != (1, 1):
        assert (label >= 2).any() and (label == 1).any() and ((label >= 26).any() == ghost)


def test_camera_options():
    """focus follows the root; hide_im / hide_expert drop a humanoid from the image and from the shadows"""
    qa, qb = poses()
    P = np.zeros((len(qa), 2, 24, 12), np.float32)
    P[:, 0], P[:, 1] = render_emu.pose(qa), render_emu.pose(qb)
    P[:, :, :, 9] += 3.0                                         # both humanoids 3 m away in x
    m = HumanoidModel()
    lab = compare(P, m, (64, 36), dict(focus=True, shift_expert=1.0), 2)
    assert (lab >= 2).any()
    lab = compare(P, m, (64, 36), dict(focus=True, hide_im=True), 2)
    assert not ((lab >= 2) & (lab < 26)).any() and (lab >= 26).any()
    lab = compare(P, m, (64, 36), dict(focus=True, hide_expert=True), 2)
    assert (lab >= 2).any() and not (lab >= 26).any()
