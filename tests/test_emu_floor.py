"""CPU: the floor measurements' per-frame code (uhc_b200/csrc/floor_core.h), compiled into the host emulation, against the numpy
restatement (tests/floor_ref.py); the audit and height-fix rules of MotionSet on clips built to trip each of them; the config refusal."""
import os

import numpy as np
import pytest

from tests import floor_ref as FR
from tests.emu import floor_emu as emu
from uhc_b200 import motion_lib as ML
from uhc_b200.model import HumanoidModel

pytestmark = pytest.mark.filterwarnings("ignore:Gimbal lock")
RTOL, ATOL = 1e-9, 1e-9      # relative, and mm absolute


def check(qpos, model=None, variants=None, variant=None):
    got = emu.floor_qpos(qpos, variants, variant)
    want = FR.floor_rows(qpos, model)
    d = np.abs(got - want)
    assert (d <= ATOL + RTOL * np.abs(want)).all(), "column %d differs by %g" % (np.argmax(d.max(0)), d.max())
    assert np.array_equal(got[:, 4], want[:, 4])
    return got


def golden(tag):
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", f"expert_{tag}.npz"))
    return z["qpos"]


def random_qpos(T, rng, z=0.9):
    q = np.zeros((T, 76))
    q[:, :3] = rng.normal(0, 0.3, (T, 3)) + [0, 0, z]
    q[:, 3:7] = rng.normal(size=(T, 4))
    q[:, 3:7] /= np.linalg.norm(q[:, 3:7], axis=1, keepdims=True)
    q[:, 7:] = rng.normal(0, 0.5, (T, 69))
    return q


@pytest.mark.parametrize("tag", ["sway", "kick"])
def test_golden_clips(tag):
    q = golden(tag)
    check(q)
    low = q.copy()
    low[:, 2] -= 0.08                      # feet in the floor: penetration and skate are exercised
    r = check(low)
    assert (r[:, 1] > 0).all() and (r[1:, 2] > 0).any()


def test_seeded_random_poses_in_every_shape_variant():
    rng = np.random.default_rng(5)
    models = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.85, 1.15, 24)), HumanoidModel(scale=rng.uniform(0.9, 1.2, 24))]
    for v, m in enumerate(models):
        q = random_qpos(40, rng, z=0.5)
        check(q, m, models, v)
    q = random_qpos(12, rng, z=0.4)         # a variant per row, the previous frame read with the row's variant
    got = emu.floor_qpos(q, models, np.arange(12) % 3)
    for i in range(1, 12):
        assert np.allclose(got[i], FR.floor_rows(q[i - 1:i + 1], models[i % 3])[1], rtol=RTOL, atol=ATOL)


def test_adversarial_frames():
    rng = np.random.default_rng(9)
    q = random_qpos(6, rng)
    q[:2, 2] = 3.0                          # no vertex below
    q[2:4, 2] = -3.0                        # every vertex below
    q[4:, 3:7] = [0.0, 1.0, 0.0, 0.0]       # root upside down
    q[4:, 2] = 0.3
    r = check(q)
    n = len(HumanoidModel().hull)
    assert (r[:2, 4] == 0).all() and (r[:2, 1] == 0).all() and (r[:2, 3] > 0).all() and (r[2:4, 4] == n).all() and r[3, 2] > 0
    first = emu.floor_qpos(q, first=[1, 0, 1, 0, 0, 1])
    assert (first[[0, 2, 5], 2] == 0).all() and np.array_equal(first[[1, 3, 4]], r[[1, 3, 4]])
    wide = np.concatenate([q, rng.normal(size=(6, 72))], 1)          # pitch 148: only the first 76 columns are read
    assert np.array_equal(emu.floor_qpos(wide), r)


def test_motion_rows_of_both_kinds_equal_the_qpos_path():
    rng = np.random.default_rng(3)
    models = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    clips = [{"pose_aa": rng.normal(0, 0.4, (T, 72)), "trans": rng.normal(0, 0.2, (T, 3)) + [0, 0, 0.85]} for T in (9, 1, 14)]
    ms, fk = ML.MotionSet(clips), [1, 0, 1]
    rows, feet = emu.EmuFloor(models).motion_floor(ms, fk)
    o = 0
    for c, v in zip(clips, fk):
        q = ML.smpl_to_qpos(c["pose_aa"], c["trans"], models[v])
        T = len(q)
        assert np.allclose(rows[o:o + T], emu.floor_qpos(q, models, v), rtol=1e-9, atol=1e-9)
        if T > 1:
            assert np.allclose(feet[o:o + T], ML.qpos_fk(q, models[v])["wbpos"].reshape(T, 24, 3)[:, [3, 7, 4, 8], 2], atol=1e-12)
        o += T
    qs = ML.MotionSet([{"qpos": ML.smpl_to_qpos(c["pose_aa"], c["trans"], models[0])} for c in clips])
    assert np.array_equal(emu.EmuFloor(models).motion_floor(qs)[0], np.concatenate([emu.floor_qpos(r) for r in np.split(qs.rows, np.cumsum(qs.lens)[:-1])]))


def standing_clip(T, lift):
    """the rest pose, upright, for T frames, its lowest hull vertex at lift[t] above the floor"""
    q = np.repeat(HumanoidModel().qpos0[None], T, 0)
    q[:, 3:7] = [0.7071067811865476, 0.7071067811865476, 0.0, 0.0]
    q[:, 2] += np.asarray(lift) - FR.hull_vertices(q[:1])[0, :, 2].min()
    return q


def hop(n, T=60):
    lift = np.zeros(T)
    lift[10:10 + n] = 0.5
    return standing_clip(T, lift)


def test_audit_rules_trip_where_the_reference_drops():
    eng = emu.EmuFloor()
    toe_z = float(ML.qpos_fk(standing_clip(2, np.zeros(2)))["wbpos"].reshape(2, 24, 3)[0, 4, 2])     # toe joint height of the standing pose
    deep = standing_clip(20, np.zeros(20))
    deep[5:, 2] -= toe_z + 0.16                                                           # toes at -0.16 from frame 5
    shallow = standing_clip(20, np.zeros(20))
    shallow[5:, 2] -= toe_z + 0.14
    clips = [hop(31), hop(30), standing_clip(10, np.full(10, 0.11)), standing_clip(10, np.full(10, 0.09)), deep, shallow]
    ms = ML.MotionSet([{"qpos": q} for q in clips])
    a = ms.floor_audit(eng)
    assert list(a["airborne_run"][:2]) == [31, 30]
    assert list(a["start_high"]) == [False, False, True, False, False, False]
    assert np.isclose(a["deepest_toe"][4], -0.16, atol=1e-9) and np.isclose(a["deepest_toe"][5], -0.14, atol=1e-9)
    assert list(a["implausible"]) == [True, False, True, False, True, False]
    assert np.allclose(a["dz_first"], [0, 0, 0.11, 0.09, 0, 0], atol=1e-12) and np.isclose(a["dz_clip"][4], -(toe_z + 0.16), atol=1e-9)
    assert not a["crawling"].any()
    kept = ms.drop(a["implausible"])
    assert list(kept.lens) == [60, 10, 20] and np.array_equal(kept.rows[:60], clips[1]) and np.array_equal(kept.rows[70:], clips[5])


def test_fix_height_puts_the_first_frame_on_the_floor():
    rng = np.random.default_rng(2)
    eng = emu.EmuFloor()
    clips = [{"pose_aa": rng.normal(0, 0.3, (T, 72)), "trans": rng.normal(0, 0.2, (T, 3)) + [0, 0, 1.1]} for T in (8, 5)]
    for ms in (ML.MotionSet(clips), ML.MotionSet([{"qpos": ML.smpl_to_qpos(c["pose_aa"], c["trans"])} for c in clips])):
        a = ms.floor_audit(eng)
        assert (np.abs(a["dz_first"]) > 0.05).all()
        off = ms.fix_height(a, "off")
        assert np.array_equal(off.rows, ms.rows) and np.array_equal(off.lens, ms.lens) and off.rows is not ms.rows
        fixed = ms.fix_height(a, "first_frame")
        assert np.abs(fixed.floor_audit(eng)["dz_first"]).max() < 1e-12
        zc = 2 if ms.kind == ms.QPOS else ms.pose_dim + 2
        other = np.delete(np.arange(ms.rows.shape[1]), zc)
        assert np.array_equal(fixed.rows[:, other], ms.rows[:, other])
        assert np.abs(ms.fix_height(a, "clip_min").floor_audit(eng)["dz_clip"]).max() < 1e-12
        assert np.allclose(ms.fix_height(a, "first_frame", offset=0.015).floor_audit(eng)["dz_first"], 0.015, atol=1e-12)
    with pytest.raises(ValueError, match="mode"):
        ms.fix_height(a, "lowest")


def test_crawling_clips_keep_their_height():
    q = standing_clip(6, np.zeros(6))
    q[:, 3:7] = [1.0, 0.0, 0.0, 0.0]                                       # the model's own frame: lying down
    q[:, 2] = 0.25
    ms = ML.MotionSet([{"qpos": q}])
    a = ms.floor_audit(emu.EmuFloor())
    assert a["crawling"][0] and abs(a["dz_first"][0]) > 1e-3
    assert np.array_equal(ms.fix_height(a, "first_frame").rows, ms.rows)
    assert not np.array_equal(ms.fix_height(a, "clip_min").rows, ms.rows)


def test_height_fix_without_device_tables_is_refused_naming_the_key(tmp_path):
    import joblib
    from uhc.data_loaders.dataset_amass_single import DatasetAMASSSingle
    rng = np.random.default_rng(0)
    path = str(tmp_path / "clips.pkl")
    pose = rng.normal(0, 0.05, (12, 72))
    pose[:, 0] += np.pi / 2                                                # upright: SMPL's y-up body turned to z-up
    hi = {"pose_aa": pose, "trans": np.tile([0.0, 0.0, 1.3], (12, 1)), "beta": np.zeros(16), "gender": "neutral"}
    ok = {"pose_aa": pose, "trans": np.tile([0.0, 0.0, 0.95], (12, 1)), "beta": np.zeros(16), "gender": "neutral"}
    joblib.dump({"high": hi, "fine": ok}, path)
    specs = dict(file_path=path, test_file_path=path, t_min=5, t_max=-1)
    for extra in (dict(fix_height="first_frame"), dict(drop_implausible=True), dict(fix_height="clip_min", expert_tables="host")):
        with pytest.raises(ValueError, match="expert_tables: device"):
            DatasetAMASSSingle(dict(specs, **extra))
    assert DatasetAMASSSingle(dict(specs)).floor_fixed                     # the default: nothing to do
    ds = DatasetAMASSSingle(dict(specs, expert_tables="device", fix_height="first_frame", drop_implausible=True))
    lines = []
    assert ds.fix_floor(emu.EmuFloor(), lines.append) and not ds.fix_floor(emu.EmuFloor(), lines.append)
    assert lines == ["Starting too high: high"] and ds.data_keys == ["fine"] and ds.get_len() == 1 and len(ds.shapes) == 1
    assert all(k == "fine" for k, _ in ds.sample_keys) and list(ds.motions.lens) == [12] and set(ds.data["trans"]) == {"fine"}
    assert abs(ds.motions.floor_audit(emu.EmuFloor())["dz_first"][0]) < 1e-12
    assert np.array_equal(ds.data["trans"]["fine"], ds.motions.rows[:, 72:75]) and ds.data["trans"]["fine"][0, 2] != 0.95
