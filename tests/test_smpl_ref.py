"""CPU: properties of the fp64 SMPL restatement (tests/smpl_ref.py) the device skinning is tested against."""
import numpy as np

from tests.smpl_ref import batch_rodrigues, floor_rows, smpl_forward
from tests.test_smpl_model import synthetic
from uhc_b200.smpl_model import validate, NJ


def model(V=50, seed=1):
    raw = synthetic(V, seed)
    m = {k: raw[k] for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "weights")}
    p = raw["kintree_table"][0].astype(np.int32)
    p[0] = -1
    m["parents"] = p
    return validate(m)


def test_rest_pose_is_the_template_plus_trans():
    m = model()
    trans = np.array([[0.3, -1.0, 2.0], [0.0, 0.0, 0.0]])
    v, j = smpl_forward(m, np.zeros((2, 72)), trans, np.zeros((2, 10)))
    assert np.abs(v - (m["v_template"][None] + trans[:, None])).max() < 1e-12
    assert np.abs(j - (m["J_regressor"] @ m["v_template"])[None] - trans[:, None]).max() < 1e-12


def test_root_rotation_is_rigid_about_joint_0():
    m = model()
    beta = np.random.RandomState(2).uniform(-3, 3, (1, 10))
    r = np.array([0.4, -1.1, 0.7])
    pose = np.zeros((1, 72))
    pose[0, :3] = r
    v0, j0 = smpl_forward(m, np.zeros((1, 72)), np.zeros((1, 3)), beta)
    v, j = smpl_forward(m, pose, np.zeros((1, 3)), beta)
    R = batch_rodrigues(r)[0]
    c = j0[0, 0]
    assert np.abs(v[0] - ((v0[0] - c) @ R.T + c)).max() < 1e-12
    assert np.abs(j[0] - ((j0[0] - c) @ R.T + c)).max() < 1e-12


def test_rodrigues_is_finite_and_orthonormal_near_0_and_pi():
    rng = np.random.RandomState(3)
    axes = rng.normal(size=(30, 3))
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    for a in (0.0, 1e-9, np.pi - 1e-6, np.pi):
        R = batch_rodrigues(axes * a)
        assert np.isfinite(R).all()
        assert np.abs(R @ R.transpose(0, 2, 1) - np.eye(3)).max() < 1e-7
    assert np.abs(batch_rodrigues(np.zeros((1, 3)))[0] - np.eye(3)).max() < 1e-15
    m = model()
    pose = np.concatenate([axes[:NJ] * a for a in (0.0, 1e-9, np.pi - 1e-6)]).reshape(3, 72)
    v, j = smpl_forward(m, pose, np.zeros((3, 3)), np.zeros((3, 10)))
    assert np.isfinite(v).all() and np.isfinite(j).all()


def test_floor_rows_follow_the_reference_rules():
    v = np.zeros((3, 4, 3))
    v[:, :, 2] = [[-0.01, 0.0, 0.2, 0.5], [-0.03, 0.0, -0.01, 0.5], [0.1, 0.2, 0.3, 0.4]]
    v[1, :, 0] = 0.003
    r = floor_rows(v)
    assert r[0, 1] == 10.0 and r[0, 4] == 1 and r[0, 2] == 0.0                     # z == 0 is not below, frame 0 has no skate
    assert abs(r[1, 1] - 20.0) < 1e-12 and r[1, 4] == 2 and abs(r[1, 2] - 3.0) < 1e-12   # both frames z <= 0: vertices 0 and 1
    assert r[2, 2] == 0.0 and abs(r[2, 3] - 100.0) < 1e-12
    assert floor_rows(v, first=[1, 1, 1])[1, 2] == 0.0
