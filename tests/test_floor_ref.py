"""CPU: the numpy restatement of the floor measurements (tests/floor_ref.py) on hand-made cases whose answers are known."""
import numpy as np

from tests import floor_ref as FR
from uhc_b200.metrics import floor_summary
from uhc_b200.model import HumanoidModel


def standing(z_lowest=0.0):
    """the rest pose, upright, with its lowest hull vertex at z_lowest"""
    q = HumanoidModel().qpos0.copy()[None]
    q[0, 3:7] = [0.7071067811865476, 0.7071067811865476, 0.0, 0.0]
    q[0, 2] -= FR.hull_vertices(q)[0, :, 2].min() - z_lowest
    return q


def test_lowered_pose_penetrates_by_the_mean_depth_of_the_vertices_below():
    q = standing(-0.02)
    z = FR.hull_vertices(q)[0, :, 2]
    r = FR.floor_rows(q)[0]
    below = z[z < 0]
    assert 0 < len(below) < len(z) and r[4] == len(below)
    assert np.isclose(r[1], -below.mean() * 1000, rtol=1e-12) and 0 < r[1] < 20
    assert np.isclose(r[0], -0.02, atol=1e-12) and r[3] == 0


def test_slide_of_one_centimetre_with_the_feet_down_skates_ten_millimetres():
    q = np.repeat(standing(-0.01), 3, 0)
    q[1, 0] += 0.01
    q[2, 0] += 0.01
    q[2, 1] -= 0.01
    r = FR.floor_rows(q)
    assert r[0, 2] == 0 and np.isclose(r[1, 2], 10.0, rtol=1e-9) and np.isclose(r[2, 2], 10.0, rtol=1e-9)
    assert np.isclose(FR.summary(q)["skate"], 10.0, rtol=1e-9) and np.isclose(floor_summary(r)["skate"], 10.0, rtol=1e-9)


def test_lifted_pose_floats_and_neither_penetrates_nor_skates():
    q = np.repeat(standing(0.05), 2, 0)
    q[1, 0] += 0.3
    r = FR.floor_rows(q)
    assert np.allclose(r[:, 3], 50.0, rtol=1e-9) and (r[:, 1] == 0).all() and (r[:, 2] == 0).all() and (r[:, 4] == 0).all()
    s = floor_summary(r)
    assert np.isclose(s["float"], 50.0, rtol=1e-9) and s["pentration"] == 0 and s["skate"] == 0
    assert FR.summary(q) == {"pentration": 0.0, "skate": 0.0, "float": s["float"]}


def test_a_vertex_exactly_on_the_floor_skates_but_does_not_penetrate():
    v = np.zeros((2, 3, 3))
    v[:, 0, 2], v[:, 1, 2], v[:, 2, 2] = 0.0, 0.25, 0.5          # vertex 0 exactly on the floor, in both frames
    v[1, :, 0] = 0.003
    assert FR.compute_penetration(v) == [0.0, 0.0]                # z < 0: nothing is below
    assert np.isclose(FR.compute_skate(v)[0], 3.0, rtol=1e-12)    # z <= 0: the vertex on the floor counts
    v[1, 0, 2] = 1e-300                                            # off the floor in the second frame: no pair
    assert FR.compute_skate(v) == [0.0]
