"""Plain numpy restatement of the floor measurements (TEST INFRASTRUCTURE): scipy rotations and the tree FK of uhc_b200/motion_lib.py place the
24 bodies, every hull vertex of uhc_b200/model.py is moved to the world, and the reference's compute_penetration / compute_skate
(uhc/smpllib/smpl_eval.py:125-149, floor_z = 0) run on those vertices as they are written there."""
import numpy as np
from scipy.spatial.transform import Rotation as sRot

from uhc_b200 import motion_lib as ML
from uhc_b200.model import HumanoidModel

FLOOR_Z = 0.0


def hull_vertices(qpos, model=None):
    """qpos [T][>= 76] -> world hull vertices [T][nvert][3]"""
    m = model or HumanoidModel()
    q = np.asarray(qpos, np.float64)[:, :76]
    T = len(q)
    bq = ML.euler_zyx_quat(q[:, 7:].reshape(T, 23, 3))
    wpos, wquat = np.zeros((T, 24, 3)), np.zeros((T, 24, 4))
    wpos[:, 0], wquat[:, 0] = q[:, :3], q[:, 3:7]
    for b in range(1, 24):                                                       # the tree FK of motion_lib.qpos_fk
        p = m.parent[b]
        wpos[:, b] = ML.qrot(wquat[:, p], np.broadcast_to(m.offset[b], (T, 3))) + wpos[:, p]
        wquat[:, b] = ML.qmul(wquat[:, p], bq[:, b - 1])
    out = np.zeros((T, len(m.hull), 3))
    for b in range(24):
        a, k = int(m.hull_adr[b]), int(m.hull_num[b])
        R = sRot.from_quat(wquat[:, b][:, [1, 2, 3, 0]]).as_matrix()            # scipy normalises, as qmat does
        out[:, a:a + k] = np.einsum("tij,vj->tvi", R, m.hull[a:a + k]) + wpos[:, b][:, None]
    return out


def compute_penetration(vert):
    pen = []
    for vert_i in vert:
        vert_z = vert_i[:, 2] - FLOOR_Z
        pind = vert_z < 0
        if np.any(pind):
            pen_i = -vert_z[pind].mean() * 1000
        else:
            pen_i = 0.0
        pen.append(pen_i)
    return pen


def compute_skate(vert):
    skate = []
    for t in range(vert.shape[0] - 1):
        cind = (vert[t, :, 2] <= FLOOR_Z) & (vert[t + 1, :, 2] <= FLOOR_Z)
        if np.any(cind):
            offset = vert[t + 1, cind, :2] - vert[t, cind, :2]
            skate_i = np.linalg.norm(offset, axis=1).mean() * 1000
        else:
            skate_i = 0.0
        skate.append(skate_i)
    return skate


def floor_rows(qpos, model=None):
    """rows [T][5] of one clip: min_z, pen_mm, skate_mm (row 0: 0), float_mm, n_below"""
    v = hull_vertices(qpos, model)
    z = v[:, :, 2]
    out = np.zeros((len(v), 5))
    out[:, 0] = z.min(1)
    out[:, 1] = compute_penetration(v)
    out[1:, 2] = compute_skate(v)
    out[:, 3] = np.maximum(out[:, 0], 0.0) * 1000
    out[:, 4] = (z < 0).sum(1)
    return out


def summary(qpos, model=None):
    """pentration / skate / float of a clip, as compute_metrics takes the means"""
    v = hull_vertices(qpos, model)
    return {"pentration": np.mean(compute_penetration(v)), "skate": np.mean(compute_skate(v)) if len(v) > 1 else 0.0,
            "float": np.mean(np.maximum(v[:, :, 2].min(1), 0.0) * 1000)}
