"""Evaluation metrics of the imitation benchmark (SURVEY.md section 8f row 2), vectorised numpy.

Restates uhc/smpllib/smpl_eval.py:24-123 (p_mpjpe, compute_metrics) and the finite-difference errors of
uhc/losses/loss_function.py:36-95 for whole episodes at once; parity: tests/test_metrics.py against outputs of the reference's own
functions (tests/golden/metrics.npz, tools/make_golden.py gen_metrics).  Units follow the reference: millimetres (per frame).
"""
import numpy as np


def quat_to_mat4(q):
    """[T,4] (w,x,y,z) -> [T,4,4] homogeneous rotation (transformation.py quaternion_matrix; quaternions are normalised by |q|^2)."""
    q = np.asarray(q, dtype=np.float64)
    n = (q * q).sum(-1)
    s = np.where(n > np.finfo(float).eps * 4.0, 2.0 / np.maximum(n, 1e-300), 0.0)
    w, x, y, z = q[:, 0], q[:, 1], q[:, 2], q[:, 3]
    M = np.zeros((len(q), 4, 4))
    M[:, 0, 0] = 1 - s * (y * y + z * z); M[:, 0, 1] = s * (x * y - z * w); M[:, 0, 2] = s * (x * z + y * w)
    M[:, 1, 0] = s * (x * y + z * w); M[:, 1, 1] = 1 - s * (x * x + z * z); M[:, 1, 2] = s * (y * z - x * w)
    M[:, 2, 0] = s * (x * z - y * w); M[:, 2, 1] = s * (y * z + x * w); M[:, 2, 2] = 1 - s * (x * x + y * y)
    M[:, 3, 3] = 1.0
    M[n <= np.finfo(float).eps * 4.0, :3, :3] = np.eye(3)
    return M


def root_dist_mm(qpos_pred, qpos_gt):
    """||I - X_pred X_gt^-1||_F per frame, divided by the number of frames (the reference's get_frobenious_norm does), in mm."""
    Xp, Xg = quat_to_mat4(qpos_pred[:, 3:7]), quat_to_mat4(qpos_gt[:, 3:7])
    Xp[:, :3, 3], Xg[:, :3, 3] = qpos_pred[:, :3], qpos_gt[:, :3]
    err = np.eye(4)[None] - Xp @ np.linalg.inv(Xg)
    return np.sqrt((err ** 2).sum((1, 2))) / len(qpos_pred) * 1000.0


def procrustes_mpjpe(pred, gt):
    """per-frame joint error after the best similarity alignment (scale, rotation, translation) of pred onto gt: [T,J,3] -> [T,J]."""
    mu_g, mu_p = gt.mean(1, keepdims=True), pred.mean(1, keepdims=True)
    G, P = gt - mu_g, pred - mu_p
    ng, npd = np.sqrt((G ** 2).sum((1, 2), keepdims=True)), np.sqrt((P ** 2).sum((1, 2), keepdims=True))
    G, P = G / ng, P / npd
    U, s, Vt = np.linalg.svd(G.transpose(0, 2, 1) @ P)
    V = Vt.transpose(0, 2, 1)
    flip = np.sign(np.linalg.det(V @ U.transpose(0, 2, 1)))          # no reflections
    V[:, :, -1] *= flip[:, None]
    s[:, -1] *= flip
    R = V @ U.transpose(0, 2, 1)
    scale = s.sum(1)[:, None, None] * ng / npd
    aligned = scale * (pred @ R) + (mu_g - scale * (mu_p @ R))
    return np.linalg.norm(aligned - gt, axis=2)


def compute_metrics(res):
    """res: pred / gt = qpos [T,76]; pred_jpos / gt_jpos = world joint positions [T,72]; percent; fail_safe.
    Returns the dict of smpl_eval.compute_metrics (per-frame arrays in mm + succ)."""
    jp = np.asarray(res["pred_jpos"], dtype=np.float64).reshape(len(res["pred"]), -1, 3)
    jg = np.asarray(res["gt_jpos"], dtype=np.float64).reshape(len(res["gt"]), -1, 3)
    qp, qg = np.asarray(res["pred"], dtype=np.float64), np.asarray(res["gt"], dtype=np.float64)
    out = {"root_dist": root_dist_mm(qp, qg)}
    vel = np.linalg.norm((jp[1:] - jp[:-1]) - (jg[1:] - jg[:-1]), axis=2).mean(1)
    acc = np.linalg.norm((jp[:-2] - 2 * jp[1:-1] + jp[2:]) - (jg[:-2] - 2 * jg[1:-1] + jg[2:]), axis=2).mean(1)
    out["mpjpe_g"] = np.linalg.norm(jp - jg, axis=2).mean(-1) * 1000.0
    root = 0 if jp.shape[1] == 24 else 7                       # 24-joint SMPL: Pelvis; 14 / 12-joint sets: index 7
    jp, jg = jp - jp[:, root:root + 1], jg - jg[:, root:root + 1]
    out["pa_mpjpe"] = procrustes_mpjpe(jp, jg).mean(-1) * 1000.0
    out["mpjpe"] = np.linalg.norm(jp - jg, axis=2).mean(-1) * 1000.0
    out["accel_dist"], out["vel_dist"] = acc * 1000.0, vel * 1000.0
    out["succ"] = np.array([(not res["fail_safe"]) and res["percent"] == 1])
    return out


def metrics_from_frames(frames, percent, fail_safe):
    """compute_metrics' dict from the per-frame rows [T][6] the device evaluation writes (uhc_b200/csrc/eval_core.h; T >= 3):
    mpjpe_g, mpjpe, pa_mpjpe, vel (valid from frame 1), accel (from frame 2), |I - X_pred X_gt^-1|_F, which root_dist_mm divides by T."""
    f = np.asarray(frames, dtype=np.float64)
    T = len(f)
    return {"root_dist": f[:, 5] / T * 1000.0, "vel_dist": f[1:, 3].copy(), "accel_dist": f[2:, 4].copy(), "mpjpe_g": f[:, 0].copy(),
            "pa_mpjpe": f[:, 2].copy(), "mpjpe": f[:, 1].copy(), "succ": np.array([(not fail_safe) and percent == 1])}
