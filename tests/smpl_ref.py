"""fp64 numpy restatement of smplx's SMPL forward (smplx/lbs.py lbs, batch_rodrigues, batch_rigid_transform; smplx/body_models.py SMPL),
the reference the device skinning (include/uhc_mesh.h) is tested against.  It shares no code with the CUDA.  smplx itself is not a
dependency, so this restatement is written from smplx's published source and has not been run beside it here."""
import numpy as np


def batch_rodrigues(r):
    """[n][3] axis-angles -> [n][3][3]; angle = |r + 1e-8| as smplx takes it, so r = 0 gives the identity"""
    r = np.asarray(r, np.float64).reshape(-1, 3)
    angle = np.linalg.norm(r + 1e-8, axis=1, keepdims=True)
    d = r / angle
    c, s = np.cos(angle)[:, :, None], np.sin(angle)[:, :, None]
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    o = np.zeros_like(x)
    K = np.stack([o, -z, y, z, o, -x, -y, x, o], 1).reshape(-1, 3, 3)
    return np.eye(3)[None] + s * K + (1.0 - c) * (K @ K)


def smpl_forward(model, pose, trans, betas):
    """model = load_smpl_model's dict; pose [n][72], trans [n][3], betas [n][10] -> (vertices [n][V][3], joints [n][24][3]) in fp64:
    smplx's vertices + transl and joints[:, :24] (J_transformed) + transl"""
    pose = np.asarray(pose, np.float64).reshape(-1, 24, 3)
    n = len(pose)
    trans = np.asarray(trans, np.float64).reshape(n, 3)
    betas = np.asarray(betas, np.float64).reshape(n, 10)
    V = model["v_template"].shape[0]
    v_shaped = model["v_template"][None] + np.einsum("bl,mkl->bmk", betas, model["shapedirs"])
    J = np.einsum("jv,bvk->bjk", model["J_regressor"], v_shaped)
    R = batch_rodrigues(pose.reshape(-1, 3)).reshape(n, 24, 3, 3)
    pose_feature = (R[:, 1:] - np.eye(3)).reshape(n, -1)                        # row-major per joint
    posedirs = model["posedirs"].reshape(-1, 207).T                             # smplx: reshape(posedirs, [-1, 207]).T
    v_posed = v_shaped + (pose_feature @ posedirs).reshape(n, V, 3)
    parents = model["parents"]
    rel = J.copy()
    rel[:, 1:] -= J[:, parents[1:]]
    Tm = np.zeros((n, 24, 4, 4))
    Tm[:, :, :3, :3], Tm[:, :, :3, 3], Tm[:, :, 3, 3] = R, rel, 1.0
    G = np.zeros_like(Tm)
    G[:, 0] = Tm[:, 0]
    for k in range(1, 24):
        G[:, k] = G[:, parents[k]] @ Tm[:, k]
    joints = G[:, :, :3, 3]
    Jh = np.concatenate([J, np.zeros((n, 24, 1))], 2)[..., None]                # pad(G . [J; 0])
    A = G - np.concatenate([np.zeros((n, 24, 4, 3)), G @ Jh], 3)
    T = np.einsum("vk,bkij->bvij", model["weights"], A)
    vh = np.concatenate([v_posed, np.ones((n, V, 1))], 2)
    verts = np.einsum("bvij,bvj->bvi", T, vh)[:, :, :3]
    return verts + trans[:, None], joints + trans[:, None]


def floor_rows(verts, first=None):
    """compute_penetration / compute_skate (uhc/smpllib/smpl_eval.py:125-149, floor_z = 0) per frame over [n][V][3] vertices, in
    include/uhc_floor.h's columns: min_z, pen_mm, skate_mm (over the row and its previous one; 0 on a row without one), float_mm, n_below.
    first = per row, 1 where it has no previous row (None: one clip)"""
    v = np.asarray(verts, np.float64)
    n = len(v)
    out = np.zeros((n, 5))
    for i in range(n):
        z = v[i, :, 2]
        b = z < 0
        out[i, 0] = z.min()
        out[i, 1] = -z[b].mean() * 1000 if b.any() else 0.0
        out[i, 3] = max(z.min(), 0.0) * 1000
        out[i, 4] = b.sum()
        if i > 0 and not (first is not None and first[i]):
            c = (v[i - 1, :, 2] <= 0) & (z <= 0)
            if c.any():
                out[i, 2] = np.linalg.norm(v[i, c, :2] - v[i - 1, c, :2], axis=1).mean() * 1000
    return out
