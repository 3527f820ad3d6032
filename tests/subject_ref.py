"""fp64 numpy restatement of the subject body builder (include/uhc_subject.h, uhc_b200/subject_body.py) for the tests.  It fits each
subject's maps directly (a least-squares solve per subject and body, not the beta basis), and derives the mass properties, offsets, hull,
spheres and invweight0 from them as DESIGN.md section 4 states; it shares no code with uhc_b200/csrc/subject_core.h or the basis fit."""
import numpy as np

from uhc_b200.model import HumanoidModel

NB = 24
Z = np.array([[1.0, 0, 0], [0, 0, -1.0], [0, 1.0, 0]])          # y-up -> z-up: (x, y, z) -> (x, -z, y)


def subject_maps(hm, neutral, model, beta):
    """(A | t) [24][3][4] of one subject whose SMPL model is `model`, by model body"""
    joint = [HumanoidModel.SMPL_BONE_ORDER.index(n) for n in hm.body_names]
    owner = neutral["weights"].argmax(1)
    vn = neutral["v_template"]
    Jn = neutral["J_regressor"] @ vn
    vg = model["v_template"] + model["shapedirs"][:, :, :10] @ np.asarray(beta, np.float64)[:10]
    Jg = model["J_regressor"] @ vg
    out = np.zeros((NB, 3, 4))
    for b in range(NB):
        j = joint[b]
        S = owner == j
        P, Q = (vn[S] - Jn[j]) @ Z.T, (vg[S] - Jg[j]) @ Z.T
        X = np.linalg.lstsq(np.hstack([P, np.ones((len(P), 1))]), Q, rcond=None)[0]
        out[b] = X.T
    return out, Jn, Jg


def subject_offsets(hm, Jn, Jg):
    joint = [HumanoidModel.SMPL_BONE_ORDER.index(n) for n in hm.body_names]
    off = hm.offset.copy()
    for b in range(NB):
        j = joint[b]
        if b == 0:
            off[b] += Z @ (Jg[j] - Jn[j])
        else:
            p = joint[hm.parent[b]]
            off[b] += Z @ ((Jg[j] - Jg[p]) - (Jn[j] - Jn[p]))
    return off


def mapped_mass(m, c, I, A, t):
    """mass, COM and inertia about the COM of a body of uniform density after x -> A x + t"""
    det = np.linalg.det(A)
    if det <= 0:
        raise ValueError("the map inverts the body (det A <= 0)")
    S = 0.5 * np.trace(I) * np.eye(3) - I
    S2 = det * A @ S @ A.T
    return m * det, A @ c + t, np.trace(S2) * np.eye(3) - S2


def invweight0(hm, offset, ipos, mass, inertia):
    """trace(Jv M^-1 Jv^T) / 3 at qpos0 for every body"""
    gpos = np.zeros((NB, 3))
    gpos[0] = offset[0]
    for b in range(1, NB):
        gpos[b] = gpos[hm.parent[b]] + offset[b]
    xi = gpos + ipos
    nv = 6 + 3 * (NB - 1)
    Jv, Jw = np.zeros((NB, 3, nv)), np.zeros((NB, 3, nv))
    for b in range(NB):
        Jv[b, :, :3] = np.eye(3)
        a = b
        chain = []
        while a > 0:
            chain.append(a)
            a = hm.parent[a]
        for k in range(3):
            e = np.eye(3)[k]
            Jw[b, :, 3 + k], Jv[b, :, 3 + k] = e, np.cross(e, xi[b] - gpos[0])
        for a in chain:
            for k, ax in enumerate(np.eye(3)[[2, 1, 0]]):
                d = 6 + 3 * (a - 1) + k
                Jw[b, :, d], Jv[b, :, d] = ax, np.cross(ax, xi[b] - gpos[a])
    M = np.diag(hm.armature.astype(np.float64))
    for b in range(NB):
        M += mass[b] * Jv[b].T @ Jv[b] + Jw[b].T @ inertia[b] @ Jw[b]
    Mi = np.linalg.inv(M)
    return np.array([np.trace(Jv[b] @ Mi @ Jv[b].T) / 3.0 for b in range(NB)])


def subject_body(hm, neutral, model, beta):
    """(body_f [24][20], hull [nvert][3], maps [24][3][4]) of one subject"""
    maps, Jn, Jg = subject_maps(hm, neutral, model, beta)
    offset = subject_offsets(hm, Jn, Jg)
    hull = hm.hull.copy()
    ipos, mass, inertia = np.zeros((NB, 3)), np.zeros(NB), np.zeros((NB, 3, 3))
    bf = np.zeros((NB, 20))
    for b in range(NB):
        A, t = maps[b, :, :3], maps[b, :, 3]
        mass[b], ipos[b], inertia[b] = mapped_mass(hm.mass[b], hm.ipos[b], hm.inertia[b], A, t)
        s = slice(hm.hull_adr[b], hm.hull_adr[b] + hm.hull_num[b])
        hull[s] = hm.hull[s] @ A.T + t
        c = hull[s].mean(0)
        bf[b, 14:17], bf[b, 17] = c, np.linalg.norm(hull[s] - c, axis=1).max() * 1.0001 + 1e-6
    bf[:, 0:3], bf[:, 3:6], bf[:, 6] = offset, ipos, mass
    bf[:, 7:13] = np.stack([inertia[:, 0, 0], inertia[:, 1, 1], inertia[:, 2, 2], inertia[:, 0, 1], inertia[:, 0, 2], inertia[:, 1, 2]], 1)
    bf[:, 13] = invweight0(hm, offset, ipos, mass, inertia)
    bf[:, 18:20] = hm.body_f[:, 18:20]
    return bf, hull, maps


def uniform_scale_model(seed=0):
    """a synthetic SMPL model built from the neutral humanoid (the hull vertices at rest, owned by their body) whose shape direction 0 is
    v_template itself: beta_0 = s - 1 scales the whole body about the origin"""
    hm = HumanoidModel()
    gpos = np.load(__import__("uhc_b200.model", fromlist=["ASSET"]).ASSET)["body_gpos"].astype(np.float64)
    order = [hm.body_names.index(n) for n in hm.SMPL_BONE_ORDER]
    inv = {b: j for j, b in enumerate(order)}
    parents = np.array([-1] + [inv[int(hm.parent[order[j]])] for j in range(1, 24)], np.int32)
    to_smpl = lambda x: x @ Z                                                 # z-up -> y-up, the inverse of Z
    J = to_smpl(gpos[order])
    vt, owner = [], []
    for j, b in enumerate(order):
        v = hm.hull[hm.hull_adr[b]:hm.hull_adr[b] + hm.hull_num[b]] + gpos[b]
        vt.append(to_smpl(v))
        owner += [j] * len(v)
    vt, owner = np.concatenate(vt), np.array(owner)
    V = len(vt)
    reg = np.zeros((24, V))
    for j in range(24):
        idx = np.nonzero(owner == j)[0]
        A = np.vstack([vt[idx].T, np.ones(len(idx))])
        reg[j, idx] = np.linalg.lstsq(A, np.append(J[j], 1.0), rcond=None)[0]
    w = np.zeros((V, 24))
    w[np.arange(V), owner] = 0.7
    w[np.arange(V)[owner > 0], parents[owner[owner > 0]]] += 0.3
    w[owner == 0, 0] = 1.0
    rng = np.random.RandomState(seed)
    sd = np.einsum("vc,ldc->vdl", vt, rng.normal(0, 0.02, (10, 3, 3))) + rng.normal(0, 1e-4, (V, 3, 10))    # smooth, as SMPL's are
    sd[:, :, 0] = vt
    return dict(v_template=vt, shapedirs=sd, posedirs=rng.normal(0, 0.003, (V, 3, 207)), J_regressor=reg, weights=w, parents=parents)


def gendered(model, seed):
    """another gender's model on the same mesh: the template moved a little, other shape directions"""
    rng = np.random.RandomState(seed)
    m = dict(model)
    vt = model["v_template"]
    m["v_template"] = vt * (1.0 + rng.normal(0, 0.02, 3)) + rng.normal(0, 5e-4, vt.shape)
    m["shapedirs"] = model["shapedirs"] + np.einsum("vc,ldc->vdl", vt, rng.normal(0, 0.005, (10, 3, 3))) + rng.normal(0, 1e-4, model["shapedirs"].shape)
    return m
