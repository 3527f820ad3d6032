"""Independent fp64 numpy ray caster of the humanoid's body hulls (TEST REFERENCE for uhc_b200/csrc/render_core.h).

Shares no code with the kernels: the face planes come from its own ConvexHull call on the model's hull vertices (no merging), the FK from
uhc_b200/motion_lib.py (pinned to the reference's qpos_fk by tests/test_motion_lib.py), the camera basis, the clip and the shading are
restated here in fp64 and vectorised over pixels.  Besides the image it reports, per pixel, whether an fp32 evaluation could decide
differently: a primary or shadow decision within TOL of flipping (a clip interval of length < TOL, two surfaces within TOL of each other,
an entering face within TOL of another one, a checker edge or the floor's far cut within TOL (relative past 1 m)).
"""
import numpy as np
from scipy.spatial import ConvexHull

from uhc_b200 import motion_lib as ML

# the scene constants render_core.h states
LIGHT = np.array([1.0, -2.0, 3.0]) / np.sqrt(14.0)
AMBIENT, DIFFUSE = 0.35, 0.65
SKY = np.array([0.62, 0.74, 0.86])
FLOOR = (0.60, 0.42)
FLOOR_FAR = 60.0
BODY = (np.array([0.70, 0.70, 0.70]), np.array([0.70, 0.0, 0.0]))
EPS = 1e-4
TOL = 1e-5


def hull_planes(model):
    """per body [k][4] (n, d) of ConvexHull(vertices).equations"""
    return [ConvexHull(model.hull[model.hull_adr[b]:model.hull_adr[b] + model.hull_num[b]]).equations for b in range(24)]


def hull_verts(model):
    return [model.hull[model.hull_adr[b]:model.hull_adr[b] + model.hull_num[b]] for b in range(24)]


def quat_mat(q):
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = (q[..., i] for i in range(4))
    return np.stack([np.stack([w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z], -1)], -2)


def pose_table(qpos, model):
    """qpos [T][>= 76] -> [T][24][12]: rotation (row-major) and position of every body, from motion_lib.qpos_fk"""
    fk = ML.qpos_fk(np.asarray(qpos, np.float64)[:, :76], model)
    T = len(qpos)
    R = quat_mat(fk["wbquat"].reshape(T, 24, 4))
    return np.concatenate([R.reshape(T, 24, 9), fk["wbpos"].reshape(T, 24, 3)], -1)


def camera(cam, W, H):
    """MuJoCo free camera: (offset of the eye from lookat, forward, right * tan * aspect, up * tan)"""
    az, el = np.radians(cam.get("azimuth", 45.0)), np.radians(cam.get("elevation", -8.0))
    th = np.tan(np.radians(cam.get("fovy", 45.0)) / 2)
    f = np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
    u = np.array([-np.sin(el) * np.cos(az), -np.sin(el) * np.sin(az), np.cos(el)])
    r = np.cross(f, u)
    return -cam.get("distance", 5.0) * f, f, r * th * W / H, u * th


def clip(o, d, pl, t_lo):
    """rays o + t d (body frame, [N][3] each) against planes [K][4]: (t_in, t_out, entering plane, the plane entered second-last and its t)"""
    den = d @ pl[:, :3].T
    nu = -(o @ pl[:, :3].T + pl[:, 3])
    with np.errstate(divide="ignore", invalid="ignore"):
        t = nu / den
    ent = np.where(den < 0, t, -np.inf)
    ext = np.where(den > 0, t, np.inf)
    order = np.argsort(ent, 1)
    k, k2 = order[:, -1], order[:, -2]
    rows = np.arange(len(o))
    t_in = np.maximum(ent[rows, k], t_lo)
    t_out = ext.min(1)
    t_out = np.where(((den == 0) & (nu < 0)).any(1), -np.inf, t_out)
    return t_in, t_out, np.where(ent[rows, k] > t_lo, k, -1), k2, ent[rows, k2]


def render(pose, model, size, cam=None, humanoids=2):
    """pose [n][2][24][12] (fp64 or fp32 values) -> dict(rgb [n][H][W][3] uint8, colour (float), depth, label, amb (bool), and per pixel
    the hit body slot, its entering plane, the world hit point and |cos| of the angle between the ray and the surface normal)"""
    cam = dict(cam or {})
    W, H = size
    n = len(pose)
    off, f, r, u = camera(cam, W, H)
    planes, verts = hull_planes(model), hull_verts(model)
    ys, xs = np.mgrid[0:H, 0:W]
    a = (2 * (xs.ravel() + 0.5) / W - 1)[:, None]
    b = (1 - 2 * (ys.ravel() + 0.5) / H)[:, None]
    d = f + a * r + b * u
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    N = len(d)
    vis = [not cam.get("hide_im", False), humanoids > 1 and not cam.get("hide_expert", False)]
    shift = cam.get("shift_expert", 0.0)
    shift = 1.0 if shift is True else float(shift)
    out = {k: [] for k in ("cos", "rgb", "colour", "depth", "label", "amb", "slot", "plane", "point", "parts")}
    for i in range(n):
        P = np.asarray(pose[i], np.float64).copy()
        P[1, :, 9] += shift
        look = np.array(cam.get("lookat", (0.0, 0.0, 1.0)), np.float64)
        if cam.get("focus", False):
            look[:2] = np.asarray(pose[i], np.float64)[0, 0, 9:11]
        o = look + off
        bodies = [(h * 24 + bb, P[h, bb, :9].reshape(3, 3), P[h, bb, 9:]) for h in range(2) if vis[h] for bb in range(24)]

        def cast(orig, dirs, t_lo):
            """every body: clip's (t_in, t_out, plane, second plane, its t) per ray, inf / -1 where it misses the bounding sphere"""
            M = len(dirs)
            orig = np.broadcast_to(orig, dirs.shape)
            res = []
            for j, R, p in bodies:
                wv = verts[j % 24] @ R.T + p
                c = wv.mean(0)
                rad = np.linalg.norm(wv - c, axis=1).max() * (1 + 1e-6) + 1e-9
                oc = c - orig
                bp = (oc * dirs).sum(1)
                dist2 = (oc * oc).sum(1) - bp * bp
                cand = np.nonzero(dist2 <= rad * rad)[0]
                ti, to, kk, k2, t2 = np.full(M, np.inf), np.full(M, -np.inf), np.full(M, -1), np.full(M, -1), np.full(M, -np.inf)
                if len(cand):
                    ob = orig[cand] - p
                    ti[cand], to[cand], kk[cand], k2[cand], t2[cand] = clip(ob @ R, dirs[cand] @ R, planes[j % 24], t_lo)
                res.append((j, R, ti, to, kk, k2, t2))
            return res

        amb = np.zeros(N, bool)
        t = np.full(N, np.inf)
        tf = np.full(N, np.inf)
        down = d[:, 2] < 0
        tf[down] = -o[2] / d[down, 2]
        floor = (tf > 0) & (tf < FLOOR_FAR)
        parts = {}
        parts["far"] = np.abs(tf - FLOOR_FAR) < TOL * np.maximum(tf, 1)
        amb |= parts["far"]
        t[floor] = tf[floor]
        label = np.where(floor, 1, 0)
        cands = [t.copy()]
        slot, plane, plane2, t2hit = np.full(N, -1), np.full(N, -1), np.full(N, -1), np.full(N, -np.inf)
        R_of = {}
        for j, R, ti, to, kk, k2, t2 in cast(o, d, 0.0):
            R_of[j] = R
            amb |= np.abs(to - ti) < TOL
            hit = ti <= to
            cands.append(np.where(hit, ti, np.inf))
            better = hit & (ti < t)
            t[better], label[better], slot[better], plane[better], plane2[better], t2hit[better] = ti[better], 2 + j, j, kk[better], k2[better], t2[better]
        cs = np.sort(np.stack(cands, 1), 1)
        parts["interval"] = amb & ~parts["far"]
        with np.errstate(invalid="ignore"):
            parts["depth"] = (cs[:, 1] - cs[:, 0] < TOL) & np.isfinite(cs[:, 0])
        amb |= parts["depth"]
        p = o + t[:, None] * d
        nw = np.zeros((N, 3))
        nw[:, 2] = 1.0
        edge_dl = np.zeros(N)          # Lambert term of the face entered second-last, where the ray hits near the edge between the two
        for j in np.unique(slot[slot >= 0]):
            m = slot == j
            nw[m] = planes[j % 24][plane[m], :3] @ R_of[j].T
            edge_dl[m] = np.maximum(planes[j % 24][plane2[m], :3] @ R_of[j].T @ LIGHT, 0)
        # near an edge between two faces an fp32 cast may take either normal: ambiguous when their shades differ by a level or more
        parts["edge"] = (slot >= 0) & (t - t2hit < TOL) & (np.abs(np.maximum(nw @ LIGHT, 0) - edge_dl) * DIFFUSE * 255 >= 1)
        amb |= parts["edge"]
        fl = label == 1
        sq = np.zeros(N)
        sq[fl] = np.floor(p[fl, 0]) + np.floor(p[fl, 1])
        fr = np.full(N, np.inf)
        fr[fl] = np.abs(p[fl, :2] - np.round(p[fl, :2])).min(1)
        parts["checker"] = (label == 1) & (fr < TOL * np.maximum(t, 1))
        amb |= parts["checker"]
        shadow = np.zeros(N, bool)
        ndl = np.maximum((nw * LIGHT).sum(1), 0.0)
        lit = np.ones(N, bool)
        sh = np.nonzero((label > 0) & (ndl > 0))[0]
        if len(sh):
            for j, R, ti, to, kk, k2, t2 in cast(p[sh], np.broadcast_to(LIGHT, (len(sh), 3)), EPS):
                shadow[sh] |= np.abs(to - ti) < TOL
                lit[sh[ti <= to]] = False
        parts["shadow"] = shadow
        amb |= shadow
        ndl = np.where(lit, ndl, 0.0)
        base = np.where(fl[:, None], np.where(np.mod(sq, 2) == 0, FLOOR[0], FLOOR[1])[:, None],
                        np.where((label >= 26)[:, None], BODY[1], BODY[0]))
        col = np.where((label == 0)[:, None], SKY, base * (AMBIENT + DIFFUSE * ndl)[:, None])
        rgb = np.floor(np.clip(col, 0, 1) * 255 + 0.5).astype(np.uint8)
        out["parts"].append({k: v.reshape(H, W) for k, v in parts.items()})
        cosi = np.abs((nw * d).sum(1))
        for k, v in (("cos", cosi.reshape(H, W)), ("rgb", rgb.reshape(H, W, 3)), ("colour", col.reshape(H, W, 3)), ("depth", t.reshape(H, W)), ("label", label.reshape(H, W)),
                     ("amb", amb.reshape(H, W)), ("slot", slot.reshape(H, W)), ("plane", plane.reshape(H, W)), ("point", p.reshape(H, W, 3))):
            out[k].append(v)
    res = {k: np.stack(v) for k, v in out.items() if k != "parts"}
    res["parts"], res["planes"] = out["parts"], planes
    return res
