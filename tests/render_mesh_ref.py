"""Independent fp64 numpy brute-force ray caster of triangle meshes (TEST REFERENCE for uhc_b200/csrc/render_mesh_core.h).

Shares no code with the kernels or with tests/render_ref.py: its own camera from MuJoCo's free-camera formulas, its own ray-triangle
intersection (Moller-Trumbore in fp64 against every face of every body whose bounding sphere the ray meets, no hierarchy), its own flat
shading and shadow rays.  Besides the image it reports, per pixel, whether an fp32 evaluation could decide differently (render_ref.py's
rules carried over to triangles): a face whose edge or vertex lies within TOL of the ray in barycentric terms where taking or losing it
changes the label, the shade by a level or the depth; two surfaces within TOL (m) of each other; a shadow decided within TOL; a checker
edge or the floor's far cut within TOL (relative past 1 m)."""
import numpy as np

LIGHT = np.array([1.0, -2.0, 3.0]) / np.sqrt(14.0)
AMBIENT, DIFFUSE = 0.35, 0.65
SKY = np.array([0.62, 0.74, 0.86])
FLOOR = (0.60, 0.42)
FLOOR_FAR = 60.0
BODY = (np.array([0.70, 0.70, 0.70]), np.array([0.70, 0.0, 0.0]))
EPS = 1e-4
TOL = 1e-5


def camera(cam, W, H):
    """eye offset from lookat, forward, right (scaled by tan(fovy / 2) W / H) and up (scaled by tan(fovy / 2)) of MuJoCo's free camera"""
    az, el = np.deg2rad(cam.get("azimuth", 45.0)), np.deg2rad(cam.get("elevation", -8.0))
    fwd = np.array([np.cos(el) * np.cos(az), np.cos(el) * np.sin(az), np.sin(el)])
    up = np.array([-np.sin(el) * np.cos(az), -np.sin(el) * np.sin(az), np.cos(el)])
    right = np.array([np.sin(az), -np.cos(az), 0.0])
    th = np.tan(np.deg2rad(cam.get("fovy", 45.0)) / 2)
    return -cam.get("distance", 5.0) * fwd, fwd, right * th * W / H, up * th


def _hits(orig, dirs, tri, t_lo):
    """rays (orig [M][3] or [3], dirs [M][3]) x triangles [K][3][3]: (ray, face, t, min barycentric) of every pair with min barycentric > -TOL
    and t > t_lo - TOL; zero-area faces never hit"""
    e1, e2 = tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]
    area = np.linalg.norm(np.cross(e1, e2), axis=1) > 0
    orig = np.broadcast_to(orig, dirs.shape)
    pv = np.cross(dirs[:, None, :], e2[None])                         # [M][K][3]
    det = (e1[None] * pv).sum(-1)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = 1.0 / det
        s = orig[:, None, :] - tri[None, :, 0]
        u = (s * pv).sum(-1) * inv
        qv = np.cross(s, e1[None])
        v = (dirs[:, None, :] * qv).sum(-1) * inv
        t = (e2[None] * qv).sum(-1) * inv
        mb = np.minimum(np.minimum(u, v), 1 - u - v)
    ok = (det != 0) & area[None] & (mb > -TOL) & (t > t_lo - TOL) & np.isfinite(t)
    r, k = np.nonzero(ok)
    return r, k, t[r, k], mb[r, k]


def _groups(faces, face_body, hs):
    """per visible (humanoid, body): (slot, face indices, world triangles [K][3][3], sphere centre, radius)"""
    out = []
    for h, V in hs:
        for b in range(24):
            idx = np.nonzero(face_body == b)[0]
            if not len(idx):
                continue
            tri = V[faces[idx]]
            pts = tri.reshape(-1, 3)
            c = pts.mean(0)
            out.append((24 * h + b, idx, tri, c, np.linalg.norm(pts - c, axis=1).max() * (1 + 1e-9) + 1e-9))
    return out


def _cast(groups, orig, dirs, t_lo):
    """every possible hit: arrays (ray, slot, face, t, min barycentric, unit normal towards the ray's origin)"""
    rec = [[], [], [], [], [], []]
    orig_b = np.broadcast_to(orig, dirs.shape)
    for slot, idx, tri, c, rad in groups:
        oc = c - orig_b
        bp = (oc * dirs).sum(1)
        d2 = (oc * oc).sum(1) - bp * bp
        cand = np.nonzero(d2 <= rad * rad + 1e-9)[0]
        for a in range(0, len(cand), 1024):
            cc = cand[a:a + 1024]
            r, k, t, mb = _hits(orig_b[cc], dirs[cc], tri, t_lo)
            n = np.cross(tri[k, 1] - tri[k, 0], tri[k, 2] - tri[k, 0])
            n /= np.linalg.norm(n, axis=1, keepdims=True)
            n = np.where(((n * dirs[cc[r]]).sum(1) > 0)[:, None], -n, n)
            for lst, x in zip(rec, (cc[r], np.full(len(r), slot), idx[k], t, mb, n)):
                lst.append(x)
    empty = (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0), np.zeros(0), np.zeros((0, 3)))
    return [np.concatenate(x) if x else e for x, e in zip(rec, empty)]


def _level(base, ndl):
    return np.floor(np.clip(base * (AMBIENT + DIFFUSE * np.asarray(ndl))[..., None], 0, 1) * 255 + 0.5)


def render(verts, faces, face_body, size, cam=None, ghost=None, root=None):
    """verts / ghost [n][V][3] (values taken in fp64), faces [F][3], face_body [F] (the model body of every face), root [n][3] (focus) ->
    dict(rgb [n][H][W][3] uint8, depth, label, amb (bool), parts: per frame the ambiguity masks by cause)"""
    cam = dict(cam or {})
    W, H = size
    faces = np.asarray(faces, np.int64)
    face_body = np.asarray(face_body)
    off, f, r, u = camera(cam, W, H)
    ys, xs = np.mgrid[0:H, 0:W]
    a = (2 * (xs.ravel() + 0.5) / W - 1)[:, None]
    b = (1 - 2 * (ys.ravel() + 0.5) / H)[:, None]
    d = f + a * r + b * u
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    N = len(d)
    shift = cam.get("shift_expert", 0.0)
    shift = 1.0 if shift is True else float(shift)
    vis = [not cam.get("hide_im", False), ghost is not None and not cam.get("hide_expert", False)]
    out = {k: [] for k in ("rgb", "depth", "label", "amb", "parts")}
    for i in range(len(verts)):
        hs = [(0, np.asarray(verts[i], np.float64))] if vis[0] else []
        if vis[1]:
            g = np.asarray(ghost[i], np.float64).copy()
            g[:, 0] += shift
            hs.append((1, g))
        groups = _groups(faces, face_body, hs)
        look = np.array(cam.get("lookat", (0.0, 0.0, 1.0)), np.float64)
        if cam.get("focus", False):
            look[:2] = np.asarray(root[i], np.float64)[:2]
        o = look + off
        tf = np.full(N, np.inf)
        down = d[:, 2] < 0
        tf[down] = -o[2] / d[down, 2]
        floor = (tf > 0) & (tf < FLOOR_FAR)
        parts = {"far": np.abs(tf - FLOOR_FAR) < TOL * np.maximum(tf, 1)}
        ray, slot, face, t, mb, nrm = _cast(groups, o, d, 0.0)
        # the fp64 decision: the nearest face with every barycentric >= 0, else the floor, else the sky
        t_ref = np.where(floor, tf, np.inf)
        lab = np.where(floor, 1, 0)
        n_ref = np.tile([0.0, 0.0, 1.0], (N, 1))
        sure = mb >= 0
        order = np.lexsort((t[sure], ray[sure]))
        rs, ts, ss, ns = ray[sure][order], t[sure][order], slot[sure][order], nrm[sure][order]
        first = np.unique(rs, return_index=True)[1]
        rs, ts, ss, ns = rs[first], ts[first], ss[first], ns[first]
        take = ts < t_ref[rs]
        t_ref[rs[take]], lab[rs[take]], n_ref[rs[take]] = ts[take], 2 + ss[take], ns[take]
        base = np.where((lab == 1)[:, None], 0.0, np.where((lab >= 26)[:, None], BODY[1], BODY[0]))
        p = o + np.where(np.isfinite(t_ref), t_ref, 0)[:, None] * d
        fl = lab == 1
        sq = np.floor(p[:, 0]) + np.floor(p[:, 1])
        base[fl] = np.where(np.mod(sq[fl], 2) == 0, FLOOR[0], FLOOR[1])[:, None]
        ndl = np.maximum(n_ref @ LIGHT, 0.0)
        # every other outcome an fp32 cast could reach: faces within TOL of the ray's edge test, surfaces within TOL of the nearest
        amb_edge = np.zeros(N, bool)
        near = (np.abs(mb) < TOL) | (np.abs(t - t_ref[ray]) < TOL * np.maximum(t_ref[ray], 1))
        near &= (t < t_ref[ray] + TOL * np.maximum(t_ref[ray], 1)) & ~((mb >= TOL) & (t == t_ref[ray]))
        level = _level(base, ndl)
        for k in np.nonzero(near)[0]:
            j = ray[k]
            if amb_edge[j]:
                continue
            alt_lab = 2 + slot[k]
            alt_base = BODY[1] if alt_lab >= 26 else BODY[0]
            alt_lvl = _level(alt_base, max(nrm[k] @ LIGHT, 0.0))
            deep = abs(t[k] - t_ref[j]) > TOL * max(t_ref[j], 1) if np.isfinite(t_ref[j]) else True
            amb_edge[j] = alt_lab != lab[j] or np.abs(alt_lvl - level[j]).max() >= 1 or deep
        parts["edge"] = amb_edge
        # the floor against a surface within TOL
        with np.errstate(invalid="ignore"):
            parts["depth"] = (lab >= 2) & floor & (np.abs(tf - t_ref) < TOL * np.maximum(t_ref, 1))
        fr = np.full(N, np.inf)
        fr[fl] = np.abs(p[fl, :2] - np.round(p[fl, :2])).min(1)
        parts["checker"] = fl & (fr < TOL * np.maximum(t_ref, 1))
        # shadow rays from the lit surface points
        lit = np.ones(N, bool)
        sh_amb = np.zeros(N, bool)
        sh = np.nonzero((lab > 0) & (ndl > 0))[0]
        if len(sh):
            sr, _, _, st, smb, _ = _cast(groups, p[sh], np.broadcast_to(LIGHT, (len(sh), 3)).copy(), EPS)
            certain = (smb > TOL) & (st > EPS + TOL)
            lit[sh[np.unique(sr[certain])]] = False
            unsure = np.zeros(len(sh), bool)
            unsure[sr[~certain]] = True
            sh_amb[sh[unsure & lit[sh]]] = True
        parts["shadow"] = sh_amb & (ndl * DIFFUSE * 255 >= 0.5)
        ndl = np.where(lit, ndl, 0.0)
        col = np.where((lab == 0)[:, None], SKY, base * (AMBIENT + DIFFUSE * ndl)[:, None])
        rgb = np.floor(np.clip(col, 0, 1) * 255 + 0.5).astype(np.uint8)
        amb = parts["far"] | parts["edge"] | parts["depth"] | parts["checker"] | parts["shadow"]
        out["rgb"].append(rgb.reshape(H, W, 3))
        out["depth"].append(t_ref.reshape(H, W))
        out["label"].append(lab.reshape(H, W))
        out["amb"].append(amb.reshape(H, W))
        out["parts"].append({k: v.reshape(H, W) for k, v in parts.items()})
    res = {k: np.stack(v) for k, v in out.items() if k != "parts"}
    res["parts"] = out["parts"]
    return res
