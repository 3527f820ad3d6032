"""Synthetic mesh scenes for the mesh renderer's tests and timing (TEST INFRASTRUCTURE).  A real SMPL file is licence-gated, so:
  - hull_mesh: the humanoid's convex body hulls triangulated (ConvexHull.simplices), posed by the hull renderer's pose table; these surfaces
    are the hulls, so the mesh renderer's labels must equal the hull renderer's;
  - smpl_sized_model: tests/test_gpu_mesh.py's synthetic SMPL model (the neutral humanoid's hull vertices at rest, skinned to the owning joint
    and its parent) with the hulls' triangles, refined by longest-edge bisection to SMPL's 6890 vertices and topped up to SMPL's 13 776 faces
    with copies of its largest faces (24 closed surfaces have 92 faces fewer than one closed surface of as many vertices)."""
import heapq

import numpy as np
from scipy.spatial import ConvexHull

from uhc_b200.model import HumanoidModel


def hull_mesh(model=None):
    """(body-frame vertices [V][3], faces [F][3], vertex body [V], weights [V][24] one-hot on the body's SMPL joint)"""
    m = model or HumanoidModel()
    verts, faces, owner = [], [], []
    o = 0
    for b in range(24):
        v = m.hull[m.hull_adr[b]:m.hull_adr[b] + m.hull_num[b]]
        faces.append(ConvexHull(v).simplices + o)
        verts.append(v); owner += [b] * len(v)
        o += len(v)
    owner = np.array(owner)
    w = np.zeros((o, 24))
    w[np.arange(o), [HumanoidModel.SMPL_BONE_ORDER.index(m.body_names[b]) for b in owner]] = 1.0
    return np.concatenate(verts), np.concatenate(faces).astype(np.int32), owner, w


def pose_verts(P, verts, owner):
    """pose table [n][2][24][12] (fp32 values) -> world vertices [n][2][V][3] fp32, world = R v + p in fp64 rounded once"""
    P = np.asarray(P, np.float64)
    R = P[:, :, owner, :9].reshape(P.shape[0], 2, len(owner), 3, 3)
    return (np.einsum("nhvij,vj->nhvi", R, verts) + P[:, :, owner, 9:]).astype(np.float32)


def smpl_sized_model(V=6890, F=13776, seed=0):
    from tests.test_gpu_mesh import humanoid_model
    m = humanoid_model(seed)
    vt = m["v_template"]
    owner = np.argmax(m["weights"], axis=1)                 # 0.7 on the owning joint, 0.3 on its parent
    faces = []
    for j in range(24):
        idx = np.nonzero(owner == j)[0]
        faces.append(idx[ConvexHull(vt[idx]).simplices])
    faces = [tuple(int(x) for x in f) for f in np.concatenate(faces)]
    attrs = {k: list(m[k]) for k in ("v_template", "shapedirs", "posedirs", "weights")}
    alive = set(range(len(faces)))
    edge_faces = {}
    for i, f in enumerate(faces):
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
            edge_faces.setdefault((min(a, b), max(a, b)), set()).add(i)
    heap = [(-np.linalg.norm(vt[a] - vt[b]), a, b) for (a, b) in edge_faces]
    heapq.heapify(heap)
    while len(attrs["v_template"]) < V:
        _, a, b = heapq.heappop(heap)
        if (a, b) not in edge_faces:
            continue
        c = len(attrs["v_template"])
        for k in attrs:
            attrs[k].append((np.asarray(attrs[k][a]) + np.asarray(attrs[k][b])) / 2)
        for i in sorted(edge_faces.pop((a, b))):
            f = faces[i]
            alive.discard(i)
            k = f.index(a) if f.index(a) == (f.index(b) + 1) % 3 else f.index(b)   # the edge's second vertex in the face's winding
            x, y, z = f[(k + 2) % 3], f[k], f[(k + 1) % 3]      # winding x -> y -> z with edge (x, y)
            for nf in ((x, c, z), (c, y, z)):
                faces.append(nf); alive.add(len(faces) - 1)
                for p, q in ((nf[0], nf[1]), (nf[1], nf[2]), (nf[2], nf[0])):
                    e = (min(p, q), max(p, q))
                    edge_faces.setdefault(e, set()).discard(i)
                    edge_faces[e].add(len(faces) - 1)
            for p in (x, y):
                e = (min(p, z), max(p, z))
                edge_faces[e].discard(i)
        pa, pb, pc = np.asarray(attrs["v_template"][a]), np.asarray(attrs["v_template"][b]), np.asarray(attrs["v_template"][c])
        for p, q, pp, pq in ((a, c, pa, pc), (c, b, pc, pb)):
            heapq.heappush(heap, (-np.linalg.norm(pp - pq), min(p, q), max(p, q)))
    fa = np.array([faces[i] for i in sorted(alive)], np.int32)
    area = np.linalg.norm(np.cross(np.asarray(attrs["v_template"])[fa[:, 1]] - np.asarray(attrs["v_template"])[fa[:, 0]],
                                   np.asarray(attrs["v_template"])[fa[:, 2]] - np.asarray(attrs["v_template"])[fa[:, 0]]), axis=1)
    fa = np.concatenate([fa, fa[np.argsort(-area, kind="stable")[:F - len(fa)]]])
    out = {k: np.asarray(v, np.float64) for k, v in attrs.items()}
    out.update(J_regressor=np.concatenate([m["J_regressor"], np.zeros((24, V - len(vt)))], 1), parents=m["parents"], faces=fa)
    return out


def seam_rays(tb, verts, owner, n_edges=600, n_verts=300, seed=0):
    """the points of a closed mesh where a leaf box could lose a ray: points along edges whose two faces lie in different leaves, and vertices
    whose faces lie in two leaves or more, each with the camera that aims the one pixel of a 1 x 1 image at it from 1.5 m straight through the
    surface (along the inward mean of its faces' normals, oriented away from their body's centre: convex hulls).  Returns [(point, camera)]."""
    lf, face = tb["leaf_first"], tb["face"].astype(np.int64)
    leaf = np.searchsorted(lf, np.arange(len(face)), side="right") - 1
    tri = verts[face].astype(np.float64)
    n = np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0])
    n /= np.linalg.norm(n, axis=1, keepdims=True)
    centre = {b: verts[owner == b].astype(np.float64).mean(0) for b in np.unique(owner)}
    out_c = np.stack([centre[owner[f[0]]] for f in face])
    n = np.where(((tri.mean(1) - out_c) * n).sum(1, keepdims=True) < 0, -n, n)
    edges, vfaces = {}, {}
    for i, f in enumerate(face):
        for a, b in ((f[0], f[1]), (f[1], f[2]), (f[2], f[0])):
            edges.setdefault((min(a, b), max(a, b)), []).append(i)
        for v in f:
            vfaces.setdefault(int(v), []).append(i)
    seams = [(e, fs) for e, fs in edges.items() if len(fs) == 2 and leaf[fs[0]] != leaf[fs[1]]]
    corners = [(v, fs) for v, fs in vfaces.items() if len(set(leaf[fs])) > 1]
    rng = np.random.default_rng(seed)
    targets = []
    for k in rng.permutation(len(seams))[:n_edges]:
        (a, b), fs = seams[k]
        for s in (0.5, 1e-3, 0.3):
            targets.append(((1 - s) * verts[a].astype(np.float64) + s * verts[b], n[fs].sum(0)))
    for k in rng.permutation(len(corners))[:n_verts]:
        v, fs = corners[k]
        targets.append((verts[v].astype(np.float64), n[fs].sum(0)))
    rays = []
    for p, m in targets:
        fwd = -m / np.linalg.norm(m)
        cam = dict(lookat=tuple(p), distance=1.5, fovy=1.0, azimuth=float(np.degrees(np.arctan2(fwd[1], fwd[0]))),
                   elevation=float(np.degrees(np.arcsin(np.clip(fwd[2], -1, 1)))))
        rays.append((p, cam))
    return rays


def cube_mesh(n=8, lo=(-0.2137, 0.1311, 0.3173), size=0.4719):
    """a closed axis-aligned cube of n x n cells per side, two triangles per cell, every face owned by body 0: a leaf inside one side is flat,
    so its box has zero thickness and a seam between two such leaves lies on both boxes' edges -- where a box test without margin loses rays.
    Returns hull_mesh's (vertices, faces, vertex body, weights)."""
    idx, verts, faces = {}, [], []

    def vid(g):
        if g not in idx:
            idx[g] = len(verts)
            verts.append(np.asarray(lo) + size * np.asarray(g, np.float64) / n)
        return idx[g]

    for axis in range(3):
        for side in (0, n):
            for i in range(n):
                for j in range(n):
                    def g(a, b):
                        c = [0, 0, 0]
                        c[axis], c[(axis + 1) % 3], c[(axis + 2) % 3] = side, a, b
                        return tuple(c)
                    q = [vid(g(i, j)), vid(g(i + 1, j)), vid(g(i + 1, j + 1)), vid(g(i, j + 1))]
                    faces += [(q[0], q[1], q[2]), (q[0], q[2], q[3])]
    V = len(verts)
    w = np.zeros((V, 24))
    w[:, 0] = 1.0
    return np.array(verts, np.float32), np.array(faces, np.int32), np.zeros(V, np.int64), w
