"""CPU: pins the fp64 reference ray caster (tests/render_ref.py) the renderer is compared against -- hits lie on their hull's boundary, the
floor is the analytic ray-plane intersection with its checker colour, the covered pixels are those inside the bodies' projected hulls --
and the renderer's plane tables (HumanoidModel.render_struct) against the hull vertices, for every shape variant."""
import os

import numpy as np
import pytest
from scipy.spatial import ConvexHull

from tests import render_ref as RF
from uhc_b200.model import HumanoidModel


def poses():
    """standing, crouching and mid-fall poses from the golden clips (the humanoid), and golden frames (the ghost)"""
    g = os.path.join(os.path.dirname(__file__), "golden")
    sway, kick = np.load(os.path.join(g, "expert_sway.npz"))["qpos"], np.load(os.path.join(g, "expert_kick.npz"))["qpos"]
    stand = sway[0].copy()
    crouch = sway[30].copy()
    crouch[2] -= 0.35
    names = HumanoidModel().body_names
    for n, ang in (("L_Hip", -1.4), ("R_Hip", -1.4), ("L_Knee", 1.8), ("R_Knee", 1.8)):     # body b's hinges z, y, x at 7 + 3 (b - 1)
        crouch[7 + 3 * (names.index(n) - 1) + 2] += ang
    fall = kick[35].copy()
    c, s = np.cos(0.6), np.sin(0.6)
    q = fall[3:7]
    fall[3:7] = [c * q[0] - s * q[1], c * q[1] + s * q[0], c * q[2] - s * q[3], c * q[3] + s * q[2]]   # tilted 69 degrees about x
    fall[2] = 0.45
    return np.stack([stand, crouch, fall]), np.stack([sway[60], kick[10], kick[60]])


def table(model, qa, qb):
    P = np.zeros((len(qa), 2, 24, 12))
    P[:, 0], P[:, 1] = RF.pose_table(qa, model), RF.pose_table(qb, model)
    return P


@pytest.fixture(scope="module")
def rendered():
    m = HumanoidModel()
    qa, qb = poses()
    cam = dict(distance=3.5, shift_expert=0.8)
    return m, table(m, qa, qb), cam, RF.render(table(m, qa, qb), m, (160, 90), cam)


def test_hits_lie_on_the_hull_boundary(rendered):
    m, P, cam, r = rendered
    sl, pl, pt = r["slot"], r["plane"], r["point"]
    assert (sl >= 0).sum() > 500
    for i in range(len(P)):
        for j in np.unique(sl[i][sl[i] >= 0]):
            msk = sl[i] == j
            R, p = P[i, j // 24, j % 24, :9].reshape(3, 3), P[i, j // 24, j % 24, 9:].copy()
            if j >= 24:
                p[0] += cam["shift_expert"]
            xb = (pt[i][msk] - p) @ R                     # body frame
            eq = r["planes"][j % 24]
            val = xb @ eq[:, :3].T + eq[:, 3]
            k = pl[i][msk]
            assert (k >= 0).all()
            assert np.abs(val[np.arange(len(k)), k]).max() <= 1e-9
            assert val.max() <= 1e-9


def test_floor_is_the_analytic_intersection_with_its_checker(rendered):
    m, P, cam, r = rendered
    W, H = 160, 90
    off, f, rr, u = RF.camera(cam, W, H)
    eye = np.array([0.0, 0.0, 1.0]) + off
    fl = r["label"] == 1
    assert fl.sum() > 1000
    ys, xs = np.nonzero(fl[0])
    d = f + (2 * (xs + 0.5) / W - 1)[:, None] * rr + (1 - 2 * (ys + 0.5) / H)[:, None] * u
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    t = -eye[2] / d[:, 2]
    assert np.allclose(r["depth"][0][ys, xs], t, rtol=1e-12, atol=0)
    hit = eye + t[:, None] * d
    assert np.abs(hit[:, 2]).max() <= 1e-12
    sq = (np.floor(hit[:, 0]) + np.floor(hit[:, 1])) % 2
    want = np.where(sq == 0, RF.FLOOR[0], RF.FLOOR[1])
    shade = r["colour"][0][ys, xs, 0] / want
    # lit floor: ambient + diffuse * L_z; shadowed floor: ambient only
    assert np.all(np.isclose(shade, RF.AMBIENT + RF.DIFFUSE * RF.LIGHT[2]) | np.isclose(shade, RF.AMBIENT))
    assert np.isclose(shade, RF.AMBIENT).sum() > 20        # the humanoids cast shadows


def test_coverage_matches_projected_hulls(rendered):
    m, P, cam, r = rendered
    W, H = 160, 90
    off, f, rr, u = RF.camera(cam, W, H)
    eye = np.array([0.0, 0.0, 1.0]) + off
    verts = RF.hull_verts(m)
    for i in range(len(P)):
        inside_any = np.zeros((H, W), bool)
        deep = np.zeros((H, W), bool)
        ys, xs = np.mgrid[0:H, 0:W]
        c = np.stack([xs.ravel() + 0.5, ys.ravel() + 0.5], 1)
        for h in range(2):
            for b in range(24):
                R, p = P[i, h, b, :9].reshape(3, 3), P[i, h, b, 9:].copy()
                if h:
                    p[0] += cam["shift_expert"]
                v = verts[b] @ R.T + p - eye
                z = v @ f
                x = (v @ rr) / (rr @ rr) / z
                y = (v @ u) / (u @ u) / z
                px = np.stack([(x + 1) * W / 2, (1 - y) * H / 2], 1)
                eq = ConvexHull(px).equations                         # n . c + d <= 0 inside, |n| = 1 (pixels)
                s = c @ eq[:, :2].T + eq[:, 2]
                inside_any |= (s.max(1) <= 1e-6).reshape(H, W)
                deep |= (s.max(1) < -1.0).reshape(H, W)
        cov = r["label"][i] >= 2
        assert deep.sum() > 50
        assert cov[deep].all()
        assert not (cov & ~inside_any).any()


@pytest.mark.parametrize("scale_seed", [None, 3, 7])
def test_plane_tables_hold_every_hull_vertex(scale_seed):
    base = HumanoidModel()
    models = [base] + ([HumanoidModel(scale=np.random.default_rng(scale_seed).uniform(0.85, 1.2, 24))] if scale_seed else [])
    base.render_struct(models)
    k = base._rkeep
    assert k["plane"].shape[1] == k["num"].sum() and (k["num"] >= 4).all()
    assert k["plane"].shape[1] * 16 < 48 * 1024
    for s, m in enumerate(models):
        pl = k["plane"][s]
        assert np.allclose(np.linalg.norm(pl[:, :3], axis=1), 1, atol=1e-12)
        for b in range(24):
            v = m.hull[m.hull_adr[b]:m.hull_adr[b] + m.hull_num[b]]
            e = pl[k["adr"][b]:k["adr"][b] + k["num"][b]]
            val = v @ e[:, :3].T + e[:, 3]
            assert val.max() <= 1e-12
            assert (np.abs(val) <= 1e-9).sum(0).min() >= 3        # every plane carries a face: at least three hull vertices on it
        sph = k["sphere"][s]
        for b in range(24):
            v = m.hull[m.hull_adr[b]:m.hull_adr[b] + m.hull_num[b]]
            assert np.linalg.norm(v - sph[b, :3], axis=1).max() < sph[b, 3]
