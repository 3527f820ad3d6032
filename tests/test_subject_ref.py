"""CPU: the subject body builder's rules (tests/subject_ref.py, uhc_b200/subject_body.py) and the host emulation of its per-item code
(uhc_b200/csrc/subject_core.h): uniform scale against HumanoidModel(scale=), the closed-form mass properties against the polytope
integrals of tools/compile_model.py, beta = 0 neutral as the shipped tables, the refusals, and the emulation against the restatement."""
import os

import numpy as np
import pytest
from scipy.spatial import ConvexHull

from tests.subject_ref import gendered, mapped_mass, subject_body, uniform_scale_model
from uhc_b200.model import HumanoidModel
from uhc_b200.subject_body import SubjectBasis

REL = 1e-12


@pytest.fixture(scope="module")
def hm():
    return HumanoidModel()


@pytest.fixture(scope="module")
def models():
    n = uniform_scale_model()
    return n, gendered(n, 1), gendered(n, 2)


@pytest.fixture(scope="module")
def basis(hm, models):
    return SubjectBasis.from_models(hm, *models)


def _close(a, b, rel=REL, atol=0.0):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return np.all(np.abs(a - b) <= rel * np.maximum(np.abs(a), np.abs(b)) + atol)


@pytest.mark.parametrize("s", [0.8, 1.0, 1.23])
def test_uniform_scale_is_the_scaled_humanoid(hm, models, s):
    beta = np.zeros(10)
    beta[0] = s - 1.0
    bf, hull, maps = subject_body(hm, models[0], models[0], beta)
    ref = HumanoidModel(scale=[s] * 24)
    assert _close(maps[:, :, :3], s * np.eye(3)[None].repeat(24, 0), atol=1e-13) and np.abs(maps[:, :, 3]).max() < 1e-13
    want = ref.body_f.copy()
    want[0, 0:3] = s * hm.body_f[0, 0:3]                 # scale= keeps the root offset, the builder moves it with J[0]
    scale = np.abs(want).max(0)                          # per column: offsets near 0 are compared on the column's scale
    for c in range(19):
        assert np.all(np.abs(bf[:, c] - want[:, c]) <= REL * 10 * scale[c]), c
    assert _close(bf[:, 13], want[:, 13]) and _close(bf[:, 6], want[:, 6])
    assert np.abs(hull - ref.hull).max() <= REL * np.abs(ref.hull).max()


def test_closed_form_mass_properties_are_the_polytope_integrals():
    import sys
    sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
    from compile_model import poly_mass_props
    rng = np.random.RandomState(3)
    for _ in range(20):
        pts = rng.normal(0, 0.1, (30, 3))
        tri = pts[ConvexHull(pts).simplices]
        tri = np.where((np.einsum("ij,ij->i", np.cross(tri[:, 1] - tri[:, 0], tri[:, 2] - tri[:, 0]), tri[:, 0] - pts.mean(0)) < 0)[:, None, None],
                       tri[:, [0, 2, 1]], tri)         # outward orientation
        vol, com, I = poly_mass_props(tri)
        m, c, I = 1000.0 * vol, com, 1000.0 * I
        A = np.eye(3) + rng.normal(0, 0.3, (3, 3))
        if np.linalg.det(A) < 0:
            A[:, 0] *= -1
        t = rng.normal(0, 0.05, 3)
        m2, c2, I2 = mapped_mass(m, c, I, A, t)
        q = pts @ A.T + t
        tq = q[ConvexHull(q).simplices]
        tq = np.where((np.einsum("ij,ij->i", np.cross(tq[:, 1] - tq[:, 0], tq[:, 2] - tq[:, 0]), tq[:, 0] - q.mean(0)) < 0)[:, None, None],
                      tq[:, [0, 2, 1]], tq)
        v3, c3, I3 = poly_mass_props(tq)
        assert abs(m2 - 1000.0 * v3) <= 1e-12 * m2 and np.abs(c2 - c3).max() <= 1e-12 * (np.abs(c3).max() + 0.1)
        assert np.abs(I2 - 1000.0 * I3).max() <= 1e-12 * np.abs(I2).max()


def test_zero_beta_neutral_is_the_shipped_body(hm, basis):
    from tests.emu.subject_emu import subject_body as emu
    bf, hull, maps = emu(basis, np.zeros(10), 0)
    assert np.array_equal(maps, np.tile(np.hstack([np.eye(3), np.zeros((3, 1))]), (24, 1, 1)))
    assert np.array_equal(hull, hm.hull)
    cols = [c for c in range(20) if c != 13]
    assert np.array_equal(bf[:, cols], hm.body_f[:, cols])
    assert _close(bf[:, 13], hm.body_f[:, 13])


def test_basis_is_the_direct_fit(hm, models, basis):
    rng = np.random.RandomState(4)
    for g in range(3):
        beta = rng.uniform(-2, 2, 10)
        _, _, maps = subject_body(hm, models[0], models[g], beta)
        got = np.einsum("btij,t->bij", basis.map[g], np.concatenate([[1.0], beta]))
        assert np.abs(got - maps).max() < 1e-12


def test_emulation_matches_the_restatement(hm, models, basis):
    from tests.emu.subject_emu import subject_body as emu
    rng = np.random.RandomState(5)
    for g in (0, 1, 2, 1, 2):
        beta = rng.uniform(-2.5, 2.5, 10)
        beta[0] = rng.uniform(-0.3, 0.3)                                             # direction 0 scales the whole body by 1 + beta_0
        bf, hull, maps = emu(basis, beta, g)
        rb, rh, rm = subject_body(hm, models[0], models[g], beta)
        assert np.abs(maps - rm).max() < 1e-12
        assert np.abs(hull - rh).max() < 1e-14 + REL * np.abs(rh).max()
        scale = np.abs(rb).max(0) + 1e-300
        assert np.all(np.abs(bf - rb) <= 10 * REL * scale), np.abs(bf - rb).max(0) / scale
        assert _close(bf[:, 13], rb[:, 13], rel=1e-10) and _close(bf[:, 6], rb[:, 6])


def test_refusals(hm, models, basis):
    from tests.emu.subject_emu import subject_body as emu
    n = models[0]
    with pytest.raises(ValueError, match="vertices"):
        short = dict(n, v_template=n["v_template"][:-1])
        SubjectBasis.from_models(hm, n, short)
    flat = dict(n, v_template=n["v_template"].copy())
    owner = n["weights"].argmax(1)
    flat["v_template"][owner == hm.SMPL_BONE_ORDER.index("Head"), 2] = 0.0           # the head's vertices in one plane
    with pytest.raises(ValueError, match="Head"):
        SubjectBasis.from_models(hm, flat)
    beta = np.zeros(10)
    beta[0] = -1.5                                                                   # s = -0.5: every body mirrored through its joint
    with pytest.raises(ValueError, match="det A"):
        emu(basis, beta, 0)
    with pytest.raises(ValueError, match="det A"):
        subject_body(hm, n, n, beta)
    only_neutral = SubjectBasis.from_models(hm, n)
    with pytest.raises(ValueError, match="gender code 2"):
        only_neutral.build(np.zeros((2, 16)), [0, 2])
    with pytest.raises(ValueError, match="gender code 5"):
        basis.build(np.zeros((1, 16)), [5])
    bad = np.zeros((3, 16))
    bad[1, 4] = np.nan
    with pytest.raises(ValueError, match="row 1 has a non-finite beta"):
        basis.build(bad, [0, 1, 2])


def test_model_file_problems_are_named(tmp_path):
    from uhc_b200.smpl_model import load_smpl_model
    n = uniform_scale_model()
    kt = np.stack([np.where(n["parents"] < 0, 4294967295, n["parents"]), np.arange(24)]).astype(np.int64)
    keys = {k: v for k, v in n.items() if k not in ("parents", "J_regressor")}
    np.savez(tmp_path / "SMPL_MALE.npz", kintree_table=kt, **keys)
    with pytest.raises(ValueError, match="J_regressor"):
        load_smpl_model(str(tmp_path / "SMPL_MALE.npz"))


def test_dedup_needs_no_device(hm, basis):
    """rows that are all beta = 0 neutral map to variant 0 without a device call"""
    variants, idx = basis.build(np.zeros((5, 16)), [0] * 5)
    assert len(variants) == 1 and variants[0] is hm and np.array_equal(idx, np.zeros(5))
