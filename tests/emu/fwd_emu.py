"""ctypes wrapper of fwd_emu.cpp: one fp32 forward pass of the step kernel's smooth phase (kin_rne_forward, project_force, collide) in the
host emulation, and the poses its golden fixture pins (TEST INFRASTRUCTURE).

  python -m tests.emu.fwd_emu --write     rewrites tests/golden/fwd_pass_fp32.npz from the current sources

The fixture was written from the sources before the forward pass was restructured; tests/test_emu_fwd_golden.py asserts that the current
sources give the same bytes.
"""
import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_fwd_emu.so")
GOLDEN = os.path.join(_HERE, "..", "golden", "fwd_pass_fp32.npz")
NB, NV, MAXCON = 24, 75, 40
FLOATS = (("xpos", (NB, 3)), ("xmat", (NB, 9)), ("xipos", (NB, 3)), ("S", (NV, 6)), ("Vb", (NB, 6)), ("Ab", (NB, 6)), ("Ib", (NB, 10)),
          ("Fb", (NB, 6)), ("C", (NV,)), ("cdist", (MAXCON,)), ("cr", (MAXCON, 3)))
INTS = (("cbody", (MAXCON,)), ("bcon_adr", (NB + 1,)), ("ncon", ()), ("upper_contact", ()), ("con_overflow", ()))
_BASE = np.array([0.7071068, 0.7071068, 0.0, 0.0])      # the upright root orientation of the Z-up world


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    srcs = [os.path.join(_HERE, "fwd_emu.cpp"), os.path.join(_HERE, "emu.cpp"), os.path.join(csrc, "sim_core.h"), os.path.join(csrc, "env_step.h"),
            os.path.join(_HERE, "..", "..", "include", "uhc_b200.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _n(shape):
    return int(np.prod(shape)) if shape else 1


class FwdEmu:
    def __init__(self, model):
        from tests.emu.emu import default_cfg
        self.lib = C.CDLL(build())
        self.lib.emu_create.restype = C.c_void_p
        self.model = model
        self._ms = model.host_struct()
        self._cfg = default_cfg(32)
        self.h = C.c_void_p(self.lib.emu_create(C.byref(self._ms), C.byref(self._cfg), C.c_int(1), C.c_int(32)))

    def close(self):
        self.lib.emu_destroy(self.h, 32)

    def run(self, qpos, qvel):
        f = np.zeros(sum(_n(s) for _, s in FLOATS), np.float32)
        i = np.zeros(sum(_n(s) for _, s in INTS), np.int32)
        q, v = np.ascontiguousarray(qpos, np.float64), np.ascontiguousarray(qvel, np.float64)
        self.lib.emu_fwd_pass(self.h, q.ctypes.data_as(C.POINTER(C.c_double)), v.ctypes.data_as(C.POINTER(C.c_double)),
                              f.ctypes.data_as(C.POINTER(C.c_float)), i.ctypes.data_as(C.POINTER(C.c_int)))
        out, o = {}, 0
        for k, s in FLOATS:
            out[k] = f[o:o + _n(s)].reshape(s); o += _n(s)
        o = 0
        for k, s in INTS:
            out[k] = i[o:o + _n(s)].reshape(s); o += _n(s)
        return out


def _qmul(a, b):
    return np.array([a[0] * b[0] - a[1:] @ b[1:], *(a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:]))])


def _axis_angle(v):
    ang = np.linalg.norm(v) + 1e-300
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * v / ang])


def tie_model():
    """the base model with, in every hull, more vertices at the height of the lowest and of the highest one (body frame z): under a rotation whose last row is
    exactly (0, 0, 1) the narrow phase's deepest vertex is a tie, decided by the lower vertex index"""
    from uhc_b200.model import HumanoidModel
    m = HumanoidModel()
    hull = m.hull.copy()
    for b in range(NB):
        a, n = int(m.hull_adr[b]), int(m.hull_num[b])
        z = hull[a:a + n, 2]
        for i in (int(np.argmin(z)), int(np.argmax(z))):   # lowest under z = +(body z), highest under z = -(body z)
            hull[a + (i + 33) % n, 2] = z[i]          # a vertex another lane scans (index +33 mod n)
            hull[a + (i + 5) % n, 2] = z[i]           # and one the same lane or a neighbouring one scans
    m.hull = hull
    return m


def cases():
    """(name, model key, qpos, qvel): the seeded states of tests/step_corpus.py's regimes, and crafted poses for what those may not reach:
    lying flat (every body a candidate, the 40 contact slots overflow), hands and head on the floor (upper_contact), an upper body near the
    floor whose deepest vertex is above the margin, and exact deepest-vertex ties"""
    from tests import step_corpus as SC
    s = SC.setup("base")
    out = []
    rng = np.random.default_rng(7)
    for r in SC.REGIMES:
        for k in range(6):
            c = SC._case(s, rng, r)
            out.append(("%s_%d" % (r, k), "base", c["qpos"], c["qvel"]))
    q0 = s.clips[0]["qpos"][0].copy()
    f32 = SC.f32
    for k, h in enumerate(np.linspace(0.02, 0.30, 8)):         # lying on the back, then on the front, root lowered step by step
        for side, ang in (("back", -np.pi / 2), ("front", np.pi / 2)):
            q = q0.copy()
            q[2] = h
            q[3:7] = _qmul(_axis_angle(np.array([0.0, ang, 0.0])), _BASE)
            q[7:] = rng.normal(0, 0.05, 69)
            out.append(("flat_%s_%d" % (side, k), "base", f32(q), f32(rng.normal(0, 0.5, 75))))
    for k, h in enumerate(np.linspace(0.55, 0.95, 9)):          # bent forward at the hips, arms down: hands (and head) reach the floor
        q = q0.copy()
        q[2] = h
        q[3:7] = _qmul(_axis_angle(np.array([0.0, np.deg2rad(75.0 + 3 * k), 0.0])), _BASE)
        q[7:] = rng.normal(0, 0.05, 69)
        out.append(("hands_%d" % k, "base", f32(q), f32(rng.normal(0, 0.5, 75))))
    for k, h in enumerate(np.linspace(0.6, 1.3, 8)):            # upside down: head and hands first, above and below the margin
        q = q0.copy()
        q[2] = h
        q[3:7] = _qmul(_axis_angle(np.array([np.pi, 0.0, 0.0])), _BASE)
        q[7:] = rng.normal(0, 0.05, 69)
        out.append(("inverted_%d" % k, "base", f32(q), f32(rng.normal(0, 0.5, 75))))
    for k, (quat, h) in enumerate(((0, 0.0), (0, 0.06), (1, 0.0), (1, 0.1), (2, 0.0), (3, 0.0), (3, 0.12))):
        q = np.zeros(76)                                        # all hinges at 0 and an axis-aligned root: every body frame is exactly the identity
        q[3 + quat] = 1.0                                       # or diag(+-1): z is +-(body-frame z) exactly, so the doctored vertices tie
        q[2] = h
        out.append(("tie_%d" % k, "tie", q, np.zeros(75)))
    return out


def run_cases():
    from uhc_b200.model import HumanoidModel
    emus = {"base": FwdEmu(HumanoidModel()), "tie": FwdEmu(tie_model())}
    res = {}
    names = []
    for name, key, q, v in cases():
        names.append(name)
        for k, x in emus[key].run(q, v).items():
            res.setdefault(k, []).append(x)
    for e in emus.values():
        e.close()
    return names, {k: np.stack(v) for k, v in res.items()}


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        sys.exit(__doc__)
    names, res = run_cases()
    np.savez_compressed(GOLDEN, names=np.array(names), **res)
    print("wrote %s: %d poses, ncon %s, overflow %d, upper %d" % (GOLDEN, len(names), np.bincount(res["ncon"]).nonzero()[0].tolist(),
                                                                  int(res["con_overflow"].sum()), int(res["upper_contact"].sum())))
