"""Every clip's own body: humanoid shape variants built on the GPU from SMPL beta and gender (include/uhc_subject.h).

The reference rebuilds its MuJoCo humanoid for every clip from the clip's beta and gender (HumanoidEnv.reset_robot ->
Robot.load_from_skeleton): joints from the SMPL J_regressor, each body the decimated convex hull of the vertices skinned to it.  That hull
has a topology of its own per subject, and the engine needs one hull graph for all its shape variants.  So this module carries the shipped
neutral humanoid onto the subject with one affine map per body instead (DESIGN.md section 4, "Subject bodies"):

  S_j   the vertices whose largest skinning weight in the neutral model is SMPL joint j (the body's joint)
  P_i = Z (v_n(0)_i - J_n(0)_j), Q_i = Z (v_g(beta)_i - J_g(beta)_j), Z the y-up -> z-up rotation (x, y, z) -> (x, -z, y)
  (A, t) the least-squares solution of Q ~ A P + t over S_j

The design matrix [P 1] does not depend on beta, so (A, t) is affine in beta: SubjectBasis.from_models fits, once per gender and body, the
constant term and the 10 beta directions.  For the neutral gender the constant term is exactly (1, 0), so beta = 0 is the shipped body.
The body offset moves by the change of the SMPL joint difference, Z [(J_g(beta)_j - J_g(beta)_p) - (J_n(0)_j - J_n(0)_p)], which is affine
in beta as well.  SubjectBasis.build evaluates the bases and everything that follows on the device."""
import ctypes as C

import numpy as np

from uhc_b200.model import BODYF, NB, HumanoidModel

NBETA, NTERM = 10, 11
RANK_TOL = 1e-8         # a body's centred source points must have singular values >= RANK_TOL * the largest
GENDERS = ("neutral", "male", "female")     # gender codes 0, 1, 2 (dataset_amass_single._gender_code)


class UhcSubjectBasis(C.Structure):
    """C mirror: include/uhc_subject.h `UhcSubjectBasis`."""
    _fields_ = [("map", C.POINTER(C.c_double) * 3), ("offset", C.POINTER(C.c_double) * 3)]


def z_up(x):
    """SMPL's y-up frame -> the model's z-up frame: (x, y, z) -> (x, -z, y)"""
    x = np.asarray(x, np.float64)
    return np.stack([x[..., 0], -x[..., 2], x[..., 1]], -1)


def subject_key(beta, gender):
    """what identifies a subject: beta[:10] (-0 read as 0) and the gender code"""
    return np.ascontiguousarray(np.asarray(beta, np.float64)[:NBETA] + 0.0).tobytes(), int(gender)


class SubjectBasis:
    """The per-gender bases of include/uhc_subject.h for one humanoid: map[g] [24][11][3][4] and offset[g] [24][11][3] (model body order),
    None for a gender without a model."""

    def __init__(self, humanoid, maps, offsets):
        self.humanoid, self.map, self.offset = humanoid, maps, offsets

    @classmethod
    def from_models(cls, humanoid, neutral, male=None, female=None):
        """fits the bases from SMPL model dicts as uhc_b200.smpl_model.load_smpl_model returns them.  ValueError when the models' vertex
        counts differ, or when a body's source points are rank deficient (naming its joint)."""
        models = [neutral, male, female]
        V = len(neutral["v_template"])
        for g, m in enumerate(models):
            if m is not None and len(m["v_template"]) != V:
                raise ValueError(f"subject bodies: the {GENDERS[g]} SMPL model has {len(m['v_template'])} vertices, the neutral one {V}: "
                                 "the models must share one mesh")
        joint = [HumanoidModel.SMPL_BONE_ORDER.index(n) for n in humanoid.body_names]          # SMPL joint of every model body
        pj = [-1] + [joint[int(humanoid.parent[b])] for b in range(1, NB)]
        owner = np.argmax(np.asarray(neutral["weights"], np.float64), axis=1)
        Jn = np.asarray(neutral["J_regressor"], np.float64) @ np.asarray(neutral["v_template"], np.float64)
        vn = np.asarray(neutral["v_template"], np.float64)
        pinv = []
        for b in range(NB):
            j = joint[b]
            idx = np.flatnonzero(owner == j)
            P = z_up(vn[idx] - Jn[j])
            sv = np.linalg.svd(P - P.mean(0), compute_uv=False) if len(idx) >= 4 else np.zeros(3)
            if len(sv) < 3 or not sv[2] >= RANK_TOL * sv[0]:
                raise ValueError(f"subject bodies: the vertices of SMPL joint {HumanoidModel.SMPL_BONE_ORDER[j]} (model body {b}) span less "
                                 f"than three dimensions (singular values {sv}, threshold {RANK_TOL:g} x the largest): no affine map fits them")
            pinv.append((idx, np.linalg.pinv(np.hstack([P, np.ones((len(idx), 1))]))))         # [4][k]
        maps, offs = [None] * 3, [None] * 3
        for g, m in enumerate(models):
            if m is None:
                continue
            vt, sd, Jr = (np.asarray(m[k], np.float64) for k in ("v_template", "shapedirs", "J_regressor"))
            J0, dJ = Jr @ vt, np.einsum("jv,vcl->ljc", Jr, sd[:, :, :NBETA])                  # [24][3], [10][24][3]
            mp, of = np.zeros((NB, NTERM, 3, 4)), np.zeros((NB, NTERM, 3))
            for b in range(NB):
                j, p = joint[b], pj[b]
                idx, pi = pinv[b]
                terms = [z_up(vt[idx] - J0[j])] + [z_up(sd[idx, :, l] - dJ[l, j]) for l in range(NBETA)]
                for k, Q in enumerate(terms):
                    mp[b, k] = (pi @ Q).T                                                       # (A | t): Q^T = [A t] [P 1]^T
                rel = (lambda J: J[j] - J[p]) if p >= 0 else (lambda J: J[j])
                of[b, 0] = z_up(rel(J0) - rel(Jn))
                for l in range(NBETA):
                    of[b, 1 + l] = z_up(rel(dJ[l]))
            if g == 0:                         # beta = 0 neutral is the shipped body exactly
                mp[:, 0] = np.hstack([np.eye(3), np.zeros((3, 1))])
                of[:, 0] = 0.0
            maps[g], offs[g] = mp, of
        return cls(humanoid, maps, offs)

    def struct(self):
        """ctypes UhcSubjectBasis (arrays kept alive on self)"""
        s = UhcSubjectBasis()
        self._keep = []
        for g in range(3):
            if self.map[g] is None:
                continue
            m, o = np.ascontiguousarray(self.map[g], np.float64), np.ascontiguousarray(self.offset[g], np.float64)
            self._keep += [m, o]
            s.map[g], s.offset[g] = m.ctypes.data_as(C.POINTER(C.c_double)), o.ctypes.data_as(C.POINTER(C.c_double))
        return s

    def bodies(self, betas, genders, device=0):
        """uhc_subject_bodies on `device` for every row: (body_f [n][24][20], hull [n][nvert][3], maps [n][24][3][4]).  ValueError for a
        refused row (the library's text)."""
        from uhc_b200.engine import _chk, load_library
        b = np.ascontiguousarray(np.asarray(betas, np.float64).reshape(len(genders), -1)[:, :NBETA])
        g = np.ascontiguousarray(genders, np.int32)
        n, hm = len(g), self.humanoid
        bf, hull, mp = np.zeros((n, NB, BODYF)), np.zeros((n, len(hm.hull), 3)), np.zeros((n, NB, 3, 4))
        had = getattr(hm, "_keep", None)                 # an engine's host_struct of the humanoid keeps its arrays there
        base, basis = hm.host_struct(), self.struct()
        keep, hm._keep = hm._keep, had
        d = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
        _chk(load_library().uhc_subject_bodies(C.c_int(device), C.byref(base), C.byref(basis), C.c_int(n), d(b), g.ctypes.data_as(C.POINTER(C.c_int)),
                                               d(bf), d(hull), d(mp)), "uhc_subject_bodies", ValueError)
        del keep
        return bf, hull, mp

    def build(self, betas, genders, device=0):
        """shape variants for rows of beta (the first 10 of each row are used) and gender code: (variants, index per row).  Identical
        (beta[:10], gender) rows share a variant; variant 0 is the humanoid itself, which beta = 0 neutral rows map to."""
        b = np.asarray(betas, np.float64).reshape(len(genders), -1)[:, :NBETA]
        g = np.asarray(genders).astype(np.int64).reshape(-1)
        if not np.isfinite(b).all():
            raise ValueError(f"subject bodies: row {int(np.flatnonzero(~np.isfinite(b).all(1))[0])} has a non-finite beta")
        for r, c in enumerate(g):
            if not 0 <= c <= 2 or self.map[c] is None:
                raise ValueError(f"subject bodies: row {r} has gender code {c}, which has no SMPL model")
        keys, index, order = {subject_key(np.zeros(NBETA), 0): 0}, np.zeros(len(g), np.int32), []
        for r in range(len(g)):
            k = subject_key(b[r], g[r])
            if k not in keys:
                keys[k] = len(keys)
                order.append(r)
            index[r] = keys[k]
        variants = [self.humanoid]
        if order:
            bf, hull, mp = self.bodies(b[order], g[order], device)
            variants += [HumanoidModel.from_tables(self.humanoid, bf[i], hull[i], mp[i]) for i in range(len(order))]
        return variants, index
