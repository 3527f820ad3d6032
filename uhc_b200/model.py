"""Host-side model tables for the batched engine.

Loads the compiled humanoid (uhc_b200/assets/smpl_neutral_model.npz, produced by tools/compile_model.py from the
reference's humanoid_smpl_neutral_mesh.xml + STL hulls) and derives the topology tables the kernels index with:
depth-first dof numbering (root 6 dofs, then 3 hinges z,y,x per body), children lists, subtree ranges, and the per-tree-level
lane-group table of the articulated-body solve.
Mirrors what SMPLConverter exposes to the reference env (uhc/smpllib/smpl_mujoco.py:259-281): kp/kd/torque-limit/diff-weight.
"""
import ctypes as C
import os

import numpy as np

ASSET = os.path.join(os.path.dirname(os.path.abspath(__file__)), "assets", "smpl_neutral_model.npz")
NB, NQ, NV, NU = 24, 76, 75, 69
BODYF = 20


class UhcModelHost(C.Structure):
    """C mirror: include/uhc_b200.h `UhcModelHost`."""
    _fields_ = [("nvert", C.c_int), ("nnbr", C.c_int),
                ("body_f", C.POINTER(C.c_double)), ("dof_f", C.POINTER(C.c_double)), ("hull", C.POINTER(C.c_double)),
                ("hull_adr", C.POINTER(C.c_int)), ("hull_num", C.POINTER(C.c_int)), ("nbr", C.POINTER(C.c_int)),
                ("nbradr", C.POINTER(C.c_int)), ("parent", C.POINTER(C.c_int)), ("depth", C.POINTER(C.c_int)),
                ("child_adr", C.POINTER(C.c_int)), ("child", C.POINTER(C.c_int)), ("body_sub_end", C.POINTER(C.c_int)),
                ("ee", C.POINTER(C.c_int)),
                ("lvl_tab", C.POINTER(C.c_int)), ("lvl_pack", C.POINTER(C.c_int)),
                ("dt", C.c_double), ("margin", C.c_double), ("mu", C.c_double), ("solref", C.c_double * 2),
                ("solimp", C.c_double * 5), ("gravz", C.c_double), ("nshape", C.c_int), ("dof_lim", C.POINTER(C.c_double))]


class UhcRenderHulls(C.Structure):
    """C mirror: include/uhc_render.h `UhcRenderHulls`."""
    _fields_ = [("nshape", C.c_int), ("nplane", C.c_int), ("plane", C.POINTER(C.c_double)), ("plane_adr", C.POINTER(C.c_int)),
                ("plane_num", C.POINTER(C.c_int)), ("sphere", C.POINTER(C.c_double))]


class HumanoidModel:
    def __init__(self, npz=ASSET, scale=None, jnt_range=None):
        """jnt_range: optional [69][2] hinge limits in radians overriding the model's (xml: +-180 deg on every hinge; smpl_robot.py:1087-1110 tightens
        knee / ankle ranges per shape)."""
        z = np.load(npz)
        self.z = {k: z[k] for k in z.files}
        self.body_names = [str(n) for n in z["body_names"]]
        self.parent = z["parent"].astype(np.int32)
        offset, ipos, mass, inertia = (z[k].astype(np.float64).copy() for k in ("body_offset", "body_ipos", "body_mass", "body_inertia"))
        hull = z["hull_vert"].astype(np.float64).copy()
        invw = z["body_invweight0"][:, 0].astype(np.float64).copy()
        self.hull_adr, self.hull_num = z["hull_vadr"].astype(np.int32), z["hull_vnum"].astype(np.int32)
        if scale is not None:  # synthetic body-shape variant: per-body isotropic limb scale (SURVEY section 8d config 4)
            s = np.asarray(scale, dtype=np.float64)
            offset[1:] *= s[self.parent[1:], None]   # bone offsets live in the parent's frame
            ipos *= s[:, None]
            mass *= s ** 3
            inertia *= (s ** 5)[:, None, None]
            for b in range(NB):
                hull[self.hull_adr[b]:self.hull_adr[b] + self.hull_num[b]] *= s[b]
            invw = None          # recomputed below from the scaled mass properties
        self.offset, self.ipos, self.mass, self.inertia, self.hull, self.invw = offset, ipos, mass, inertia, hull, invw
        self.diffw = z["diffw"].astype(np.float64)
        self.jkp, self.jkd, self.torque_lim = (z[k].astype(np.float64) for k in ("jkp", "jkd", "torque_lim"))
        self.armature = z["armature"].astype(np.float64)
        self.ee = z["ee_body"].astype(np.int32)
        self.nbr, self.nbradr = z["hull_nbr"].astype(np.int32), z["hull_nbradr"].astype(np.int32)
        self.dt = float(z["timestep"])
        self.margin, self.mu = float(z["margin"]), float(z["friction"])
        self.solref, self.solimp, self.gravz = z["solref"], z["solimp"], float(z["gravity"][2])
        self.qpos0 = np.zeros(NQ)
        self.qpos0[:3] = z["body_gpos"][0]
        self.qpos0[3] = 1.0
        self.root_offset = z["body_gpos"][0].copy()  # mj_model.body_pos[1] in smpl_to_qpose (count_offset)
        self.jnt_range = np.asarray(jnt_range if jnt_range is not None else z["jnt_range"], dtype=np.float64).reshape(NV - 6, 2)
        self.dof_invweight0 = z["dof_invweight0"].astype(np.float64)
        self._topology()
        if self.invw is None:
            self.invw = self._invweight0()
        self._pack()

    @classmethod
    def from_tables(cls, base, body_f, hull, maps):
        """a shape variant of `base` from its tables (uhc_b200/subject_body.py): body_f [24][20] and hull [nvert][3] taken as they are (invweight0
        and the bounding spheres included), maps [24][3][4] the per-body affine maps (A | t) that carry base's hulls onto this one.  Shares the
        base's topology, dof tables and joint limits."""
        m = cls.__new__(cls)
        m.__dict__.update({k: v for k, v in base.__dict__.items() if k not in ("_keep", "_rkeep")})
        bf = np.array(body_f, np.float64).reshape(NB, BODYF)
        m.hull = np.array(hull, np.float64).reshape(len(base.hull), 3)
        m.maps = np.array(maps, np.float64).reshape(NB, 3, 4)
        m.offset, m.ipos, m.mass, m.invw = bf[:, 0:3].copy(), bf[:, 3:6].copy(), bf[:, 6].copy(), bf[:, 13].copy()
        q = bf[:, 7:13]
        m.inertia = np.stack([np.stack([q[:, 0], q[:, 3], q[:, 4]], 1), np.stack([q[:, 3], q[:, 1], q[:, 5]], 1),
                              np.stack([q[:, 4], q[:, 5], q[:, 2]], 1)], 1)
        m.body_f = np.ascontiguousarray(bf)
        m.root_offset = bf[0, 0:3].copy()            # the root body's offset: where smpl_to_qpos puts the pelvis, as the device FK does
        m.qpos0 = base.qpos0.copy()
        m.qpos0[:3] = m.root_offset
        return m

    def _topology(self):
        p = self.parent
        self.depth = np.zeros(NB, np.int32)
        for b in range(1, NB):
            self.depth[b] = self.depth[p[b]] + 1
        ch = [[c for c in range(NB) if p[c] == b] for b in range(NB)]
        self.child_adr = np.concatenate([[0], np.cumsum([len(c) for c in ch])]).astype(np.int32)
        self.child = np.array([c for cs in ch for c in cs], np.int32)
        sub_end = np.arange(NB)
        for b in range(NB - 1, 0, -1):
            sub_end[p[b]] = max(sub_end[p[b]], sub_end[b])
        self.body_sub_end = sub_end.astype(np.int32)
        # Elimination tree of the articulated-body solve.  The joint-space matrix only needs A tree of bodies and joints, not the
        # kinematic root: hanging the same tree from its centre (Spine2 for SMPL) gives 7 levels of <= 5 bodies instead of 9.
        # Joints on the path centre -> Pelvis are traversed against their kinematic direction (sign bit); the Pelvis free joint
        # becomes an external wrench on the Pelvis body (its armature must be 0) and the centre body carries 6 virtual dofs.
        # Per level and lane group (<= 5): body, parent's group, groups of <= 3 children, joint block (first dof / 3), sign.
        nbrs = [[c for c in range(NB) if p[c] == b] + ([int(p[b])] if b > 0 else []) for b in range(NB)]

        def hang(root):
            par, dep, order = {root: -1}, {root: 0}, [root]
            for b in order:
                for c in sorted(nbrs[b]):
                    if c not in par:
                        par[c], dep[c] = b, dep[b] + 1
                        order.append(c)
            return par, dep
        root = min(range(NB), key=lambda r: (max(hang(r)[1].values()), r))
        par2, dep2 = hang(root)
        nlev = max(dep2.values()) + 1
        ch2 = [[c for c in range(NB) if par2[c] == b] for b in range(NB)]
        groups = [[b for b in range(NB) if dep2[b] == L] for L in range(9)]
        assert nlev <= 9 and max(len(g) for g in groups) <= 5 and max(len(c) for c in ch2) <= 3
        assert np.all(self.armature[:6] == 0), "the solve re-roots the tree: the free joint must have no armature"
        grp = {b: g.index(b) for g in groups for b in g}
        tab = -np.ones((9, 5, 7), np.int32)
        for L, g in enumerate(groups):
            for gi, b in enumerate(g):
                tab[L, gi, 0] = b
                tab[L, gi, 1] = grp[par2[b]] if par2[b] >= 0 else 0
                for k, c in enumerate(ch2[b]):
                    tab[L, gi, 2 + k] = grp[c]
                if par2[b] < 0:
                    tab[L, gi, 5], tab[L, gi, 6] = NV // 3, 0            # virtual dofs NV .. NV+5 of the centre body
                elif p[b] == par2[b]:
                    tab[L, gi, 5], tab[L, gi, 6] = 1 + b, 0              # own joint: dofs 3 + 3 b ..
                else:
                    tab[L, gi, 5], tab[L, gi, 6] = 1 + par2[b], 1        # the tree parent's joint, traversed backwards
        self.solve_root, self.solve_levels = root, nlev
        self.lvl_tab = np.ascontiguousarray(tab[:, :, :5].reshape(-1))
        nslot = (tab[:, :, 2:5] >= 0).sum(axis=2).max(axis=1)          # most children any body of the level has (uniform per level)
        self.lvl_pack = np.ascontiguousarray(((tab[:, :, 0] + 1) | (np.maximum(tab[:, :, 1], 0) << 6) | ((tab[:, :, 2] + 1) << 9) | ((tab[:, :, 3] + 1) << 12) | ((tab[:, :, 4] + 1) << 15)
                                              | (nslot[:, None] << 18) | (np.maximum(tab[:, :, 5], 0) << 20) | (np.maximum(tab[:, :, 6], 0) << 25) | (nlev << 26)).astype(np.int32).reshape(-1))
        self.dof_body = np.array([0] * 6 + [1 + d // 3 for d in range(NU)], np.int32)

    def _invweight0(self):
        """body_invweight0 (translational): trace(Jv M^-1 Jv^T) / 3 at qpos0 (rest pose, all rotations identity) -- tools/compile_model.py."""
        p = self.parent
        gpos = np.zeros((NB, 3))
        gpos[0] = self.z["body_gpos"][0]
        for b in range(1, NB):
            gpos[b] = gpos[p[b]] + self.offset[b]
        axes = np.eye(3)[[2, 1, 0]]
        xipos = gpos + self.ipos
        Jv, Jw = np.zeros((NB, 3, NV)), np.zeros((NB, 3, NV))
        for b in range(NB):
            Jv[b, :, 0:3] = np.eye(3)
            for k in range(3):
                Jw[b, :, 3 + k] = np.eye(3)[k]
                Jv[b, :, 3 + k] = np.cross(np.eye(3)[k], xipos[b] - gpos[0])
            a = b
            while a > 0:
                for k in range(3):
                    d = 6 + 3 * (a - 1) + k
                    Jw[b, :, d] = axes[k]
                    Jv[b, :, d] = np.cross(axes[k], xipos[b] - gpos[a])
                a = p[a]
        M = np.diag(self.armature)
        for b in range(NB):
            M += self.mass[b] * Jv[b].T @ Jv[b] + Jw[b].T @ self.inertia[b] @ Jw[b]
        Minv = np.linalg.inv(M)
        return np.array([np.trace(Jv[b] @ Minv @ Jv[b].T) / 3 for b in range(NB)])

    def _pack(self):
        bf = np.zeros((NB, BODYF))
        bf[:, 0:3], bf[:, 3:6], bf[:, 6] = self.offset, self.ipos, self.mass
        I = self.inertia
        bf[:, 7:13] = np.stack([I[:, 0, 0], I[:, 1, 1], I[:, 2, 2], I[:, 0, 1], I[:, 0, 2], I[:, 1, 2]], 1)
        bf[:, 13] = self.invw
        for b in range(NB):  # bounding sphere of the hull about its vertex centroid
            v = self.hull[self.hull_adr[b]:self.hull_adr[b] + self.hull_num[b]]
            c = v.mean(0)
            bf[b, 14:17], bf[b, 17] = c, np.linalg.norm(v - c, axis=1).max() * 1.0001 + 1e-6
        bf[:, 18] = self.diffw
        df = np.zeros((NV, 4))
        df[:, 0] = self.armature
        df[6:, 1], df[6:, 2], df[6:, 3] = self.jkp, self.jkd, self.torque_lim
        self.body_f, self.dof_f = np.ascontiguousarray(bf), np.ascontiguousarray(df)
        # joint-limit table [NV][4]: lower, upper (rad), dof_invweight0 (diagApprox of a limit row), pad; the free joint has no limits
        dl = np.zeros((NV, 4))
        dl[:6, 0], dl[:6, 1] = -1e30, 1e30
        dl[6:, 0:2] = self.jnt_range
        dl[:, 2] = self.dof_invweight0
        self.dof_lim = np.ascontiguousarray(dl)

    # residual-force slot order of the explicit mode: vf_bodies = SMPL_BONE_ORDER_NAMES (humanoid_im.py:236-237, smpl_parser.py:11-36)
    SMPL_BONE_ORDER = ("Pelvis", "L_Hip", "R_Hip", "Torso", "L_Knee", "R_Knee", "Spine", "L_Ankle", "R_Ankle", "Chest", "L_Toe", "R_Toe", "Neck", "L_Thorax",
                       "R_Thorax", "Head", "L_Shoulder", "R_Shoulder", "L_Elbow", "R_Elbow", "L_Wrist", "R_Wrist", "L_Hand", "R_Hand")

    def vf_slot(self):
        """residual-force slot of every model body (bodies are numbered depth-first, the slots follow the SMPL joint order)"""
        return [self.SMPL_BONE_ORDER.index(n) for n in self.body_names]

    def hull_planes(self):
        """face planes of every body hull in body frame, [nplane][4] (unit outward normal n, offset d; n . x + d <= 0 inside), from
        scipy's ConvexHull(...).equations with faces coplanar to 1e-9 merged, and per body plane_adr / plane_num [24]"""
        from scipy.spatial import ConvexHull
        planes, num = [], []
        for b in range(NB):
            eq = ConvexHull(self.hull[self.hull_adr[b]:self.hull_adr[b] + self.hull_num[b]]).equations
            keep = []
            for e in eq:
                if not any(np.abs(e - k).max() <= 1e-9 for k in keep):
                    keep.append(e)
            planes.append(np.array(keep))
            num.append(len(keep))
        return np.concatenate(planes), np.concatenate([[0], np.cumsum(num)[:-1]]).astype(np.int32), np.array(num, np.int32)

    def mapped_planes(self, planes):
        """hull_planes() of a variant built by from_tables, as the images of its base's `planes` under the body maps instead of a hull per
        body: x -> A x + t takes n . x + d <= 0 to (A^-T n) . x' + d - (A^-T n) . t <= 0, renormalised"""
        pl, adr, num = planes
        out = np.empty_like(pl)
        for b in range(NB):
            A, t = self.maps[b, :, :3], self.maps[b, :, 3]
            rows = pl[adr[b]:adr[b] + num[b]]
            n = np.linalg.solve(A.T, rows[:, :3].T).T
            d = rows[:, 3] - n @ t
            s = np.linalg.norm(n, axis=1)
            out[adr[b]:adr[b] + num[b]] = np.hstack([n / s[:, None], (d / s)[:, None]])
        return out, adr, num

    def render_struct(self, variants=None):
        """ctypes UhcRenderHulls of the shape variants host_struct(variants) builds, in the same order (arrays kept alive on self).  Variants
        share plane_adr / plane_num: a body whose hull has fewer merged faces in one variant repeats its last plane, which clips nothing more."""
        models = variants or [self]
        assert models[0] is self
        own = self.hull_planes()
        per = [own if s == 0 else m.mapped_planes(own) if getattr(m, "maps", None) is not None else m.hull_planes() for s, m in enumerate(models)]
        num = np.max([p[2] for p in per], axis=0).astype(np.int32)
        adr = np.concatenate([[0], np.cumsum(num)[:-1]]).astype(np.int32)
        plane = np.zeros((len(models), int(num.sum()), 4))
        for s, (pl, a, k) in enumerate(per):
            for b in range(NB):
                rows = pl[a[b]:a[b] + k[b]]
                plane[s, adr[b]:adr[b] + num[b]] = np.concatenate([rows, np.repeat(rows[-1:], num[b] - k[b], 0)])
        sphere = np.ascontiguousarray(np.stack([m.body_f[:, 14:18] for m in models]))
        keep = self._rkeep = dict(plane=np.ascontiguousarray(plane), adr=adr, num=num, sphere=sphere)
        h = UhcRenderHulls()
        h.nshape, h.nplane = len(models), plane.shape[1]
        h.plane = keep["plane"].ctypes.data_as(C.POINTER(C.c_double))
        h.plane_adr, h.plane_num = adr.ctypes.data_as(C.POINTER(C.c_int)), num.ctypes.data_as(C.POINTER(C.c_int))
        h.sphere = sphere.ctypes.data_as(C.POINTER(C.c_double))
        return h

    def host_struct(self, variants=None):
        """ctypes struct of host pointers for uhc_engine_create / the emulation (arrays kept alive on self).
        variants: optional list of HumanoidModel shape variants (same topology); variant 0 must be `self`."""
        h = UhcModelHost()
        keep = self._keep = {}
        models = variants or [self]
        assert models[0] is self and all(len(m.hull) == len(self.hull) for m in models)
        body_f = np.concatenate([m.body_f for m in models])
        hull = np.concatenate([m.hull for m in models])

        def ptr(name, arr, ct):
            a = np.ascontiguousarray(arr)
            keep[name] = a
            return a.ctypes.data_as(C.POINTER(ct))

        h.nvert, h.nnbr = len(self.hull), len(self.nbr)
        h.body_f, h.dof_f, h.hull = ptr("bf", body_f, C.c_double), ptr("df", self.dof_f, C.c_double), ptr("hull", hull, C.c_double)
        h.nshape = len(models)
        h.dof_lim = ptr("dof_lim", self.dof_lim, C.c_double)
        for n in ("hull_adr", "hull_num", "nbr", "nbradr", "parent", "depth", "child_adr", "child", "body_sub_end", "ee", "lvl_tab", "lvl_pack"):
            setattr(h, n, ptr(n, getattr(self, n).astype(np.int32), C.c_int))
        h.dt, h.margin, h.mu, h.gravz = self.dt, self.margin, self.mu, self.gravz
        h.solref = (C.c_double * 2)(*self.solref)
        h.solimp = (C.c_double * 5)(*self.solimp)
        return h
