"""Motion library: SMPL pose sequences -> expert tables for the batched engine (SURVEY.md section 8a row a9 / 8f row 1).

Host-side, vectorised numpy (fp64), run once per clip instead of once per episode:
  smpl_to_qpos   uhc/smpllib/smpl_mujoco.py:543-607   axis-angle -> per-joint ZYX euler in MuJoCo body order, root quaternion,
                                                      root position = trans + body_pos[1]
  qpos_fk        uhc/smpllib/torch_smpl_humanoid.py:155-261  tree FK, finite-difference qvel / body angular velocity @30 Hz
Parity: tests/test_motion_lib.py against tests/golden/expert_*.npz (generated from the reference's own functions).
"""
import numpy as np
from scipy.spatial.transform import Rotation as sRot

from .model import HumanoidModel

# uhc/smpllib/smpl_parser.py:11-36 (SMPL joint order) -> MuJoCo depth-first body order (model.body_names)
SMPL_BONE_ORDER_NAMES = ["Pelvis", "L_Hip", "R_Hip", "Torso", "L_Knee", "R_Knee", "Spine", "L_Ankle", "R_Ankle", "Chest", "L_Toe",
                         "R_Toe", "Neck", "L_Thorax", "R_Thorax", "Head", "L_Shoulder", "R_Shoulder", "L_Elbow", "R_Elbow", "L_Wrist",
                         "R_Wrist", "L_Hand", "R_Hand"]
EXPERT_KEYS = ("qpos", "qvel", "wbpos", "wbquat", "bquat", "bangvel", "ee_wpos", "com")


def qmul(a, b):
    w0, x0, y0, z0 = (a[..., i] for i in range(4))
    w1, x1, y1, z1 = (b[..., i] for i in range(4))
    return np.stack([w0 * w1 - x0 * x1 - y0 * y1 - z0 * z1, w0 * x1 + x0 * w1 + y0 * z1 - z0 * y1,
                     w0 * y1 - x0 * z1 + y0 * w1 + z0 * x1, w0 * z1 + x0 * y1 - y0 * x1 + z0 * w1], -1)


def qinv(q):
    c = q * np.array([1.0, -1.0, -1.0, -1.0])
    return c / (q * q).sum(-1, keepdims=True)


def qrot(q, v):
    """rotate v by quaternion q (quat_mul_vec_batch, torch_utils)."""
    qv = q[..., 1:]
    uv = np.cross(qv, v)
    uuv = np.cross(qv, uv)
    return v + 2 * (q[..., :1] * uv + uuv)


def qmat(q):
    q = q / np.linalg.norm(q, axis=-1, keepdims=True)
    w, x, y, z = (q[..., i] for i in range(4))
    return np.stack([np.stack([1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], -1),
                     np.stack([2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)], -1),
                     np.stack([2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)], -1)], -2)


def euler_zyx_quat(e):
    """quaternion_from_euler(e0, e1, e2, 'rzyx') = Rz(e0) Ry(e1) Rx(e2)."""
    h = 0.5 * e
    c, s = np.cos(h), np.sin(h)
    z = np.zeros_like(c[..., 0])
    qz = np.stack([c[..., 0], z, z, s[..., 0]], -1)
    qy = np.stack([c[..., 1], z, s[..., 1], z], -1)
    qx = np.stack([c[..., 2], s[..., 2], z, z], -1)
    return qmul(qmul(qz, qy), qx)


def rot_from_quat(q, separate=False):
    """rotation_from_quaternion_batch (uhc/utils/torch_utils.py:142-167)."""
    ac = np.arccos(np.clip(q[..., 0], -1.0 + 1e-7, 1.0 - 1e-7))
    sn = np.sin(ac)
    cond = np.abs(sn) < 1e-5
    axis = np.where(cond[..., None], np.array([1.0, 0.0, 0.0]), q[..., 1:4] / np.where(cond, 1.0, sn)[..., None])
    angle = np.where(cond, 0.0, 2 * ac)
    return (axis, angle) if separate else axis * angle[..., None]


def smpl_to_qpos(pose_aa, trans, model=None):
    m = model or HumanoidModel()
    pose = np.asarray(pose_aa, dtype=np.float64)
    T = pose.shape[0]
    if pose.shape[-1] == 156:  # smplh_to_smpl (smpl_mujoco.py:533-535): keep 22 joints, zero the hands
        pose = np.concatenate([pose[:, :66], np.zeros((T, 6))], 1)
    pose = pose.reshape(T, 24, 3)
    if trans is None:
        trans = np.tile([0.0, 0.0, 0.91437225], (T, 1))
    R = sRot.from_rotvec(pose.reshape(-1, 3))
    eul = R.as_euler("ZYX").reshape(T, 24, 3)
    order = [SMPL_BONE_ORDER_NAMES.index(n) for n in m.body_names]
    eul = eul[:, order]
    rq = sRot.from_rotvec(pose[:, 0]).as_quat()[:, [3, 0, 1, 2]]
    rq = np.where(rq[:, :1] < 0, -rq, rq)
    qpos = np.concatenate([np.asarray(trans, dtype=np.float64).reshape(T, 3) + m.root_offset, rq, eul[:, 1:].reshape(T, 69)], 1)
    return qpos


def qpos_fk(qpos, model=None, dt=1.0 / 30):
    m = model or HumanoidModel()
    qpos = np.asarray(qpos, dtype=np.float64)
    T = qpos.shape[0]
    rootq, rootp = qpos[:, 3:7], qpos[:, :3]
    bq_local = euler_zyx_quat(qpos[:, 7:].reshape(T, 23, 3))
    wpos, wquat, wcom = [None] * 24, [None] * 24, [None] * 24
    for b in range(24):
        if b == 0:
            wpos[0], wquat[0] = rootp, rootq
        else:
            p = m.parent[b]
            wpos[b] = qrot(wquat[p], np.broadcast_to(m.offset[b], (T, 3))) + wpos[p]
            wquat[b] = qmul(wquat[p], bq_local[:, b - 1])
        wcom[b] = qrot(wquat[b], np.broadcast_to(m.ipos[b], (T, 3))) + wpos[b]
    wbpos, wbquat, body_com = np.stack(wpos, 1), np.stack(wquat, 1), np.stack(wcom, 1)
    bquat = np.concatenate([rootq[:, None], bq_local], 1)
    if T > 1:  # get_qvel_fd_batch (torch_utils.py:368-386)
        cur, nxt = qpos[:-1], qpos[1:]
        v = (nxt[:, :3] - cur[:, :3]) / dt
        axis, angle = rot_from_quat(qmul(nxt[:, 3:7], qinv(cur[:, 3:7])), True)
        angle = np.where(angle > np.pi, angle - 2 * np.pi, angle)
        angle = np.where(angle < -np.pi, angle + 2 * np.pi, angle)
        rv = axis * angle[:, None] / dt
        rv = np.einsum("tji,tj->ti", qmat(cur[:, 3:7]), rv)
        qvel = np.concatenate([v, rv, (nxt[:, 7:] - cur[:, 7:]) / dt], 1)
        bang = rot_from_quat(qmul(bquat[1:], qinv(bquat[:-1]))) / dt
    else:
        qvel, bang = np.zeros((0, 75)), np.zeros((0, 24, 3))
    qvel = np.clip(np.concatenate([qvel[:1], qvel], 0), -10.0, 10.0)
    bang = np.concatenate([bang[:1], bang], 0)
    ee = wbpos[:, m.ee]
    return {"qpos": qpos, "qvel": qvel, "wbpos": wbpos.reshape(T, 72), "wbquat": wbquat.reshape(T, 96), "bquat": bquat.reshape(T, 96),
            "body_com": body_com.reshape(T, 72), "bangvel": bang.reshape(T, 72), "ee_wpos": ee.reshape(T, 15), "com": body_com[:, 0],
            "height_lb": qpos[:, 2].min(), "len": T}


def make_expert(pose_aa, trans, model=None):
    m = model or HumanoidModel()
    return qpos_fk(smpl_to_qpos(pose_aa, trans, m), m)


class MotionSet:
    """Raw motion of a dataset, for Engine.load_motions: the expert tables are built on the GPU from it (uhc_b200/csrc/motion_lib.cu),
    so the host never holds them.  clips: list of {pose_aa [T][72 | 156], trans [T][3] (None: the default height)} or of {qpos [T][76]}
    dicts, all of one kind.  Keeps the concatenated rows [sum T][pose_dim + 3 | 76] (fp64) and the clip lengths.  A set that mixes 72- and
    156-wide poses is stored 72 wide with the SMPL-H conversion applied (columns 66:72 zeroed), which smpl_to_qpos would do per clip."""
    SMPL, QPOS = 0, 1          # include/uhc_b200.h UHC_MOTION_SMPL / UHC_MOTION_QPOS

    def __init__(self, clips):
        clips = list(clips)
        assert clips, "MotionSet: no clips"
        if all("qpos" in c and "pose_aa" not in c for c in clips):
            self.kind, self.pose_dim = self.QPOS, 76
            rows = [np.asarray(c["qpos"], dtype=np.float64).reshape(-1, 76) for c in clips]
        else:
            assert all("pose_aa" in c for c in clips), "MotionSet: every clip needs pose_aa (+ trans), or every clip qpos"
            poses = [np.asarray(c["pose_aa"], dtype=np.float64) for c in clips]
            poses = [p.reshape(p.shape[0], -1) for p in poses]
            widths = {p.shape[1] for p in poses}
            assert widths <= {72, 156}, "MotionSet: pose_aa rows are 72 (SMPL) or 156 (SMPL-H) wide"
            if len(widths) > 1:
                poses = [p if p.shape[1] == 72 else np.concatenate([p[:, :66], np.zeros((len(p), 6))], 1) for p in poses]
            self.kind, self.pose_dim = self.SMPL, poses[0].shape[1]
            rows = []
            for p, c in zip(poses, clips):
                tr = c.get("trans")
                tr = np.tile([0.0, 0.0, 0.91437225], (len(p), 1)) if tr is None else np.asarray(tr, dtype=np.float64).reshape(len(p), 3)
                rows.append(np.concatenate([p, tr], 1))
        self.lens = np.array([len(r) for r in rows], np.int32)
        self.rows = np.ascontiguousarray(np.concatenate(rows))

    def __len__(self):
        return len(self.lens)

    @property
    def num_frames(self):
        return int(self.lens.sum())

    @classmethod
    def _from_rows(cls, kind, pose_dim, rows, lens):
        ms = object.__new__(cls)
        ms.kind, ms.pose_dim = kind, pose_dim
        ms.rows, ms.lens = np.ascontiguousarray(rows, np.float64), np.asarray(lens, np.int32)
        return ms

    # ---- height against the floor, before the tables are built (include/uhc_floor.h uhc_motion_floor).  The reference fixes the height off
    # line with the SMPL mesh (uhc/data_process/process_amass_db.py:126-219); here the surface is the body hulls, which are coarser.
    START_HIGH, AIRBORNE_Z, AIRBORNE_RUN, TOE_DEPTH, CRAWL_ROOT, CRAWL_FEET = 0.1, 0.2, 30, -0.15, 0.3, -0.1

    def floor_audit(self, engine, fk_models=None):
        """Per clip, from one device pass over the raw rows (Engine.motion_floor; fk_models = shape variant per clip), arrays [C]:
          dz_first      lowest hull vertex of frame 0 (m): fix_height_smpl_vanilla's gp
          dz_clip       lowest hull vertex of the whole clip
          start_high    dz_first > 0.1 (fix_height_smpl drops these)
          airborne_run  longest run of frames with both feet above 0.2 m once the clip is lowered by dz_first (fix_height_smpl drops runs
                        above 30; it reads SMPL joints 10 and 11, which this model names L_Toe and R_Toe)
          deepest_toe   lowest toe of the clip once lowered by dz_first (fix_height drops clips below -0.15)
          crawling      root below 0.3 m with both toes above -0.1 m at frame 0 (fix_height leaves these clips alone)
          implausible   start_high, or airborne_run > 30, or deepest_toe < -0.15: the clips drop_implausible removes"""
        rows, feet = engine.motion_floor(self, fk_models)
        rows, feet = (np.asarray(x.cpu() if hasattr(x, "cpu") else x, dtype=np.float64) for x in (rows, feet))
        C = len(self)
        adr = np.concatenate([[0], np.cumsum(self.lens)])
        models = getattr(engine, "variants", None) or [engine.model]
        fk = np.zeros(C, np.int32) if fk_models is None else np.asarray(fk_models, np.int32).reshape(C)
        out = {k: np.zeros(C) for k in ("dz_first", "dz_clip", "deepest_toe")}
        out.update(airborne_run=np.zeros(C, np.int64), crawling=np.zeros(C, bool))
        for c in range(C):
            a, b = int(adr[c]), int(adr[c + 1])
            dz = rows[a, 0]
            toes = feet[a:b, 2:4] - dz
            up = np.concatenate([[0], (toes > self.AIRBORNE_Z).all(1).astype(np.int64), [0]])
            edges = np.flatnonzero(np.diff(up))
            root_z = self.rows[a, 2] if self.kind == self.QPOS else self.rows[a, self.pose_dim + 2] + models[fk[c]].root_offset[2]
            out["dz_first"][c], out["dz_clip"][c], out["deepest_toe"][c] = dz, rows[a:b, 0].min(), toes.min()
            out["airborne_run"][c] = (edges[1::2] - edges[::2]).max() if len(edges) else 0
            out["crawling"][c] = root_z < self.CRAWL_ROOT and feet[a, 2:4].min() > self.CRAWL_FEET
        out["start_high"] = out["dz_first"] > self.START_HIGH
        out["implausible"] = out["start_high"] | (out["airborne_run"] > self.AIRBORNE_RUN) | (out["deepest_toe"] < self.TOE_DEPTH)
        return out

    def fix_height(self, audit, mode="first_frame", offset=0.0):
        """a new set with every clip's translation z (trans of SMPL rows, qpos[2] of qpos rows) lowered so that the lowest hull vertex of
        frame 0 (mode "first_frame", fix_height_smpl_vanilla; crawling clips are left alone, as fix_height does) or of the whole clip
        ("clip_min") sits at `offset` above the floor; "off" returns the rows unchanged.  audit: floor_audit's result for this set."""
        if mode not in ("first_frame", "clip_min", "off"):
            raise ValueError(f"fix_height: mode must be first_frame, clip_min or off, not {mode!r}")
        rows = self.rows.copy()
        if mode != "off":
            dz = np.asarray(audit["dz_first" if mode == "first_frame" else "dz_clip"], np.float64) - float(offset)
            if mode == "first_frame":
                dz = np.where(audit["crawling"], 0.0, dz)
            assert len(dz) == len(self), "fix_height: the audit is of another set"
            rows[:, 2 if self.kind == self.QPOS else self.pose_dim + 2] -= np.repeat(dz, self.lens)
        return self._from_rows(self.kind, self.pose_dim, rows, self.lens.copy())

    def drop(self, mask):
        """a new set without the clips where mask is true"""
        keep = ~np.asarray(mask, bool).reshape(len(self))
        assert keep.any(), "MotionSet.drop: no clip left"
        return self._from_rows(self.kind, self.pose_dim, self.rows[np.repeat(keep, self.lens)], self.lens[keep])


def synthetic_clip(T, rng, model=None, kind="normal"):
    """AMASS-shaped synthetic motion (SURVEY.md section 8d config 5): 30 fps, joint angles = sum of 3 low-frequency sinusoids
    (amplitude <= 0.5 rad, f <= 1.5 Hz), slow root walk; `kind` sets the root-height profile."""
    m = model or HumanoidModel()
    t = np.arange(T) / 30.0
    ang = np.zeros((T, 69))
    for _ in range(3):
        amp = rng.uniform(0.0, 0.5 / 3, 69) * (rng.uniform(size=69) < 0.6)
        ang += amp * np.sin(2 * np.pi * rng.uniform(0.1, 1.5, 69) * t[:, None] + rng.uniform(0, 2 * np.pi, 69))
    ang[:, 9:12] *= 0.2
    ang[:, 21:24] *= 0.2                     # toes
    qpos = np.zeros((T, 76))
    speed, head = rng.uniform(0, 1.0), rng.uniform(0, 2 * np.pi)
    qpos[:, 0], qpos[:, 1] = speed * t * np.cos(head), speed * t * np.sin(head)
    z = 0.93 + 0.01 * np.sin(2 * np.pi * 0.5 * t)
    if kind == "sitting":
        z = 0.93 - 0.45 * np.clip(t / 2.0, 0, 1)
    elif kind == "airborne":
        z = 0.93 + 0.3 * np.abs(np.sin(2 * np.pi * 0.8 * t))
    qpos[:, 2] = z
    yaw = head + 0.3 * np.sin(2 * np.pi * 0.2 * t)
    base = np.array([0.7071068, 0.7071068, 0.0, 0.0])
    qyaw = np.stack([np.cos(yaw / 2), np.zeros(T), np.zeros(T), np.sin(yaw / 2)], 1)
    qpos[:, 3:7] = qmul(qyaw, np.broadcast_to(base, (T, 4)))
    qpos[:, 7:] = ang
    return qpos_fk(qpos, m)
