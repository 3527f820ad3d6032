"""ctypes binding of libuhc_b200.so (include/uhc_b200.h) -- the batched humanoid-imitation engine.

PyTorch is plumbing here: it owns the device buffers handed to the C ABI and the CUDA stream.  There is NO CPU fallback:
if the CUDA library is missing or no GPU is visible this module raises.
"""
import ctypes as C
import os

import numpy as np

from .model import HumanoidModel, UhcModelHost

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.environ.get("UHC_B200_SO") or os.path.join(_HERE, "libuhc_b200.so")   # override: scratch builds of kernel variants
OBS_DIM, ACT_DIM, NQ, NV, NU, EX_SIZE = 657, 105, 76, 75, 69, 576
EXPERT_FIELDS = (("qpos", 76), ("qvel", 75), ("wbpos", 72), ("wbquat", 96), ("bquat", 96), ("bangvel", 72), ("ee_wpos", 15), ("com", 3))


class UhcEnvCfg(C.Structure):
    _fields_ = [("base_rot", C.c_double * 4), ("rfc_scale", C.c_double), ("rfc_lim", C.c_double), ("rfc_rate", C.c_double),
                ("body_diff_thresh", C.c_double), ("meta_pd", C.c_int), ("env_episode_len", C.c_int), ("trail_steps", C.c_int),
                ("newton_max_iter", C.c_int), ("w", C.c_double * 5), ("k", C.c_double * 5), ("newton_tol", C.c_double),
                ("auto_reset", C.c_int), ("t_min", C.c_int), ("t_max", C.c_int), ("reactive_v", C.c_int), ("reset_seed", C.c_ulonglong),
                ("reactive_rate", C.c_double), ("rfc_mode", C.c_int), ("vf_slot", C.c_int * 24), ("obs_v", C.c_int), ("fut_frames", C.c_int), ("fut_skip", C.c_int), ("no_shape", C.c_int), ("term_body", C.c_int), ("head_body", C.c_int), ("reward_mul", C.c_int)]


class UhcEvalClip(C.Structure):
    """include/uhc_eval.h UhcEvalClip"""
    _fields_ = [("frames", C.c_int), ("last_t", C.c_int), ("fail_any", C.c_int), ("reserved", C.c_int), ("reward_sum", C.c_double)]


class UhcEvalOut(C.Structure):
    """include/uhc_eval.h UhcEvalOut"""
    _fields_ = [("frames_host", C.c_void_p), ("clips_host", C.c_void_p), ("states_host_or_null", C.c_void_p), ("smpl_host_or_null", C.c_void_p),
                ("floor_host_or_null", C.c_void_p)]


class UhcFloorHulls(C.Structure):
    """include/uhc_floor.h UhcFloorHulls"""
    _fields_ = [("nshape", C.c_int), ("nvert", C.c_int), ("hull", C.POINTER(C.c_double)), ("hull_adr", C.POINTER(C.c_int)), ("hull_num", C.POINTER(C.c_int))]


class UhcSmplModel(C.Structure):
    """include/uhc_mesh.h UhcSmplModel"""
    _fields_ = [("nvert", C.c_int), ("v_template", C.POINTER(C.c_double)), ("shapedirs", C.POINTER(C.c_double)), ("posedirs", C.POINTER(C.c_double)),
                ("J_regressor", C.POINTER(C.c_double)), ("weights", C.POINTER(C.c_double)), ("parents", C.POINTER(C.c_int))]


EVAL_SMPL = 75      # include/uhc_eval.h UHC_EVAL_SMPL: pose 72, trans 3
FLOOR_NCOL = 5      # include/uhc_floor.h UHC_FLOOR_NCOL: min_z (m), pen_mm, skate_mm, float_mm, n_below
FLOOR_NFEET = 4     # UHC_FLOOR_NFEET: z of L_Ankle, R_Ankle, L_Toe, R_Toe


class UhcRenderCamera(C.Structure):
    """include/uhc_render.h UhcRenderCamera"""
    _fields_ = [("lookat", C.c_double * 3), ("azimuth", C.c_double), ("elevation", C.c_double), ("distance", C.c_double), ("fovy", C.c_double),
                ("focus", C.c_int), ("hide_im", C.c_int), ("hide_expert", C.c_int), ("shift_expert", C.c_double)]


class UhcRenderMesh(C.Structure):
    """include/uhc_render.h UhcRenderMesh"""
    _fields_ = [("nvert", C.c_int), ("nface", C.c_int), ("nleaf", C.c_int), ("face", C.POINTER(C.c_int)), ("face_body", C.POINTER(C.c_int)),
                ("leaf_first", C.POINTER(C.c_int)), ("body_leaf", C.POINTER(C.c_int))]

    @classmethod
    def of(cls, tables, nvert):
        """over the arrays of uhc_b200.render_mesh.build_tables (kept alive by the struct)"""
        keep = {k: np.ascontiguousarray(tables[k], np.int32) for k in ("face", "face_body", "leaf_first", "body_leaf")}
        m = cls(int(nvert), len(keep["face"]), len(keep["leaf_first"]) - 1, *(_ip_out(keep[k]) for k in ("face", "face_body", "leaf_first", "body_leaf")))
        m._keep = keep
        return m


def make_camera(camera=None):
    """UhcRenderCamera from a dict (or None): CopycatVisualizer.setup_viewing_angle's view by default -- lookat (0, 0, 1), azimuth 45,
    elevation -8, distance 5, fovy 45 (MuJoCo's default) -- with focus / hide_im / hide_expert (bools) and shift_expert (x offset of the
    ghost in m; True means update_pose's 1 m)."""
    c = dict(lookat=(0.0, 0.0, 1.0), azimuth=45.0, elevation=-8.0, distance=5.0, fovy=45.0, focus=False, hide_im=False, hide_expert=False,
             shift_expert=0.0)
    unknown = set(camera or {}) - set(c)
    if unknown:
        raise ValueError(f"camera: unknown keys {sorted(unknown)}")
    c.update(camera or {})
    s = c["shift_expert"]
    cam = UhcRenderCamera()
    cam.lookat = (C.c_double * 3)(*[float(x) for x in c["lookat"]])
    cam.azimuth, cam.elevation, cam.distance, cam.fovy = (float(c[k]) for k in ("azimuth", "elevation", "distance", "fovy"))
    cam.focus, cam.hide_im, cam.hide_expert = (int(bool(c[k])) for k in ("focus", "hide_im", "hide_expert"))
    cam.shift_expert = 1.0 if s is True else float(s)
    return cam


def make_cfg(precision=32, base_rot=(0.7071, 0.7071, 0.0, 0.0), rfc_scale=100.0, rfc_lim=100.0, rfc_rate=1.0, body_diff_thresh=0.5,
             meta_pd=1, env_episode_len=100000, trail_steps=0, w=(0.3, 0.1, 0.45, 0.1, 0.05), k=(2.0, 0.005, 5.0, 100.0, 1.0),
             newton_max_iter=None, newton_tol=None, auto_reset=0, t_min=5, t_max=300, reset_seed=1, reactive_v=0, reactive_rate=0.3,
             rfc_mode="implicit", vf_slot=None, obs_v=2, fut_frames=10, fut_skip=10, has_shape=True, term_body="body", head_body=13, reward_mul=False):
    """Defaults = config/release/uhc_implicit_shape.yml + copycat_config.py defaults of the reference."""
    c = UhcEnvCfg()
    c.base_rot = (C.c_double * 4)(*base_rot)
    c.rfc_scale, c.rfc_lim, c.rfc_rate, c.body_diff_thresh = rfc_scale, rfc_lim, rfc_rate, body_diff_thresh
    c.meta_pd, c.env_episode_len, c.trail_steps = int(meta_pd), int(env_episode_len), int(trail_steps)
    c.newton_max_iter = newton_max_iter or (20 if precision == 64 else 12)
    c.newton_tol = newton_tol or (1e-11 if precision == 64 else 1e-5)
    c.w, c.k = (C.c_double * 5)(*w), (C.c_double * 5)(*k)
    c.auto_reset, c.t_min, c.t_max, c.reset_seed = int(auto_reset), int(t_min), int(t_max), int(reset_seed)
    c.reactive_v, c.reactive_rate = int(reactive_v), float(reactive_rate)
    # cfg.residual_force_mode: "implicit" (6 action dims: root wrench) | "explicit" (24 x 9: contact point, force, torque per body, mj_applyFT)
    c.rfc_mode = 1 if rfc_mode in (1, "explicit") else (2 if rfc_mode in (2, "none", None, False) else 0)      # "none": cfg.residual_force false
    c.vf_slot = (C.c_int * 24)(*(list(vf_slot) if vf_slot is not None else range(24)))
    assert int(obs_v) in (1, 2, 3, 5, 6), "obs_v: 1 (get_full_obs_v1), 2 (get_full_obs_v2), 3 (get_full_obs_v3: fut_frames v2 blocks, skip frames apart), 5 / 6 (get_full_obs_v5 / v6)"
    c.obs_v, c.fut_frames, c.fut_skip, c.no_shape = int(obs_v), int(fut_frames), int(fut_skip), int(not has_shape)
    # cfg.env_term_body: "body" | "root" | "Head" (humanoid_im.py:1223-1229); head_body = model body of "Head" (13 in the SMPL humanoid)
    c.term_body = {"body": 0, "root": 1, "Head": 2, "head": 2, 0: 0, 1: 1, 2: 2}[term_body]
    c.head_body = int(head_body)
    c.reward_mul = int(bool(reward_mul))          # reward_id world_rfc_implicit_v1_mul
    return c


def obs_dim_of(cfg):
    """env.obs_dim: 657 (obs v2 with the shape vector) or 784 (obs v1)"""
    block = OBS_DIM - (17 if cfg.no_shape else 0)
    if cfg.obs_v in (5, 6):
        return (636 if cfg.obs_v == 5 else 384) + (0 if cfg.no_shape else 17)
    return 784 if cfg.obs_v == 1 else (block * (cfg.fut_frames if cfg.fut_frames > 0 else 10) if cfg.obs_v == 3 else block)


def act_dim_of(cfg):
    """env.action_dim (humanoid_im.py:250)"""
    return NU + {0: 6, 1: 216, 2: 0}[cfg.rfc_mode] + (30 if cfg.meta_pd else 0)


def pack_expert(ex):
    """expert dict -> [T][576] frame records (layout: include/uhc_b200.h UHC_EX_SIZE).  body_com (72, obs v1) starts where com (its first 3
    values: the root body's centre of mass) sits; an expert dict without body_com (obs v2 only) leaves the rest zero."""
    T = len(ex["qpos"])
    out = np.zeros((T, EX_SIZE))
    o = 0
    for k, n in EXPERT_FIELDS:
        out[:, o:o + n] = np.asarray(ex[k], dtype=np.float64).reshape(T, n)
        o += n
    if "body_com" in ex:
        bc = np.asarray(ex["body_com"], dtype=np.float64).reshape(T, 72)
        assert np.abs(bc[:, :3] - out[:, 502:505]).max() < 1e-9, "expert['com'] must be the root body's body_com"
        out[:, 502:574] = bc
    return out


def unpack_expert(rec):
    """[T][576] frame records -> dict with the fields of motion_lib.qpos_fk (the inverse of pack_expert)"""
    rec = np.asarray(rec, dtype=np.float64)
    T, ex, o = len(rec), {}, 0
    for k, n in EXPERT_FIELDS:
        ex[k] = rec[:, o:o + n].copy()
        o += n
    ex["body_com"] = rec[:, 502:574].copy()
    ex["height_lb"] = ex["qpos"][:, 2].min() if T else np.nan
    ex["len"] = T
    return ex


_lib = None


def load_library():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            raise RuntimeError(f"{_SO} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                               "(there is no CPU fallback for the engine)")
        L = C.CDLL(_SO)
        L.uhc_last_error.restype = C.c_char_p
        _lib = L
    return _lib


def _chk(rc, who="uhc_b200", invalid=RuntimeError):
    """raises `who: <the library's error text>` for a non-zero return code: `invalid` for -2 (a refused argument), RuntimeError otherwise"""
    if rc != 0:
        raise (invalid if rc == -2 else RuntimeError)(f"{who}: " + load_library().uhc_last_error().decode())


def _ip(a):
    return np.ascontiguousarray(a, dtype=np.int32).ctypes.data_as(C.POINTER(C.c_int))


def _ip_out(a):
    assert a.dtype == np.int32 and a.flags.c_contiguous
    return a.ctypes.data_as(C.POINTER(C.c_int))


class Engine:
    """E environments on one GPU.  Mirrors HumanoidEnv.reset/step (+ the agent's custom_reward) for all envs at once."""

    def __init__(self, num_envs, model=None, device=0, precision=32, variants=None, **cfg):
        import torch
        if not torch.cuda.is_available():
            raise RuntimeError("uhc_b200.Engine needs a CUDA device (no CPU fallback)")
        self.torch = torch
        self.lib = load_library()
        self.E, self.device, self.precision = int(num_envs), int(device), precision
        self.model = model or HumanoidModel()
        self.variants = variants
        self._ms = self.model.host_struct(variants)
        if cfg.get("rfc_mode") in (1, "explicit") and cfg.get("vf_slot") is None:
            cfg["vf_slot"] = self.model.vf_slot()                 # slot order of the reference: SMPL_BONE_ORDER_NAMES
        self._cfg_kw = dict(cfg)
        self._cfg = make_cfg(precision, **cfg)
        self.act_dim, self.obs_dim = act_dim_of(self._cfg), obs_dim_of(self._cfg)
        h = C.c_void_p()
        _chk(self.lib.uhc_engine_create(C.byref(self._ms), C.byref(self._cfg), C.c_int(self.E), C.c_int(self.device), C.c_int(precision), C.byref(h)))
        self.h = h
        dev = torch.device("cuda", self.device)
        f = dict(device=dev, dtype=torch.float32)
        self.obs = torch.zeros(self.E, self.obs_dim, **f)
        self.reward = torch.zeros(self.E, **f)
        self.cinfo = torch.zeros(self.E, 5, **f)
        self.percent = torch.zeros(self.E, **f)
        self.fail = torch.zeros(self.E, device=dev, dtype=torch.int32)
        self.end = torch.zeros(self.E, device=dev, dtype=torch.int32)
        self.clip_len = self.clip_models = None
        self._render_ready = self._floor_ready = False
        self.cur_cfg = None            # device curriculum parameters while it is enabled (curriculum_enable)
        if int(cfg.get("reactive_v", 0)) == 1:
            self.set_neutral_pose()

    def set_neutral_pose(self, qpos=None, qvel=None):
        """standing-neutral pose of the reactive starts; default = the bundled copy of the reference's sample_data/standing_neutral.pkl"""
        if qpos is None:
            z = np.load(os.path.join(_HERE, "assets", "standing_neutral.npz"))
            qpos, qvel = z["qpos"], z["qvel"]
        q, v = np.ascontiguousarray(qpos, np.float64), np.ascontiguousarray(qvel, np.float64)
        _chk(self.lib.uhc_set_neutral_pose(self.h, q.ctypes.data_as(C.POINTER(C.c_double)), v.ctypes.data_as(C.POINTER(C.c_double))))
        self.neutral = (q.copy(), v.copy())

    def close(self):
        if getattr(self, "h", None):
            self.lib.uhc_eval_release(self.h)
            self.lib.uhc_track_end(self.h)
            self.lib.uhc_render_release(self.h)
            self.lib.uhc_video_release(self.h)
            self.lib.uhc_floor_release(self.h)
            self.lib.uhc_mesh_release(self.h)
            self.lib.uhc_rollout_release(self.h)
            self.lib.uhc_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def set_cfg(self, **cfg):
        self._cfg_kw = dict(getattr(self, "_cfg_kw", {}), **cfg)
        self._cfg = make_cfg(self.precision, **self._cfg_kw)
        assert obs_dim_of(self._cfg) == self.obs_dim, "obs_v cannot change on a live engine (buffers are sized at creation)"
        self.act_dim = act_dim_of(self._cfg)
        _chk(self.lib.uhc_engine_set_cfg(self.h, C.byref(self._cfg)))

    def load_clips(self, experts, shapes=None, clip_models=None):
        """experts: list of dicts with the fields of Humanoid.qpos_fk (torch_smpl_humanoid.py:234-260); shapes: [C][17]."""
        lens = np.array([len(e["qpos"]) for e in experts], np.int32)
        frames = np.ascontiguousarray(np.concatenate([pack_expert(e) for e in experts]))
        shp = np.zeros((len(experts), 17)) if shapes is None else np.asarray(shapes, dtype=np.float64).reshape(len(experts), 17)
        shp = np.ascontiguousarray(shp)
        _chk(self.lib.uhc_load_clips(self.h, C.c_int(len(experts)), _ip(lens), frames.ctypes.data_as(C.POINTER(C.c_double)),
                                     shp.ctypes.data_as(C.POINTER(C.c_double))))
        self._table_loaded(lens, clip_models)
        if clip_models is not None:
            _chk(self.lib.uhc_set_clip_models(self.h, C.c_int(len(experts)), _ip(clip_models)))

    def load_motions(self, motions, shapes=None, clip_models=None, fk_models=None, chunk_frames=0):
        """Expert tables built on the GPU (uhc_load_motions) from a motion_lib.MotionSet: the same table load_clips gets from
        [motion_lib.make_expert | qpos_fk per clip], without building it on the host.  fk_models: shape variant per clip used by the FK
        (None: variant 0, as make_expert's default model); clip_models: the simulated body per clip (uhc_set_clip_models); chunk_frames:
        frames per host-to-device chunk (0: the library's default)."""
        n = len(motions)
        lens = np.ascontiguousarray(motions.lens, np.int32)
        rows = np.ascontiguousarray(motions.rows, np.float64)
        shp = np.zeros((n, 17)) if shapes is None else np.asarray(shapes, dtype=np.float64).reshape(n, 17)
        shp = np.ascontiguousarray(shp)
        fk = None if fk_models is None else np.ascontiguousarray(fk_models, np.int32).reshape(n)
        _chk(self.lib.uhc_load_motions(self.h, C.c_int(n), _ip(lens), C.c_int(motions.kind), C.c_int(motions.pose_dim),
                                       rows.ctypes.data_as(C.POINTER(C.c_double)), shp.ctypes.data_as(C.POINTER(C.c_double)),
                                       None if fk is None else _ip(fk), C.c_int(int(chunk_frames))))
        self._table_loaded(lens.copy(), clip_models)
        if clip_models is not None:
            _chk(self.lib.uhc_set_clip_models(self.h, C.c_int(n), _ip(clip_models)))

    def _table_loaded(self, lens, clip_models=None):
        self.clip_models = None if clip_models is None else np.array(clip_models, np.int32).reshape(len(lens))
        if self.cur_cfg is not None and (self.clip_len is None or len(lens) != len(self.clip_len)):
            self.cur_cfg = None        # the engine disabled the curriculum: its histories belonged to the old clips
        self.clip_len = lens

    @property
    def load_motions_time(self):
        """device time of the last load_motions from CUDA events (ms): its kernels and its host-to-device row copies"""
        out = np.zeros(2, np.float32)
        _chk(self.lib.uhc_load_motions_time(self.h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return dict(kernel_ms=float(out[0]), copy_ms=float(out[1]))

    def clip_frames(self, clip, first=0, n=None):
        """rows first .. first + n - 1 of a loaded clip (uhc_get_clip_frames), in the engine's precision, as a dict with the field
        names and shapes of motion_lib.qpos_fk (height_lb and len are those of the rows read)."""
        n = int(self.clip_len[clip]) - first if n is None else int(n)
        out = np.zeros((n, EX_SIZE))
        _chk(self.lib.uhc_get_clip_frames(self.h, C.c_int(int(clip)), C.c_int(int(first)), C.c_int(n), out.ctypes.data_as(C.POINTER(C.c_double))))
        return unpack_expert(out)

    def _stream(self):
        return C.c_void_p(self.torch.cuda.current_stream(self.device).cuda_stream)

    def reset(self, env_ids=None, clip=None, start=None, length=None, qpos=None, qvel=None):
        """env.reset() for the listed envs; returns the (whole) obs tensor [E,657] (rows of env_ids refreshed)."""
        t = self.torch
        ids = np.arange(self.E, dtype=np.int32) if env_ids is None else np.asarray(env_ids, dtype=np.int32)
        n = len(ids)
        clip = np.zeros(n, np.int32) if clip is None else np.broadcast_to(np.asarray(clip, np.int32), (n,))
        start = np.zeros(n, np.int32) if start is None else np.broadcast_to(np.asarray(start, np.int32), (n,))
        length = (self.clip_len[clip] - start) if length is None else np.broadcast_to(np.asarray(length, np.int32), (n,))
        qd = vd = None
        if qpos is not None:
            qd = t.as_tensor(np.asarray(qpos, np.float32).reshape(n, NQ)).to(self.obs.device).contiguous()
            vd = t.as_tensor(np.asarray(qvel, np.float32).reshape(n, NV)).to(self.obs.device).contiguous()
        _chk(self.lib.uhc_env_reset(self.h, C.c_int(n), _ip(ids), _ip(clip), _ip(start), _ip(length),
                                    C.c_void_p(qd.data_ptr() if qd is not None else None), C.c_void_p(vd.data_ptr() if vd is not None else None),
                                    C.c_void_p(self.obs.data_ptr()), self._stream()))
        return self.obs

    def step(self, actions, torque_out=None, reward_out=None):
        """env.step(a) + custom_reward for all envs.  actions: float32 cuda tensor [E,105].  Returns views of the engine's
        output tensors (obs, reward, cinfo, fail, end, percent)."""
        t = self.torch
        assert actions.is_cuda and actions.dtype == t.float32 and actions.is_contiguous() and tuple(actions.shape) == (self.E, self.act_dim)
        rew = self.reward if reward_out is None else reward_out
        _chk(self.lib.uhc_env_step(self.h, C.c_void_p(actions.data_ptr()), C.c_void_p(self.obs.data_ptr()), C.c_void_p(rew.data_ptr()),
                                   C.c_void_p(self.cinfo.data_ptr()), C.c_void_p(self.fail.data_ptr()), C.c_void_p(self.end.data_ptr()),
                                   C.c_void_p(self.percent.data_ptr()), C.c_void_p(torque_out.data_ptr() if torque_out is not None else None),
                                   self._stream()))
        return self.obs, rew, self.cinfo, self.fail, self.end, self.percent

    def step_host(self, actions, obs=None, reward=None, cinfo=None, fail=None, end=None, percent=None):
        """Host-buffer entry (H2D of actions and D2H of every requested output inside the call)."""
        a = np.ascontiguousarray(actions, dtype=np.float32).reshape(self.E, self.act_dim)
        obs = np.empty((self.E, self.obs_dim), np.float32) if obs is None else obs
        reward = np.empty(self.E, np.float32) if reward is None else reward
        cinfo = np.empty((self.E, 5), np.float32) if cinfo is None else cinfo
        fail = np.empty(self.E, np.int32) if fail is None else fail
        end = np.empty(self.E, np.int32) if end is None else end
        percent = np.empty(self.E, np.float32) if percent is None else percent
        p = lambda x: C.c_void_p(x.ctypes.data)
        _chk(self.lib.uhc_env_step_host(self.h, p(a), p(obs), p(reward), p(cinfo), p(fail), p(end), p(percent)))
        return obs, reward, cinfo, fail, end, percent

    def get_state(self, env=0):
        q, v, xp, bq, ist = np.zeros(NQ), np.zeros(NV), np.zeros(72), np.zeros(96), np.zeros(8, np.int32)
        d = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
        _chk(self.lib.uhc_env_get_state(self.h, C.c_int(env), d(q), d(v), d(xp), d(bq), ist.ctypes.data_as(C.POINTER(C.c_int))))
        return dict(qpos=q, qvel=v, xpos=xp.reshape(24, 3), bquat=bq, cur_t=int(ist[0]), clip=int(ist[1]), start=int(ist[2]), len=int(ist[3]),
                    newton_iters=int(ist[6]), ncon=int(ist[7]))

    def get_states(self, env_ids=None):
        """state of many envs with one gather launch + one copy (evaluation / parity hook): dict of arrays [n, ...]."""
        ids = np.arange(self.E, dtype=np.int32) if env_ids is None else np.ascontiguousarray(env_ids, dtype=np.int32)
        n = len(ids)
        out, ist = np.zeros((n, 319)), np.zeros((n, 8), np.int32)
        _chk(self.lib.uhc_env_get_state_batch(self.h, C.c_int(n), _ip(ids), out.ctypes.data_as(C.POINTER(C.c_double)), ist.ctypes.data_as(C.POINTER(C.c_int))))
        return dict(qpos=out[:, :76], qvel=out[:, 76:151], xpos=out[:, 151:223].reshape(n, 24, 3), bquat=out[:, 223:319], cur_t=ist[:, 0], clip=ist[:, 1],
                    start=ist[:, 2], len=ist[:, 3], episode=ist[:, 4], flags=ist[:, 5], newton_iters=ist[:, 6], ncon=ist[:, 7])

    def set_state(self, env, qpos, qvel):
        self.set_states([env], np.asarray(qpos)[None], np.asarray(qvel)[None])

    def set_states(self, env_ids, qpos, qvel):
        """fail_safe for many envs at once (humanoid_im.py:902-905): one reset-with-override launch."""
        ids = np.ascontiguousarray(env_ids, dtype=np.int32)
        q = np.ascontiguousarray(qpos, np.float64).reshape(len(ids), NQ)
        v = np.ascontiguousarray(qvel, np.float64).reshape(len(ids), NV)
        _chk(self.lib.uhc_env_set_state_batch(self.h, C.c_int(len(ids)), _ip(ids), q.ctypes.data_as(C.POINTER(C.c_double)), v.ctypes.data_as(C.POINTER(C.c_double))))

    def eval_run(self, clips, policy, log_std, zfilter_stats, zclip=5.0, fail_safe=False, window=32, record_states=False, export_smpl=False, floor=False):
        """device evaluation of up to E clips (uhc_eval_run, include/uhc_eval.h): envs 0..n-1 roll out clips[i] from frame 0 with the mean
        action under the current cfg.  policy: nn.mlp_struct / nn.mcp_struct of the policy; zfilter_stats: the ZFilter's device statistics.
        Returns dict(frames=[n][max(len)-1][6] per-frame rows (rows past `nframes` unspecified), nframes, last_t, fail_any, reward_sum,
        states=[n][max(len)-1][148] recorded qpos + xpos when record_states, else None, and with export_smpl pose_aa=[n][max(len)-1][72] and
        trans=[n][max(len)-1][3], every recorded qpos as SMPL (uhc_eval_run_ex), else None, and with floor floor=[n][max(len)-1][5], every recorded
        frame's hulls against the floor (include/uhc_floor.h: min_z, pen_mm, skate_mm, float_mm, n_below), else None)."""
        t = self.torch
        clips = np.ascontiguousarray(clips, dtype=np.int32).reshape(-1)
        n = len(clips)
        ok = 0 < n <= self.E and self.clip_len is not None and ((clips >= 0) & (clips < len(self.clip_len))).all()
        T = int(self.clip_len[clips].max()) - 1 if ok else 1
        frames = t.empty((max(n, 1), T, 6), dtype=t.float64, pin_memory=True)
        states = t.empty((max(n, 1), T, 148), dtype=t.float64, pin_memory=True) if record_states else None
        smpl = t.empty((max(n, 1), T, EVAL_SMPL), dtype=t.float64, pin_memory=True) if export_smpl else None
        fl = self._floor_buf(max(n, 1), T) if floor else None
        rec = (UhcEvalClip * max(n, 1))()
        out = self._eval_out(frames, rec, states, smpl, fl)
        from .nn import UhcMcp
        fn = self.lib.uhc_eval_run_mcp_ex if isinstance(policy, UhcMcp) else self.lib.uhc_eval_run_ex
        rc = fn(self.h, C.c_int(n), _ip(clips), C.byref(policy), C.c_void_p(log_std.data_ptr()), C.c_void_p(zfilter_stats.data_ptr()), C.c_float(zclip),
                C.c_int(int(bool(fail_safe))), C.c_int(int(window)), C.byref(out), self._stream())
        _chk(rc, "uhc_eval_run", ValueError)
        return self._eval_result(rec, 0, n, frames.numpy(), states.numpy() if states is not None else None, smpl.numpy() if smpl is not None else None,
                                 fl.numpy() if fl is not None else None)

    def _floor_buf(self, n, T):
        self._floor_init()
        return self.torch.empty((n, T, FLOOR_NCOL), dtype=self.torch.float64, pin_memory=True)

    @staticmethod
    def _eval_out(frames, rec, states, smpl, floor=None):
        o = UhcEvalOut()
        o.frames_host, o.clips_host = frames.data_ptr(), C.addressof(rec)
        o.states_host_or_null = states.data_ptr() if states is not None else None
        o.smpl_host_or_null = smpl.data_ptr() if smpl is not None else None
        o.floor_host_or_null = floor.data_ptr() if floor is not None else None
        return o

    @staticmethod
    def _eval_result(rec, o, k, fr, st, sm, fl=None):
        r = rec[o:o + k]
        return dict(frames=fr[o:o + k], nframes=np.array([x.frames for x in r]), last_t=np.array([x.last_t for x in r]),
                    fail_any=np.array([bool(x.fail_any) for x in r]), reward_sum=np.array([x.reward_sum for x in r]),
                    states=st[o:o + k] if st is not None else None,
                    pose_aa=sm[o:o + k, :, :72] if sm is not None else None, trans=sm[o:o + k, :, 72:] if sm is not None else None,
                    floor=fl[o:o + k] if fl is not None else None)

    def eval_run_groups(self, groups, zclip=5.0, fail_safe=False, window=32, record_states=False, export_smpl=False, floor=False):
        """several policies of one architecture in one device evaluation (uhc_eval_run_groups): groups = [(clips, policy, zfilter_stats)], group g
        on the envs after those of groups 0 .. g-1.  Returns one eval_run dict per group, bit-identical to eval_run(clips, policy, ...) of that
        group alone (any finite log_std).  export_smpl, floor: as eval_run's."""
        t = self.torch
        from .nn import UhcMcp, UhcMlp
        G = len(groups)
        clips = [np.ascontiguousarray(c, dtype=np.int32).reshape(-1) for c, _, _ in groups]
        sizes = np.array([len(c) for c in clips], np.int32)
        allc = np.concatenate(clips) if G else np.zeros(0, np.int32)
        n = int(sizes.sum())
        ok = 0 < n <= self.E and self.clip_len is not None and ((allc >= 0) & (allc < len(self.clip_len))).all()
        T = int(self.clip_len[allc].max()) - 1 if ok else 1
        frames = t.empty((max(n, 1), T, 6), dtype=t.float64, pin_memory=True)
        states = t.empty((max(n, 1), T, 148), dtype=t.float64, pin_memory=True) if record_states else None
        smpl = t.empty((max(n, 1), T, EVAL_SMPL), dtype=t.float64, pin_memory=True) if export_smpl else None
        fl = self._floor_buf(max(n, 1), T) if floor else None
        rec = (UhcEvalClip * max(n, 1))()
        out = self._eval_out(frames, rec, states, smpl, fl)
        mcp = G > 0 and isinstance(groups[0][1], UhcMcp)
        pols = ((UhcMcp if mcp else UhcMlp) * max(G, 1))(*[p for _, p, _ in groups])
        zs = (C.c_void_p * max(G, 1))(*[z.data_ptr() for _, _, z in groups])
        fn = self.lib.uhc_eval_run_groups_mcp_ex if mcp else self.lib.uhc_eval_run_groups_ex
        rc = fn(self.h, C.c_int(G), _ip(sizes), _ip(allc), pols, zs, C.c_float(zclip), C.c_int(int(bool(fail_safe))), C.c_int(int(window)),
                C.byref(out), self._stream())
        _chk(rc, "uhc_eval_run_groups", ValueError)
        fr, st, sm = frames.numpy(), states.numpy() if states is not None else None, smpl.numpy() if smpl is not None else None
        fl = fl.numpy() if fl is not None else None
        res, o = [], 0
        for k in sizes:
            res.append(self._eval_result(rec, o, int(k), fr, st, sm, fl))
            o += int(k)
        return res

    # ---- the SMPL export (include/uhc_export.h)
    def qpos_to_smpl(self, qpos, variants=None):
        """qpos_to_smpl (uhc/smpllib/smpl_mujoco.py:738-752) on the device (uhc_qpos_to_smpl): qpos = a cuda tensor [n][>= 76] of float32 | float64
        whose rows are contiguous (its first 76 columns are read, in place) or anything numpy takes (copied to the device as float64); variants =
        shape variant per row (None: 0), the root offset trans is taken against.  Returns (pose_aa [n][72], trans [n][3]), float64 cuda tensors."""
        t = self.torch
        dev = self.obs.device
        q = qpos if t.is_tensor(qpos) and qpos.is_cuda else t.as_tensor(np.ascontiguousarray(qpos, np.float64), device=dev)
        if q.dim() != 2 or q.dtype not in (t.float32, t.float64) or q.shape[1] < 76 or q.stride(1) != 1:
            raise ValueError("qpos_to_smpl: qpos must be [n][>= 76] contiguous rows of float32 | float64")
        n = q.shape[0]
        v = None if variants is None else t.as_tensor(np.array(np.broadcast_to(np.asarray(variants, np.int32), (n,))), device=dev)
        pose, trans = t.empty(n, 72, dtype=t.float64, device=dev), t.empty(n, 3, dtype=t.float64, device=dev)
        _chk(self.lib.uhc_qpos_to_smpl(self.h, C.c_void_p(q.data_ptr()), C.c_int(32 if q.dtype == t.float32 else 64), C.c_long(n),
                                       C.c_long(q.stride(0) if n > 1 else q.shape[1]), C.c_void_p(v.data_ptr() if v is not None else None),
                                       C.c_void_p(pose.data_ptr()), C.c_void_p(trans.data_ptr()), self._stream()), "uhc_qpos_to_smpl", ValueError)
        return pose, trans

    def track_smpl(self, state_out, pose=None, trans=None):
        """the tracker's state_out [E][223] as SMPL (uhc_track_smpl), env e with the shape variant of uhc_track_begin's fk_models; stream-ordered,
        no synchronise.  Returns (pose_aa [E][72], trans [E][3]) float64 cuda tensors (written into pose / trans when given)."""
        t = self.torch
        dev = self.obs.device
        pose = t.empty(self.E, 72, dtype=t.float64, device=dev) if pose is None else pose
        trans = t.empty(self.E, 3, dtype=t.float64, device=dev) if trans is None else trans
        assert state_out.is_cuda and state_out.is_contiguous() and tuple(state_out.shape) == (self.E, 223)
        assert state_out.dtype == (t.float32 if self.precision == 32 else t.float64)
        _chk(self.lib.uhc_track_smpl(self.h, C.c_void_p(state_out.data_ptr()), C.c_void_p(pose.data_ptr()), C.c_void_p(trans.data_ptr()),
                                     self._stream()), "uhc_track_smpl", ValueError)
        return pose, trans

    # ---- the floor measurements (include/uhc_floor.h)
    def _floor_init(self):
        if not self._floor_ready:
            models = self.variants or [self.model]
            m = self.model
            keep = self._fkeep = dict(hull=np.ascontiguousarray(np.stack([v.hull for v in models]), np.float64),
                                      adr=np.ascontiguousarray(m.hull_adr, np.int32), num=np.ascontiguousarray(m.hull_num, np.int32))
            h = UhcFloorHulls()
            h.nshape, h.nvert = len(models), len(m.hull)
            h.hull = keep["hull"].ctypes.data_as(C.POINTER(C.c_double))
            h.hull_adr, h.hull_num = _ip_out(keep["adr"]), _ip_out(keep["num"])
            _chk(self.lib.uhc_floor_init(self.h, C.byref(h)), "uhc_floor_init", ValueError)
            self._floor_ready = True

    def floor_qpos(self, qpos, variants=None, first=None):
        """the body hulls against the floor z = 0 on the device (uhc_floor_qpos): qpos = a cuda tensor [n][>= 76] of float32 | float64 whose rows
        are contiguous (its first 76 columns are read, in place: a state record of 148 or the tracker's state_out of 223 as they are) or anything
        numpy takes (copied as float64); variants = shape variant per row (None: 0); first = per row, 1 where the row has no previous frame
        (None: the rows are one clip).  Returns [n][5] float64 on the device: min_z (m), pen_mm, skate_mm, float_mm, n_below."""
        t = self.torch
        self._floor_init()
        q = self._rows(qpos, who="floor_qpos")
        n = q.shape[0]
        v = self._variant_arg(variants, n)
        f = self._variant_arg(first, n)
        out = t.empty(n, FLOOR_NCOL, dtype=t.float64, device=self.obs.device)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(self.lib.uhc_floor_qpos(self.h, p(q), C.c_int(32 if q.dtype == t.float32 else 64), C.c_long(n), C.c_long(q.stride(0) if n > 1 else q.shape[1]),
                                     p(v), p(f), p(out), self._stream()), "uhc_floor_qpos", ValueError)
        return out

    def track_floor(self, state_out, out=None):
        """the tracker's state_out [E][223] against the floor (uhc_track_floor), env e with the shape variant of uhc_track_begin's fk_models and no
        previous frame; stream-ordered, no synchronise.  Returns [E][5] float64 on the device (written into out when given)."""
        t = self.torch
        self._floor_init()
        out = t.empty(self.E, FLOOR_NCOL, dtype=t.float64, device=self.obs.device) if out is None else out
        assert state_out.is_cuda and state_out.is_contiguous() and tuple(state_out.shape) == (self.E, 223)
        assert state_out.dtype == (t.float32 if self.precision == 32 else t.float64)
        _chk(self.lib.uhc_track_floor(self.h, C.c_void_p(state_out.data_ptr()), C.c_void_p(out.data_ptr()), self._stream()), "uhc_track_floor", ValueError)
        return out

    def motion_floor(self, motions, fk_models=None, chunk_frames=0):
        """uhc_floor_qpos' reduction over the raw rows of a motion_lib.MotionSet (uhc_motion_floor), before any table is built: returns
        (rows [frames][5], feet [frames][4] = z of L_Ankle, R_Ankle, L_Toe, R_Toe), float64 cuda tensors; fk_models: shape variant per clip."""
        t = self.torch
        self._floor_init()
        n = len(motions)
        lens = np.ascontiguousarray(motions.lens, np.int32)
        rows = np.ascontiguousarray(motions.rows, np.float64)
        fk = None if fk_models is None else np.ascontiguousarray(fk_models, np.int32).reshape(n)
        out = t.empty(int(lens.sum()), FLOOR_NCOL, dtype=t.float64, device=self.obs.device)
        feet = t.empty(int(lens.sum()), FLOOR_NFEET, dtype=t.float64, device=self.obs.device)
        _chk(self.lib.uhc_motion_floor(self.h, C.c_int(n), _ip(lens), C.c_int(motions.kind), C.c_int(motions.pose_dim),
                                       rows.ctypes.data_as(C.POINTER(C.c_double)), None if fk is None else _ip(fk), C.c_int(int(chunk_frames)),
                                       C.c_void_p(out.data_ptr()), C.c_void_p(feet.data_ptr())), "uhc_motion_floor", ValueError)
        return out, feet

    # ---- the SMPL mesh (include/uhc_mesh.h)
    def mesh_init(self, model):
        """uploads an SMPL model (uhc_mesh_init): a dict as uhc_b200.smpl_model.load_smpl_model returns it, or a path it reads.  A later call
        replaces the model; a failed one leaves the previous model in place."""
        from uhc_b200.smpl_model import as_model
        m = as_model(model)
        keep = {k: np.ascontiguousarray(m[k], np.float64) for k in ("v_template", "shapedirs", "posedirs", "J_regressor", "weights")}
        keep["parents"] = np.ascontiguousarray(m["parents"], np.int32)
        d = lambda k: keep[k].ctypes.data_as(C.POINTER(C.c_double))
        h = UhcSmplModel(len(keep["v_template"]), d("v_template"), d("shapedirs"), d("posedirs"), d("J_regressor"), d("weights"), _ip_out(keep["parents"]))
        _chk(self.lib.uhc_mesh_init(self.h, C.byref(h)), "uhc_mesh_init", ValueError)
        self.smpl_nvert = len(keep["v_template"])

    def _smpl_args(self, pose, trans, betas, beta_idx):
        t = self.torch
        dev = self.obs.device
        f64 = lambda x: x if t.is_tensor(x) and x.is_cuda and x.dtype == t.float64 and x.is_contiguous() else \
            t.as_tensor(np.ascontiguousarray(x.cpu().numpy() if t.is_tensor(x) else x, np.float64), device=dev)
        pose, trans, betas = f64(pose), f64(trans), f64(betas)
        n = pose.shape[0]
        betas = betas[None] if betas.dim() == 1 else betas
        if pose.dim() != 2 or pose.shape[1] != 72 or tuple(trans.shape) != (n, 3) or betas.dim() != 2 or betas.shape[1] != 10:
            raise ValueError("smpl_mesh: pose [n][72], trans [n][3] and betas [nb][10] float64")
        return pose, trans, betas, self._variant_arg(beta_idx, n)

    def smpl_mesh(self, pose, trans, betas, beta_idx=None, vertices=True, joints=True):
        """SMPL linear blend skinning on the device (uhc_smpl_mesh) after mesh_init: pose [n][72] axis-angles and trans [n][3] (qpos_to_smpl's
        outputs, used in place when they are float64 cuda tensors), betas [nb][10], beta_idx = the betas row of each row (None: row 0).
        Returns (vertices [n][V][3] float32, joints [n][24][3] float64) cuda tensors, None for what is not asked for."""
        t = self.torch
        pose, trans, betas, bi = self._smpl_args(pose, trans, betas, beta_idx)
        n = pose.shape[0]
        dev = self.obs.device
        V = getattr(self, "smpl_nvert", 0)
        vo = t.empty(n, V, 3, dtype=t.float32, device=dev) if vertices else None
        jo = t.empty(n, 24, 3, dtype=t.float64, device=dev) if joints else None
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(self.lib.uhc_smpl_mesh(self.h, C.c_long(n), p(pose), p(trans), C.c_int(betas.shape[0]), p(betas), p(bi), p(vo), p(jo), self._stream()),
             "uhc_smpl_mesh", ValueError)
        return vo, jo

    def smpl_floor(self, pose, trans, betas, beta_idx=None, first=None):
        """the SMPL mesh of the same rows against the floor z = 0 (uhc_smpl_floor), no vertex written: first = per row, 1 where it has no
        previous row (None: one clip).  Returns [n][5] float64 on the device: min_z (m), pen_mm, skate_mm, float_mm, n_below."""
        t = self.torch
        pose, trans, betas, bi = self._smpl_args(pose, trans, betas, beta_idx)
        n = pose.shape[0]
        f = self._variant_arg(first, n)
        out = t.empty(n, FLOOR_NCOL, dtype=t.float64, device=self.obs.device)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(self.lib.uhc_smpl_floor(self.h, C.c_long(n), p(pose), p(trans), C.c_int(betas.shape[0]), p(betas), p(bi), p(f), p(out), self._stream()),
             "uhc_smpl_floor", ValueError)
        return out

    def qpos_mesh(self, qpos, betas, beta_idx=None, variants=None, vertices=True, joints=True, floor=False, first=None):
        """qpos rows -> SMPL (qpos_to_smpl with `variants`) -> the mesh, without leaving the device: smpl_mesh's (vertices, joints), or with
        floor=True smpl_floor's rows"""
        pose, trans = self.qpos_to_smpl(qpos, variants)
        if floor:
            return self.smpl_floor(pose, trans, betas, beta_idx, first)
        return self.smpl_mesh(pose, trans, betas, beta_idx, vertices, joints)

    @property
    def eval_graph_count(self):
        """CUDA graphs the evaluation holds for this engine now (uhc_eval_graph_count)"""
        return int(self.lib.uhc_eval_graph_count(self.h))

    # ---- the renderer (include/uhc_render.h)
    def _render_init(self):
        if not self._render_ready:
            self._rhulls = self.model.render_struct(self.variants)
            _chk(self.lib.uhc_render_init(self.h, C.byref(self._rhulls)), "uhc_render_init", ValueError)
            self._render_ready = True

    def _rows(self, q, n=None, who="render"):
        """a cuda tensor [n][>= 76] of float32 | float64 with contiguous rows (read in place), or anything numpy takes (copied as float64)"""
        t = self.torch
        q = q if t.is_tensor(q) and q.is_cuda else t.as_tensor(np.ascontiguousarray(q, np.float64), device=self.obs.device)
        if q.dim() != 2 or q.dtype not in (t.float32, t.float64) or q.shape[1] < NQ or q.stride(1) != 1 or (n is not None and q.shape[0] != n):
            raise ValueError(who + ": qpos rows must be [n][>= 76] contiguous rows of float32 | float64 (the ghost as many as qpos)")
        return q

    def _variant_arg(self, variants, n):
        if variants is None:
            return None
        t = self.torch
        if t.is_tensor(variants) and variants.is_cuda and variants.dtype == t.int32 and variants.is_contiguous() and tuple(variants.shape) == (n,):
            return variants                        # already on the device: used in place
        return self.torch.as_tensor(np.array(np.broadcast_to(np.asarray(variants, np.int32), (n,))), device=self.obs.device)

    def render_pose(self, qpos, ghost=None, variants=None):
        """the renderer's pose table (uhc_render_pose) [n][2][24][12] float32: per body the world rotation (row-major) and position of qpos row
        i (humanoid 0) and ghost row i (humanoid 1, zero without a ghost), from the fp64 FK with shape variant variants[i] (None: 0)"""
        t = self.torch
        q = self._rows(qpos)
        n = q.shape[0]
        g = None if ghost is None else self._rows(ghost, n)
        v = self._variant_arg(variants, n)
        pose = t.zeros(n, 2, 24, 12, dtype=t.float32, device=self.obs.device)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        pitch = lambda x: C.c_long(x.stride(0) if x is not None and x.shape[0] > 1 else (x.shape[1] if x is not None else NQ))
        _chk(self.lib.uhc_render_pose(self.h, C.c_long(n), p(q), C.c_int(32 if q.dtype == t.float32 else 64), pitch(q), p(g), pitch(g), p(v),
                                      p(pose), self._stream()), "uhc_render_pose", ValueError)
        return pose

    def _render_out(self, n, size, depth, label):
        t = self.torch
        W, H = (int(x) for x in size)
        dev = self.obs.device
        rgb = t.empty(n, H, W, 3, dtype=t.uint8, device=dev)
        dep = t.empty(n, H, W, dtype=t.float32, device=dev) if depth else None
        lab = t.empty(n, H, W, dtype=t.uint8, device=dev) if label else None
        return W, H, rgb, dep, lab

    def render(self, qpos, ghost=None, variants=None, camera=None, size=(640, 360), depth=False, label=False):
        """n frames of W x H pixels (uhc_render_qpos): frame i shows the humanoid at qpos row i (grey) and, with a ghost, the ghost at ghost row i
        (red).  qpos / ghost: cuda tensors [n][>= 76] of float32 | float64 read in place (a state record of 148 or the tracker's state_out of 223
        as they are), or arrays numpy takes.  variants: shape variant per frame (None: 0).  camera: a dict for make_camera (MuJoCo's free camera
        with focus / hide_im / hide_expert / shift_expert).  Returns (rgb [n][H][W][3] uint8, depth [n][H][W] float32 (m along the ray, inf on
        sky) or None, label [n][H][W] uint8 (0 sky, 1 floor, 2 + b body b, 26 + b the ghost's body b) or None), cuda tensors."""
        t = self.torch
        self._render_init()
        q = self._rows(qpos)
        n = q.shape[0]
        g = None if ghost is None else self._rows(ghost, n)
        v = self._variant_arg(variants, n)
        W, H, rgb, dep, lab = self._render_out(n, size, depth, label)
        cam = make_camera(camera)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        pitch = lambda x: C.c_long(x.stride(0) if x is not None and x.shape[0] > 1 else (x.shape[1] if x is not None else NQ))
        _chk(self.lib.uhc_render_qpos(self.h, C.byref(cam), C.c_int(W), C.c_int(H), C.c_long(n), p(q), C.c_int(32 if q.dtype == t.float32 else 64),
                                      pitch(q), p(g), pitch(g), p(v), p(rgb), p(dep), p(lab), self._stream()), "uhc_render_qpos", ValueError)
        return rgb, dep, lab

    def render_bodies(self, pose, humanoids=2, variants=None, camera=None, size=(640, 360), depth=False, label=False):
        """render() from a pose table [n][2][24][12] float32 cuda tensor (render_pose's layout) instead of qpos (uhc_render_bodies)"""
        t = self.torch
        self._render_init()
        assert pose.is_cuda and pose.dtype == t.float32 and pose.is_contiguous() and pose.dim() == 4 and tuple(pose.shape[1:]) == (2, 24, 12)
        n = pose.shape[0]
        v = self._variant_arg(variants, n)
        W, H, rgb, dep, lab = self._render_out(n, size, depth, label)
        cam = make_camera(camera)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(self.lib.uhc_render_bodies(self.h, C.byref(cam), C.c_int(W), C.c_int(H), C.c_long(n), p(pose), C.c_int(int(humanoids)), p(v),
                                        p(rgb), p(dep), p(lab), self._stream()), "uhc_render_bodies", ValueError)
        return rgb, dep, lab

    # ---- the mesh renderer (include/uhc_render.h uhc_render_mesh*)
    def render_mesh_init(self, model):
        """uploads the mesh renderer's topology (uhc_render_mesh_init) of an SMPL model with faces: a dict as
        uhc_b200.smpl_model.load_smpl_model returns it, or a path it reads.  The tables are built on the host (uhc_b200.render_mesh); a later
        call replaces them, a failed one leaves the previous ones."""
        from uhc_b200.render_mesh import build_tables
        from uhc_b200.smpl_model import as_model
        m = as_model(model)
        if m.get("faces") is None:
            raise ValueError("render_mesh_init: the SMPL model has no faces (key f)")
        self._rmesh = UhcRenderMesh.of(build_tables(m["faces"], m["weights"], m["v_template"], self.model.body_names), len(m["v_template"]))
        _chk(self.lib.uhc_render_mesh_init(self.h, C.byref(self._rmesh)), "uhc_render_mesh_init", ValueError)

    def render_mesh(self, verts, ghost_verts=None, root=None, camera=None, size=(640, 360), depth=False, label=False):
        """n frames of W x H pixels of the skinned mesh (uhc_render_mesh) after render_mesh_init: verts / ghost_verts = [n][V][3] (smpl_mesh's
        vertices: contiguous float32 cuda tensors are read in place, anything else is copied as float32), root = [n][3] where a camera with focus looks (the first humanoid's root).  Outputs, labels
        and the camera as render()."""
        t = self.torch
        dev = self.obs.device
        verts = t.as_tensor(verts, dtype=t.float32, device=dev).contiguous()          # in place when already a contiguous float32 cuda tensor
        ghost_verts = None if ghost_verts is None else t.as_tensor(ghost_verts, dtype=t.float32, device=dev).contiguous()
        if verts.dim() != 3 or verts.shape[2] != 3 or (ghost_verts is not None and ghost_verts.shape != verts.shape):
            raise ValueError("render_mesh: verts and ghost_verts must be [n][V][3] of one shape")
        n, V = int(verts.shape[0]), int(verts.shape[1])
        if root is not None:
            root = t.as_tensor(root, dtype=t.float32, device=self.obs.device).contiguous()
            if tuple(root.shape) != (n, 3):
                raise ValueError("render_mesh: root must be [n][3]")
        W, H, rgb, dep, lab = self._render_out(n, size, depth, label)
        cam = make_camera(camera)
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(self.lib.uhc_render_mesh(self.h, C.byref(cam), C.c_int(W), C.c_int(H), C.c_long(n), p(verts), p(ghost_verts), p(root), C.c_int(V),
                                      p(rgb), p(dep), p(lab), self._stream()), "uhc_render_mesh", ValueError)
        return rgb, dep, lab

    def render_smpl(self, qpos, ghost=None, betas=None, beta_idx=None, variants=None, camera=None, size=(640, 360), depth=False, label=False):
        """qpos rows (and the ghost's) -> SMPL (qpos_to_smpl with `variants`) -> the skinned mesh (smpl_mesh with betas [nb][10] and beta_idx per
        row, shared by both humanoids) -> render_mesh, without leaving the device; needs mesh_init and render_mesh_init of the same model.  The
        focus root is qpos[:, :3], the hull renderer's root, so a mesh frame is framed exactly like render()'s frame of the same qpos."""
        if betas is None:
            raise ValueError("render_smpl: betas [nb][10] are required")
        q = self._rows(qpos, who="render_smpl")
        g = None if ghost is None else self._rows(ghost, q.shape[0], who="render_smpl")
        verts = self.qpos_mesh(q, betas, beta_idx, variants, joints=False)[0]
        gverts = None if g is None else self.qpos_mesh(g, betas, beta_idx, variants, joints=False)[0]
        root = q[:, :3].to(self.torch.float32).contiguous()
        return self.render_mesh(verts, gverts, root, camera, size, depth, label)

    # ---- the JPEG encoder (include/uhc_video.h)
    def encode_jpeg(self, rgb, quality=90):
        """frames rgb [n][H][W][3] (a contiguous cuda uint8 tensor, render()'s layout) -> (data, offsets): one baseline JPEG file per frame
        (uhc_jpeg_encode), packed in the cuda uint8 tensor data, file i = data[offsets[i]:offsets[i + 1]] with offsets a cuda int64 tensor [n + 1]"""
        t = self.torch
        if not (t.is_tensor(rgb) and rgb.is_cuda and rgb.dtype == t.uint8 and rgb.dim() == 4 and rgb.shape[3] == 3 and rgb.is_contiguous()):
            raise ValueError("encode_jpeg: rgb must be a contiguous cuda uint8 tensor [n][H][W][3]")
        n, H, W = (int(x) for x in rgb.shape[:3])
        dev = rgb.device
        offsets = t.empty(n + 1, dtype=t.int64, device=dev)
        hints = self.__dict__.setdefault("_jpeg_hint", {})
        key = (W, H, int(quality))
        cap = max(1, n * hints.get(key, W * H // 4 + 1024))           # bytes per frame seen so far at this size and quality, with a margin
        total = C.c_size_t(0)
        for _ in range(2):
            data = t.empty(cap, dtype=t.uint8, device=dev)
            rc = self.lib.uhc_jpeg_encode(self.h, C.c_void_p(rgb.data_ptr()), C.c_long(n), C.c_int(W), C.c_int(H), C.c_int(int(quality)),
                                          C.c_void_p(data.data_ptr()), C.c_size_t(cap), C.c_void_p(offsets.data_ptr()), C.byref(total),
                                          self._stream())
            if rc != -3:
                break
            cap = int(total.value)                                     # too small: the call reported the size it needs
        _chk(rc, "uhc_jpeg_encode", ValueError)
        if n:
            hints[key] = max(hints.get(key, 0), int(total.value) * 5 // (4 * n) + 1)
        return data[:int(total.value)], offsets

    # ---- the batched physics tracker (include/uhc_track.h uhc_track_*)
    def track_begin(self, window=8, kind="qpos", pose_dim=None, fk_models=None, shapes=None):
        """tracking mode: env e follows a stream of raw target frames (kind "qpos": qpos rows of 76; "smpl": pose_aa (pose_dim 72 | 156) then
        trans) held in a window of `window` expert-table rows.  fk_models: shape variant per env (FK and simulated body), shapes: [E][17]."""
        k = {"qpos": 1, "smpl": 0, 1: 1, 0: 0}[kind]
        pose_dim = (NQ if k == 1 else 72) if pose_dim is None else int(pose_dim)
        fk = None if fk_models is None else np.ascontiguousarray(fk_models, np.int32).reshape(self.E)
        shp = None if shapes is None else np.ascontiguousarray(np.asarray(shapes, np.float64).reshape(self.E, 17))
        _chk(self.lib.uhc_track_begin(self.h, C.c_int(int(window)), C.c_int(k), C.c_int(pose_dim), None if fk is None else _ip_out(fk),
                                      None if shp is None else shp.ctypes.data_as(C.POINTER(C.c_double))), "uhc_track_begin", ValueError)
        self.track_row_w = NQ if k == 1 else pose_dim + 3
        self._table_loaded(np.full(self.E, int(window), np.int32), fk)

    def track_reset(self, env_ids, frames, qpos=None, qvel=None):
        """frames: float64 cuda tensor [n][2][row width], target frames 0 and 1 of each listed env; qpos / qvel: optional fp32 cuda overrides"""
        t = self.torch
        ids = np.ascontiguousarray(env_ids, np.int32).reshape(-1)
        assert frames.is_cuda and frames.dtype == t.float64 and frames.is_contiguous() and tuple(frames.shape) == (len(ids), 2, self.track_row_w)
        for x, w in ((qpos, NQ), (qvel, NV)):
            assert x is None or (x.is_cuda and x.dtype == t.float32 and x.is_contiguous() and tuple(x.shape) == (len(ids), w))
        _chk(self.lib.uhc_track_reset(self.h, C.c_int(len(ids)), _ip_out(ids), C.c_void_p(frames.data_ptr()),
                                      C.c_void_p(qpos.data_ptr() if qpos is not None else None), C.c_void_p(qvel.data_ptr() if qvel is not None else None),
                                      self._stream()), "uhc_track_reset", ValueError)

    def track_step(self, next_frames, mask, policy, log_std, zfilter_stats, zclip, fail_safe, state_out, reward_out, fail_out):
        """one tracker step of every env (uhc_track_step): next_frames float64 [E][row width] or None, mask int32 [E] or None; the outputs
        are written into state_out [E][223] (engine precision: qpos 76 | qvel 75 | xpos 72), reward_out [E] fp32, fail_out [E] int32"""
        t = self.torch
        if next_frames is not None:
            assert next_frames.is_cuda and next_frames.dtype == t.float64 and next_frames.is_contiguous() and tuple(next_frames.shape) == (self.E, self.track_row_w)
        if mask is not None:
            assert mask.is_cuda and mask.dtype == t.int32 and mask.is_contiguous() and tuple(mask.shape) == (self.E,)
        from .nn import UhcMcp
        fn = self.lib.uhc_track_step_mcp if isinstance(policy, UhcMcp) else self.lib.uhc_track_step
        p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
        _chk(fn(self.h, p(next_frames), p(mask), C.byref(policy), p(log_std), p(zfilter_stats), C.c_float(zclip), C.c_int(int(bool(fail_safe))),
                p(state_out), p(reward_out), p(fail_out), self._stream()), "uhc_track_step", ValueError)

    def track_push(self, next_frames, mask=None):
        """append a frame to every (masked-in) env's stream without stepping (uhc_track_push)"""
        t = self.torch
        assert next_frames.is_cuda and next_frames.dtype == t.float64 and next_frames.is_contiguous() and tuple(next_frames.shape) == (self.E, self.track_row_w)
        assert mask is None or (mask.is_cuda and mask.dtype == t.int32 and mask.is_contiguous() and tuple(mask.shape) == (self.E,))
        _chk(self.lib.uhc_track_push(self.h, C.c_void_p(next_frames.data_ptr()), C.c_void_p(mask.data_ptr() if mask is not None else None),
                                     self._stream()), "uhc_track_push", ValueError)

    def track_obs(self, out=None):
        """the observation the next track_step feeds the policy (uhc_track_obs), [E][obs_dim] fp32"""
        out = self.torch.empty(self.E, self.obs_dim, device=self.obs.device) if out is None else out
        _chk(self.lib.uhc_track_obs(self.h, C.c_void_p(out.data_ptr()), self._stream()), "uhc_track_obs", ValueError)
        return out

    def track_state(self):
        """per env: steps since its reset, cur_t in the window, rows held, pushes dropped on a full window (synchronises)"""
        out = np.zeros((self.E, 4), np.int32)
        _chk(self.lib.uhc_track_state(self.h, _ip_out(out)), "uhc_track_state", ValueError)
        return dict(steps=out[:, 0], cur_t=out[:, 1], rows=out[:, 2], dropped=out[:, 3])

    def track_end(self):
        self.lib.uhc_track_end(self.h)

    @property
    def track_graph_count(self):
        """CUDA graphs the tracker holds for this engine now (uhc_track_graph_count)"""
        return int(self.lib.uhc_track_graph_count(self.h))

    def track_subjects_enable(self, basis):
        """run-time subjects (uhc_track_subjects_enable): one extra shape variant per env, filled by track_set_subjects; basis = a
        subject_body.SubjectBasis of this engine's model.  Before track_begin."""
        s = basis.struct()
        _chk(self.lib.uhc_track_subjects_enable(self.h, C.byref(s)), "uhc_track_subjects_enable", ValueError)

    def track_subject_tables(self, env):
        """env's run-time subject slot (uhc_track_subject_tables): dict(body_f [24][20], hull [nvert][3]) in the engine's precision widened to
        float64, fk_body [24][6] and hull64 [nvert][3] in float64"""
        nv = len(self.model.hull)
        out = dict(body_f=np.zeros((24, 20)), hull=np.zeros((nv, 3)), fk_body=np.zeros((24, 6)), hull64=np.zeros((nv, 3)))
        d = lambda k: out[k].ctypes.data_as(C.POINTER(C.c_double))
        _chk(self.lib.uhc_track_subject_tables(self.h, C.c_int(int(env)), d("body_f"), d("hull"), d("fk_body"), d("hull64")),
             "uhc_track_subject_tables", ValueError)
        return out

    def track_set_subjects(self, env_ids, shapes):
        """each listed env's own body from its shape row [17] = beta 16, gender code (uhc_track_set_subjects); track_reset those envs next"""
        ids = np.ascontiguousarray(env_ids, np.int32).reshape(-1)
        shp = np.ascontiguousarray(np.asarray(shapes, np.float64).reshape(len(ids), 17))
        _chk(self.lib.uhc_track_set_subjects(self.h, C.c_int(len(ids)), _ip_out(ids), shp.ctypes.data_as(C.POINTER(C.c_double)), self._stream()),
             "uhc_track_set_subjects", ValueError)

    def set_clip_weights(self, weights=None):
        """sampling weights of the in-kernel re-seeding (None = the reference's sample_keys rule)."""
        if weights is None:
            _chk(self.lib.uhc_set_clip_weights(self.h, C.c_int(len(self.clip_len)), None))
        else:
            w = np.ascontiguousarray(weights, dtype=np.float32)
            _chk(self.lib.uhc_set_clip_weights(self.h, C.c_int(len(w)), w.ctypes.data_as(C.POINTER(C.c_float))))

    # ---- the failure-weighted curriculum on the device (include/uhc_rollout.h uhc_curriculum_*)
    def curriculum_enable(self, max_freq=50, temp=0.2, freq=0.5, prec_freq=0.0, fit_clip=-1):
        """per-clip outcome rings of max_freq entries on the device; from here on the curriculum owns the clip CDF.  Called again with the
        same max_freq it keeps the history; max_freq = 0 turns it off."""
        _chk(self.lib.uhc_curriculum_enable(self.h, C.c_int(int(max_freq)), C.c_double(float(temp)), C.c_double(float(freq)),
                                            C.c_double(float(prec_freq)), C.c_int(int(fit_clip))), "uhc_curriculum_enable", ValueError)
        self.cur_cfg = dict(max_freq=int(max_freq), temp=float(temp), freq=float(freq), prec_freq=float(prec_freq), fit_clip=int(fit_clip)) if max_freq else None

    def curriculum_update(self, buf, T):
        """append the episodes that ended in rows 0 .. T-1 of a RolloutBuffer and rewrite the clip CDF, stream-ordered, no synchronise"""
        from .agent import UhcRolloutBuf
        b = UhcRolloutBuf()
        b.ep_clip, b.ep_pct, b.ep_start, b.T_cap = buf.ep_clip.data_ptr(), buf.ep_pct.data_ptr(), buf.ep_start.data_ptr(), buf.T
        _chk(self.lib.uhc_curriculum_update(self.h, C.byref(b), C.c_int(int(T)), self._stream()), "uhc_curriculum_update", ValueError)

    def curriculum_push(self, clips, pct, starts):
        clips = np.ascontiguousarray(clips, np.int32).reshape(-1)
        p = np.ascontiguousarray(pct, np.float32).reshape(-1)
        s = np.ascontiguousarray(starts, np.int32).reshape(-1)
        assert len(clips) == len(p) == len(s)
        _chk(self.lib.uhc_curriculum_push(self.h, C.c_int(len(clips)), _ip(clips), p.ctypes.data_as(C.POINTER(C.c_float)), _ip(s)),
             "uhc_curriculum_push", ValueError)

    def curriculum_get(self):
        """every clip's history, oldest first: (len [C], percent [C][max_freq], start [C][max_freq])"""
        n, M = len(self.clip_len), self.cur_cfg["max_freq"]
        ln, p, s = np.zeros(n, np.int32), np.zeros((n, M), np.float32), np.zeros((n, M), np.int32)
        _chk(self.lib.uhc_curriculum_get(self.h, _ip_out(ln), p.ctypes.data_as(C.POINTER(C.c_float)), _ip_out(s)), "uhc_curriculum_get", ValueError)
        return ln, p, s

    def curriculum_set(self, lens, pct, starts):
        n, M = len(self.clip_len), self.cur_cfg["max_freq"]
        ln = np.ascontiguousarray(lens, np.int32).reshape(n)
        p = np.ascontiguousarray(pct, np.float32).reshape(n, M)
        s = np.ascontiguousarray(starts, np.int32).reshape(n, M)
        _chk(self.lib.uhc_curriculum_set(self.h, _ip(ln), p.ctypes.data_as(C.POINTER(C.c_float)), _ip(s)), "uhc_curriculum_set", ValueError)

    def clip_cdf(self):
        """the sampler's cumulative clip weights [C] (fp32)"""
        out = np.zeros(len(self.clip_len), np.float32)
        _chk(self.lib.uhc_get_clip_cdf(self.h, out.ctypes.data_as(C.POINTER(C.c_float))))
        return out

    def curriculum_reseed(self):
        """re-seed every env through the in-kernel sampler; returns the obs tensor with the reset rows"""
        _chk(self.lib.uhc_curriculum_reseed(self.h, C.c_void_p(self.obs.data_ptr()), self._stream()), "uhc_curriculum_reseed", ValueError)
        return self.obs

    @property
    def counters(self):
        out = np.zeros(4, np.int32)
        _chk(self.lib.uhc_engine_counters(self.h, out.ctypes.data_as(C.POINTER(C.c_int))))
        return dict(contact_overflow_steps=int(out[0]), invalid_env_steps=int(out[1]))

    @property
    def kernel_launches(self):
        return self.lib.uhc_kernel_launches(self.h)
