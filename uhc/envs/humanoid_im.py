"""HumanoidEnv: single-environment facade with the reference's env surface (uhc/envs/humanoid_im.py:50, khrylib
mujoco_env.py:95-113) over one environment of the batched engine.  Used by evaluation / debugging code that wants the
classic gym-style loop; training uses uhc_b200.agent.BatchedAgent (thousands of envs in lock-step).

    env = HumanoidEnv(cfg, init_expert, data_specs, mode)     # init_expert: a dataset sample dict (pose_aa, trans, beta, gender, ...)
    obs = env.reset()                                          # np.ndarray[657] float64
    obs, reward(=1.0), done, info = env.step(a[105])           # info: fail / end / percent   (humanoid_im.py:1243)
"""
import numpy as np

from uhc_b200 import motion_lib
from uhc_b200.engine import Engine
from uhc_b200.model import HumanoidModel


class _Space:
    def __init__(self, n):
        self.shape = (n,)
        self.low, self.high = -np.ones(n), np.ones(n)


class _RobotShim:
    smpl_model = "smpl"

    def export_vis_string(self):
        raise NotImplementedError("the batched engine has no MuJoCo XML to export; rendering is out of scope")


class _ModelShim:
    """The few mujoco_py model attributes the agent / reward code reads (agent_copycat.py:139, humanoid_im.py:917)."""

    def __init__(self, tables):
        self.body_names = list(tables.body_names)
        self._body_name2id = {n: i for i, n in enumerate(self.body_names)}
        self.actuator_names = [f"{b}_{ax}" for b in self.body_names[1:] for ax in "zyx"]   # three hinges z, y, x per non-root body


class _DataShim:
    """data.qpos / data.qvel / data.body_xpos views of the engine state (read-only copies)."""

    def __init__(self, env):
        self._env = env

    qpos = property(lambda self: self._env.engine.get_state(0)["qpos"])
    qvel = property(lambda self: self._env.engine.get_state(0)["qvel"])
    body_xpos = property(lambda self: self._env.engine.get_state(0)["xpos"])


def _quat_rot(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def _transform_vec(v, q, trans="root"):
    """uhc/utils/math_utils.py:103-115."""
    q = np.asarray(q, dtype=np.float64).copy()
    if trans == "heading":
        q[1] = q[2] = 0.0
    else:
        assert trans == "root"
    return _quat_rot(q).T.dot(v)


class HumanoidEnv:
    def __init__(self, cfg, init_expert, data_specs, mode="train", no_root=False, device=0, precision=32):
        import torch
        self.torch = torch
        self.cc_cfg, self.mode = cfg, mode
        self.model_tables = HumanoidModel()
        rw = cfg.reward_weights or {}
        w = [rw.get(k, d) for k, d in (("w_p", 0.6), ("w_v", 0.1), ("w_e", 0.2), ("w_c", 0.1), ("w_vf", 0.0))]
        k = [rw.get(k, d) for k, d in (("k_p", 2), ("k_v", 0.005), ("k_e", 20), ("k_c", 1000), ("k_vf", 1))]
        self.engine = Engine(1, self.model_tables, device=device, precision=precision, base_rot=data_specs.get("base_rot", [0.7071, 0.7071, 0.0, 0.0]),
                             rfc_scale=cfg.residual_force_scale, rfc_lim=cfg.residual_force_lim, rfc_rate=0.0 if cfg.rfc_decay else 1.0,
                             body_diff_thresh=cfg.get("body_diff_thresh", 0.5) if mode == "train" else cfg.get("body_diff_thresh_test", 0.5),
                             meta_pd=int(cfg.meta_pd), env_episode_len=cfg.env_episode_len, trail_steps=cfg.env_expert_trail_steps, w=w, k=k,
                             rfc_mode=cfg.get("residual_force_mode", "implicit") if cfg.residual_force else "none", obs_v=int(cfg.get("obs_v", 2)),
                             fut_frames=int(cfg.get("fut_frames", 10)), fut_skip=int(cfg.get("skip", 10)),
                             has_shape=bool(cfg.get("has_shape", False)) and bool(cfg.get("has_shape_obs", True)),
                             term_body=cfg.get("env_term_body", "body") if cfg.get("env_term_body", "body") in ("root", "Head") else "body",
                             head_body=self.model_tables.body_names.index("Head"), reward_mul=cfg.get("reward_id", "") == "world_rfc_implicit_v1_mul")
        self.dt = self.model_tables.dt * 15
        # set_action_spaces (humanoid_im.py:226-255): implicit = 6 residual-force dims, explicit = 9 per body x 24 bodies
        explicit = cfg.get("residual_force_mode", "implicit") == "explicit"
        self.ndof, self.vf_dim, self.meta_pd_dim = 69, (216 if explicit else 6) if cfg.residual_force else 0, 30 if cfg.meta_pd else 0
        self.body_vf_dim, self.vf_bodies = 9, list(self.model_tables.SMPL_BONE_ORDER)
        ACT_DIM = self.engine.act_dim
        assert ACT_DIM == self.ndof + self.vf_dim + self.meta_pd_dim
        OBS_DIM = self.engine.obs_dim
        self.action_dim, self.obs_dim = ACT_DIM, OBS_DIM
        self.action_space, self.observation_space = _Space(ACT_DIM), _Space(OBS_DIM)
        self.body_diffw, self.jpos_diffw = self.model_tables.diffw[1:], self.model_tables.diffw[:, None]
        self.smpl_robot, self.np_random = _RobotShim(), np.random.RandomState(0)
        self.model, self.data, self.converter = _ModelShim(self.model_tables), _DataShim(self), None
        self.prev_bquat = None
        self.cur_t, self.start_ind, self.end_reward, self.rfc_rate = 0, 0, 0.0, 1.0
        self.last_reward, self.last_cinfo = 0.0, np.zeros(5)
        self._act = torch.zeros(1, ACT_DIM, device=self.engine.obs.device, dtype=torch.float32)
        self.load_expert(init_expert)

    def seed(self, seed=None):
        self.np_random = np.random.RandomState(seed)
        return [seed]

    def set_mode(self, mode):
        self.mode = mode

    def load_expert(self, expert_data, reload_robot=True):
        """humanoid_im.py:182-215: pose_aa/trans -> qpos -> expert dict (plus the pass-through keys)."""
        self.expert = dict(expert_data)
        self.expert.update(motion_lib.make_expert(expert_data["pose_aa"], np.asarray(expert_data["trans"]).squeeze(), self.model_tables))
        self.expert["meta"] = {"cyclic": False, "seq_name": expert_data.get("seq_name", "")}
        beta = np.asarray(expert_data.get("beta", np.zeros((1, 16))))[0]
        gender = float(np.asarray(expert_data.get("gender", [0]))[0])
        self.engine.load_clips([self.expert], [np.concatenate([beta, [gender]])])

    def reset(self):
        self.cur_t = 0
        qpos = None
        if self.mode == "train" and self.cc_cfg.env_init_noise > 0:   # humanoid_im.py:1253
            qpos = self.expert["qpos"][0].copy()
            qpos[7:] += self.np_random.normal(0.0, self.cc_cfg.env_init_noise, 69)
        obs = self.engine.reset([0], 0, 0, None, qpos=qpos[None] if qpos is not None else None,
                                qvel=self.expert["qvel"][:1] if qpos is not None else None)
        self.prev_bquat = None            # humanoid_im.py:95 / :1198: set at the start of each step
        return obs[0].double().cpu().numpy()

    def step(self, a):
        self.prev_bquat = self.get_body_quat().copy()
        self._act.copy_(self.torch.as_tensor(np.asarray(a, dtype=np.float32)).reshape(1, self.action_dim))
        obs, rew, cinfo, fail, end, pct = self.engine.step(self._act)
        self.cur_t += 1
        self.last_reward, self.last_cinfo = float(rew[0]), cinfo[0].cpu().numpy()
        f, e = bool(fail[0]), bool(end[0])
        return obs[0].double().cpu().numpy(), 1.0, f or e, {"fail": f, "end": e, "percent": float(pct[0])}

    # ---- getters the agent / reward code of the reference touches (humanoid_im.py:1322-1415)
    def get_expert_index(self, t):
        return min(self.start_ind + t, self.expert["len"] - 1)

    def get_expert_attr(self, attr, ind):
        return np.asarray(self.expert[attr][ind]).copy()

    def get_expert_qpos(self, delta_t=0):
        return self.get_expert_attr("qpos", self.get_expert_index(self.cur_t + delta_t))

    def get_expert_qvel(self, delta_t=0):
        return self.get_expert_attr("qvel", self.get_expert_index(self.cur_t + delta_t))

    def get_humanoid_qpos(self):
        return self.engine.get_state(0)["qpos"]

    def get_humanoid_qvel(self):
        return self.engine.get_state(0)["qvel"]

    def get_wbody_pos(self, selectList=None):
        return self.engine.get_state(0)["xpos"].ravel()

    def get_body_quat(self):
        return self.engine.get_state(0)["bquat"]

    @property
    def bquat(self):
        return self.get_body_quat()

    def get_ee_pos(self, transform):
        """humanoid_im.py:910-923: the five end effectors, world frame or relative to the root in its root / heading frame."""
        st = self.engine.get_state(0)
        out = []
        for b in self.model_tables.ee:
            v = st["xpos"][int(b)].copy()
            if transform is not None:
                v = _transform_vec(v - st["qpos"][:3], st["qpos"][3:7], transform)
            out.append(v)
        return np.concatenate(out)

    def get_com(self):
        """humanoid_im.py:962-965: data.get_body_xipos("Pelvis")."""
        st = self.engine.get_state(0)
        return st["xpos"][0] + _quat_rot(st["qpos"][3:7]).dot(self.model_tables.ipos[0])

    def render(self, *a, **k):
        raise NotImplementedError("rendering needs MuJoCo; the batched engine has no viewer")

    def calc_body_diff(self):
        cur = self.engine.get_state(0)["xpos"]
        e = self.get_expert_attr("wbpos", self.get_expert_index(self.cur_t)).reshape(-1, 3)
        d = (cur - e) * self.jpos_diffw
        return np.linalg.norm(d[self.jpos_diffw.squeeze().astype(bool)], axis=1).mean()

    def fail_safe(self):
        """humanoid_im.py:902-905: snap the simulator onto the expert and run sim.forward()."""
        self.engine.set_state(0, self.get_expert_qpos(), self.get_expert_qvel())
