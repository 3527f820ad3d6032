"""The trained controller as a batched physics tracker (include/uhc_track.h): every env follows target poses that exist only once the
previous step has run, the role the UHC policy plays inside HumanoidKinEnv.step (uhc/envs/humanoid_kin_v1.py:297-370).

    trk = agent.tracker(window=8, kind="qpos")
    trk.reset(f0, f1)                  # target frames 0 and 1 of every env, float64 cuda [E][76]
    state, reward, fail = trk.step()   # the first step tracks frame 1, which the reset supplied
    while ...:
        state, reward, fail = trk.step(kin(state))   # frame t + 1 from the simulated state

Each step is one CUDA-graph replay on the device: the new frame's expert record, the observation against it, the policy mean, the
physics step and fail_safe.  The returned tensors are the tracker's own buffers, overwritten by the next step.

With subjects= (a subject_body.SubjectBasis, e.g. SubjectBasis.from_models over the user's SMPL files) every env can be given its own body
while the tracker runs, as the reference's reset_robot rebuilds the humanoid for each sequence:

    trk = agent.tracker(window=8, kind="smpl", subjects=basis)
    trk.set_subjects([3], betas=[beta], genders=["female"])   # env 3's body, built on the GPU
    trk.reset(f0[3:4], f1[3:4], env_ids=[3])                  # its rows from the new body's FK; the other envs keep stepping
"""
import numpy as np

from . import nn


class Tracker:
    def __init__(self, agent, window=8, kind="qpos", fail_safe=True, pose_dim=None, fk_models=None, shapes=None, subjects=None):
        import torch
        self.torch, self.agent, self.engine = torch, agent, agent.engine
        self.E, self.fail_safe = agent.E, bool(fail_safe)
        if subjects is not None:
            self.engine.track_subjects_enable(subjects)
        self.engine.track_begin(window, kind, pose_dim, fk_models, shapes)
        self.row_w = self.engine.track_row_w
        dev = agent.dev
        self.state = torch.zeros(self.E, 223, device=dev, dtype=torch.float32 if self.engine.precision == 32 else torch.float64)
        self.reward = torch.zeros(self.E, device=dev, dtype=torch.float32)
        self.fail = torch.zeros(self.E, device=dev, dtype=torch.int32)

    def _policy(self):
        a = self.agent
        return nn.mcp_struct(a.policy) if a.actor_type == "mcp" else nn.mlp_struct(a.policy)

    def reset(self, f0, f1, env_ids=None, qpos=None, qvel=None):
        """frames 0 and 1 ([n][row width] each) of the listed envs (default: all); the envs start on frame 0 (or the fp32 overrides)"""
        t = self.torch
        ids = np.arange(self.E, dtype=np.int32) if env_ids is None else np.asarray(env_ids, np.int32).reshape(-1)
        frames = t.stack([t.as_tensor(f0), t.as_tensor(f1)], 1).to(device=self.state.device, dtype=t.float64).contiguous()
        cvt = lambda x: None if x is None else t.as_tensor(x).to(device=self.state.device, dtype=t.float32).contiguous()
        self.engine.track_reset(ids, frames, cvt(qpos), cvt(qvel))
        self.agent.obs = None          # the envs left whatever episode they were on

    def set_subjects(self, env_ids, betas, genders):
        """gives each listed env its own body, built on the device from betas [n][10 .. 16] (the first 10 shape the body, all of them up to 16
        go into the shape observation) and genders [n] (0 / "neutral", 1 / "male", 2 / "female", DatasetAMASSSingle's codes).  Needs subjects=
        at construction.  The envs do not step again until reset(..., env_ids=...) gives them frames; the others are untouched."""
        from uhc.data_loaders.dataset_amass_single import _gender_code
        ids = np.asarray(env_ids, np.int32).reshape(-1)
        b = np.asarray(betas, np.float64).reshape(len(ids), -1)
        if b.shape[1] < 10 or b.shape[1] > 16:
            raise ValueError("set_subjects: betas must be [n][10 .. 16]")
        g = [x if isinstance(x, (int, np.integer)) else _gender_code(x) for x in np.asarray(genders, object).reshape(-1)]
        shapes = np.zeros((len(ids), 17))
        shapes[:, :b.shape[1]], shapes[:, 16] = b, g
        self.engine.track_set_subjects(ids, shapes)

    def step(self, next_frames=None, mask=None):
        """next_frames: target frame t + 1 of every env ([E][row width], None on the first step after a reset); mask: int32 [E], 0 = this
        env gets no frame.  Returns (state [E][223] = qpos 76 | qvel 75 | xpos 72 as the step left it, reward [E], fail [E])."""
        t = self.torch
        nf = None if next_frames is None else t.as_tensor(next_frames).to(device=self.state.device, dtype=t.float64).contiguous()
        mk = None if mask is None else t.as_tensor(mask).to(device=self.state.device, dtype=t.int32).contiguous()
        a = self.agent
        self.engine.track_step(nf, mk, self._policy(), a.log_std, a.running_state.stats, a.running_state.clip, self.fail_safe,
                               self.state, self.reward, self.fail)
        return self.state, self.reward, self.fail

    @property
    def qpos(self):
        return self.state[:, :76]

    @property
    def qvel(self):
        return self.state[:, 76:151]

    @property
    def xpos(self):
        return self.state[:, 151:223].reshape(self.E, 24, 3)

    def smpl(self):
        """the state of the last step as SMPL (qpos_to_smpl on the device, each env with its fk_models shape variant or its set_subjects body), enqueued on the tracker's
        stream with no host synchronise.  Returns (pose_aa [E][72], trans [E][3]), float64 tensors overwritten by the next call."""
        if getattr(self, "_smpl", None) is None:
            t = self.torch
            self._smpl = (t.empty(self.E, 72, device=self.state.device, dtype=t.float64), t.empty(self.E, 3, device=self.state.device, dtype=t.float64))
        return self.engine.track_smpl(self.state, *self._smpl)

    def floor(self):
        """the body hulls of the last step's state against the floor (uhc_floor_qpos' kernel at pitch 223, each env with its fk_models shape variant
        or its set_subjects body
        and no previous frame: the envs are unrelated rows, so skate_mm is 0).  Returns [E][5] float64 on the device: min_z (m), pen_mm,
        skate_mm, float_mm, n_below, a tensor overwritten by the next call.  The variants were range-checked by track_begin, so nothing synchronises
        (as smpl())."""
        if getattr(self, "_floor", None) is None:
            self._floor = self.torch.empty(self.E, 5, device=self.state.device, dtype=self.torch.float64)
        return self.engine.track_floor(self.state, self._floor)

    def steps(self):
        """control steps each env has taken since its reset (synchronises)"""
        return self.engine.track_state()["steps"]

    def close(self):
        self.engine.track_end()
