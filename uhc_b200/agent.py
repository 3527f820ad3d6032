"""Batched rollout + PPO driver on the engine (SURVEY.md section 8a rows a11, a15-a17).

Replaces the reference's fork-per-iteration CPU workers (uhc/agents/agent_copycat.py:496-605, khrylib/rl/agents/agent.py:42-126)
by E device-resident environments stepped in lock-step: per control step one obs-normaliser pass, one policy forward
(tensor cores), one Gaussian sample, one fused physics/task kernel, and the transition lands in a time-major [T][E] buffer
in HBM.  Episode semantics follow Appendix C of SURVEY.md: an env that fails or reaches the end of its clip slice gets
mask 0 and is re-seeded with a freshly sampled (clip, start) slice (dataset_amass_single.py:172-253); rollouts cut mid-episode
are bootstrapped with V(s_T) (the reference never truncates, so this is the one semantic addition, documented in DESIGN.md).
Multi-GPU: envs are sharded, one process per GPU; the flat gradient tensor of each net is all-reduced once per optimisation step
(nn.GradComm, overlapped with the other net's backward); nothing else crosses GPUs.
"""
import ctypes as C
import time

import numpy as np

from . import nn
from .engine import EVAL_SMPL, Engine, _chk
from .motion_lib import MotionSet


class UhcRolloutBuf(C.Structure):
    """include/uhc_rollout.h UhcRolloutBuf"""
    _fields_ = [(k, C.c_void_p) for k in ("states", "actions", "rewards", "masks", "exps", "logp", "fails", "obs_cur", "ep_clip", "ep_pct")] + \
               [("T_cap", C.c_int), ("reserved", C.c_int), ("ep_start", C.c_void_p)]


def ewma(x, alpha=0.05):
    """uhc/utils/math_utils.py:25-29"""
    avg = float(x[0])
    for i in x[1:]:
        avg = alpha * float(i) + (1 - alpha) * avg
    return avg


def failure_weights(success_hist, sampling_temp=0.2, sampling_freq=0.5):
    """Per-clip sampling weights of the training loop (DatasetAMASSSingle.sample_seq with freq_dict, dataset_amass_single.py:183-186):
    with probability sampling_freq the clip is drawn from p ~ exp(-ewma(success history) / temp) (0 for an empty history), else
    uniformly over the clips.  success_hist: one list of 0/1 outcomes per clip (freq_dict[k][:, 0] == 1).  Returns the mixture
    weights w = sampling_freq * p + (1 - sampling_freq) / C for uhc_set_clip_weights."""
    s = np.array([ewma(np.asarray(h, dtype=np.float64) == 1) if len(h) > 0 else 0.0 for h in success_hist])
    p = np.exp(-s / sampling_temp)
    p = p / p.sum()
    return (sampling_freq * p + (1.0 - sampling_freq) / len(p)).astype(np.float32)


MAX_EVAL_GROUPS = 64       # include/uhc_eval.h UHC_EVAL_MAX_GROUPS


def pack_groups(K, n, E, max_groups=MAX_EVAL_GROUPS):
    """calls of a K-checkpoint x n-clip sweep on E envs: the K * n (checkpoint, clip) pairs, checkpoint-major, cut into calls of at most E envs
    and max_groups groups, a group being one checkpoint's run of consecutive clips inside a call.  Returns [[(k, c0, c1), ...] per call]."""
    assert K >= 1 and n >= 1 and E >= 1 and max_groups >= 1
    calls, cur, used = [], [], 0
    for k in range(K):
        c0 = 0
        while c0 < n:
            if used == E or len(cur) == max_groups:
                calls.append(cur)
                cur, used = [], 0
            c1 = min(n, c0 + E - used)
            cur.append((k, c0, c1))
            used += c1 - c0
            c0 = c1
    calls.append(cur)
    return calls


def call_env_steps(lens):
    """env-steps of one evaluation call over clips of these lengths: every env of the call steps until its longest clip ends"""
    lens = np.asarray(lens, np.int64).reshape(-1)
    return int(len(lens) * (lens.max() - 1)) if len(lens) else 0


def assign_clips(clip_len, world, E):
    """the evaluation's clips of every rank, each split into its device calls of at most E clips: [[clips of one call, ...] per rank].
    World 1 keeps the contiguous chunks c0 .. c0 + E - 1.  Otherwise the clips, longest first, are cut into calls of
    min(E, ceil(n / world)) consecutive clips, so the clips of a call have similar lengths and few padded steps, and each call in turn goes to
    the rank with the fewest env-steps (call_env_steps) so far, the lower rank on a tie.  Every env's roll-out is independent of the others
    and of its slot, so a clip's result does not depend on where it runs.  A caller that hands a rank's clips to a method which re-chunks them
    (evaluate_policies, export_motion) gets the same clips per rank, but not these calls."""
    lens = np.asarray(clip_len, np.int64).reshape(-1)
    n = len(lens)
    assert world >= 1 and E >= 1
    if world == 1:
        return [[np.arange(c0, min(n, c0 + E), dtype=np.int32) for c0 in range(0, n, E)]]
    order = np.argsort(-lens, kind="stable").astype(np.int32)
    b = max(1, min(E, -(-n // world)))
    calls, load = [[] for _ in range(world)], [0] * world
    for k in range(0, n, b):
        r = load.index(min(load))
        calls[r].append(order[k:k + b])
        load[r] += call_env_steps(lens[order[k:k + b]])
    return calls


def shard_clips(clip_len, world, rank, E):
    """this rank's calls of assign_clips"""
    return assign_clips(clip_len, world, E)[rank]


class ClipSampler:
    """DatasetAMASSSingle.sample_seq / get_sample_from_key (dataset_amass_single.py:172-253): uniform clip choice (or
    failure-weighted when freq stats are given), start ~ U[0, len - t_min), slice length min(t_max, len - start)."""

    def __init__(self, clip_lens, t_min=5, t_max=300, seed=0):
        self.lens, self.t_min, self.t_max = np.asarray(clip_lens), t_min, t_max
        self.rng = np.random.RandomState(seed)
        self.probs = None

    def set_failure_weights(self, success_ewma, temp=0.1):
        p = np.exp(-np.asarray(success_ewma) / temp)
        self.probs = p / p.sum()

    def sample(self, n, freq=0.5):
        if self.probs is not None:
            pick_w = self.rng.binomial(1, freq, n).astype(bool)
            clip = np.where(pick_w, self.rng.choice(len(self.lens), n, p=self.probs), self.rng.randint(0, len(self.lens), n))
        else:
            clip = self.rng.randint(0, len(self.lens), n)
        L = self.lens[clip]
        start = (self.rng.random_sample(n) * np.maximum(L - self.t_min, 1)).astype(np.int64)
        length = np.minimum(self.t_max if self.t_max > 0 else L, L - start)
        return clip.astype(np.int32), start.astype(np.int32), length.astype(np.int32)


class RolloutBuffer:
    def __init__(self, T, E, device, act_dim=105, obs_dim=657):
        import torch
        f = dict(device=device, dtype=torch.float32)
        self.T, self.E = T, E
        self.states = torch.empty(T, E, obs_dim, **f)
        self.actions = torch.empty(T, E, act_dim, **f)
        self.rewards, self.masks, self.exps, self.logp = (torch.empty(T, E, **f) for _ in range(4))
        self.last_obs = torch.empty(E, obs_dim, **f)
        self.last_alive = torch.empty(E, **f)
        self.fails = torch.zeros(T, E, device=device, dtype=torch.int32)
        self.ep_clip = torch.full((T, E), -1, device=device, dtype=torch.int32)      # clip of the episode that ended at (t, e), -1 = none
        self.ep_pct = torch.zeros(T, E, **f)                                         # its completed fraction (info["percent"])
        self.ep_start = torch.zeros(T, E, device=device, dtype=torch.int32)          # and its start frame (fr_start)

    def c_struct(self, obs_cur):
        b = UhcRolloutBuf()
        for k in ("states", "actions", "rewards", "masks", "exps", "logp", "fails", "ep_clip", "ep_pct", "ep_start"):
            setattr(b, k, getattr(self, k).data_ptr())
        b.obs_cur, b.T_cap = obs_cur.data_ptr(), self.T
        return b

    # TrajBatch-compatible flat views (khrylib/rl/core/trajbatch.py)
    def flat(self, name):
        t = getattr(self, name)
        return t.reshape(self.T * self.E, *t.shape[2:])


class BatchedAgent:
    def __init__(self, num_envs, clips, shapes=None, device=0, seed=1, precision=32, policy_hsize=(2048, 1024, 512),
                 value_hsize=(2048, 1024, 512), htype="gelu", log_std=-2.3, policy_lr=5e-5, value_lr=3e-4, gamma=0.95, tau=0.95,
                 clip_epsilon=0.2, num_optim_epoch=10, grad_clip=40.0, t_min=5, t_max=300, noise_rate=1.0, rank=0, world=1,
                 grad_sync=None, model=None, update_tc=True, variants=None, clip_models=None, c_update=True, actor_type="gauss", num_primitive=8,
                 composer_dim=(300, 200), subject_of=None, curriculum_global=False, **env_cfg):
        """curriculum_global: one failure-weighted curriculum across the ranks of a data-parallel run (turns the device curriculum on with its
        default parameters): every rank's episode log rides the first gradient all-reduce of update_params, and every rank merges all of them
        into bit-identical rings.  At world 1 it is the device curriculum."""
        import torch
        self.torch = torch
        self.dev = torch.device("cuda", device)
        torch.cuda.set_device(self.dev)
        if world > 1 and not update_tc:
            raise ValueError("BatchedAgent: the fp32 update (update_tc=False) is single-GPU only: it has no gradient all-reduce")
        self.E, self.seed, self.rank, self.world = num_envs, seed, rank, world
        self.auto_reset = bool(env_cfg.pop("auto_reset", True))
        self.engine = Engine(num_envs, model=model, device=device, precision=precision, variants=variants, auto_reset=int(self.auto_reset), t_min=t_min, t_max=t_max,
                             reset_seed=seed * 7919 + rank * 104729 + 1, **env_cfg)
        if callable(clips):                                  # clips(engine) -> (MotionSet, shapes): raw motion that needs the engine before it is
            clips, shapes = clips(self.engine)               # loaded (a height fix measured on the GPU); the sampler below sees what it returns
        fk_models = None
        if subject_of is not None:                           # subject_of(shapes [C][17]) -> the variant of each clip: its simulated body and the
            assert isinstance(clips, MotionSet), "subject_of needs raw motion: the expert FK runs on each clip's body on the GPU"
            clip_models = fk_models = subject_of(shapes)     # body of its expert FK (AgentCopycat's subject_bodies)
        if isinstance(clips, MotionSet):                     # raw motion: the expert tables are built on the GPU
            self.engine.load_motions(clips, shapes, clip_models, fk_models=fk_models)
        else:
            self.engine.load_clips(clips, shapes, clip_models)   # clip_models: body-shape variant per clip (the reference rebuilds the robot per clip)
        self.sampler = ClipSampler(self.engine.clip_len, t_min, t_max, seed=seed * 9973 + rank)
        A = self.act_dim = self.engine.act_dim          # env.action_dim (humanoid_im.py:250): 69 + (6 | 216) + (30 if meta_pd)
        D = self.obs_dim = self.engine.obs_dim          # env.obs_dim: 657 (obs v2) or 784 (obs v1)
        assert actor_type in ("gauss", "mcp"), "actor_type: gauss (PolicyGaussian) | mcp (PolicyMCP)"
        self.actor_type = actor_type
        if actor_type == "mcp":        # policy_mcp.py:9-37 (config/release/uhc_implicit.yml): runs through uhc_rollout_mcp / uhc_ppo_trainer_create_mcp only
            assert c_update and update_tc and bool(env_cfg.get("auto_reset", True)), "the PolicyMCP actor runs on the C-side rollout / update paths"
            self.policy = nn.MCPNet(D, policy_hsize, A, htype, num_primitive=num_primitive, composer_dim=composer_dim, device=self.dev, seed=seed)
        else:
            self.policy = nn.MLPNet(D, policy_hsize, A, htype, device=self.dev, head_name="action_mean", seed=seed)
        self.value = nn.MLPNet(D, value_hsize, 1, htype, device=self.dev, head_name="value_head", seed=seed + 1)
        self.log_std = torch.full((A,), float(log_std), device=self.dev, dtype=torch.float32)
        self.running_state = nn.ZFilter(D, clip=5.0, device=self.dev)
        self.opt_p, self.opt_v = nn.Adam(self.policy.params(), policy_lr, net=self.policy), nn.Adam(self.value.params(), value_lr, net=self.value)
        self.comm = nn.GradComm(world)
        self.gamma, self.tau, self.clip_epsilon, self.epochs, self.grad_clip = gamma, tau, clip_epsilon, num_optim_epoch, grad_clip
        self.noise_rate, self.grad_sync, self.update_tc = noise_rate, grad_sync, update_tc
        self.c_update, self._ctrainer, self._nccl = c_update, None, None      # uhc_ppo_update (include/uhc_ppo.h): the update behind one C-ABI call
        self.global_step = 0
        self.obs = None
        self.ep_len = torch.zeros(num_envs, device=self.dev, dtype=torch.float32)
        self.ep_ret = torch.zeros(num_envs, device=self.dev, dtype=torch.float32)
        self.nn_launches = 0
        self._notdone = torch.zeros(num_envs, device=self.dev, dtype=torch.bool)
        self.curriculum_global = bool(curriculum_global)
        self._cur_staged = None           # T of the rollout whose episode log waits in _cur_slots for the next update_params (global curriculum)
        if self.curriculum_global:
            self.curriculum_enable()

    # ---- env.reset for a subset with freshly sampled clip slices
    def reset_envs(self, ids=None):
        ids = np.arange(self.E, dtype=np.int32) if ids is None else np.asarray(ids, dtype=np.int32)
        clip, start, length = self.sampler.sample(len(ids))
        self.obs = self.engine.reset(ids, clip, start, length)
        return self.obs

    def policy_step(self, obs, update_filter=True, mean_action=None, use_tc=True, out_state=None, out_action=None, out_logp=None):
        """running_state -> policy -> sample.  Returns (normalised state, action, logp); the out_* tensors (rows of the rollout
        buffer) are written in place by the kernels."""
        s = self.running_state(obs, update=update_filter, out=out_state)
        mean = self.policy.forward_tc(s) if use_tc else self.policy.forward(s)
        a, lp = nn.gaussian_sample(mean, self.log_std, self.seed * 1000003 + self.rank, self.global_step, mean_action, out_action, out_logp)
        self.nn_launches += (3 if update_filter else 1) + (1 + len(self.policy.W) if use_tc else len(self.policy.W)) + 1
        return s, a, lp

    def step_once(self, buf, k, use_tc=True):
        """one lock-step control step of every env: normalise, policy, sample, physics+task kernel, buffer write, re-seed ended episodes."""
        t = self.torch
        mean_action = None
        if self.noise_rate < 1.0:
            mean_action = (t.rand(self.E, device=self.dev, dtype=t.float32) < (1.0 - self.noise_rate)).to(t.uint8)
        s, a, lp = self.policy_step(self.obs, True, mean_action, use_tc, buf.states[k], buf.actions[k], buf.logp[k])
        if mean_action is not None:
            buf.exps[k].copy_(1.0 - mean_action.float())
        elif not getattr(buf, "_exps_ones", False):
            buf.exps.fill_(1.0)
            buf._exps_ones = True
        obs, rew, cinfo, fail, end, pct = self.engine.step(a, reward_out=buf.rewards[k])
        done = (fail | end) != 0
        t.logical_not(done, out=self._notdone)
        buf.masks[k].copy_(self._notdone)
        self.global_step += 1
        buf.fails[k].copy_(fail)
        if self.auto_reset:
            return            # finished episodes were re-seeded inside the step kernel (no host round trip)
        ids = done.nonzero().flatten()
        if ids.numel():
            self.reset_envs(ids.cpu().numpy().astype(np.int32))

    def rollout(self, buf, T, row0=0, use_graph=True):
        """T control steps through the C-side loop (uhc_rollout, include/uhc_rollout.h): the same kernels as step_once, enqueued from C and
        replayed as one CUDA graph.  Needs auto_reset (finished episodes are re-seeded inside the step kernel)."""
        assert self.auto_reset, "uhc_rollout re-seeds finished episodes in the step kernel: build the agent with auto_reset=True"
        L = self.engine.lib
        mcp = self.actor_type == "mcp"
        if self.policy._bf16 is None or getattr(self, "_mlp_c", None) is None:
            self._mlp_c = nn.mcp_struct(self.policy) if mcp else nn.mlp_struct(self.policy)
        if getattr(self, "_ro_step", None) != self.global_step:
            L.uhc_rollout_set_step(self.engine.h, C.c_ulonglong(self.global_step))
        bs = buf.c_struct(self.obs)
        st = C.c_void_p(self.torch.cuda.current_stream(self.dev).cuda_stream)
        rc = (L.uhc_rollout_mcp if mcp else L.uhc_rollout)(self.engine.h, C.c_int(T), C.c_int(row0), C.byref(self._mlp_c), C.c_void_p(self.log_std.data_ptr()),
                           C.c_void_p(self.running_state.stats.data_ptr()), C.c_float(self.running_state.clip), C.c_int(1),
                           C.c_ulonglong(self.seed * 1000003 + self.rank), C.c_float(self.noise_rate), C.byref(bs), C.c_int(int(use_graph)), st)
        _chk(rc, "uhc_rollout")
        self.global_step += T
        self._ro_step = self.global_step
        self.nn_launches += T * (L.uhc_rollout_launches_per_step(self.engine.h) - 1)      # the env-step launch is counted by the engine

    def sample(self, T, buf=None, use_tc=True, c_loop=None):
        """agent.sample(): T lock-step control steps of all envs.  Returns (buffer, log).  c_loop (default: whenever auto_reset is on):
        the loop runs behind the C ABI as one CUDA graph; otherwise the Python loop over step_once (identical kernels and results)."""
        t = self.torch
        staging = self.engine.cur_cfg is not None and self._merges_across_ranks()
        if staging and self._cur_staged is not None:
            raise RuntimeError("the global curriculum merges a rollout's episode log in the update that follows it: call update_params before the next sample")
        if self.obs is None:
            if self.engine.cur_cfg is not None:               # the device curriculum's sampler (fit_clip / precision starts) seeds the first episodes too
                self.obs = self.engine.curriculum_reseed()
            else:
                self.reset_envs()
        buf = buf or RolloutBuffer(T, self.E, self.dev, self.act_dim, self.obs_dim)
        t0 = time.time()
        len0, ret0 = self.ep_len.clone(), self.ep_ret.clone()
        if c_loop is None:
            c_loop = self.auto_reset and use_tc
        if self.engine.cur_cfg is not None and not c_loop:
            raise RuntimeError("the device curriculum is fed by the C-side rollout's episode log (c_loop): the Python step loop does not record it")
        if c_loop:
            self.rollout(buf, T)
        else:
            for k in range(T):
                self.step_once(buf, k, use_tc)
        buf.last_obs.copy_(self.obs)
        if self.engine.cur_cfg is not None and c_loop:
            if staging:
                self._stage_curriculum(buf, T)
            else:
                self.curriculum_update(buf, T)
        # episode statistics from the buffer (one sync at the end of the rollout): segment the [T][E] masks per env
        m, r = buf.masks[:T], buf.rewards[:T]
        done = m == 0
        n_eps = int(done.sum())
        run_len = t.zeros(self.E, device=self.dev, dtype=t.float32); run_ret = t.zeros(self.E, device=self.dev, dtype=t.float32)
        run_len += len0; run_ret += ret0
        tot_len = t.zeros((), device=self.dev, dtype=t.float32); tot_ret = t.zeros((), device=self.dev, dtype=t.float32)
        for k in range(T):
            run_len += 1; run_ret += r[k]
            d = done[k]
            tot_len += (run_len * d).sum(); tot_ret += (run_ret * d).sum()
            run_len *= ~d; run_ret *= ~d
        self.ep_len, self.ep_ret = run_len, run_ret
        n_fail = int(((buf.fails[:T] != 0) & done).sum())
        log = dict(num_steps=T * self.E, num_episodes=n_eps, avg_episode_len=float(tot_len) / max(n_eps, 1),
                   avg_episode_reward=float(tot_ret) / max(n_eps, 1), fail_rate=n_fail / max(n_eps, 1),
                   avg_reward=float(r.mean()), sample_time=time.time() - t0)
        return buf, log

    def update_params(self, buf):
        """AgentPG.update_params (agent_pg.py:39-56): V(s), GAE (+bootstrap), advantage normalisation, PPO epochs -- all on the
        tensor-core path.  Multi-GPU (envs sharded by rank): the ONLY collective is the all-reduce of the flat gradient tensors; the
        global-batch statistics the reference's full-batch semantics need (advantage sum / sum of squares / count, the number of
        selected rows, the ZFilter increments of every rank) ride in the tail of the first one (SURVEY.md section 8e)."""
        t = self.torch
        L = nn._lib()
        ev = [t.cuda.Event(enable_timing=True) for _ in range(3)]
        ev[0].record()
        staged, self._cur_staged = getattr(self, "_cur_staged", None), None    # a failed update drops the log: the rings stay as they were
        T, E = buf.T, buf.E
        N = T * E
        states = buf.flat("states")
        if not self.update_tc:               # fp32 SIMT parity path (single GPU)
            t0 = time.time()
            values = self.value.forward(states).reshape(T, E)
            last_v = self.value.forward(self.running_state(buf.last_obs, update=False)).reshape(E)
            adv, ret = nn.gae(buf.rewards, buf.masks, values, last_v, self.gamma, self.tau, normalize=True)
            losses = nn.ppo_update(self.policy, self.value, self.log_std, self.opt_p, self.opt_v, states, buf.flat("actions"), ret.reshape(-1),
                                   adv.reshape(-1), buf.flat("exps"), self.clip_epsilon, self.epochs, self.grad_clip, use_tc=False)
            t.cuda.synchronize()
            self._mlp_c = None
            return dict(update_time=time.time() - t0, surr_loss=float(losses[0]), value_loss=float(losses[1]))
        if self.c_update:
            return self._update_params_c(buf, ev, staged)
        tp = getattr(self.policy, "_tc_trainer", None) or nn.TCTrainer(self.policy)
        tv = getattr(self.value, "_tc_trainer", None) or nn.TCTrainer(self.value)
        self.policy._tc_trainer, self.value._tc_trainer = tp, tv
        xb, xT = tp.prepare_input(states)
        tv.cache["xb"], tv.cache["xT"] = xb, xT
        v0, ctx0 = tv.forward(xb)                                                   # V(s): GAE input and epoch 0's value forward
        last_v = self.value.forward_tc(self.running_state(buf.last_obs, update=False)).reshape(E)
        adv, ret = nn.gae(buf.rewards, buf.masks, v0.reshape(T, E), last_v, self.gamma, self.tau, normalize=False)
        adv, ret, exps = adv.reshape(-1), ret.reshape(-1), buf.flat("exps")
        mom = t.zeros(2, device=self.dev, dtype=t.float64)
        nn._chk(L.uhc_adv_moments(nn._p(adv), C.c_long(N), nn._p(mom), nn._stream(adv)))
        cnt = (exps != 0).sum().to(t.float64).reshape(1)
        inv_count = t.zeros(1, device=self.dev, dtype=t.float32)
        after = None
        if self.world <= 1:
            nn._chk(L.uhc_adv_normalize(nn._p(adv), C.c_long(N), nn._p(mom), None, nn._stream(adv)))
            inv_count.copy_(1.0 / t.clamp(cnt, min=1.0))
        else:
            D = self.obs_dim
            zs = self.running_state.stats
            if getattr(self, "_z_sync", None) is None:                               # fresh agent: every rank starts from empty statistics
                self._z_sync = t.zeros_like(zs)                                      # additive form of the statistics every rank agreed on last
            d = t.cat([mom, t.full((1,), float(N), device=self.dev, dtype=t.float64), cnt, nn.zfilter_to_sums(zs, D) - self._z_sync])
            nd = d.numel()
            extra = self._cur_slots if staged is not None else None                  # the global curriculum's episode logs ride behind the statistics
            self.value.ensure_grad_tail(nn.stats_tail_floats(D) + (0 if extra is None else extra.numel()))
            nn.pack_stats_tail(self.value.gfull[self.value.nflat:], d, extra)       # [5, nd] exact fixed-point digits (fp32), then the payload
            ntot = t.zeros(1, device=self.dev, dtype=t.float64)

            def after(tail_r):
                g, ex = nn.unpack_stats_tail(tail_r, nd, 0 if extra is None else extra.numel())   # summed over the ranks by the gradient all-reduce
                if extra is not None:
                    self._cur_sum.copy_(ex)
                ntot.copy_(g[2:3])
                gm = g[0:2].contiguous()
                nn._chk(L.uhc_adv_normalize(nn._p(adv), C.c_long(N), nn._p(gm), nn._p(ntot), nn._stream(adv)))
                inv_count.copy_(1.0 / t.clamp(g[3:4], min=1.0))
                self._z_sync = self._z_sync + g[4:]
                zs.copy_(nn.zfilter_from_sums(self._z_sync, D))                     # every rank now holds the same running_state
        ev[1].record()
        losses = nn.ppo_epochs_tc(self.policy, self.value, self.log_std, self.opt_p, self.opt_v, xb, xT, buf.flat("actions"), ret, adv, exps,
                                  self.clip_epsilon, self.epochs, self.grad_clip, comm=self.comm, first_value=(v0, ctx0), after_first_reduce=after,
                                  inv_count_dev=inv_count, world=self.world)
        if staged is not None:
            self.engine.curriculum_update_gathered(self._cur_sum, staged, self.world)
        ev[2].record()
        t.cuda.synchronize()
        self._mlp_c = None
        out = dict(update_time=1e-3 * ev[0].elapsed_time(ev[2]), gae_ms=ev[0].elapsed_time(ev[1]), epochs_ms=ev[1].elapsed_time(ev[2]),
                   surr_loss=float(losses[0]), value_loss=float(losses[1]))
        if self.world > 1:
            out.update(allreduce_ms=self.comm.pop_ms(), allreduce_bytes=self.comm.bytes, allreduce_calls=self.comm.calls)
            self.comm.bytes = self.comm.calls = 0
        return out

    def _update_params_c(self, buf, ev, staged=None):
        """the production update: ONE call of uhc_ppo_update (include/uhc_ppo.h) -- V(s) and V(s_T), GAE, global advantage normalisation, the
        epochs of both nets, Adam, and (world > 1) the gradient all-reduces on this job's ncclComm_t with the statistics tail.  staged: T of the
        rollout whose episode log the global curriculum carries in that tail (uhc_ppo_update_ex) and merges afterwards."""
        t = self.torch
        T, E = buf.T, buf.E
        if staged is not None:
            self.value.ensure_grad_tail(nn.stats_tail_floats(self.obs_dim) + self._cur_slots.numel())
        if (self._ctrainer is None or self._ctrainer.max_rows < T * E or self._ctrainer.max_envs < E or self._ctrainer.dv.gtail != self.value.grad_tail
                or self._ctrainer.dv.gfull != self.value.gfull.data_ptr()):
            fn = None
            if self._ctrainer is not None:
                fn = self._ctrainer.all_reduce          # an installed collective stays with the rebuilt trainer
                self._ctrainer.close()
            self._ctrainer = nn.CPpoTrainer(self.policy, self.value, self.opt_p, self.opt_v, T * E, E, self.dev, all_reduce=fn)
        zs = zsync = None
        if self.world > 1:
            if self._nccl is None:
                self._nccl = nn.make_nccl_comm(self.rank, self.world, self.dev)
            zs = self.running_state.stats
            if getattr(self, "_z_sync", None) is None:
                self._z_sync = t.zeros_like(zs)
            zsync = self._z_sync
        last_s = self.running_state(buf.last_obs, update=False)
        if getattr(self, "_losses", None) is None:
            self._losses = t.zeros(2, device=self.dev, dtype=t.float32)
        ev[1].record()
        self._ctrainer.update(buf.flat("states"), last_s, buf.flat("actions"), buf.rewards, buf.masks, buf.flat("exps"), self.log_std, T, E, self.gamma,
                              self.tau, self.clip_epsilon, self.epochs, self.grad_clip, self._losses, zfilter=zs, z_sync=zsync, comm=self._nccl, world=self.world,
                              extra_in=self._cur_slots if staged is not None else None, extra_out=self._cur_sum if staged is not None else None)
        if staged is not None:
            self.engine.curriculum_update_gathered(self._cur_sum, staged, self.world)
        ev[2].record()
        t.cuda.synchronize()
        out = dict(update_time=1e-3 * ev[0].elapsed_time(ev[2]), gae_ms=0.0, epochs_ms=ev[1].elapsed_time(ev[2]),      # GAE runs inside the call
                   surr_loss=float(self._losses[0]), value_loss=float(self._losses[1]))
        if self.world > 1:
            ms, by, calls = self._ctrainer.comm_stats()
            out.update(allreduce_ms=ms, allreduce_bytes=by, allreduce_calls=calls)
        return out

    # ---- the failure-weighted curriculum on the device (Engine.curriculum_*): updated after every C-side rollout
    def curriculum_enable(self, max_freq=50, temp=0.2, freq=0.5, prec_freq=0.0, fit_clip=-1):
        old = self.engine.cur_cfg
        self.engine.curriculum_enable(max_freq, temp, freq, prec_freq, fit_clip)
        if max_freq and (old is None or old["fit_clip"] != int(fit_clip)) and self.obs is not None:
            self.obs = self.engine.curriculum_reseed()      # the new fit_clip applies to every env from the next rollout on

    @property
    def fit_clip(self):
        return -1 if self.engine.cur_cfg is None else self.engine.cur_cfg["fit_clip"]

    @fit_clip.setter
    def fit_clip(self, clip):
        """the clip every re-seed uses (-1: off); turns the device curriculum on (default parameters) if it is off"""
        c = dict(self.engine.cur_cfg or dict(max_freq=50, temp=0.2, freq=0.5, prec_freq=0.0))
        c["fit_clip"] = int(clip)
        self.curriculum_enable(**c)

    def curriculum_update(self, buf, T):
        self.engine.curriculum_update(buf, T)

    def _merges_across_ranks(self):
        return getattr(self, "curriculum_global", False) and self.world > 1

    def _stage_curriculum(self, buf, T):
        """the global curriculum: this rank's episode log into its slot of the payload update_params' first all-reduce sums"""
        n = self.world * T * self.E * 3
        if getattr(self, "_cur_slots", None) is None or self._cur_slots.numel() != n:
            self._cur_slots = self.torch.empty(n, device=self.dev, dtype=self.torch.float32)
            self._cur_sum = self.torch.empty_like(self._cur_slots)
        self.engine.curriculum_stage(buf, T, self.rank, self.world, self._cur_slots)
        self._cur_staged = T

    def curriculum_push(self, clips, pct, starts):
        self.engine.curriculum_push(clips, pct, starts)

    def curriculum_get(self):
        return self.engine.curriculum_get()

    def curriculum_set(self, lens, pct, starts):
        self.engine.curriculum_set(lens, pct, starts)

    def evaluate(self, clips, fail_safe, window=32, record_states=False, export_smpl=False, floor=False):
        """deterministic roll-out of every listed clip from frame 0 on the device (Engine.eval_run, one call per chunk of E clips) under
        the engine's current cfg.  Returns one dict per clip: frames = [nframes][6] per-frame rows (uhc_b200/metrics.py
        metrics_from_frames), last_t, fail_any, reward_sum (and states = [nframes][148] when record_states; pose_aa = [nframes][72] and
        trans = [nframes][3], the simulated motion as SMPL, when export_smpl; floor = [nframes][5], the body hulls against the floor per frame
        (include/uhc_floor.h; metrics.floor_summary), when floor)."""
        clips = np.asarray(clips, dtype=np.int32).reshape(-1)
        out = []
        for c0 in range(0, len(clips), self.E):
            out += self._evaluate_call(clips[c0:c0 + self.E], fail_safe, window, record_states, export_smpl, floor)
        self.obs = None       # every env was reset onto an evaluation clip
        return out

    def _evaluate_call(self, clips, fail_safe, window, record_states, export_smpl, floor=False):
        pol = nn.mcp_struct(self.policy) if self.actor_type == "mcp" else nn.mlp_struct(self.policy)
        r = self.engine.eval_run(clips, pol, self.log_std, self.running_state.stats, self.running_state.clip, fail_safe, window, record_states, export_smpl,
                                 floor)
        out = []
        for i, nf in enumerate(r["nframes"]):
            d = dict(frames=r["frames"][i, :nf].copy(), last_t=int(r["last_t"][i]), fail_any=bool(r["fail_any"][i]), reward_sum=float(r["reward_sum"][i]))
            if record_states:
                d["states"] = r["states"][i, :nf].copy()
            if export_smpl:
                d["pose_aa"], d["trans"] = r["pose_aa"][i, :nf].copy(), r["trans"][i, :nf].copy()
            if floor:
                d["floor"] = r["floor"][i, :nf].copy()
            out.append(d)
        return out

    def export_motion(self, clips, fail_safe, window=32, max_bytes=1 << 30, floor=False):
        """the simulated motion of every listed clip, as evaluate() rolls it out: per clip pred = [nframes][76] qpos, pred_jpos = [nframes][72]
        world body positions, pose_aa = [nframes][72] and trans = [nframes][3] (the qpos as SMPL, uhc_qpos_to_smpl on the device) and evaluate()'s
        summary (frames, last_t, fail_any, reward_sum; floor = [nframes][5] with floor=True), in the caller's order.  Clips of similar length share a device call; a call takes at most
        E clips and as many as keep its pinned state and SMPL arrays, n * (max(len) - 1) * (148 + 75) * 8 bytes, within max_bytes (a clip that
        alone needs more runs on its own).  Every env is independent of the others, so a clip's result does not depend on the chunking.  Needs
        the engine's test-mode cfg (auto_reset off, as eval_policy sets it): with auto_reset an ended env would re-seed itself from the sampler,
        whose draws depend on the env it runs on."""
        if self.engine._cfg.auto_reset:
            raise ValueError("export_motion needs the test-mode cfg: engine.set_cfg(auto_reset=0) first")
        clips = np.asarray(clips, dtype=np.int32).reshape(-1)
        per_frame = (148 + EVAL_SMPL) * 8
        order = np.argsort(self.engine.clip_len[clips], kind="stable")
        out = [None] * len(clips)
        k = 0
        while k < len(clips):
            m = 1
            while k + m < len(clips) and m < self.E and (m + 1) * (int(self.engine.clip_len[clips[order[k + m]]]) - 1) * per_frame <= max_bytes:
                m += 1
            idx = order[k:k + m]
            for i, d in zip(idx, self._evaluate_call(clips[idx], fail_safe, window, True, True, floor)):
                st = d.pop("states")
                d["pred"], d["pred_jpos"] = st[:, :76], st[:, 76:]
                out[i] = d
            k += m
        self.obs = None
        return out

    def render_motion(self, clips, fail_safe, size=(640, 360), camera=None, ghost=True, max_bytes=1 << 30, writer=None, window=32, encode=None,
                      quality=90, body="hulls", betas=None):
        """export_motion's evaluation of every listed clip, drawn on the device (Engine.render): frame k of clip i shows the simulated qpos
        pred[k] (grey) and, with ghost, the expert frame eval_seq pairs it with, gt[k] = qpos[min(k + 1, len - 1)] (red), with the clip's
        shape variant.  Frames come to the host in chunks of at most max_bytes of rgb (at least one frame).  writer(i, chunks) is called once
        per clip, in the caller's order, with an iterator over its uint8 chunks [k][H][W][3], rendered as it is consumed; without a writer
        the frames are returned.  Returns per clip export_motion's dict plus gt (and frames without a writer).  self.render_times holds the
        seconds spent in evaluation, rendering, device-to-host copies and the writer.  With encode="jpeg" every chunk is compressed on the
        device (Engine.encode_jpeg at `quality`) and only the JPEG files come to the host: a chunk, and frames, are then lists of bytes, one
        file per frame, and render_times also holds the seconds of encoding.  body="mesh" draws the skinned SMPL mesh instead of the hulls
        (Engine.render_smpl, after the engine's mesh_init and render_mesh_init): clip i's pred and gt are both shaped by betas[i] (betas =
        [len(clips)][10] in the caller's order; None: zeros), and the vertices of a chunk count against max_bytes beside its rgb."""
        if encode not in (None, "jpeg"):
            raise ValueError('render_motion: encode must be None or "jpeg"')
        if body not in ("hulls", "mesh"):
            raise ValueError('render_motion: body must be "hulls" or "mesh"')
        W, H = (int(x) for x in size)
        per_frame = W * H * 3
        if body == "mesh":
            if getattr(self.engine, "smpl_nvert", None) is None:
                raise ValueError('render_motion: body="mesh" needs the engine\'s mesh_init and render_mesh_init')
            nclip = len(np.atleast_1d(clips))
            betas = np.zeros((nclip, 10)) if betas is None else np.asarray(betas, np.float64)
            if betas.shape != (nclip, 10):
                raise ValueError(f"render_motion: betas must be [len(clips)][10] = [{nclip}][10], got {list(betas.shape)}")
            per_frame += (2 if ghost else 1) * self.engine.smpl_nvert * 12
        step = max(1, int(max_bytes) // per_frame)
        t0 = time.perf_counter()
        mot = self.export_motion(clips, fail_safe, window, max_bytes)
        times = self.render_times = dict(evaluation=time.perf_counter() - t0, rendering=0.0, copy=0.0, writer=0.0)
        if encode:
            times["encoding"] = 0.0
        eng, clips = self.engine, np.asarray(clips, dtype=np.int32).reshape(-1)

        def chunks(d, var, beta):
            for k0 in range(0, len(d["pred"]), step):
                t1 = time.perf_counter()
                pred, gt = d["pred"][k0:k0 + step], d["gt"][k0:k0 + step] if ghost else None
                if body == "mesh":
                    rgb = eng.render_smpl(pred, gt, beta, variants=var, camera=camera, size=(W, H))[0]
                else:
                    rgb = eng.render(pred, gt, var, camera, (W, H))[0]
                self.torch.cuda.synchronize(self.dev)
                t2 = time.perf_counter()
                times["rendering"] += t2 - t1
                if encode:
                    data, offsets = eng.encode_jpeg(rgb, quality)        # synchronises
                    t3 = time.perf_counter()
                    times["encoding"] += t3 - t2
                    data, o = data.cpu().numpy(), offsets.cpu().numpy()
                    host = [data[o[i]:o[i + 1]].tobytes() for i in range(len(o) - 1)]
                else:
                    t3 = t2
                    host = rgb.cpu().numpy()
                times["copy"] += time.perf_counter() - t3
                yield host

        for i, (c, d) in enumerate(zip(clips, mot)):
            nf, L = len(d["pred"]), int(eng.clip_len[c])
            d["gt"] = eng.clip_frames(int(c))["qpos"][np.minimum(np.arange(1, nf + 1), L - 1)]
            var = None if eng.clip_models is None else int(eng.clip_models[c])
            beta = None if betas is None else betas[i]
            if writer is None:
                if encode:
                    d["frames"] = [f for ch in chunks(d, var, beta) for f in ch]
                else:
                    d["frames"] = np.concatenate(list(chunks(d, var, beta))) if nf else np.zeros((0, H, W, 3), np.uint8)
            else:
                inside = lambda: times["rendering"] + times["copy"] + times.get("encoding", 0.0)
                t1, inner = time.perf_counter(), inside()
                writer(i, chunks(d, var, beta))
                times["writer"] += time.perf_counter() - t1 - (inside() - inner)
        return mot

    def _checkpoint_policy(self, k, cp):
        """(policy net, ZFilter) slot k of the evaluation pool, beside the agent's own (which stay untouched), loaded from a checkpoint in the
        reference's wire format.  The pool is kept: its tensors keep their addresses, so a repeated sweep replays its captured graphs."""
        pool = self.__dict__.setdefault("_eval_pool", [])
        pol = self.policy
        while len(pool) <= k:
            if self.actor_type == "mcp":
                net = nn.MCPNet(self.obs_dim, pol.dims[1:-1], self.act_dim, pol.htype, num_primitive=pol.num_primitive,
                                composer_dim=tuple(pol.composer.dims[1:-1]), device=self.dev, seed=0)
            else:
                net = nn.MLPNet(self.obs_dim, pol.dims[1:-1], self.act_dim, pol.htype, device=self.dev, head_name="action_mean", seed=0)
            pool.append((net, nn.ZFilter(self.obs_dim, clip=self.running_state.clip, device=self.dev)))
        net, zf = pool[k]
        net.load_state_dict(cp["policy_dict"])
        rs = cp.get("running_state")
        if isinstance(rs, dict):
            zf.load(rs["n"], rs["mean"], rs["std"])
        elif rs is not None:
            zf.load_sums(rs.rs._n, rs.rs._M, rs.rs._S)
        else:                 # as load_state_dicts: a checkpoint without statistics is normalised by the agent's
            zf.stats.copy_(self.running_state.stats)
        return net, zf

    def evaluate_policies(self, checkpoints, clips, fail_safe, window=32, record_states=False, floor=False):
        """evaluate() of every listed clip for each checkpoint ({"policy_dict", "running_state"}, what state_dicts writes), with the checkpoints
        side by side in each device call (Engine.eval_run_groups, packed by pack_groups).  Returns one list per checkpoint, each equal to
        what load_state_dicts(cp) + evaluate(clips, ...) returns.  The agent's own weights, log_std and running_state are not touched."""
        clips = np.asarray(clips, dtype=np.int32).reshape(-1)
        K, n = len(checkpoints), len(clips)
        out = [[] for _ in range(K)]
        if K == 0 or n == 0:
            return out
        mcp = self.actor_type == "mcp"
        pols = [self._checkpoint_policy(k, cp) for k, cp in enumerate(checkpoints)]
        structs = [(nn.mcp_struct(net) if mcp else nn.mlp_struct(net), zf) for net, zf in pols]
        for call in pack_groups(K, n, self.E):
            groups = [(clips[c0:c1], structs[k][0], structs[k][1].stats) for k, c0, c1 in call]
            res = self.engine.eval_run_groups(groups, self.running_state.clip, fail_safe, window, record_states, floor=floor)
            for (k, _, _), r in zip(call, res):
                for i, nf in enumerate(r["nframes"]):
                    d = dict(frames=r["frames"][i, :nf].copy(), last_t=int(r["last_t"][i]), fail_any=bool(r["fail_any"][i]), reward_sum=float(r["reward_sum"][i]))
                    if record_states:
                        d["states"] = r["states"][i, :nf].copy()
                    if floor:
                        d["floor"] = r["floor"][i, :nf].copy()
                    out[k].append(d)
        self.obs = None       # every env was reset onto an evaluation clip
        return out

    def tracker(self, window=8, kind="qpos", fail_safe=True, **kw):
        """this agent's policy as a batched physics tracker of streamed target frames (uhc_b200/tracker.py); it takes over the engine's
        clip table until the next load_clips / load_motions.  The cfg must be a test-mode one: auto_reset off, trail_steps >= 1.  subjects=
        a subject_body.SubjectBasis lets Tracker.set_subjects give each env its own body at run time."""
        from .tracker import Tracker
        return Tracker(self, window, kind, fail_safe, **kw)

    def optimize_policy(self, T):
        buf, log = self.sample(T)
        log.update(self.update_params(buf))
        return log

    # checkpoint in the reference's wire format (agent_copycat.py:190-201): policy_dict / value_dict / running_state
    def state_dicts(self):
        pd = self.policy.state_dict()
        pd["action_log_std"] = self.log_std.detach().cpu().reshape(1, -1)
        # `running_state` in the reference's wire format: a ZFilter object (agent_copycat.py:194-200 pickles the object itself and
        # load_checkpoint assigns it back, :249-260), filled from the device statistics
        from uhc.khrylib.utils.zfilter import ZFilter as HostZFilter
        st = self.running_state.stats.cpu().numpy()
        D = self.running_state.dim
        return {"policy_dict": pd, "value_dict": self.value.state_dict(),
                "running_state": HostZFilter.from_stats(st[0], st[1:1 + D], st[1 + D:], clip=self.running_state.clip)}

    def load_state_dicts(self, cp):
        t = self.torch
        self.policy.load_state_dict(cp["policy_dict"])
        self.value.load_state_dict(cp["value_dict"])
        if "action_log_std" in cp["policy_dict"]:
            self.log_std.copy_(t.as_tensor(np.asarray(cp["policy_dict"]["action_log_std"]), dtype=t.float32).reshape(-1))
        rs = cp.get("running_state")
        if rs is not None:
            if isinstance(rs, dict):          # round-1 checkpoints of this repo
                self.running_state.load(rs["n"], rs["mean"], rs["std"])
            else:                             # a pickled khrylib ZFilter (reference checkpoints and this repo's)
                self.running_state.load_sums(rs.rs._n, rs.rs._M, rs.rs._S)
            # a loaded normaliser is common to every rank: the cross-rank merge (update_params) only exchanges what is added from here on
            self._z_sync = nn.zfilter_to_sums(self.running_state.stats, self.running_state.dim).clone()


def make_nccl_grad_sync(world):
    """flatten -> one torch.distributed all_reduce(sum) -> unflatten, averaged over ranks (full-batch mean semantics)."""
    import torch
    import torch.distributed as dist

    def sync(grads):
        flat = torch.cat([g.reshape(-1) for g in grads])
        dist.all_reduce(flat, op=dist.ReduceOp.SUM)
        flat.div_(world)
        out, o = [], 0
        for g in grads:
            n = g.numel()
            out.append(flat[o:o + n].view_as(g))
            o += n
        return out
    return sync
