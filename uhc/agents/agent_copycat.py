"""AgentCopycat with the reference's surface (uhc/agents/agent_copycat.py:51-605) on the batched engine.

  AgentCopycat(cfg, dtype, device, training=True, checkpoint_epoch=0)
  .optimize_policy(epoch)   per_epoch_update -> sample -> update_params -> checkpoint / eval every save_n_epochs -> log   (:326-352)
  .sample(min_batch_size)   -> (batch, log)      batch: states / actions / masks / rewards / exps (device resident, numpy on demand)
  .update_params(batch)     GAE + PPO epochs (khrylib agent_pg.py:39-56, agent_ppo.py:16-51)
  .eval_policy(epoch, dump) deterministic roll-out of every clip, coverage / error statistics                               (:354-494)
  .eval_checkpoints(epochs, dump)   eval_policy of several saved checkpoints at once (device evaluation, checkpoints side by side)
  .save_checkpoint / .load_checkpoint   pickle {"policy_dict", "value_dict", "running_state"} at models/iter_%04d.p        (:190-260)

Differences that are inherent to the batched design are listed in DESIGN.md (lock-step horizon with value bootstrap, batched
ZFilter merge, clip sampling without the per-clip failure history unless eval statistics are available).
"""
import logging
import math
import os
import os.path as osp
import pickle
import time
from collections import defaultdict

import joblib
import numpy as np

from uhc.data_loaders.dataset_amass_single import DatasetAMASSSingle
from uhc.envs.humanoid_im import HumanoidEnv
from uhc.losses.reward_function import reward_func
from uhc_b200 import nn
from uhc_b200.agent import BatchedAgent, RolloutBuffer, make_nccl_grad_sync, shard_clips
from uhc_b200.model import HumanoidModel


class _Batch:
    """TrajBatch-compatible view (khrylib/rl/core/trajbatch.py:4-15) over the device rollout buffer."""

    def __init__(self, buf):
        self.buf = buf

    def __getattr__(self, name):
        if name in ("states", "actions", "rewards", "masks", "exps"):
            return self.buf.flat(name).cpu().numpy()
        raise AttributeError(name)


class _Log(dict):
    __getattr__ = dict.get


# per-clip result keys that hold a clip's trajectory (eval_dump_motion, full_eval with dump): only rank 0, which writes the dumps, receives them
TRAJECTORY_KEYS = frozenset(("gt", "pred", "gt_jpos", "pred_jpos", "pose_aa", "trans", "pred_vertices", "pred_joints", "gt_vertices", "gt_joints"))


def exchange(work):
    """this rank's share of a sharded evaluation, work() -> a picklable value, all-gathered over the job's torch.distributed group:
    returns every rank's value in rank order.  A rank whose work raises still joins the all-gather, with its error in place of the
    value, and then every rank raises, so no rank waits on one that stopped; the all-gather itself runs under the group's timeout."""
    import torch.distributed as dist
    err = None
    try:
        val = work()
    except Exception as e:
        val, err = None, e
    out = [None] * dist.get_world_size()
    dist.all_gather_object(out, (None if err is None else f"{type(err).__name__}: {err}", val))
    bad = [f"rank {r}: {e}" for r, (e, _) in enumerate(out) if e is not None]
    if bad:
        raise RuntimeError("sharded evaluation failed on " + "; ".join(bad)) from err
    return [v for _, v in out]


def merge_results(parts, keys):
    """every rank's {key: result} of one table as one dict in the table's clip order, the order world 1 builds it in"""
    got = {}
    for p in parts:
        got.update(p)
    assert len(got) == len(keys) and all(k in got for k in keys), "every clip must be evaluated by exactly one rank"
    return {k: got[k] for k in keys}


def merge_outcomes(parts):
    """every rank's eval outcomes (table clip, training clip, outcome) in table clip order, the order world 1 applies them in"""
    return sorted((o for p in parts for o in p), key=lambda o: o[0])


def clip_betas(shapes, clips):
    """beta[:10] of each listed clip's shape row: [len(clips)][10], also for a rank whose shard is empty"""
    return np.array([np.asarray(shapes[c], np.float64)[:10] for c in clips], np.float64).reshape(len(clips), 10)


def gather_to_root(local, max_bytes):
    """every rank's {key: result} on rank 0, sent in pieces of at most max_bytes of arrays (at least one clip): rank 0 returns all of
    them, every other rank its own `local`, and no rank other than 0 ever holds more than its own results"""
    import torch.distributed as dist
    rank, world = dist.get_rank(), dist.get_world_size()
    pieces, size = [{}], 0
    for k, r in local.items():
        b = sum(v.nbytes for v in r.values() if isinstance(v, np.ndarray))
        if pieces[-1] and size + b > max_bytes:
            pieces.append({})
            size = 0
        pieces[-1][k] = r
        size += b
    counts = [None] * world
    dist.all_gather_object(counts, 0 if rank == 0 else len(pieces))
    out = dict(local)
    for j in range(max(counts)):
        got = [None] * world if rank == 0 else None
        dist.gather_object(pieces[j] if rank and j < len(pieces) else None, got, dst=0)
        if rank == 0:
            for p in got:
                out.update(p or {})
    return out if rank == 0 else local


def supported_variant(cfg):
    """The reference configuration keys this engine implements; returns the residual-force mode ("implicit" | "explicit" | "none").  `cfg` needs `.get(key, default)`
    and the attributes obs_v, actor_type, reward_id, fix_std, residual_force (uhc/utils/config_utils/copycat_config.py).  Everything else raises an AssertionError
    naming the key: of the reference's 115 yaml files 86 pass (tests/test_shim_cpu.py counts them); the others use explicit residual forces with contact gating /
    projection / body subsets (10), the six-term world_rfc_implicit_v2 / _v3 rewards (8), obs_v 0 / 4 (6), a trained log_std (2), ..."""
    assert cfg.obs_v in (1, 2, 3, 5, 6) and cfg.actor_type in ("gauss", "mcp") and cfg.reward_id in reward_func, \
        "the batched engine implements obs_v 1 | 2 | 3 | 5 | 6, the gauss and mcp actors, world_rfc_implicit (_v1_mul) / world_rfc_explicit (obs_v 0/4, reward v2/v3: SURVEY.md section 8f, next)"
    assert cfg.get("obs_vel", "full") == "full" and cfg.get("obs_coord", "root") == "root" and not cfg.get("obs_phase", False), "obs_vel full / obs_coord root / no phase only"
    if cfg.obs_v == 1:
        assert not cfg.get("has_shape", False), "obs_v 1 carries no shape vector (has_shape: false in config/release/uhc_implicit.yml)"
    # variants the batched engine does not implement must not be accepted silently (ADVICE r1)
    assert cfg.fix_std, "log_std is not a trained parameter in this engine (fix_std: true in every released config)"
    assert cfg.get("env_term_body", "body") in ("body", "root", "Head"), "env_term_body: 'body' (calc_body_diff), 'root' or 'Head' (humanoid_im.py:1223-1229)"
    rfc_mode = cfg.get("residual_force_mode", "implicit") if cfg.residual_force else "none"     # residual_force: false -> no residual-force dims (humanoid_im.py:231-243)
    assert rfc_mode in ("implicit", "explicit", "none"), "residual_force_mode: implicit | explicit"
    if rfc_mode == "explicit":      # the kernel restates the release settings of the explicit mode (config/release/uhc_explicit.yml)
        assert cfg.get("residual_force_bodies", "all") == "all" and cfg.get("residual_force_torque", True) and int(cfg.get("residual_force_bodies_num", 1)) == 1 \
            and not cfg.get("residual_contact_only", False) and not cfg.get("residual_contact_projection", False), \
            "explicit residual force: only residual_force_bodies = all, one point per body, torque on, no contact gating / projection"
    # the fused reward follows the residual-force mode (world_rfc_implicit :12-88 / world_rfc_explicit :253-341), as the released configs pair them
    assert cfg.reward_id in (("world_rfc_explicit",) if rfc_mode == "explicit" else ("world_rfc_implicit", "world_rfc_implicit_v1_mul")), "reward_id must match residual_force_mode"
    assert float(cfg.get("env_init_noise", 0.0)) == 0.0, "env_init_noise > 0 is not implemented"
    return rfc_mode


class AgentCopycat:
    def __init__(self, cfg, dtype, device, training=True, checkpoint_epoch=0):
        import torch
        self.cfg = self.cc_cfg = cfg
        self.dtype, self.device, self.training = dtype, device, training
        self.epoch, self.max_freq = 0, 50
        dev_index = device.index if getattr(device, "type", "cpu") == "cuda" and device.index is not None else int(getattr(cfg, "gpu_index", 0) or 0)
        if not torch.cuda.is_available():
            raise RuntimeError("the batched engine needs a CUDA device (the reference's CPU sampling path is replaced, not kept as a fallback)")
        self.model_tables = HumanoidModel()
        # data (setup_data_loader :128-134)
        self.data_loader = DatasetAMASSSingle(cfg.data_specs, data_mode="train", model=self.model_tables)
        self.test_data_loaders = [self.data_loader]
        if len(cfg.data_specs.get("test_file_path", [])) > 0:
            self.test_data_loaders.append(DatasetAMASSSingle(cfg.data_specs, data_mode="test", model=self.model_tables))
        self.logger = logging.getLogger(f"uhc_b200.{cfg.id}")
        if not self.logger.handlers:
            logging.basicConfig(level=logging.INFO, format="%(message)s")
        rw = cfg.reward_weights or {}
        w = [rw.get(k, d) for k, d in (("w_p", 0.6), ("w_v", 0.1), ("w_e", 0.2), ("w_c", 0.1), ("w_vf", 0.0))]
        kk = [rw.get(k, d) for k, d in (("k_p", 2), ("k_v", 0.005), ("k_e", 20), ("k_c", 1000), ("k_vf", 1))]
        self.num_envs = int(cfg.get("num_envs", 4096))
        self.horizon = max(2, int(math.ceil(cfg.min_batch_size / self.num_envs)))
        world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
        sync = None
        if world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                dist.init_process_group("nccl")
            sync = make_nccl_grad_sync(world)
        rfc_mode = supported_variant(cfg)       # refuses (AssertionError) what the batched engine does not implement instead of accepting it silently (ADVICE r1)
        self._subjects = self._subject_bodies(dev_index) if cfg.get("subject_bodies", False) else None
        def fixed_motions(engine):
            """data_specs.fix_height / drop_implausible (DatasetAMASSSingle.fix_floor): the raw motion is measured on the GPU, so it runs between
            the engine's creation and the first table load; the clip table, the clip sampler and the history keys are all built from what is left"""
            self.data_loader.fix_floor(engine, self.logger.info)
            return self.data_loader.motions, self.data_loader.shapes
        self.agent = BatchedAgent(
            self.num_envs, fixed_motions if self._device_tables(self.data_loader) else self.data_loader.experts, self.data_loader.shapes, device=dev_index, seed=cfg.seed, policy_hsize=cfg.policy_hsize,
            value_hsize=cfg.value_hsize, htype=cfg.policy_htype, log_std=cfg.log_std, policy_lr=cfg.policy_lr, value_lr=cfg.value_lr,
            gamma=cfg.gamma, tau=cfg.tau, clip_epsilon=cfg.clip_epsilon, num_optim_epoch=cfg.num_optim_epoch, grad_clip=40.0,
            t_min=cfg.data_specs.get("t_min", 90), t_max=cfg.data_specs.get("t_max", -1), rank=rank, world=world, grad_sync=sync,
            model=self.model_tables, base_rot=cfg.data_specs.get("base_rot", [0.7071, 0.7071, 0.0, 0.0]), rfc_scale=cfg.residual_force_scale,
            rfc_lim=cfg.residual_force_lim, rfc_rate=0.0 if cfg.rfc_decay else 1.0, body_diff_thresh=cfg.get("body_diff_thresh", 0.5),
            meta_pd=int(cfg.meta_pd), env_episode_len=cfg.env_episode_len, trail_steps=cfg.env_expert_trail_steps, w=w, k=kk, rfc_mode=rfc_mode,
            obs_v=int(cfg.obs_v), fut_frames=int(cfg.get("fut_frames", 10)), fut_skip=int(cfg.get("skip", 10)),
            has_shape=bool(cfg.get("has_shape", False)) and bool(cfg.get("has_shape_obs", True)), actor_type=cfg.actor_type, num_primitive=int(cfg.get("num_primitive", 8)), composer_dim=tuple(cfg.get("composer_dim", [300, 200])),
            reactive_v=int(cfg.get("reactive_v", 0)), reactive_rate=float(cfg.get("reactive_rate", 0.3)),
            term_body=cfg.get("env_term_body", "body"), head_body=self.model_tables.body_names.index("Head"), reward_mul=cfg.reward_id == "world_rfc_implicit_v1_mul",
            variants=self._subjects and self._subjects[0], subject_of=self._subjects and self._subject_of, curriculum_global=bool(cfg.get("curriculum_global", False)))
        self.policy_net, self.value_net, self.running_state = self.agent.policy, self.agent.value, self.agent.running_state
        self.state_dim, self.action_dim = self.agent.obs_dim, self.agent.act_dim
        self.expert_reward = reward_func[cfg.reward_id]
        self.env = None   # single-env facade, built lazily (eval_seq / visualisation code paths)
        self.freq_dict = {k: [] for k in self.data_loader.data_keys}
        for loader in self.test_data_loaders:                   # a separate test set: fixed here, before any evaluation reads its length
            loader.fix_floor(self.agent.engine, self.logger.info)
        # the failure-weighted curriculum (freq_dict): on the host (default) or, with curriculum_on_device, in device rings updated after
        # every rollout (Engine.curriculum_*).  precision_mode and fit_single_key need the device curriculum and turn it on, and so does
        # curriculum_global: one history across the ranks of a multi-GPU run, merged from every rank's episodes in each update
        self._precision_mode = bool(cfg.get("precision_mode", False))
        self._fit_single_key = ""
        self.curriculum_on_device = bool(cfg.get("curriculum_on_device", False)) or self._precision_mode or self.agent.curriculum_global
        if self.curriculum_on_device:
            self._enable_device_curriculum()
        if checkpoint_epoch > 0:
            self.load_checkpoint(checkpoint_epoch)
            self.epoch = checkpoint_epoch

    # ---------------------------------------------------------------- device curriculum (agent_copycat.py:503-517, dataset_amass_single.py:172-232)
    @property
    def precision_mode(self):
        return self._precision_mode

    @precision_mode.setter
    def precision_mode(self, on):      # assignable as scripts/fit_uhc.py does
        self._precision_mode = bool(on)
        if self._precision_mode and not self.curriculum_on_device:
            self.curriculum_on_device = True
        if self.curriculum_on_device:
            self._enable_device_curriculum()

    @property
    def fit_single_key(self):
        return self._fit_single_key

    @fit_single_key.setter
    def fit_single_key(self, key):
        self._fit_single_key = key or ""
        if self._fit_single_key and not self.curriculum_on_device:
            self.curriculum_on_device = True
        if self.curriculum_on_device:
            self._enable_device_curriculum()

    def _curriculum_params(self):
        """the sampler's parameters: sample_seq passes sampling_freq to both of its draws; with fit_single_key get_sample_from_key runs
        with its default sampling_freq 0.75 (agent_copycat.py:504-510)"""
        cfg, fit = self.cfg, self._fit_single_key
        freq = float(cfg.get("sampling_freq", 0.5))
        prec = (0.75 if fit else freq) if self._precision_mode else 0.0
        return dict(max_freq=self.max_freq, temp=float(cfg.get("sampling_temp", 0.2)), freq=freq, prec_freq=prec,
                    fit_clip=self.data_loader.data_keys.index(fit) if fit else -1)

    def _enable_device_curriculum(self):
        fresh = self.agent.engine.cur_cfg is None
        self.agent.curriculum_enable(**self._curriculum_params())
        if fresh:
            self._freq_dict_to_device(self.freq_dict)

    def _freq_dict_to_device(self, fd):
        keys, M = self.data_loader.data_keys, self.max_freq
        ln, p, st = np.zeros(len(keys), np.int32), np.zeros((len(keys), M), np.float32), np.zeros((len(keys), M), np.int32)
        for c, k in enumerate(keys):
            h = list(fd.get(k, []))[-M:]
            ln[c] = len(h)
            for j, r in enumerate(h):
                p[c, j], st[c, j] = float(r[0]), int(r[1])
        self.agent.curriculum_set(ln, p, st)

    def _freq_dict_from_device(self):
        ln, p, st = self.agent.curriculum_get()
        return {k: [[float(p[c, j]), int(st[c, j])] for j in range(ln[c])] for c, k in enumerate(self.data_loader.data_keys)}

    def get_freq_dict(self):
        """{key: [[percent, start], ...]} -- the host history, or the device rings read back"""
        return self._freq_dict_from_device() if self.curriculum_on_device else self.freq_dict

    # ---------------------------------------------------------------- schedules (:279-297)
    def per_epoch_update(self, epoch):
        cfg = self.cfg
        cfg.update_adaptive_params(epoch)
        self.agent.noise_rate = cfg.adp_noise_rate
        self.agent.opt_p.lr = cfg.adp_policy_lr
        if cfg.rfc_decay:
            rate = float(np.clip(1 - epoch / cfg.get("rfc_decay_max", 10000), 0, 1))
            self.agent.engine.set_cfg(rfc_rate=rate)
        if cfg.fix_std:
            self.agent.log_std.fill_(float(cfg.adp_log_std))

    # ---------------------------------------------------------------- sampling / update
    def sample(self, min_batch_size=None):
        T = self.horizon if min_batch_size is None else max(2, int(math.ceil(min_batch_size / self.num_envs)))
        buf, log = self.agent.sample(T)
        if not self.curriculum_on_device:           # the device curriculum was updated inside agent.sample
            self._update_freq_dict(buf)
        log = _Log(log)
        log.update(avg_c_reward=log["avg_reward"], avg_episode_c_reward=log["avg_episode_reward"])
        return _Batch(buf), log

    def _update_freq_dict(self, buf):
        """per-clip success history from the episodes that ended in this rollout ([percent, fr_start] per episode, agent_copycat.py:561,
        590-603, capped at max_freq entries), then the device sampler's weights (dataset_amass_single.py:183-186)."""
        clip = buf.ep_clip.cpu().numpy().reshape(-1)
        pct = buf.ep_pct.cpu().numpy().reshape(-1)
        sel = clip >= 0
        keys = self.data_loader.data_keys
        for c, p in zip(clip[sel], pct[sel]):
            self.freq_dict[keys[c]].append([float(p), 0])
        self.freq_dict = {k: v[-self.max_freq:] for k, v in self.freq_dict.items()}
        self._push_clip_weights()

    def _push_clip_weights(self):
        from uhc_b200.agent import failure_weights
        cfg = self.cfg
        hist = [[r[0] for r in self.freq_dict[k]] for k in self.data_loader.data_keys]
        if any(len(h) for h in hist):
            self.agent.engine.set_clip_weights(failure_weights(hist, cfg.get("sampling_temp", 0.2), cfg.get("sampling_freq", 0.5)))

    def update_params(self, batch):
        return self.agent.update_params(batch.buf)["update_time"]

    def optimize_policy(self, epoch, save_model=True):
        cfg = self.cfg
        self.epoch = epoch
        t0 = time.time()
        self.per_epoch_update(epoch)
        batch, log = self.sample(cfg.min_batch_size)
        t1 = time.time()
        self.update_params(batch)
        t2 = time.time()
        info = {"log": log, "T_sample": t1 - t0, "T_update": t2 - t1, "T_total": t2 - t0}
        if save_model and (self.epoch + 1) % cfg.save_n_epochs == 0:
            self.save_checkpoint(epoch)
            info["log_eval"] = self.eval_policy(epoch)
        self.log_train(info)
        return info

    def log_train(self, info):
        log = info["log"]
        self.logger.info(f"{self.cfg.id} | {self.epoch:4d} | T_s {info['T_sample']:.2f} T_u {info['T_update']:.2f} | steps {log['num_steps']} "
                         f"({log['num_steps'] / max(info['T_sample'], 1e-9):.0f}/s) | eps_len {log['avg_episode_len']:.1f} | avg_r {log['avg_reward']:.4f} "
                         f"| eps_r {log['avg_episode_reward']:.2f} | fail {log['fail_rate']:.2f}")
        if not getattr(self.cfg, "no_log", True):
            try:
                import wandb
                wandb.log({"rewards": log["avg_reward"], "eps_len": log["avg_episode_len"], "avg_rwd": log["avg_episode_reward"]}, step=self.epoch)
                if "log_eval" in info:
                    [wandb.log(t, step=self.epoch) for t in info["log_eval"]]
            except Exception:
                pass

    # ---------------------------------------------------------------- evaluation (:354-494), batched: one env per clip
    def eval_policy(self, epoch=0, dump=False, max_bytes=1 << 30):
        """eval_policy / eval_seq (agent_copycat.py:354-494) for every clip at once: env i imitates clip c0 + i from frame 0 with the
        deterministic policy; per step ONE batched state read (uhc_env_get_state_batch) feeds the reference's metrics
        (smpl_eval.compute_metrics: mpjpe / pa-mpjpe / accel / vel / root distance, restated in uhc_b200/metrics.py); fail_safe re-seats a
        failed humanoid on the expert pose with one batched set_state (humanoid_im.py:902-905).

        With several ranks each rank evaluates its own clips (uhc_b200.agent.assign_clips), and every rank then holds every clip's metrics,
        logs the same coverage lines, returns what one rank would return and applies every eval outcome to its curriculum in clip order.
        Rank 0 alone writes the dumps; the trajectories they hold (eval_dump_motion, full_eval) reach it in pieces of at most max_bytes."""
        world = self.agent.world
        res_dicts = []
        for loader in self.test_data_loaders:
            if world == 1:
                res, pending = self._eval_loader(loader, dump)
            else:
                local = {}

                def shard(loader=loader):
                    r, p = self._eval_loader(loader, dump)
                    local.update(r)
                    return {k: {m: v for m, v in d.items() if m not in TRAJECTORY_KEYS} for k, d in r.items()}, p
                parts = exchange(shard)
                res, pending = merge_results([p[0] for p in parts], loader.data_keys), merge_outcomes([p[1] for p in parts])
                if dump and (self._full_eval() or self.cfg.get("eval_dump_motion", False)):
                    full = gather_to_root(local, max_bytes)         # a collective: every rank takes part, rank 0 keeps the result
                    if self.agent.rank == 0:
                        res = merge_results([full], loader.data_keys)
            self._apply_outcomes(pending)
            res_dicts.append(self._coverage(loader, res, epoch, dump))
        if not self.curriculum_on_device:
            self._push_clip_weights()
        return res_dicts

    def _apply_outcomes(self, pending):
        """eval outcomes (table clip, training clip, outcome) fed to the failure-weighted sampler like training episodes ([outcome, 0]):
        appended to freq_dict, or pushed in one call to the device curriculum"""
        if self.curriculum_on_device:
            if pending:
                self.agent.curriculum_push([i for _, i, _ in pending], [o for _, _, o in pending], [0] * len(pending))
            return
        keys = self.data_loader.data_keys
        for _, i, o in pending:
            self.freq_dict[keys[i]] = (self.freq_dict[keys[i]] + [[o, 0]])[-self.max_freq:]

    def _my_clips(self):
        """this rank's clips of the loaded table, in the order of its evaluation calls (every clip in order at world 1)"""
        calls = shard_clips(self.agent.engine.clip_len, self.agent.world, self.agent.rank, self.num_envs)
        return np.concatenate([np.zeros(0, np.int32)] + calls)

    def _eval_loader(self, loader, dump):
        """eval_policy's roll-out of this rank's clips of one loader: ({key: result}, [(table clip, training clip, outcome)])"""
        import torch
        from uhc_b200.metrics import compute_metrics, metrics_from_frames
        cfg = self.cfg
        on_device = bool(cfg.get("eval_on_device", False))     # opt-in: BatchedAgent.evaluate (uhc_eval_run) instead of the host loop below
        motion = dump and bool(cfg.get("eval_dump_motion", False))   # opt-in: the dump also holds eval_seq's trajectories + SMPL per clip
        floor = bool(cfg.get("eval_floor_metrics", False))           # opt-in: pentration / skate / float of the body hulls per clip (_add_floor)
        full = self._full_eval()                                     # opt-in: the SMPL mesh of every clip, pentration / skate from it (_add_mesh)
        if full and floor:
            raise ValueError("full_eval and eval_floor_metrics both write pentration / skate: enable one of them")
        if full:
            self._mesh_model()
        eng = self.agent.engine
        E = self.num_envs
        pending = []        # this loader's eval outcomes, applied once the training tables are back (the device curriculum's are lost on a load)
        device_tables = self._device_tables(loader)
        if loader is not self.data_loader:
            saved = self._freq_dict_from_device() if self.curriculum_on_device else None
            self._load_tables(loader)      # invalidates every env record: only the envs reset below are stepped
        eng.set_cfg(**self._env_cfg(test=True))
        res = {}
        for clips in shard_clips(eng.clip_len, self.agent.world, self.agent.rank, E):
            ids = np.arange(len(clips), dtype=np.int32)
            lens = eng.clip_len[clips]
            if on_device:                                      # the same roll-out as the loop below, as CUDA-graph replays with the metrics on the device
                kw = dict(record_states=True, export_smpl=True) if motion else (dict(record_states=True) if full else {})
                dev = self.agent.evaluate(clips, bool(cfg.fail_safe), window=32, floor=floor, **kw)
                last_t = np.array([d["last_t"] for d in dev], np.int64); fail_any = np.array([d["fail_any"] for d in dev], bool)
                rsum = np.array([d["reward_sum"] for d in dev]); nrec = [len(d["frames"]) for d in dev]
                self._eval_results(res, loader, clips, ids, lens, last_t, fail_any, rsum, nrec,
                                   lambda i, pct, fs: metrics_from_frames(dev[i]["frames"], pct, fs), pending)
                if floor:
                    for i in ids:
                        self._add_floor(res[loader.data_keys[clips[i]]], loader, int(clips[i]), dev[i]["floor"], np.arange(1, len(dev[i]["frames"]) + 1))
                if full:
                    self._add_mesh(res, loader, ids, clips, [dev[i]["states"][:, :76] for i in ids],
                                   [np.arange(1, len(dev[i]["frames"]) + 1) for i in ids], dump)
                if motion:
                    for i in ids:
                        d = dev[i]
                        self._add_motion(res[loader.data_keys[clips[i]]], loader, int(clips[i]), d["states"][:, :76], d["states"][:, 76:148],
                                         d["pose_aa"], d["trans"], np.arange(1, len(d["frames"]) + 1), bool(d["fail_any"]))
                continue
            if len(ids) < E:                                   # idle envs: park them on the call's first clip so every record is valid (their outputs are ignored)
                eng.reset(np.arange(len(ids), E, dtype=np.int32), np.full(E - len(ids), clips[0], np.int32), 0, None)
            obs = eng.reset(ids, clips, 0, None)
            alive = np.ones(len(ids), bool); fail_any = np.zeros(len(ids), bool)
            rsum = np.zeros(len(ids)); last_t = np.zeros(len(ids), np.int64)
            traj = [dict(pred=[], pred_jpos=[], t=[]) for _ in ids]
            gt = {}

            def expert(i):
                """expert table of clips[i]: the host-built one, or the device-built one read back once (in the engine's precision)"""
                if not device_tables:
                    return loader.experts[clips[i]]
                if i not in gt:
                    gt[i] = eng.clip_frames(clips[i])
                return gt[i]
            det = torch.ones(E, dtype=torch.uint8, device=obs.device)
            for t in range(int(lens.max()) - 1):
                s = self.running_state(obs, update=False)
                mean = self.policy_net.forward_tc(s)
                a, _ = nn.gaussian_sample(mean, self.agent.log_std, 0, 0, det)
                obs, rew, ci, fail, end, pct = eng.step(a)
                f, e, r = fail.cpu().numpy()[ids] != 0, end.cpu().numpy()[ids] != 0, rew.cpu().numpy()[ids]
                live = np.nonzero(alive)[0]
                st = eng.get_states(ids[live])
                for j, i in enumerate(live):
                    traj[i]["pred"].append(st["qpos"][j].copy()); traj[i]["pred_jpos"].append(st["xpos"][j].reshape(-1).copy()); traj[i]["t"].append(int(st["cur_t"][j]))
                    last_t[i] = st["cur_t"][j]
                rsum[live] += r[live]
                failed = live[f[live]]
                fail_any[failed] = True
                if len(failed):
                    if cfg.fail_safe:
                        tt = [min(int(last_t[i]), expert(i)["len"] - 1) for i in failed]
                        eng.set_states(ids[failed], np.stack([expert(i)["qpos"][k] for i, k in zip(failed, tt)]),
                                       np.stack([expert(i)["qvel"][k] for i, k in zip(failed, tt)]))
                    else:
                        alive[failed] = False
                alive[live[e[live]]] = False
                if not alive.any():
                    break
            def host_metrics(i, pct, fs):
                ex = expert(i)
                tt = np.minimum(np.array(traj[i]["t"], dtype=np.int64), ex["len"] - 1)
                return compute_metrics({"pred": np.array(traj[i]["pred"]), "gt": np.asarray(ex["qpos"])[tt], "pred_jpos": np.array(traj[i]["pred_jpos"]),
                                        "gt_jpos": np.asarray(ex["wbpos"])[tt], "percent": pct, "fail_safe": fs})
            self._eval_results(res, loader, clips, ids, lens, last_t, fail_any, rsum, [len(traj[i]["t"]) for i in ids], host_metrics, pending)
            if floor:                           # the host loop's recorded qpos through the device measurement
                for i in ids:
                    if traj[i]["t"]:
                        var = None if eng.clip_models is None else int(eng.clip_models[clips[i]])
                        rows = eng.floor_qpos(np.array(traj[i]["pred"]).reshape(-1, 76), variants=var).cpu().numpy()
                        self._add_floor(res[loader.data_keys[clips[i]]], loader, int(clips[i]), rows, np.array(traj[i]["t"], np.int64))
            if full:
                self._add_mesh(res, loader, ids, clips, [np.array(traj[i]["pred"]).reshape(-1, 76) for i in ids],
                               [np.array(traj[i]["t"], np.int64) for i in ids], dump)
            if motion:                          # the host loop's recorded qpos as SMPL through the device conversion
                for i in ids:
                    pred = np.array(traj[i]["pred"]).reshape(-1, 76)
                    pose, trans = eng.qpos_to_smpl(pred)
                    self._add_motion(res[loader.data_keys[clips[i]]], loader, int(clips[i]), pred, np.array(traj[i]["pred_jpos"]).reshape(-1, 72),
                                     pose.cpu().numpy(), trans.cpu().numpy(), np.array(traj[i]["t"], np.int64), bool(fail_any[i]), expert(i))
        if loader is not self.data_loader:
            self._load_tables(self.data_loader)
            if saved is not None:          # a table of another clip count disabled the device curriculum: restore it
                self._restore_device_curriculum(saved)
        eng.set_cfg(**self._env_cfg(test=False))
        self.agent.obs = None
        return res, pending

    def _coverage(self, loader, res, epoch, dump):
        """the coverage line and metric dict of one loader's results (and with dump its {epoch}_{loader}_coverage_full.pkl, written by rank 0)"""
        n = loader.get_len()
        names = ("succ", "reward", "mpjpe", "mpjpe_g", "pa_mpjpe", "accel_dist", "vel_dist", "root_dist")
        if bool(self.cfg.get("eval_floor_metrics", False)):
            names += ("pentration", "skate", "float", "pentration_gt", "skate_gt", "float_gt")
        elif self._full_eval():
            names += ("pentration", "skate", "pentration_gt", "skate_gt")
        metrics = {m: float(np.mean([np.mean(r[m]) for r in res.values() if m in r])) if any(m in r for r in res.values()) else float("nan") for m in names}
        coverage = int(round(metrics["succ"] * n))
        self.logger.info(f"Coverage {loader.name} of {coverage} out of {n} | " + " \t".join(f"{k}: {v:.3f}" for k, v in metrics.items()))
        metrics.update(mean_coverage=coverage / n, num_coverage=coverage, all_coverage=n)
        del metrics["succ"]
        if dump and self.agent.rank == 0:
            joblib.dump(res, osp.join(self.cfg.output_dir, f"{epoch}_{loader.name}_coverage_full.pkl"))
        return {f"coverage_{loader.name}": metrics}

    def eval_checkpoints(self, epochs, dump=False):
        """eval_policy(eval_on_device: true) of several saved checkpoints (models/iter_%04d.p) at once: every test loader is evaluated for all
        of them in shared device calls (BatchedAgent.evaluate_policies).  Returns {epoch: res_dicts}, each what load_checkpoint(epoch) +
        eval_policy(epoch, dump) gives, and logs the same coverage lines.  Comparing checkpoints is not training: no outcome reaches freq_dict
        or the device curriculum, and the agent's weights, log_std and running_state stay as they are.  With several ranks each evaluates
        its own clips and every rank returns every clip's results, as eval_policy does."""
        from uhc_b200.metrics import metrics_from_frames
        cfg, eng = self.cfg, self.agent.engine
        epochs = list(epochs)
        cps = []
        for epoch in epochs:
            path = "%s/iter_%04d.p" % (cfg.model_dir, epoch)
            self.logger.info("loading model from checkpoint: %s" % path)
            with open(path, "rb") as f:
                cps.append(pickle.load(f))
        out = {epoch: [] for epoch in epochs}
        for loader in self.test_data_loaders:
            def work(loader=loader):
                saved = None
                if loader is not self.data_loader:
                    saved = self._freq_dict_from_device() if self.curriculum_on_device else None
                    self._load_tables(loader)
                eng.set_cfg(**self._env_cfg(test=True))
                clips = self._my_clips()
                lens = eng.clip_len[clips]
                per_cp = self.agent.evaluate_policies(cps, clips, bool(cfg.fail_safe), window=32)
                if loader is not self.data_loader:
                    self._load_tables(self.data_loader)
                    if saved is not None:
                        self._restore_device_curriculum(saved)
                eng.set_cfg(**self._env_cfg(test=False))
                self.agent.obs = None
                per_res = []
                for dev in per_cp:
                    last_t = np.array([d["last_t"] for d in dev], np.int64); fail_any = np.array([d["fail_any"] for d in dev], bool)
                    rsum = np.array([d["reward_sum"] for d in dev])
                    res = {}
                    for i, c in enumerate(clips):
                        res[loader.data_keys[c]] = self._clip_result(lens[i], last_t[i], fail_any[i], rsum[i], len(dev[i]["frames"]),
                                                                     lambda pct, fs, d=dev[i]: metrics_from_frames(d["frames"], pct, fs))
                    per_res.append(res)
                return per_res
            if self.agent.world == 1:
                per_res = work()
            else:
                parts = exchange(work)
                per_res = [merge_results([p[j] for p in parts], loader.data_keys) for j in range(len(epochs))]
            for epoch, res in zip(epochs, per_res):
                out[epoch].append(self._coverage(loader, res, epoch, dump))
        if not self.curriculum_on_device:
            self._push_clip_weights()          # a test table load reset the sampler's clip weights: put the training ones back
        return out

    def _add_motion(self, r, loader, clip, pred, pred_jpos, pose_aa, trans, t, fail_any, gt=None):
        """eval_seq's trajectory keys (gt / pred qpos, gt_jpos / pred_jpos world joint positions, fail_safe) and the SMPL pose / trans of one
        clip's recorded frames into its result dict r; t = cur_t after each recorded step (the expert frame min(t, len - 1) it is compared with)"""
        if gt is None:
            gt = self.agent.engine.clip_frames(clip) if self._device_tables(loader) else loader.experts[clip]
        tt = np.minimum(np.asarray(t, np.int64), int(self.agent.engine.clip_len[clip]) - 1)
        r.update(gt=np.asarray(gt["qpos"])[tt], pred=np.array(pred), gt_jpos=np.asarray(gt["wbpos"])[tt].reshape(len(tt), -1), pred_jpos=np.array(pred_jpos),
                 pose_aa=np.array(pose_aa), trans=np.array(trans), fail_safe=bool(fail_any and self.cfg.fail_safe))

    def export_motion(self, epoch=0, loaders=None, dump=True, max_bytes=1 << 30):
        """the simulated motion of every clip of the test loaders (or `loaders`), from the device evaluation (BatchedAgent.export_motion):
        {loader name: {key: eval_seq's dict (gt, pred, gt_jpos, pred_jpos, percent, fail_safe, reward and compute_metrics' keys with succ) plus
        pose_aa [frames][72] and trans [frames][3]}}; with dump each loader's dict goes to {epoch}_{loader}_motion.pkl.  Like eval_checkpoints
        it is not training: no outcome reaches freq_dict or the device curriculum, and the training tables and cfg are restored.  max_bytes
        bounds the host memory of one device call (BatchedAgent.export_motion).

        With several ranks each rank evaluates its own clips and sends them to rank 0 in pieces of at most max_bytes: rank 0 returns
        (and with dump writes) every clip, in clip order, and every other rank returns only its own clips."""
        from uhc_b200.metrics import metrics_from_frames
        cfg, eng = self.cfg, self.agent.engine
        out = {}
        for loader in (self.test_data_loaders if loaders is None else loaders):
            def work(loader=loader):
                saved = None
                if loader is not self.data_loader:
                    saved = self._freq_dict_from_device() if self.curriculum_on_device else None
                    self._load_tables(loader)
                eng.set_cfg(**self._env_cfg(test=True))
                clips = self._my_clips()
                lens = eng.clip_len[clips].copy()
                mot = self.agent.export_motion(clips, bool(cfg.fail_safe), window=32, max_bytes=max_bytes)
                res = {}
                for c, L, d in zip(clips, lens, mot):
                    r = res[loader.data_keys[c]] = self._clip_result(L, d["last_t"], d["fail_any"], d["reward_sum"], len(d["frames"]),
                                                                     lambda pct, fs, d=d: metrics_from_frames(d["frames"], pct, fs))
                    self._add_motion(r, loader, int(c), d["pred"], d["pred_jpos"], d["pose_aa"], d["trans"], np.arange(1, len(d["frames"]) + 1), d["fail_any"])
                if loader is not self.data_loader:
                    self._load_tables(self.data_loader)
                    if saved is not None:
                        self._restore_device_curriculum(saved)
                eng.set_cfg(**self._env_cfg(test=False))
                self.agent.obs = None
                return res
            if self.agent.world == 1:
                res = work()
            else:
                local = {}
                exchange(lambda: local.update(work()))
                res = gather_to_root(local, max_bytes)
                keys = loader.data_keys if self.agent.rank == 0 else [k for k in loader.data_keys if k in res]
                res = merge_results([res], keys)
            if dump and self.agent.rank == 0:
                joblib.dump(res, osp.join(cfg.output_dir, f"{epoch}_{loader.name}_motion.pkl"))
            out[loader.name] = res
        if not self.curriculum_on_device:
            self._push_clip_weights()          # a test table load reset the sampler's clip weights: put the training ones back
        return out

    def render_motion(self, epoch=0, loaders=None, out_dir=None, size=(1920, 1080), video="mp4", body="hulls"):
        """CopycatVisualizer's render_video without MuJoCo: every clip of the test loaders (or `loaders`) evaluated on the device and drawn
        there (BatchedAgent.render_motion), the simulated `pred` beside the expert `gt` as eval_seq pairs them, one mp4 per clip written by
        write_frames_to_video to {out_dir or cfg.output}/{take_key}_{cfg.id}_{epoch}_0.mp4 (the visualizer's video_path).  The view follows cfg's
        hide_im / hide_expert / shift_expert / focus as update_pose does.  Returns {loader name: {take_key: path}}; clips of two loaders with
        the same key share a file name, as in the visualizer, so such loaders want one call each with their own out_dir.  Like export_motion it is
        not training: no outcome reaches freq_dict or the device curriculum, and the training tables and cfg are restored.  video="mjpeg"
        compresses the frames on the device (BatchedAgent.render_motion's encode="jpeg") and writes {take_key}_{cfg.id}_{epoch}_0.avi, a
        Motion-JPEG AVI (uhc_b200.video.write_mjpeg_avi), instead.  body="mesh" draws the skinned SMPL mesh instead of the body hulls:
        the neutral model data/smpl/SMPL_NEUTRAL.{pkl,npz} (as full_eval loads it, and it must hold the faces `f`), each clip shaped by its
        beta[:10] under has_shape and zeros otherwise.  With several ranks each rank renders and writes the files of its own clips."""
        from uhc.utils.image_utils import write_frames_to_video
        from uhc_b200.video import write_mjpeg_avi
        if video not in ("mp4", "mjpeg"):
            raise ValueError('render_motion: video must be "mp4" or "mjpeg"')
        ext, W, H = ("mp4" if video == "mp4" else "avi"), int(size[0]), int(size[1])
        cfg, eng = self.cfg, self.agent.engine
        out_dir = out_dir or getattr(cfg, "output", None) or cfg.output_dir
        os.makedirs(out_dir, exist_ok=True)
        if body == "mesh":
            self._mesh_model(render=True)
        cam = {k: bool(getattr(cfg, k, False)) for k in ("hide_im", "hide_expert", "focus")}
        cam["shift_expert"] = 1.0 if getattr(cfg, "shift_expert", False) else 0.0
        out = {}
        for loader in (self.test_data_loaders if loaders is None else loaders):
            paths = {k: osp.join(out_dir, f"{k}_{cfg.id}_{epoch}_0.{ext}") for k in loader.data_keys}

            def work(loader=loader, paths=paths):
                saved = None
                if loader is not self.data_loader:
                    saved = self._freq_dict_from_device() if self.curriculum_on_device else None
                    self._load_tables(loader)
                eng.set_cfg(**self._env_cfg(test=True))
                ids = self._my_clips()

                def writer(i, chunks, keys=loader.data_keys, paths=paths):
                    if video == "mp4":
                        write_frames_to_video((f for ch in chunks for f in ch), paths[keys[ids[i]]])
                    else:
                        write_mjpeg_avi(paths[keys[ids[i]]], (f for ch in chunks for f in ch), W, H)

                betas = None
                if body == "mesh" and self.cfg.get("has_shape", False):
                    betas = clip_betas(loader.shapes, ids)
                self.agent.render_motion(ids, bool(cfg.fail_safe), size, cam, writer=writer, encode=None if video == "mp4" else "jpeg", body=body,
                                         betas=betas)
                if loader is not self.data_loader:
                    self._load_tables(self.data_loader)
                    if saved is not None:
                        self._restore_device_curriculum(saved)
                eng.set_cfg(**self._env_cfg(test=False))
                self.agent.obs = None
            if self.agent.world == 1:
                work()
            else:
                exchange(work)           # each rank writes its own clips' files; every rank returns every path once all are written
            out[loader.name] = paths
        if not self.curriculum_on_device:
            self._push_clip_weights()
        return out

    def _restore_device_curriculum(self, fd):
        if self.agent.engine.cur_cfg is None:
            self.agent.curriculum_enable(**self._curriculum_params())
        self._freq_dict_to_device(fd)

    def eval_seq(self, take_key, loader):
        """eval_seq (agent_copycat.py:435-493) for one clip on the device evaluation (BatchedAgent.evaluate with the state record):
        gt / pred (qpos), gt_jpos / pred_jpos (world joint positions), reward, percent, fail_safe and compute_metrics' keys with succ --
        the values eval_policy(eval_on_device=True) computes for that clip.  The training tables and cfg are restored afterwards."""
        from uhc_b200.metrics import metrics_from_frames
        cfg, eng = self.cfg, self.agent.engine
        c = loader.data_keys.index(take_key)
        saved = None
        if loader is not self.data_loader:
            saved = self._freq_dict_from_device() if self.curriculum_on_device else None
            self._load_tables(loader)
        eng.set_cfg(**self._env_cfg(test=True))
        d = self.agent.evaluate(np.array([c], np.int32), bool(cfg.fail_safe), window=32, record_states=True)[0]
        L = int(eng.clip_len[c])
        gt = eng.clip_frames(c) if self._device_tables(loader) else loader.experts[c]
        tt = np.minimum(np.arange(1, len(d["frames"]) + 1), L - 1)
        out = self._clip_result(L, d["last_t"], d["fail_any"], d["reward_sum"], len(d["frames"]), lambda pct, fs: metrics_from_frames(d["frames"], pct, fs))
        st = d["states"]
        out.update(gt=np.asarray(gt["qpos"])[tt], pred=st[:, :76].copy(), gt_jpos=np.asarray(gt["wbpos"])[tt].reshape(len(tt), -1),
                   pred_jpos=st[:, 76:148].copy(), fail_safe=bool(d["fail_any"] and cfg.fail_safe))
        out["percent"] = float(d["last_t"]) / float(max(L - 1, 1))
        if loader is not self.data_loader:
            self._load_tables(self.data_loader)
            if saved is not None:
                self._restore_device_curriculum(saved)
        eng.set_cfg(**self._env_cfg(test=False))
        self.agent.obs = None
        return out

    def _add_floor(self, m, loader, clip, rows, t):
        """eval_floor_metrics: pentration / skate / float (smpl_eval.compute_metrics' keys, from the body hulls instead of the SMPL mesh:
        uhc_b200/metrics.py floor_summary) of a clip's simulated frames (rows = their [n][5] floor rows) and, as *_gt, of the expert frames
        min(t, len - 1) they are paired with, measured by the same kernel"""
        from uhc_b200.metrics import floor_summary
        if not len(rows):
            return
        eng = self.agent.engine
        gt = eng.clip_frames(clip) if self._device_tables(loader) else loader.experts[clip]
        var = None if eng.clip_models is None else int(eng.clip_models[clip])
        g = eng.floor_qpos(np.asarray(gt["qpos"])[np.minimum(t, int(eng.clip_len[clip]) - 1)], variants=var).cpu().numpy()
        m.update(floor_summary(rows))
        m.update({k + "_gt": v for k, v in floor_summary(g).items()})

    def _full_eval(self):
        """full_eval (the reference's --full_eval flag or full_eval: true in the yml)"""
        return bool(self.cfg.get("full_eval", False) or getattr(self.cfg, "full_eval", False))

    def _mesh_model(self, render=False):
        """full_eval's model: SMPL_NEUTRAL.{pkl,npz} in data/smpl relative to the working directory, where the reference's
        SMPL_Robot(data_dir="data/smpl") reads it (convert_2_smpl_params passes no gender), uploaded once; with render also the mesh
        renderer's topology of it (render_motion(body="mesh"))"""
        path = osp.join("data", "smpl")
        if not getattr(self, "_mesh_ready", False):
            if not any(osp.exists(osp.join(path, "SMPL_NEUTRAL." + e)) for e in ("pkl", "npz")):
                raise FileNotFoundError(f"the SMPL mesh (full_eval, render_motion(body='mesh')) needs the model {osp.join(path, 'SMPL_NEUTRAL.pkl')} (or .npz), relative to the working directory")
            self.agent.engine.mesh_init(path)
            self._mesh_ready = True
        if render and not getattr(self, "_render_mesh_ready", False):
            self.agent.engine.render_mesh_init(path)
            self._render_mesh_ready = True

    def _add_mesh(self, res, loader, ids, clips, preds, ts, dump, max_bytes=1 << 30):
        """full_eval: convert_2_smpl_params (humanoid_im.py:127-150) and compute_metrics' mesh keys (smpl_eval.py:113-121) for one evaluation
        chunk.  Every clip's simulated rows preds[k] and the expert rows min(t, len - 1) they are paired with go qpos -> SMPL -> mesh on the
        device (Engine.qpos_mesh) through the neutral model (_mesh_model), with the clip's beta[:10] when has_shape and zeros otherwise; pentration / skate (and *_gt for the expert rows)
        come from the mesh against the floor (metrics.floor_summary).  With dump, pred_vertices / gt_vertices [T][V][3] float32 and
        pred_joints / gt_joints [T][24][3] join the result, computed in device calls of at most max_bytes of vertices."""
        from uhc_b200.metrics import floor_summary
        eng = self.agent.engine
        segs = []                                      # (result dict, key prefix, qpos rows, beta, variant)
        for i, q, t in zip(ids, preds, ts):
            if not len(t):
                continue
            c = int(clips[i])
            gt = eng.clip_frames(c) if self._device_tables(loader) else loader.experts[c]
            beta = np.asarray(loader.shapes[c], np.float64)[:10] if self.cfg.get("has_shape", False) else np.zeros(10)
            var = 0 if eng.clip_models is None else int(eng.clip_models[c])
            tt = np.minimum(np.asarray(t, np.int64), int(eng.clip_len[c]) - 1)
            r = res[loader.data_keys[c]]
            segs += [(r, "pred", np.asarray(q, np.float64).reshape(-1, 76), beta, var), (r, "gt", np.asarray(gt["qpos"], np.float64)[tt], beta, var)]
        if not segs:
            return
        betas, bseg = np.unique(np.stack([s[3] for s in segs]), axis=0, return_inverse=True)
        lens = [len(s[2]) for s in segs]
        q = np.concatenate([s[2] for s in segs])
        bidx = np.repeat(bseg.reshape(-1), lens).astype(np.int32)
        var = np.repeat([s[4] for s in segs], lens).astype(np.int32)
        first = np.zeros(len(q), np.int32)
        first[np.cumsum([0] + lens[:-1])] = 1
        rows = eng.qpos_mesh(q, betas, bidx, variants=var, floor=True, first=first).cpu().numpy()
        o = 0
        for (r, who, qs, _, _), n in zip(segs, lens):
            f = floor_summary(rows[o:o + n])
            sfx = "" if who == "pred" else "_gt"
            r["pentration" + sfx], r["skate" + sfx] = f["pentration"], f["skate"]
            if dump:
                verts, joints = np.empty((n, eng.smpl_nvert, 3), np.float32), np.empty((n, 24, 3))
                step = max(1, max_bytes // (eng.smpl_nvert * 12))
                for a in range(0, n, step):
                    v, j = eng.qpos_mesh(q[o + a:o + min(n, a + step)], betas, bidx[o + a:o + min(n, a + step)], variants=var[o + a:o + min(n, a + step)],
                                         first=None)
                    verts[a:a + step], joints[a:a + step] = v.cpu().numpy(), j.cpu().numpy()
                r[who + "_vertices"], r[who + "_joints"] = verts, joints
            o += n

    def _clip_result(self, L, last_t, fail_any, rsum, nrec, metrics_of):
        """res[key] of one evaluated clip of L frames, from either roll-out: the percent / succ rules of eval_seq and the reward average.
        metrics_of(percent, fail_safe) -> compute_metrics' dict."""
        percent = float(last_t) / float(max(L - 1, 1))
        pct = 1.0 if (percent >= 1.0 and not fail_any) else min(percent, 0.999)
        m = metrics_of(pct, bool(fail_any and self.cfg.fail_safe)) if nrec >= 3 else {"succ": np.array([False])}
        m["succ"] = np.array([bool(m["succ"][0]) and not fail_any])
        m["reward"] = rsum / max(L - 1, 1)
        m["percent"] = percent
        return m

    def _eval_results(self, res, loader, clips, ids, lens, last_t, fail_any, rsum, nrec, metrics_of, pending):
        """res[key] of every clip of one evaluation call (_clip_result), and the eval outcome of every clip the training table holds,
        collected in `pending` as (table clip, training clip, outcome) for _apply_outcomes.  metrics_of(i, percent, fail_safe) -> compute_metrics' dict."""
        index = {k: c for c, k in enumerate(self.data_loader.data_keys)}
        for i in ids:
            k = loader.data_keys[clips[i]]
            m = res[k] = self._clip_result(lens[i], last_t[i], fail_any[i], rsum[i], nrec[i], lambda pct, fs: metrics_of(i, pct, fs))
            if k not in index:
                continue
            pending.append((int(clips[i]), index[k], 1.0 if m["succ"][0] else min(m["percent"], 0.999)))

    @staticmethod
    def _device_tables(loader):
        """data_specs.expert_tables: device -- the loader keeps the raw motion and the engine builds the expert tables on the GPU"""
        return getattr(loader, "expert_tables", "host") == "device"

    def _subject_bodies(self, device):
        """subject_bodies: every clip is simulated with its own subject's body, as the reference's reset_robot rebuilds the humanoid per clip
        (humanoid_im.py:154-180).  Loads data/smpl/SMPL_{NEUTRAL,MALE,FEMALE}.{pkl,npz} from the working directory, where the reference's
        Robot reads all three, and builds one shape variant per distinct (beta[:10], gender) of every loader's clips on the GPU
        (uhc_b200/subject_body.py).  Returns (variants, {subject key: variant})."""
        from uhc_b200.smpl_model import load_smpl_model
        from uhc_b200.subject_body import SubjectBasis, subject_key
        assert all(self._device_tables(l) for l in self.test_data_loaders), \
            "subject_bodies needs data_specs.expert_tables: device (the expert FK then runs on each clip's own body); expert_tables: host builds neutral-body tables"
        path, models = osp.join("data", "smpl"), []
        for g in ("NEUTRAL", "MALE", "FEMALE"):
            f = [osp.join(path, f"SMPL_{g}.{e}") for e in ("pkl", "npz") if osp.exists(osp.join(path, f"SMPL_{g}.{e}"))]
            if not f:
                raise FileNotFoundError(f"subject_bodies needs the SMPL model {osp.join(path, f'SMPL_{g}.pkl')} (or .npz), relative to the working directory")
            models.append(load_smpl_model(f[0]))
        basis = SubjectBasis.from_models(self.model_tables, *models)
        shapes = np.concatenate([np.asarray(l.shapes, np.float64).reshape(-1, 17) for l in self.test_data_loaders])
        variants, idx = basis.build(shapes[:, :10], shapes[:, 16], device=device)
        self.logger.info(f"subject_bodies: {len(variants)} bodies for {len(shapes)} clips")
        return variants, {subject_key(r[:10], r[16]): int(v) for r, v in zip(shapes, idx)}

    def _subject_of(self, shapes):
        """the shape variant of every clip of a loader (subject_bodies), from its shape rows [C][17]"""
        from uhc_b200.subject_body import subject_key
        return np.array([self._subjects[1][subject_key(r[:10], r[16])] for r in np.asarray(shapes, np.float64).reshape(-1, 17)], np.int32)

    def _load_tables(self, loader):
        if self._device_tables(loader) and self._subjects is not None:
            v = self._subject_of(loader.shapes)
            self.agent.engine.load_motions(loader.motions, loader.shapes, v, fk_models=v)
        elif self._device_tables(loader):
            self.agent.engine.load_motions(loader.motions, loader.shapes)
        else:
            self.agent.engine.load_clips(loader.experts, loader.shapes)

    def _env_cfg(self, test):
        cfg = self.cfg
        rw = cfg.reward_weights or {}
        return dict(base_rot=cfg.data_specs.get("base_rot", [0.7071, 0.7071, 0.0, 0.0]), rfc_scale=cfg.residual_force_scale, rfc_lim=cfg.residual_force_lim,
                    rfc_rate=0.0 if cfg.rfc_decay else 1.0, body_diff_thresh=cfg.get("body_diff_thresh_test" if test else "body_diff_thresh", 0.5),
                    meta_pd=int(cfg.meta_pd), env_episode_len=cfg.env_episode_len, trail_steps=cfg.env_expert_trail_steps, auto_reset=0 if test else 1,
                    rfc_mode=cfg.get("residual_force_mode", "implicit") if cfg.residual_force else "none", obs_v=int(cfg.obs_v),
                    fut_frames=int(cfg.get("fut_frames", 10)), fut_skip=int(cfg.get("skip", 10)),
                    has_shape=bool(cfg.get("has_shape", False)) and bool(cfg.get("has_shape_obs", True)),
                    term_body=cfg.get("env_term_body", "body"), head_body=self.model_tables.body_names.index("Head"), reward_mul=cfg.reward_id == "world_rfc_implicit_v1_mul",
                    w=[rw.get(k, d) for k, d in (("w_p", 0.6), ("w_v", 0.1), ("w_e", 0.2), ("w_c", 0.1), ("w_vf", 0.0))],
                    k=[rw.get(k, d) for k, d in (("k_p", 2), ("k_v", 0.005), ("k_e", 20), ("k_c", 1000), ("k_vf", 1))])

    def make_env(self, init_expert=None, mode="test"):
        """single-env facade (HumanoidEnv) for gym-style loops"""
        if init_expert is None:
            init_expert = self.data_loader.get_sample_from_key(self.data_loader.data_keys[0], full_sample=True)
        self.env = HumanoidEnv(self.cfg, init_expert, self.cfg.data_specs, mode=mode)
        return self.env

    # ---------------------------------------------------------------- checkpoints (:190-260)
    def save_checkpoint(self, epoch):
        """pickle {"policy_dict", "value_dict", "running_state": ZFilter} (agent_copycat.py:190-201).  Multi-GPU: every rank holds identical
        weights and running_state (uhc_b200/agent.py update_params), so rank 0 alone writes the file; with curriculum_global its freq_dict.pt
        is every rank's history too, otherwise rank 0's own."""
        cfg = self.cfg
        path = "%s/iter_%04d.p" % (cfg.model_dir, epoch + 1)
        if int(os.environ.get("RANK", "0")) == 0:
            with open(path, "wb") as f:
                pickle.dump(self.agent.state_dicts(), f)
            joblib.dump(self.get_freq_dict(), osp.join(cfg.result_dir, "freq_dict.pt"))
        return path

    # ---------------------------------------------------------------- single-clip fitting (scripts/fit_uhc.py; agent_copycat.py:203-236)
    def _write_cp(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.agent.state_dicts(), f)

    def save_singles(self, epoch, key):
        """{model_dir}_singles/{key}.p: policy_dict / value_dict / running_state"""
        self._write_cp(f"{self.cfg.model_dir}_singles/{key}.p")

    def save_curr(self):
        """{model_dir}/iter_best.p"""
        self._write_cp(f"{self.cfg.model_dir}/iter_best.p")

    def load_curr(self):
        path = f"{self.cfg.model_dir}/iter_best.p"
        self.logger.info("loading model from checkpoint: %s" % path)
        with open(path, "rb") as f:
            self.agent.load_state_dicts(pickle.load(f))

    def load_checkpoint(self, epoch):
        cfg = self.cfg
        path = "%s/iter_%04d.p" % (cfg.model_dir, epoch) if isinstance(epoch, int) else epoch
        self.logger.info("loading model from checkpoint: %s" % path)
        cp = pickle.load(open(path, "rb"))
        self.agent.load_state_dicts(cp)
        fd = osp.join(cfg.result_dir, "freq_dict.pt")
        if osp.exists(fd):
            self.freq_dict = joblib.load(fd)
            if self.curriculum_on_device:
                self._freq_dict_to_device(self.freq_dict)
