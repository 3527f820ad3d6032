"""Time the failure-weighted curriculum's per-iteration bookkeeping, host against device, on one GPU.

  host    what AgentCopycat does after every rollout by default: copy the [T][E] episode log to the host, append [percent, 0] per
          ended episode to freq_dict in a Python loop, trim every clip's list to 50, failure_weights (a Python ewma per clip), and
          uhc_set_clip_weights (a device synchronise and the CDF rebuilt on the host)
  device  uhc_curriculum_update on the stream (bucketing into the per-clip rings, ewma, weights, CDF in place), no host synchronise

The drop-in AgentCopycat's own methods run on a BatchedAgent built here (the agent's constructor would read a dataset pickle).  For each
clip count it reports each path's wall time to a device synchronise: the bookkeeping of one rollout (`_update_freq_dict` on the host;
`uhc_curriculum_update`, also from CUDA events, on the device), a whole training iteration (`AgentCopycat.sample` with its bookkeeping +
`update_params`), and the eval outcomes of one `eval_policy` over every clip (`_eval_results` + `_apply_outcomes`: the freq_dict appends; one `uhc_curriculum_push`), with 4096 envs, T = 32 and the production 657-(2048,1024,512)-105
policy with seeded weights.  The clips are synthetic qpos motion (60-200 frames, expert tables built on the GPU); short slices
(t_max = 12) make episodes end often.  Prints the card name and power limit, then one JSON line.
Usage: python scripts/curriculum_time.py [--envs 4096] [--T 32] [--clips 10,3334,11000] [--iters 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def qpos_clip(T, rng):
    t = np.arange(T) / 30.0
    q = np.zeros((T, 76))
    for _ in range(3):
        amp = rng.uniform(0.0, 0.5 / 3, 69) * (rng.uniform(size=69) < 0.6)
        q[:, 7:] += amp * np.sin(2 * np.pi * rng.uniform(0.1, 1.5, 69) * t[:, None] + rng.uniform(0, 2 * np.pi, 69))
    q[:, 2] = 0.93
    q[:, 3:7] = [0.7071068, 0.7071068, 0.0, 0.0]
    return q


class _Cfg(dict):
    __getattr__ = dict.get


def dropin_agent(ag, C, T, device_curriculum):
    """an AgentCopycat around an existing BatchedAgent (its constructor would load a dataset pickle): the real sample /
    _update_freq_dict / _push_clip_weights / update_params / eval outcome methods run on it"""
    from uhc.agents.agent_copycat import AgentCopycat
    a = object.__new__(AgentCopycat)
    a.cfg = a.cc_cfg = _Cfg(sampling_temp=0.2, sampling_freq=0.5, min_batch_size=T * ag.E, fail_safe=False)
    a.agent, a.num_envs, a.horizon, a.max_freq = ag, ag.E, T, 50
    a.data_loader = types.SimpleNamespace(data_keys=[f"clip{i}" for i in range(C)])
    a.freq_dict = {k: [] for k in a.data_loader.data_keys}
    a.curriculum_on_device = device_curriculum
    if device_curriculum:
        ag.curriculum_enable(50, 0.2, 0.5, 0.0, -1)
    return a


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--T", type=int, default=32)
    ap.add_argument("--clips", default="10,3334,11000")
    ap.add_argument("--iters", type=int, default=5)
    a = ap.parse_args()
    import torch
    from uhc_b200.agent import BatchedAgent, RolloutBuffer
    from uhc_b200.motion_lib import MotionSet
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print("GPU:", gpu)
    rng = np.random.RandomState(0)
    pool = [qpos_clip(200, rng) for _ in range(32)]
    out = dict(gpu=gpu, envs=a.envs, T=a.T, rows=[])
    for C in [int(x) for x in a.clips.split(",")]:
        lens = rng.randint(60, 201, C)
        ms = MotionSet([{"qpos": pool[i % len(pool)][:L]} for i, L in enumerate(lens)])
        keys = [f"clip{i}" for i in range(C)]
        row = dict(clips=C)
        for mode in ("host", "device"):
            ag = BatchedAgent(a.envs, ms, None, seed=1, t_min=2, t_max=12)
            dropin = dropin_agent(ag, C, a.T, mode == "device")
            it_t, book, book_ev, ends = [], [], [], 0
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            for i in range(a.iters + 2):            # whole iterations: AgentCopycat.sample (rollout + the curriculum's bookkeeping) + update_params
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                batch, _ = dropin.sample(a.T * a.envs)
                dropin.update_params(batch)
                torch.cuda.synchronize()
                if i >= 2:
                    it_t.append((time.perf_counter() - t0) * 1e3)
                    ends += int((batch.buf.ep_clip >= 0).sum())
            for i in range(a.iters):                # the bookkeeping alone, on the next rollouts' logs (each log appended once)
                buf, _ = ag.sample(a.T) if mode == "host" else (None, None)
                if mode == "device":
                    real = ag.curriculum_update
                    ag.curriculum_update = lambda b, T: None       # the rollout without its update, then the update alone
                    buf, _ = ag.sample(a.T)
                    ag.curriculum_update = real
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                if mode == "host":
                    dropin._update_freq_dict(buf)
                else:
                    e0.record()
                    ag.curriculum_update(buf, a.T)
                    e1.record()
                torch.cuda.synchronize()
                book.append((time.perf_counter() - t1) * 1e3)
                if mode == "device":
                    book_ev.append(e0.elapsed_time(e1))
            # the eval outcomes of one eval_policy over every clip: C appends to freq_dict on the host, one uhc_curriculum_push on the device
            lens_c, ids = np.asarray(ag.engine.clip_len), np.arange(C, dtype=np.int32)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            pend = []
            dropin._eval_results({}, dropin.data_loader, ids, ids, lens_c, lens_c - 1, np.zeros(C, bool), np.zeros(C), np.zeros(C, int),
                                 lambda i, pct, fs: {"succ": np.array([True])}, pend)
            dropin._apply_outcomes(pend)
            torch.cuda.synchronize()
            row[mode] = dict(bookkeeping_ms=float(np.median(book)), iteration_ms=float(np.median(it_t)), ends_per_iter=ends / a.iters,
                             eval_outcomes_ms=(time.perf_counter() - t2) * 1e3)
            if book_ev:
                row[mode]["update_event_ms"] = float(np.median(book_ev))
            ag.engine.close()
            del ag, dropin
            torch.cuda.empty_cache()
        print(f"C={C:6d}  host bookkeeping {row['host']['bookkeeping_ms']:9.2f} ms  device update {row['device']['bookkeeping_ms']:7.3f} ms "
              f"(events {row['device']['update_event_ms']:.3f} ms)  iteration host {row['host']['iteration_ms']:8.1f} ms  device {row['device']['iteration_ms']:8.1f} ms  "
              f"ends/iter {row['host']['ends_per_iter']:.0f}  eval outcomes host {row['host']['eval_outcomes_ms']:.2f} ms device {row['device']['eval_outcomes_ms']:.2f} ms")
        out["rows"].append(row)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
