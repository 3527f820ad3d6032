"""Time evaluating a motion dataset, host loop against device path, on one GPU.

  host    AgentCopycat.eval_policy's default loop: per control step policy + env step launched from Python, a state read of every live
          env, per-clip lists on the host, then uhc_b200/metrics.py per clip
  device  the same eval_policy with eval_on_device: true (BatchedAgent.evaluate -> uhc_eval_run: CUDA-graph replays, metrics on the GPU)

Both run the same fp32 engine of --envs envs, the production 657-(2048,1024,512)-105 policy with seeded random weights, and --clips
synthetic clips (motion_lib.synthetic_clip in bench.py's occlusion class mix, normal / sitting / airborne = 13 / 8 / 3, 150-300 frames),
with fail_safe on.  Prints the card name and power limit, each path's wall time to a device synchronise, its time per env-step, its peak
host RSS growth (current RSS sampled every 5 ms during the path, peak minus the value at its start), the worst per-frame metric
difference between the two paths, and, from one more device run under torch.profiler, the device time of each kernel of the
evaluation step (k_env_step, k_eval_frame, k_eval_reseat, the policy GEMMs); then one JSON line.
Usage: python scripts/eval_time.py [--envs 4096] [--clips 4096] [--window 32]
"""
import argparse
import json
import logging
import os
import resource
import subprocess
import sys
import tempfile
import threading
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class _Cfg(dict):
    __getattr__ = dict.get


def rss_mb():
    """current resident set size (not the lifetime peak ru_maxrss keeps)"""
    with open("/proc/self/statm") as f:
        return int(f.read().split()[1]) * resource.getpagesize() / 2 ** 20


class PeakRss:
    """peak of the current RSS while the block runs, sampled by a thread"""

    def __enter__(self):
        self.start = self.peak = rss_mb()
        self._stop = threading.Event()
        self._t = threading.Thread(target=self._run, daemon=True)
        self._t.start()
        return self

    def _run(self):
        while not self._stop.wait(0.005):
            self.peak = max(self.peak, rss_mb())

    def __exit__(self, *exc):
        self._stop.set()
        self._t.join()
        self.peak = max(self.peak, rss_mb())
        self.growth = self.peak - self.start


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_clips(n, seed=7):
    from uhc_b200 import motion_lib
    rng = np.random.default_rng(seed)
    kinds = (["normal"] * 13 + ["sitting"] * 8 + ["airborne"] * 3)
    return [motion_lib.synthetic_clip(int(rng.integers(150, 301)), rng, kind=kinds[i % len(kinds)]) for i in range(n)]


def copycat(agent, loader, out_dir, on_device, window):
    """an AgentCopycat around an existing BatchedAgent: eval_policy's code paths without a config file or a dataset pickle"""
    from uhc.agents.agent_copycat import AgentCopycat
    a = object.__new__(AgentCopycat)
    a.cfg = _Cfg(fail_safe=True, eval_on_device=on_device, output_dir=out_dir)
    a.agent, a.num_envs, a.running_state, a.policy_net = agent, agent.E, agent.running_state, agent.policy
    a.data_loader, a.test_data_loaders, a.freq_dict, a.max_freq = loader, [loader], {k: [] for k in loader.data_keys}, 50
    a.curriculum_on_device = False
    a.logger = logging.getLogger("eval_time")
    a._env_cfg = lambda test: dict(auto_reset=0 if test else 1)
    a._push_clip_weights = lambda: None
    if on_device:
        ev = agent.evaluate
        agent.evaluate = lambda clips, fail_safe, **kw: ev(clips, fail_safe, window=window)
    return a


def profile_device(agent, loader, out_dir, window):
    """device time per kernel name (ms, launches) of one device-path evaluation under torch.profiler (CUPTI records graph-launched kernels)"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    a = copycat(agent, loader, out_dir, True, window)
    os.makedirs(out_dir)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        a.eval_policy(epoch=0, dump=False)
        torch.cuda.synchronize()
    names = {"k_env_step": "k_env_step", "k_eval_frame": "k_eval_frame", "k_eval_reseat": "k_eval_reseat", "k_linear_tc": "policy GEMMs",
             "k_zfilter_apply_bf16": "k_zfilter_apply_bf16", "k_gauss_sample_dev": "k_gauss_sample_dev", "k_env_reset": "k_env_reset"}
    out = {}
    for ev in prof.key_averages():
        for key, label in names.items():
            if key in ev.key:
                ms, cnt = out.get(label, (0.0, 0))
                dev_us = getattr(ev, "device_time_total", None)
                if dev_us is None:
                    dev_us = getattr(ev, "cuda_time_total", 0.0)
                out[label] = (ms + dev_us / 1e3, cnt + ev.count)
                break
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=4096)
    ap.add_argument("--window", type=int, default=32)
    args = ap.parse_args()
    import joblib
    import torch
    from uhc_b200.agent import BatchedAgent
    clips = make_clips(args.clips)
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300)
    loader = types.SimpleNamespace(name="synthetic", data_keys=[f"clip_{i}" for i in range(len(clips))], experts=clips, get_len=lambda: len(clips))
    name = torch.cuda.get_device_name(0)
    print(f"{name}, power limit {power_limit()}; {args.envs} envs, {len(clips)} clips of {min(len(c['qpos']) for c in clips)}-"
          f"{max(len(c['qpos']) for c in clips)} frames, fp32 engine, 657-(2048,1024,512)-105 policy, window {args.window}")
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for path in ("device", "host"):      # device first: the host path's peak RSS is the larger one
            a = copycat(agent, loader, os.path.join(tmp, path), path == "device", args.window)
            os.makedirs(a.cfg.output_dir)
            torch.cuda.synchronize()
            with PeakRss() as rss:
                t0 = time.perf_counter()
                a.eval_policy(epoch=0, dump=True)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
            res = joblib.load(os.path.join(a.cfg.output_dir, "0_synthetic_coverage_full.pkl"))
            out[path] = dict(wall_s=wall, rss_growth_mb=rss.growth, res=res)
        kernels = profile_device(agent, loader, os.path.join(tmp, "profiled"), args.window)
    env_steps = sum(len(c["qpos"]) - 1 for c in clips)
    worst = 0.0
    for k, m in out["host"]["res"].items():
        for key in ("root_dist", "mpjpe_g", "mpjpe", "pa_mpjpe", "vel_dist", "accel_dist"):
            if key in m:
                a, b = np.asarray(m[key]), np.asarray(out["device"]["res"][k][key])
                assert a.shape == b.shape, (k, key)
                worst = max(worst, float((np.abs(a - b) / np.maximum(np.abs(a), 1.0)).max()) if a.size else 0.0)
    summary = {"gpu": name, "power_limit": power_limit(), "envs": args.envs, "clips": len(clips), "env_steps": env_steps, "window": args.window,
               "worst_metric_rel_diff": worst}
    for path in ("host", "device"):
        o = out[path]
        summary[f"{path}_wall_s"] = round(o["wall_s"], 3)
        summary[f"{path}_us_per_env_step"] = round(1e6 * o["wall_s"] / env_steps, 3)
        summary[f"{path}_rss_growth_mb"] = round(o["rss_growth_mb"], 1)
        print(f"{path:6s}: {o['wall_s']:.2f} s to a device synchronise, {1e6 * o['wall_s'] / env_steps:.2f} us per env-step, peak RSS growth {o['rss_growth_mb']:.0f} MB")
    print(f"worst per-frame metric difference, device vs host: {worst:.2e} (relative, mm floor 1)")
    nsteps = max(kernels.get("k_env_step", (0, 0))[1], 1)
    for k, (ms, cnt) in sorted(kernels.items(), key=lambda kv: -kv[1][0]):
        print(f"  {k:22s} {ms:9.1f} ms in {cnt:6d} launches, {1e3 * ms / nsteps:8.1f} us per step")
    if not kernels:
        print("  (torch.profiler recorded no kernels of the graph replays: per-kernel times not measured)")
    summary["device_kernel_us_per_step"] = {k: round(1e3 * ms / nsteps, 2) for k, (ms, cnt) in kernels.items()}
    print(json.dumps(summary))


if __name__ == "__main__":
    main()
