"""Checkpoint sweep timing: one BatchedAgent.evaluate_policies call (K checkpoints side by side, uhc_eval_run_groups) against K sequential
load_state_dicts + evaluate calls (uhc_eval_run), on K seeded production-size checkpoints (657-(2048,1024,512)-105, fp32 engine,
fail_safe on, window 32) over n synthetic clips of 150-300 frames.  Wall time to a device synchronise, after one warm-up of each
configuration (graph capture); both sides include loading the checkpoints.  A torch.profiler run of one configuration splits a control
step's kernel time into the grouped GEMMs, k_env_step and the rest.  Prints one JSON line (and writes it to --out)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--ns", default="16,128,512")
    ap.add_argument("--ks", default="1,4,16,32")
    ap.add_argument("--profile", default="128,16", help="n,K of the torch.profiler run ('' to skip)")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    import torch
    from uhc_b200 import nn
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.motion_lib import synthetic_clip
    ns, ks = [int(x) for x in a.ns.split(",")], [int(x) for x in a.ks.split(",")]
    rng = np.random.default_rng(0)
    clips = [synthetic_clip(int(rng.integers(150, 301)), rng) for _ in range(max(ns))]
    ag = BatchedAgent(a.envs, clips, [np.zeros(17)] * len(clips), seed=1, auto_reset=False)
    cps = []
    for k in range(max(ks)):
        net = nn.MLPNet(ag.obs_dim, (2048, 1024, 512), ag.act_dim, "gelu", head_name="action_mean", seed=100 + k)
        ag.policy.load_state_dict(net.state_dict())
        r = np.random.default_rng(k)
        ag.running_state.load_sums(1e5, r.normal(0, 0.3, ag.obs_dim), r.uniform(0.1, 2.0, ag.obs_dim) * 1e5)
        cps.append(ag.state_dicts())
        del net

    def sequential(n, K):
        out = []
        for cp in cps[:K]:
            ag.load_state_dicts(cp)
            out.append(ag.evaluate(np.arange(n), True, window=32))
        torch.cuda.synchronize()
        return out

    def grouped(n, K):
        out = ag.evaluate_policies(cps[:K], np.arange(n), True, window=32)
        torch.cuda.synchronize()
        return out

    rows = []
    for n in ns:
        for K in ks:
            res = {}
            for name, fn in (("sequential", sequential), ("grouped", grouped)):
                fn(n, K)                             # warm-up: graph capture, pool allocation
                t0 = time.perf_counter()
                got = fn(n, K)
                res[name] = time.perf_counter() - t0
                res[name + "_out"] = got
            same = all(a["last_t"] == b["last_t"] and a["reward_sum"] == b["reward_sum"] and np.array_equal(a["frames"], b["frames"])
                       for x, y in zip(res["sequential_out"], res["grouped_out"]) for a, b in zip(x, y))
            steps = max(len(d["frames"]) for d in res["grouped_out"][0])
            row = dict(n=n, K=K, sequential_s=round(res["sequential"], 4), grouped_s=round(res["grouped"], 4),
                       speedup=round(res["sequential"] / res["grouped"], 2), steps=steps, identical=bool(same))
            print(json.dumps(row), flush=True)
            rows.append(row)
    prof = None
    if a.profile:
        n, K = (int(x) for x in a.profile.split(","))
        from torch.profiler import ProfilerActivity, profile
        prof = {}
        for name, fn in (("grouped", grouped), ("sequential", sequential)):
            fn(n, K)
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                out = fn(n, K)
            steps = sum(max(len(d["frames"]) for d in o) for o in out) if name == "sequential" else max(len(d["frames"]) for d in out[0])
            tot = {}
            for ev in p.key_averages():
                if ev.device_type.name == "CUDA" or getattr(ev, "self_device_time_total", 0) > 0:
                    key = "gemm" if "k_linear_tc" in ev.key else ("env_step" if "k_env_step" in ev.key else "other")
                    tot[key] = tot.get(key, 0.0) + getattr(ev, "self_device_time_total", getattr(ev, "self_cuda_time_total", 0.0))
            per = {k: round(v / 1e3 / max(steps, 1), 4) for k, v in tot.items()}   # ms per control step of the call(s)
            prof[name] = dict(n=n, K=K, control_steps=steps, ms_per_step=per)
        print(json.dumps(dict(profile=prof)), flush=True)
    result = dict(gpu=gpu_info(), envs=a.envs, rows=rows, profile=prof)
    print(json.dumps(result))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)
    ag.engine.close()


if __name__ == "__main__":
    main()
