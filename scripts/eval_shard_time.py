"""The evaluation sharded over W ranks (uhc_b200.agent.assign_clips): its env-step counts, and its shards timed one at a time on one GPU.

  counts   for W = 1, 2, 4, 8: the env-steps of each rank's device calls (call_env_steps: n clips x (max(len) - 1) per call), their sum over
           the ranks beside the W = 1 count, and the balance bound every rank stays within (the sum / W plus the largest call)
  timing   on this one GPU: the wall time of the W = 1 evaluation, and of each rank's shard evaluated alone (BatchedAgent.evaluate of its calls,
           to a device synchronise).  The largest shard time is the projected evaluation wall time at W GPUs; a W-GPU run itself is not
           measured here.  Every shard's per-clip results are checked equal to the W = 1 results.

The clips are synthetic (motion_lib.synthetic_clip) in bench.py's multi-GPU clip mix: normal / sitting / airborne = 13 / 8 / 3, 60-299
frames.  The engine is fp32 with --envs envs, the policy the production 657-(2048,1024,512)-105 net with seeded random weights, fail_safe on.
Prints the card name and power limit beside the times, then one JSON line.
Usage: python scripts/eval_shard_time.py [--envs 4096] [--clips 4096] [--window 32]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORLDS = (1, 2, 4, 8)


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def make_clips(n, seed=7):
    from uhc_b200 import motion_lib
    rng = np.random.default_rng(seed)
    kinds = ["normal"] * 13 + ["sitting"] * 8 + ["airborne"] * 3
    return [motion_lib.synthetic_clip(int(rng.integers(60, 300)), rng, kind=kinds[i % len(kinds)]) for i in range(n)]


def counts(lens, E):
    from uhc_b200.agent import assign_clips, call_env_steps
    out = {}
    for W in WORLDS:
        calls = assign_clips(lens, W, E)
        per_rank = [sum(call_env_steps(lens[c]) for c in rank) for rank in calls]
        largest = max(call_env_steps(lens[c]) for rank in calls for c in rank)
        bound = sum(per_rank) / W + largest
        assert max(per_rank) <= bound, (W, per_rank, bound)
        out[W] = dict(per_rank=per_rank, sum=sum(per_rank), bound=bound, calls=[len(r) for r in calls])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=4096)
    ap.add_argument("--window", type=int, default=32)
    args = ap.parse_args()
    clips = make_clips(args.clips)
    lens = np.array([len(c["qpos"]) for c in clips], np.int64)
    steps = counts(lens, args.envs)
    one = steps[1]["sum"]
    print(f"{len(clips)} clips of {lens.min()}-{lens.max()} frames, {args.envs} envs per rank; env-steps of each rank's calls:")
    for W, s in steps.items():
        print(f"  W={W}: per rank {s['per_rank']} (calls {s['calls']}), max {max(s['per_rank'])} <= bound {s['bound']:.0f}; "
              f"sum over ranks {s['sum']} vs W=1 {one} ({s['sum'] / one:.4f}x)")

    import torch
    from uhc_b200.agent import assign_clips
    from uhc_b200.agent import BatchedAgent
    if not torch.cuda.is_available():
        raise SystemExit("eval_shard_time: the timing needs a CUDA device")
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300)
    agent.engine.set_cfg(auto_reset=0)                    # the evaluation's test-mode cfg, as eval_policy sets it
    name, plim = torch.cuda.get_device_name(0), power_limit()
    print(f"{name}, power limit {plim}")

    def run(calls):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = [d for c in calls for d in agent.evaluate(c, True, window=args.window)]
        torch.cuda.synchronize()
        return time.perf_counter() - t0, out

    run(assign_clips(lens, 1, args.envs)[0])              # warm-up: graph capture, module loads
    times = {}
    for W in WORLDS:
        per = []
        for rank, calls in enumerate(assign_clips(lens, W, args.envs)):
            t, out = run(calls)
            per.append(t)
            if W == 1:
                ref = out
            else:                                         # a clip's result does not depend on the rank or call it runs in
                for c, d in zip(np.concatenate(calls), out):
                    r = ref[c]
                    assert d["last_t"] == r["last_t"] and d["fail_any"] == r["fail_any"] and d["reward_sum"] == r["reward_sum"] \
                        and np.array_equal(d["frames"], r["frames"]), (W, rank, int(c))
        times[W] = per
        print(f"  W={W}: shard wall times {[round(t, 3) for t in per]} s; largest {max(per):.3f} s = projected evaluation wall time at {W} GPUs "
              f"(W=1 {times[1][0]:.3f} s; multi-GPU wall time not measured)")
    print(json.dumps({"gpu": name, "power_limit": plim, "envs": args.envs, "clips": len(clips), "w1_env_steps": one,
                      "env_steps": {W: s["per_rank"] for W, s in steps.items()}, "env_steps_sum": {W: s["sum"] for W, s in steps.items()},
                      "bound": {W: round(s["bound"], 1) for W, s in steps.items()},
                      "shard_wall_s": {W: [round(t, 4) for t in per] for W, per in times.items()},
                      "projected_wall_s": {W: round(max(per), 4) for W, per in times.items()}, "multi_gpu_wall": "not measured"}))


if __name__ == "__main__":
    main()
