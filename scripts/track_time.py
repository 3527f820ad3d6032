"""Time one tracker step (target frames streamed at run time) against the same loop written with the engine's other entry points.

  tracker   Tracker.step (uhc_track_step): push of the frame, observation, ZFilter + policy mean, k_env_step, fail_safe, as one graph replay
  baseline  what the same loop costs without the stream: per step the state is read back (get_states), the frame pair (previous, next)
            of every env is loaded as a 2-frame clip table (uhc_load_motions), every env is reset onto it with its own state as the
            override (uhc_env_reset, which also writes the observation against the new target), then uhc_policy_forward (mean action)
            and uhc_env_step.  The reset re-runs the forward pass and drops the solver's warm start, so it is not even the same physics.

Both run the fp32 engine with the production 657-(2048,1024,512)-105 policy (seeded random weights) on synthetic clips
(motion_lib.synthetic_clip), fail_safe on, at --envs (default 1, 16, 256, 4096 envs).  The targets are the clips' next qpos frames, already
on the device.  Each size runs --warmup untimed steps, then --steps (tracker) / --base-steps (baseline) steps between two device
synchronises; the time per step is that wall time over the steps.  Prints the card name and power limit, then one JSON line.
Usage: python scripts/track_time.py [--envs 1,16,256,4096] [--steps 200] [--base-steps 20] [--warmup 5] [--window 8]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def gpu_info():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip()
    except Exception as e:          # noqa: BLE001 -- the timing does not depend on it
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", default="1,16,256,4096")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--base-steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--window", type=int, default=8)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("track_time.py measures the GPU: no CUDA device")
    from uhc_b200 import motion_lib as ML
    from uhc_b200 import nn
    from uhc_b200.agent import BatchedAgent
    info = gpu_info()
    print(info, flush=True)
    T = args.warmup + max(args.steps, args.base_steps) + 3
    rng = np.random.default_rng(0)
    clips = [ML.synthetic_clip(T, rng, kind=k) for k in ("normal", "sitting", "airborne", "normal")]
    out = {"gpu": info, "window": args.window, "policy": "657-(2048,1024,512)-105", "results": []}
    for E in [int(x) for x in args.envs.split(",")]:
        agent = BatchedAgent(E, clips, auto_reset=False, trail_steps=1, body_diff_thresh=0.5, seed=1)
        eng = agent.engine
        ref = torch.tensor(np.stack([clips[e % len(clips)]["qpos"] for e in range(E)]), device="cuda")        # [E][T][76]
        # ---- tracker
        trk = agent.tracker(window=args.window, kind="qpos", fail_safe=True)
        trk.reset(ref[:, 0], ref[:, 1])
        trk.step()
        k = 1
        for _ in range(args.warmup):
            trk.step(ref[:, k + 1]); k += 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            trk.step(ref[:, k + 1]); k += 1
        torch.cuda.synchronize()
        tr_ms = (time.perf_counter() - t0) / args.steps * 1e3
        assert (trk.steps() == k).all()
        trk.close()
        # ---- baseline: existing entry points, one 2-frame table per step
        pol = nn.mlp_struct(agent.policy)
        ones = torch.ones(E, dtype=torch.uint8, device="cuda")
        act = torch.empty(E, eng.act_dim, device="cuda")
        ids = np.arange(E, dtype=np.int32)

        def base_step(k):
            st = eng.get_states()
            ms = ML.MotionSet([{"qpos": np.stack([clips[e % len(clips)]["qpos"][k], clips[e % len(clips)]["qpos"][k + 1]])} for e in range(E)])
            eng.load_motions(ms)
            obs = eng.reset(ids, clip=ids, start=0, length=2, qpos=st["qpos"], qvel=st["qvel"])
            rc = eng.lib.uhc_policy_forward(eng.h, nn.C.c_void_p(obs.data_ptr()), nn.C.byref(pol), nn.C.c_void_p(agent.log_std.data_ptr()),
                                            nn.C.c_void_p(agent.running_state.stats.data_ptr()), nn.C.c_float(agent.running_state.clip), 0,
                                            nn.C.c_ulonglong(0), nn.C.c_void_p(ones.data_ptr()), None, nn.C.c_void_p(act.data_ptr()), None, eng._stream())
            assert rc == 0
            eng.step(act)

        eng.load_motions(ML.MotionSet([{"qpos": clips[e % len(clips)]["qpos"][:2]} for e in range(E)]))
        eng.reset(ids, clip=ids, start=0, length=2)
        k = 0
        for _ in range(args.warmup):
            base_step(k); k += 1
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.base_steps):
            base_step(k); k += 1
        torch.cuda.synchronize()
        base_ms = (time.perf_counter() - t0) / args.base_steps * 1e3
        r = {"envs": E, "tracker_ms_per_step": round(tr_ms, 4), "baseline_ms_per_step": round(base_ms, 3), "speedup": round(base_ms / tr_ms, 2),
             "tracker_steps": args.steps, "baseline_steps": args.base_steps}
        print(f"E={E}: tracker {tr_ms:.3f} ms/step, baseline {base_ms:.2f} ms/step ({base_ms / tr_ms:.1f}x)", flush=True)
        out["results"].append(r)
        eng.close()
        del agent
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
