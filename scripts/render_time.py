"""Time the renderer on one GPU.

  trace          uhc_render_qpos (pose pass + trace) on --frames qpos rows at 640x360 and 1920x1080, with one humanoid and with the ghost:
                 CUDA events around --reps calls after a warm-up, reported as frames/s
  render_motion  BatchedAgent.render_motion over --clips synthetic clips of 150-300 frames (scripts/eval_time.py's clips, engine of --envs
                 envs, the seeded 657-(2048,1024,512)-105 policy, fail_safe on) at --size, each clip written to an mp4 in a temporary
                 directory; wall time split into evaluation, rendering (to a device synchronise), device-to-host copy and mp4 encoding

Prints the card name and power limit, the numbers, then one JSON line.
Usage: python scripts/render_time.py [--frames 1024] [--reps 5] [--envs 4096] [--clips 64] [--size 640x360]
"""
import argparse
import json
import os
import sys
import tempfile
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.eval_time import make_clips, power_limit  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--size", default="640x360")
    args = ap.parse_args()
    import torch
    from uhc_b200.agent import BatchedAgent
    from uhc.utils.image_utils import write_frames_to_video
    clips = make_clips(args.clips)
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300, auto_reset=False)
    eng = agent.engine
    name = torch.cuda.get_device_name(0)
    print(f"{name}, power limit {power_limit()}")
    q = np.concatenate([c["qpos"] for c in clips])
    rows = torch.tensor(q[np.arange(args.frames) % len(q)], device="cuda")
    ghost = torch.tensor(q[(np.arange(args.frames) + 7) % len(q)], device="cuda")
    out = {"trace": {}}
    cam = dict(focus=True, shift_expert=1.0)
    for W, H in ((640, 360), (1920, 1080)):
        for g in (None, ghost):
            eng.render(rows, g, camera=cam, size=(W, H))                      # warm-up: plane upload, pose scratch, output allocation
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                rgb = eng.render(rows, g, camera=cam, size=(W, H))[0]
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            key = f"{W}x{H}_{1 if g is None else 2}"
            out["trace"][key] = dict(ms_per_call=round(ms, 2), frames_per_s=round(args.frames / ms * 1e3, 1))
            print(f"uhc_render_qpos {W}x{H}, {1 if g is None else 2} humanoid(s): {ms:.1f} ms for {args.frames} frames = "
                  f"{args.frames / ms * 1e3:.0f} frames/s (mean of {args.reps})")
            del rgb
    W, H = (int(x) for x in args.size.split("x"))
    ids = np.arange(len(clips), dtype=np.int32)
    agent.export_motion(ids[:4], True)                                        # warm-up: evaluation graphs
    with tempfile.TemporaryDirectory() as tmp:
        def writer(i, chunks):
            write_frames_to_video((f for ch in chunks for f in ch), os.path.join(tmp, f"{i}.mp4"))

        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = agent.render_motion(ids, True, (W, H), cam, writer=writer)
        wall = time.perf_counter() - t0
        files = len(os.listdir(tmp))
    frames = sum(len(r["pred"]) for r in res)
    split = {k: round(v, 3) for k, v in agent.render_times.items()}
    out["render_motion"] = dict(size=f"{W}x{H}", clips=len(clips), frames=frames, wall_s=round(wall, 3), mp4_files=files, **split)
    print(f"render_motion {W}x{H}: {len(clips)} clips, {frames} frames in {wall:.2f} s -- evaluation {split['evaluation']:.2f} s, rendering "
          f"{split['rendering']:.2f} s, device-to-host {split['copy']:.2f} s, mp4 encoding {split['writer']:.2f} s")
    print(json.dumps(dict(gpu=name, power_limit=power_limit(), envs=args.envs, frames=args.frames, **out)))
    eng.close()


if __name__ == "__main__":
    main()
