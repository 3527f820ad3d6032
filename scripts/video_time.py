"""Time the JPEG encoder on one GPU.

  encode         Engine.encode_jpeg of --frames rendered frames (scripts/eval_time.py's clips beside their ghost, focus on) at 640x360 and
                 1920x1080, q = 90: CUDA events around --reps calls after a warm-up, reported as frames/s, with the mean bytes per frame
  render_motion  BatchedAgent.render_motion over --clips synthetic clips of 150-300 frames (scripts/render_time.py's setup) at --size with the
                 ghost, one file per clip in a temporary directory: mp4 through write_frames_to_video, and mjpeg (encode="jpeg" into
                 write_mjpeg_avi), alternating mjpeg, mp4, mjpeg; the render_times split of each run

Prints the card name and power limit, the numbers, then one JSON line.
Usage: python scripts/video_time.py [--frames 512] [--reps 5] [--envs 4096] [--clips 64] [--size 640x360]
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
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--size", default="640x360")
    args = ap.parse_args()
    import torch
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.video import write_mjpeg_avi
    from uhc.utils.image_utils import write_frames_to_video
    clips = make_clips(args.clips)
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300, auto_reset=False)
    eng = agent.engine
    name = torch.cuda.get_device_name(0)
    print(f"{name}, power limit {power_limit()}")
    q = np.concatenate([c["qpos"] for c in clips])
    rows = torch.tensor(q[np.arange(args.frames) % len(q)], device="cuda")
    ghost = torch.tensor(q[(np.arange(args.frames) + 7) % len(q)], device="cuda")
    cam = dict(focus=True, shift_expert=1.0)
    out = {"encode": {}}
    for W, H in ((640, 360), (1920, 1080)):
        rgb = eng.render(rows, ghost, camera=cam, size=(W, H))[0]
        data, offs = eng.encode_jpeg(rgb, 90)                                   # warm-up: scratch and the size hint
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            data, offs = eng.encode_jpeg(rgb, 90)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        bpf = data.numel() / args.frames
        out["encode"][f"{W}x{H}"] = dict(ms_per_call=round(ms, 2), frames_per_s=round(args.frames / ms * 1e3, 1), bytes_per_frame=round(bpf))
        print(f"encode_jpeg {W}x{H} q=90: {ms:.1f} ms for {args.frames} frames = {args.frames / ms * 1e3:.0f} frames/s (mean of {args.reps}), "
              f"{bpf / 1e3:.1f} KB per frame, rgb {W * H * 3 / 1e3:.0f} KB")
        del rgb, data, offs
    W, H = (int(x) for x in args.size.split("x"))
    ids = np.arange(len(clips), dtype=np.int32)
    agent.export_motion(ids[:4], True)                                          # warm-up: evaluation graphs
    out["render_motion"] = []
    for video in ("mjpeg", "mp4", "mjpeg"):
        with tempfile.TemporaryDirectory() as tmp:
            def writer(i, chunks):
                if video == "mp4":
                    write_frames_to_video((f for ch in chunks for f in ch), os.path.join(tmp, f"{i}.mp4"))
                else:
                    write_mjpeg_avi(os.path.join(tmp, f"{i}.avi"), (f for ch in chunks for f in ch), W, H)

            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = agent.render_motion(ids, True, (W, H), cam, writer=writer, encode="jpeg" if video == "mjpeg" else None)
            wall = time.perf_counter() - t0
            files = len(os.listdir(tmp))
            size = sum(os.path.getsize(os.path.join(tmp, f)) for f in os.listdir(tmp))
        frames = sum(len(r["pred"]) for r in res)
        split = {k: round(v, 3) for k, v in agent.render_times.items()}
        out["render_motion"].append(dict(video=video, size=f"{W}x{H}", clips=len(clips), frames=frames, wall_s=round(wall, 3), files=files,
                                         file_bytes=size, **split))
        print(f"render_motion {video} {W}x{H}: {len(clips)} clips, {frames} frames in {wall:.2f} s -- " + ", ".join(f"{k} {v:.2f} s" for k, v in split.items())
              + f"; {size / 1e6:.1f} MB of files")
    print(json.dumps(dict(gpu=name, power_limit=power_limit(), envs=args.envs, frames=args.frames, **out)))
    eng.close()


if __name__ == "__main__":
    main()
