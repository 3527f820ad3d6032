"""Time exporting the simulated motion of a dataset on one GPU.

  evaluate     BatchedAgent.evaluate over every clip (uhc_eval_run, no state record, no export): the evaluation alone
  export       BatchedAgent.export_motion over the same clips (uhc_eval_run_ex with the state record and the SMPL export, chunked within
               --max-bytes of pinned host arrays): the difference to `evaluate` is the cost of the export stream and its copies
  eval_seq     one clip per device call (BatchedAgent.evaluate of one clip with the state record, what AgentCopycat.eval_seq runs) on --seq
               clips, EXTRAPOLATED per clip to the whole dataset
  qpos_to_smpl uhc_qpos_to_smpl on --frames random qpos rows (CUDA events around the kernel, after a warm-up) against scipy's Rotation calls
               of the reference's qpos_to_smpl on the host

Clips, engine and policy are those of scripts/eval_time.py (--clips synthetic clips of 150-300 frames, fp32 engine of --envs envs, the seeded
657-(2048,1024,512)-105 policy, fail_safe on).  Prints the card name and power limit, each wall time to a device synchronise, the peak host
RSS growth of the evaluate and export runs (current RSS sampled every 5 ms), then one JSON line.
Usage: python scripts/export_time.py [--envs 4096] [--clips 4096] [--window 32] [--max-bytes 1073741824] [--seq 16] [--frames 1000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.eval_time import PeakRss, make_clips, power_limit  # noqa: E402


def scipy_qpos_to_smpl(q, root_offset):
    """the reference's qpos_to_smpl (smpl_mujoco.py:738-752) on numpy rows: the root with from_quat, each hinge triple with from_euler("ZYX")"""
    from scipy.spatial.transform import Rotation as sRot
    order = [0, 1, 4, 7, 10, 2, 5, 8, 11, 3, 6, 9, 12, 15, 13, 16, 18, 20, 22, 14, 17, 19, 21, 23]
    pose = np.zeros((len(q), 24, 3))
    pose[:, 0] = sRot.from_quat(q[:, [4, 5, 6, 3]]).as_rotvec()
    for b in range(1, 24):
        pose[:, order[b]] = sRot.from_euler("ZYX", q[:, 7 + 3 * (b - 1):10 + 3 * (b - 1)]).as_rotvec()
    return pose.reshape(len(q), 72), q[:, :3] - root_offset


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=4096)
    ap.add_argument("--window", type=int, default=32)
    ap.add_argument("--max-bytes", type=int, default=1 << 30)
    ap.add_argument("--seq", type=int, default=16)
    ap.add_argument("--frames", type=int, default=1_000_000)
    args = ap.parse_args()
    import torch
    from uhc_b200.agent import BatchedAgent
    clips = make_clips(args.clips)
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300, auto_reset=False)
    name = torch.cuda.get_device_name(0)
    print(f"{name}, power limit {power_limit()}; {args.envs} envs, {len(clips)} clips of {min(len(c['qpos']) for c in clips)}-"
          f"{max(len(c['qpos']) for c in clips)} frames, fp32 engine, 657-(2048,1024,512)-105 policy, window {args.window}")
    ids = np.arange(len(clips), dtype=np.int32)
    agent.evaluate(ids[:args.envs], True, window=args.window)                       # warm-up: graphs, pinned allocations
    agent.export_motion(ids[:args.envs], True, window=args.window, max_bytes=args.max_bytes)
    out = {}
    for path in ("evaluate", "export"):
        torch.cuda.synchronize()
        with PeakRss() as rss:
            t0 = time.perf_counter()
            if path == "evaluate":
                res = agent.evaluate(ids, True, window=args.window)
            else:
                res = agent.export_motion(ids, True, window=args.window, max_bytes=args.max_bytes)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
        frames = sum(len(r["frames"]) for r in res)
        out[path] = dict(wall_s=round(wall, 3), rss_growth_mb=round(rss.growth, 1), frames=frames)
        print(f"{path:8s}: {wall:.2f} s for {frames} frames, peak RSS growth {rss.growth:.0f} MB")
        del res
    seq = ids[:args.seq]
    agent.evaluate(seq[:1], True, window=32, record_states=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c in seq:
        agent.evaluate(seq[c:c + 1], True, window=32, record_states=True)
    torch.cuda.synchronize()
    per_clip = (time.perf_counter() - t0) / len(seq)
    out["eval_seq"] = dict(s_per_clip=round(per_clip, 4), extrapolated_dataset_s=round(per_clip * len(clips), 1))
    print(f"eval_seq: {per_clip:.3f} s per clip over {len(seq)} clips; EXTRAPOLATED to {len(clips)} clips: {per_clip * len(clips):.0f} s")
    eng = agent.engine
    rng = np.random.default_rng(0)
    q = np.zeros((args.frames, 76))
    q[:, :3] = rng.normal(0, 0.5, (args.frames, 3))
    q[:, 3:7] = rng.normal(size=(args.frames, 4))
    q[:, 3:7] /= np.linalg.norm(q[:, 3:7], axis=1, keepdims=True)
    q[:, 7:] = rng.uniform(-np.pi, np.pi, (args.frames, 69))
    qd = torch.tensor(q, device="cuda")
    eng.qpos_to_smpl(qd)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        pose, trans = eng.qpos_to_smpl(qd)
    e1.record()
    torch.cuda.synchronize()
    gpu_ms = e0.elapsed_time(e1) / reps
    t0 = time.perf_counter()
    sp, st = scipy_qpos_to_smpl(q, eng.model.body_f[0, :3])
    cpu_s = time.perf_counter() - t0
    worst = float(np.abs(pose.cpu().numpy() - sp).max())
    out["qpos_to_smpl"] = dict(frames=args.frames, gpu_ms=round(gpu_ms, 3), scipy_s=round(cpu_s, 3), worst_abs_diff=worst)
    print(f"qpos_to_smpl: {args.frames} frames in {gpu_ms:.2f} ms on the GPU (mean of {reps}), {cpu_s:.2f} s with scipy on the host; "
          f"worst |pose difference| {worst:.2e}")
    print(json.dumps(dict(gpu=name, power_limit=power_limit(), envs=args.envs, clips=len(clips), window=args.window, max_bytes=args.max_bytes, **out)))


if __name__ == "__main__":
    main()
