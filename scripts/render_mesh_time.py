"""Time the mesh renderer on one GPU, beside the hull renderer.

The mesh is synthetic with SMPL's counts (tests/mesh_scenes.py smpl_sized_model: 6890 vertices, 13 776 faces, the neutral humanoid's hull
triangles refined by longest-edge bisection); a real SMPL file is licence-gated, so numbers on it are not measured here.
  trace          per size (640x360, 1920x1080) and humanoids (1, 2): uhc_render_mesh on --frames skinned frames, and uhc_render_qpos on the same
                 qpos rows, CUDA events around --reps calls after a warm-up, as frames/s; then k_mesh_refit and k_render_mesh_trace kernel
                 times from torch.profiler in a run of their own
  render_motion  BatchedAgent.render_motion(encode="jpeg") over --clips synthetic clips (scripts/eval_time.py's clips, an engine of --envs
                 envs) at --size, body="hulls" and body="mesh", the JPEG files dropped; wall time split into evaluation, rendering, encoding,
                 copy and writer

Prints the card name and power limit, the numbers, then one JSON line.
Usage: python scripts/render_mesh_time.py [--frames 256] [--reps 5] [--envs 4096] [--clips 64] [--size 640x360]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.eval_time import make_clips, power_limit  # noqa: E402


def events(fn, reps):
    import torch
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def kernel_ms(fn, names, reps):
    """mean device ms per call of each named kernel, from torch.profiler over reps calls after a warm-up"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
    out = {k: 0.0 for k in names}
    for ev in prof.key_averages():
        for k in names:
            if k in ev.key:
                out[k] += ev.device_time_total / 1e3 / reps
    return {k: round(v, 3) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clips", type=int, default=64)
    ap.add_argument("--size", default="640x360")
    args = ap.parse_args()
    import torch
    from tests.mesh_scenes import smpl_sized_model
    from uhc_b200.agent import BatchedAgent
    clips = make_clips(args.clips)
    agent = BatchedAgent(args.envs, clips, [np.zeros(17)] * len(clips), seed=1, t_min=15, t_max=300, auto_reset=False)
    eng = agent.engine
    model = smpl_sized_model()
    eng.mesh_init(model)
    eng.render_mesh_init(model)
    name = torch.cuda.get_device_name(0)
    print(f"{name}, power limit {power_limit()}, mesh {len(model['v_template'])} vertices {len(model['faces'])} faces")
    q = np.concatenate([c["qpos"] for c in clips])
    rows = torch.tensor(q[np.arange(args.frames) % len(q)], device="cuda")
    ghost = torch.tensor(q[(np.arange(args.frames) + 7) % len(q)], device="cuda")
    betas = np.zeros((1, 10))
    verts = eng.qpos_mesh(rows, betas, joints=False)[0]
    gverts = eng.qpos_mesh(ghost, betas, joints=False)[0]
    root = rows[:, :3].float().contiguous()
    cam = dict(focus=True, shift_expert=1.0)
    out = {"trace": {}}
    for W, H in ((640, 360), (1920, 1080)):
        for nh in (1, 2):
            g, gv = (None, None) if nh == 1 else (ghost, gverts)
            ms_mesh = events(lambda: eng.render_mesh(verts, gv, root, cam, (W, H)), args.reps)
            ms_hull = events(lambda: eng.render(rows, g, camera=cam, size=(W, H)), args.reps)
            split = kernel_ms(lambda: eng.render_mesh(verts, gv, root, cam, (W, H)), ("k_mesh_refit", "k_render_mesh_trace"), args.reps)
            key = f"{W}x{H}_{nh}"
            out["trace"][key] = dict(mesh_ms=round(ms_mesh, 2), mesh_frames_per_s=round(args.frames / ms_mesh * 1e3, 1), hull_ms=round(ms_hull, 2),
                                     hull_frames_per_s=round(args.frames / ms_hull * 1e3, 1), refit_ms=split["k_mesh_refit"],
                                     mesh_trace_ms=split["k_render_mesh_trace"])
            print(f"{W}x{H}, {nh} humanoid(s), {args.frames} frames: uhc_render_mesh {ms_mesh:.1f} ms ({args.frames / ms_mesh * 1e3:.0f} frames/s; "
                  f"refit {split['k_mesh_refit']:.2f} ms, trace {split['k_render_mesh_trace']:.1f} ms), uhc_render_qpos {ms_hull:.1f} ms "
                  f"({args.frames / ms_hull * 1e3:.0f} frames/s)")
    W, H = (int(x) for x in args.size.split("x"))
    ids = np.arange(len(clips), dtype=np.int32)
    agent.export_motion(ids[:4], True)                                        # warm-up: evaluation graphs
    out["render_motion"] = {}
    for body in ("hulls", "mesh", "hulls", "mesh"):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = agent.render_motion(ids, True, (W, H), cam, encode="jpeg", writer=lambda i, chunks: [None for _ in chunks], body=body)
        wall = time.perf_counter() - t0
        frames = sum(len(r["pred"]) for r in res)
        split = {k: round(v, 3) for k, v in agent.render_times.items()}
        out["render_motion"][body] = dict(size=f"{W}x{H}", clips=len(clips), frames=frames, wall_s=round(wall, 3), **split)
        print(f"render_motion body={body} {W}x{H} jpeg: {len(clips)} clips, {frames} frames in {wall:.2f} s -- " +
              ", ".join(f"{k} {v:.2f} s" for k, v in split.items()))
    print(json.dumps(dict(gpu=name, power_limit=power_limit(), envs=args.envs, frames=args.frames, **out)))
    eng.close()


if __name__ == "__main__":
    main()
