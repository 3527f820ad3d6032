"""SMPL mesh timing (include/uhc_mesh.h), one process, after a warm-up:
  smpl_floor     uhc_smpl_floor over --frames rows (pose / trans already on the device), CUDA events
  smpl_mesh      uhc_smpl_mesh with the vertex output over --mesh-frames rows, CUDA events
  evaluation     BatchedAgent.evaluate of --clips synthetic clips of 150-300 frames with the state record, alone and followed by the mesh pass
                 of full_eval (qpos -> SMPL -> floor rows of every simulated row and its paired expert row), alternating; host clock around
                 work that ends in a synchronise
  host           the fp64 numpy restatement (tests/smpl_ref.py) on --host-frames rows: a host figure, not smplx's
The model is --smpl PATH (load_smpl_model), else a synthetic one of SMPL's size (6890 vertices, at most 4 joints per vertex).  Prints one
JSON line with the card's name, power limit and clocks read in the same process.

    python scripts/mesh_time.py [--smpl data/smpl] [--frames 1048576] [--mesh-frames 65536] [--clips 4096] [--reps 5]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))


def synthetic_model(V=6890, seed=0):
    rng = np.random.default_rng(seed)
    parents = np.array([-1, 0, 0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 9, 9, 12, 13, 14, 16, 17, 18, 19, 20, 21], np.int32)
    w = np.zeros((V, 24))
    for v in range(V):
        k = rng.choice(24, 4, replace=False)
        w[v, k] = rng.dirichlet(np.ones(4))
    return dict(v_template=rng.normal(0, 0.3, (V, 3)), shapedirs=rng.normal(0, 0.01, (V, 3, 10)), posedirs=rng.normal(0, 0.005, (V, 3, 207)),
                J_regressor=rng.dirichlet(np.ones(V), 24), weights=w, parents=parents)


def main():
    from floor_time import card, events_ms
    ap = argparse.ArgumentParser()
    ap.add_argument("--smpl", default=None)
    ap.add_argument("--frames", type=int, default=1 << 20)
    ap.add_argument("--mesh-frames", type=int, default=65536)
    ap.add_argument("--clips", type=int, default=4096)
    ap.add_argument("--host-frames", type=int, default=64)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from tests.smpl_ref import smpl_forward
    from uhc_b200 import motion_lib as ML
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.smpl_model import load_smpl_model
    model = load_smpl_model(a.smpl) if a.smpl else synthetic_model()
    rng = np.random.default_rng(1)
    lens = rng.integers(150, 301, 32)
    base = [ML.synthetic_clip(int(n), rng)["qpos"] for n in lens]
    agent = BatchedAgent(a.clips, [ML.qpos_fk(q) for q in base], policy_hsize=(2048, 1024, 512), value_hsize=(64, 32), auto_reset=False,
                         body_diff_thresh=0.2)
    eng = agent.engine
    eng.mesh_init(model)
    V = len(model["v_template"])
    res = dict(card=card(), model=a.smpl or "synthetic", nvert=V)
    # rows from the clips' qpos, as the evaluation's mesh pass sees them
    allq = np.concatenate(base)
    pose, trans = eng.qpos_to_smpl(allq[np.arange(a.frames) % len(allq)])
    betas = torch.tensor(rng.uniform(-2, 2, (1, 10)), device="cuda")
    t = events_ms(torch, lambda: eng.smpl_floor(pose, trans, betas), a.reps)
    res["smpl_floor_frames"], res["smpl_floor_ms"] = a.frames, [round(x, 2) for x in t]
    res["smpl_floor_Mframes_per_s"] = round(a.frames / min(t) / 1e3, 3)
    p2, t2 = pose[:a.mesh_frames].contiguous(), trans[:a.mesh_frames].contiguous()
    out = torch.empty(a.mesh_frames, V, 3, dtype=torch.float32, device="cuda")
    ptr = lambda x: C.c_void_p(x.data_ptr())
    t = events_ms(torch, lambda: eng.lib.uhc_smpl_mesh(eng.h, C.c_long(a.mesh_frames), ptr(p2), ptr(t2), 1, ptr(betas), None, ptr(out), None, None),
                  a.reps)                                     # into one preallocated output: the kernels, not the allocator
    res["smpl_mesh_frames"], res["smpl_mesh_ms"] = a.mesh_frames, [round(x, 2) for x in t]
    res["smpl_mesh_Mframes_per_s"] = round(a.mesh_frames / min(t) / 1e3, 3)
    flop = 2 * 207 * 3 * V                                     # the pose-blend contraction per frame; skinning and the chain come on top
    res["pose_blend_TFLOP_per_s_floor"] = round(flop * a.frames / (min(res["smpl_floor_ms"]) * 1e-3) / 1e12, 2)
    del out
    # the evaluation alone, then with full_eval's mesh pass
    clips = (np.arange(a.clips) % 32).astype(np.int32)
    gtq = [eng.clip_frames(c)["qpos"] for c in range(32)]

    def evaluate(mesh):
        t0 = time.perf_counter()
        dev = agent.evaluate(clips, True, window=32, record_states=True)
        rows = 0
        if mesh:
            q, first = [], []
            for i, d in enumerate(dev):
                tt = np.minimum(np.arange(1, len(d["frames"]) + 1), len(gtq[clips[i]]) - 1)
                for x in (d["states"][:, :76], gtq[clips[i]][tt]):
                    q.append(x); first += [1] + [0] * (len(x) - 1)
            q = np.concatenate(q)
            rows = len(q)
            eng.qpos_mesh(q, betas, floor=True, first=np.array(first, np.int32)).cpu()
        torch.cuda.synchronize()
        return time.perf_counter() - t0, rows
    evaluate(False), evaluate(True)
    plain, mesh = [], []
    for _ in range(a.reps):
        plain.append(evaluate(False)[0])
        s, rows = evaluate(True)
        mesh.append(s)
    res["eval_clips"], res["eval_mesh_rows"] = a.clips, rows
    res["eval_s"], res["eval_with_mesh_s"] = [round(x, 3) for x in plain], [round(x, 3) for x in mesh]
    res["mesh_pass_s_median"] = round(float(np.median(mesh) - np.median(plain)), 3)
    # the host restatement, on a sample
    hp, ht = pose[:a.host_frames].cpu().numpy(), trans[:a.host_frames].cpu().numpy()
    t0 = time.perf_counter()
    smpl_forward(model, hp, ht, np.repeat(betas.cpu().numpy(), a.host_frames, 0))
    res["host_numpy_fp64_frames_per_s"] = round(a.host_frames / (time.perf_counter() - t0), 1)
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
