"""Subject bodies on the GPU: builder throughput and what per-clip bodies cost the rollout.

  python scripts/subject_time.py [--out results.json] [--steps 40] [--rounds 3]

1. uhc_subject_bodies (SubjectBasis.bodies) in subjects/s at 1 000 and 16 384 rows, and the numpy restatement (tests/subject_ref.py) on the
   host for comparison.  Synthetic SMPL models (the neutral humanoid's hulls as a mesh, three genders), random beta.
2. Rollout env-steps/s at 4096 envs with the production policy (2048, 1024, 512): 4096 clips of one motion, every clip on variant 0, against
   the same clips each on its own subject (4097 variants).  Same clips and seed; the two agents' timed windows alternate in one process.
The card's name and power limit are read in the same run and written beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def models():
    from tests.subject_ref import gendered, uniform_scale_model
    n = uniform_scale_model()
    n["shapedirs"][:, :, 0] *= 0.05
    return n, gendered(n, 1), gendered(n, 2)


def subjects(n, seed):
    rng = np.random.RandomState(seed)
    return rng.normal(0, 1.0, (n, 10)), rng.randint(0, 3, n).astype(np.int32)


def builder(basis, ms, hm):
    import torch
    from tests.subject_ref import subject_body
    out = {}
    for n in (1000, 16384):
        b, g = subjects(n, n)
        basis.bodies(b[:8], g[:8])                             # module load, first launch
        ts = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            basis.bodies(b, g)                                 # synchronous: the outputs are on the host when it returns
            ts.append(time.perf_counter() - t0)
        out[f"gpu_rows_per_s_{n}"] = n / min(ts)
        out[f"gpu_s_{n}"] = sorted(ts)
    b, g = subjects(40, 7)
    t0 = time.perf_counter()
    for r in range(len(g)):
        subject_body(hm, ms[0], ms[g[r]], b[r])
    out["host_numpy_rows_per_s"] = len(g) / (time.perf_counter() - t0)
    return out


def rollout(basis, hm, steps, rounds):
    import torch
    from bench import make_clip
    from uhc_b200.agent import BatchedAgent, RolloutBuffer
    E = 4096
    ex, shape = make_clip()
    clips, shapes = [ex] * E, [shape] * E
    b, g = subjects(E, 11)
    variants, idx = basis.build(b, g)
    assert len(variants) == E + 1
    arms = {"variant0": BatchedAgent(E, clips, shapes, seed=1, model=hm, variants=variants, clip_models=np.zeros(E, np.int32)),
            "per_clip_subject": BatchedAgent(E, clips, shapes, seed=1, model=hm, variants=variants, clip_models=idx)}
    bufs = {}
    for k, a in arms.items():
        a.reset_envs()
        bufs[k] = RolloutBuffer(1, E, a.dev, a.act_dim, a.obs_dim)
        for _ in range(5):
            a.rollout(bufs[k], 1, 0)
    torch.cuda.synchronize()
    rates = {k: [] for k in arms}
    for _ in range(rounds):
        for k, a in arms.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                a.rollout(bufs[k], 1, 0)
            e1.record()
            torch.cuda.synchronize()
            rates[k].append(E * steps / (e0.elapsed_time(e1) * 1e-3))
    used = len(np.unique(idx))
    for a in arms.values():
        a.engine.close()
    return dict(envs=E, steps_per_window=steps, rounds=rounds, env_steps_per_s={k: v for k, v in rates.items()},
                median={k: float(np.median(v)) for k, v in rates.items()}, distinct_variants=int(used))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file (default: print it only)")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("subject_time.py measures the GPU: no CUDA device")
    from uhc_b200.model import HumanoidModel
    from uhc_b200.subject_body import SubjectBasis
    hm = HumanoidModel()
    ms = models()
    basis = SubjectBasis.from_models(hm, *ms)
    res = dict(card=card(), builder=builder(basis, ms, hm), rollout=rollout(basis, hm, args.steps, args.rounds), card_after=card())
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
