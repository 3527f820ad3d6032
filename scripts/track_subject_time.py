"""Run-time subjects of the tracker: what giving envs new bodies costs, against rebuilding the agent with those bodies.

  python scripts/track_subject_time.py [--out results.json] [--repeats 5]

A 4096-env BatchedAgent (the production policy, synthetic SMPL models of tests/subject_ref.py) tracks a qpos stream.  For n = 1, 64 and 4096
envs, each with a new random subject:
  run_time   Tracker.set_subjects + Tracker.reset of the n envs (the bodies built on the GPU into the live tracker), then one step (a graph
             replay); host wall time up to a device synchronise, best and median of --repeats
  rebuild    the same bodies the only way there was before: SubjectBasis.build of the n subjects, a new BatchedAgent over the variants, a new
             tracker with fk_models / shapes, its reset, and its first step (which captures the step graph); best of 2
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

E, T = 4096, 40
TRACK_KW = dict(trail_steps=1, body_diff_thresh=0.2, auto_reset=False)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def subjects(n, seed):
    rng = np.random.RandomState(seed)
    b = rng.normal(0, 1.0, (n, 16))
    b[:, 0] = rng.uniform(-0.2, 0.2, n)
    return b, rng.randint(0, 3, n).astype(np.int32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="also write the JSON result to this file (default: print it only)")
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("track_subject_time.py measures the GPU: no CUDA device")
    from tests.subject_ref import gendered, uniform_scale_model
    from uhc_b200 import motion_lib as ML
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.model import HumanoidModel
    from uhc_b200.subject_body import SubjectBasis
    hm = HumanoidModel()
    n0 = uniform_scale_model()
    basis = SubjectBasis.from_models(hm, n0, gendered(n0, 1), gendered(n0, 2))
    clip = ML.synthetic_clip(T, np.random.default_rng(1))
    ref = torch.tensor(np.repeat(clip["qpos"][None], E, 0), device="cuda")          # [E][T][76]
    res = dict(card=card(), envs=E, run_time={}, rebuild={})

    agent = BatchedAgent(E, [clip], seed=1, model=hm, **TRACK_KW)
    trk = agent.tracker(window=8, kind="qpos", subjects=basis)
    trk.reset(ref[:, 0], ref[:, 1])
    trk.step()
    trk.step(ref[:, 2].contiguous())
    torch.cuda.synchronize()
    for n in (1, 64, E):
        ids = np.arange(n)
        idt = torch.as_tensor(ids, device="cuda")
        f0, f1 = ref[idt, 0].contiguous(), ref[idt, 1].contiguous()
        mask = torch.ones(E, dtype=torch.int32, device="cuda")
        mask[idt] = 0
        nxt = ref[:, 2].contiguous()
        set_reset, with_step = [], []
        for r in range(args.repeats + 1):
            b, g = subjects(n, 100 * n + r)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            trk.set_subjects(ids, b, g)
            trk.reset(f0, f1, env_ids=ids)
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            trk.step(nxt, mask)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if r:                                      # the first round sizes the staging and captures the masked step's graph
                set_reset.append(t1 - t0)
                with_step.append(t2 - t0)
        res["run_time"][str(n)] = dict(set_reset_s_best=min(set_reset), set_reset_s_median=float(np.median(set_reset)),
                                       with_step_s_best=min(with_step), with_step_s_median=float(np.median(with_step)))
    agent.engine.close()
    del trk, agent

    for n in (1, 64, E):
        ts = []
        for r in range(2):
            b, g = subjects(n, 7 * n + r)
            shapes = np.zeros((E, 17))
            shapes[:n, :16], shapes[:n, 16] = b, g
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            variants, idx = basis.build(shapes[:, :10], shapes[:, 16].astype(np.int32))
            a = BatchedAgent(E, [clip], seed=1, model=hm, variants=variants if len(variants) > 1 else None, **TRACK_KW)
            tr = a.tracker(window=8, kind="qpos", fk_models=idx, shapes=shapes)
            tr.reset(ref[:, 0], ref[:, 1])
            tr.step()
            torch.cuda.synchronize()
            ts.append(time.perf_counter() - t0)
            a.engine.close()
            del tr, a
        res["rebuild"][str(n)] = dict(s_best=min(ts), s=ts)
    res["card_after"] = card()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
