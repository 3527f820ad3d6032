"""Floor-measurement timing (include/uhc_floor.h), one process, CUDA events after a warm-up:
  floor_qpos    uhc_floor_qpos over every frame of the synthetic set of scripts/motion_load_time.py (fp64 qpos rows already on the device)
  motion_floor  uhc_motion_floor over the same set's raw rows on the host (pinned chunks: copies included)
  evaluation    uhc_eval_run_ex of E clips with and without floor_host, alternating, the policy and engine of scripts/eval_time.py's size
Prints one JSON line with the card's name, power limit and clocks read in the same process.

    python scripts/floor_time.py [--frames 1000000] [--envs 4096] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
        return dict(zip(q.split(","), [x.strip() for x in out.split(",")]))
    except Exception as e:                                   # the numbers are still printed, marked as of an unknown card
        return {"name": f"unknown ({e})"}


def events_ms(torch, fn, reps, calls=1):
    """ms per call, `reps` samples of `calls` back-to-back calls each (short calls are timed several at a time), after one warm-up call"""
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ms = []
    for _ in range(reps):
        a.record()
        for _ in range(calls):
            fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b) / calls)
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1_000_000)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--clip-len", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    import torch
    from uhc_b200 import motion_lib as ML, nn
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.motion_lib import MotionSet
    rng = np.random.default_rng(0)
    base = [ML.synthetic_clip(a.clip_len, rng)["qpos"] for _ in range(32)]
    nclip = max(1, a.frames // a.clip_len)
    ms = MotionSet([{"qpos": base[c % 32]} for c in range(nclip)])
    agent = BatchedAgent(a.envs, [ML.qpos_fk(q) for q in base], policy_hsize=(2048, 1024, 512), value_hsize=(64, 32), auto_reset=False,
                         body_diff_thresh=0.2)
    eng = agent.engine
    res = dict(card=card(), frames=ms.num_frames, envs=a.envs, clip_len=a.clip_len)
    q = torch.tensor(ms.rows, device="cuda")
    first = np.zeros(ms.num_frames, np.int32)
    first[np.concatenate([[0], np.cumsum(ms.lens)[:-1]])] = 1
    first = torch.tensor(first, device="cuda")
    t = events_ms(torch, lambda: eng.floor_qpos(q, first=first), a.reps, calls=10)         # 10 calls of about 60 ms per sample
    res["floor_qpos_ms"] = [round(x, 3) for x in t]
    res["floor_qpos_Mframes_per_s"] = round(ms.num_frames / min(t) / 1e3, 2)
    t = events_ms(torch, lambda: eng.motion_floor(ms), a.reps, calls=4)
    res["motion_floor_ms"] = [round(x, 3) for x in t]
    clips = np.arange(a.envs) % 32
    ev = lambda fl: agent.evaluate(clips, True, window=32, floor=fl)
    ev(False), ev(True)                                      # both graphs captured before anything is timed
    plain, floor = [], []
    for _ in range(a.reps):                                  # alternating, so a drift of the clocks falls on both
        plain += events_ms(torch, lambda: ev(False), 1)
        floor += events_ms(torch, lambda: ev(True), 1)
    res["eval_ms"], res["eval_floor_ms"] = [round(x, 2) for x in plain], [round(x, 2) for x in floor]
    res["eval_floor_overhead_pct"] = round((np.median(floor) / np.median(plain) - 1) * 100, 2)
    print(json.dumps(res))
    eng.close()


if __name__ == "__main__":
    main()
