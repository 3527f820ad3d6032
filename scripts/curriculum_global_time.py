"""Time what the global curriculum adds to a data-parallel PPO update, on one GPU.

  payload  every rank's episode log rides the first value all-reduce: world * T * E * 3 fp32 (clip, percent, start per log entry)
  update   uhc_ppo_update (the flag off) against uhc_ppo_update_ex with that payload (the flag on), W ranks of the production
           657-(2048,1024,512)-105 policy and value nets, E envs x T steps each, 10 epochs, on seeded buffers
  merge    uhc_curriculum_stage of one rank plus uhc_curriculum_update_gathered of the summed payload, on an engine of E envs and C clips

The W ranks are host threads on ONE GPU joined by the in-process all-reduce of tests/loopback_comm.py, so an update time is the wall time of
all W ranks' updates to a device synchronise, the ranks' kernels sharing the card, and the collective is a loopback copy-and-add: these are
loopback times, not NCCL times.  The all-reduce over NVLink (torchrun, several GPUs) is not measured here.  Prints the card name and power
limit, then one JSON line per world size.
Usage: python scripts/curriculum_global_time.py [--worlds 2,8] [--envs 4096] [--T 12] [--clips 3334] [--reps 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,8")
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--T", type=int, default=12)
    ap.add_argument("--clips", type=int, default=3334)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    from tests.loopback_comm import LoopbackGroup
    from uhc_b200 import nn
    from uhc_b200.agent import RolloutBuffer
    from uhc_b200.engine import Engine
    print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"], capture_output=True, text=True).stdout.strip())
    D, A, hs, T, E = 657, 105, (2048, 1024, 512), a.T, a.envs
    g = torch.Generator().manual_seed(0)

    # merge: stage + gathered update on one engine (the payload of W ranks, W - 1 of them zero slots: the kernels' work does not depend on it)
    z = np.load(os.path.join(ROOT, "tests", "golden", "expert_sway.npz"))
    ex = {k: z[k] for k in z.files}
    so = np.concatenate([ex["beta"][0], [ex["gender"][0]]])
    eng = Engine(E, auto_reset=1, t_min=2, t_max=12)
    n0 = len(ex["qpos"])
    short = {k: (np.asarray(v)[np.arange(30) % n0] if np.ndim(v) > 0 and len(v) == n0 else v) for k, v in ex.items()}   # 30-frame clips
    eng.load_clips([short] * a.clips, [so] * a.clips)
    eng.curriculum_enable(50, 0.2, 0.5, 0.0, -1)
    buf = RolloutBuffer(T, E, torch.device("cuda"), 105, D)
    buf.ep_clip.copy_(torch.where(torch.rand(T, E, generator=g) < 0.3, torch.randint(0, a.clips, (T, E), generator=g), torch.full((T, E), -1)).int())
    buf.ep_pct.copy_(torch.rand(T, E, generator=g))
    buf.ep_start.copy_(torch.randint(0, 20, (T, E), generator=g).int())

    for W in (int(w) for w in a.worlds.split(",")):
        n = W * T * E * 3
        slots = torch.empty(n, device="cuda")
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for i in range(a.reps + 1):
            if i == 1:
                e0.record()
            eng.curriculum_stage(buf, T, 0, W, slots)
            eng.curriculum_update_gathered(slots, T, W)
        e1.record()
        torch.cuda.synchronize()
        merge_ms = e0.elapsed_time(e1) / a.reps

        group = LoopbackGroup(W, timeout=600.0)
        reps, trs = [], []
        for r in range(W):
            pol = nn.MLPNet(D, hs, A, "gelu", device="cuda", head_name="action_mean", seed=41)
            val = nn.MLPNet(D, hs, 1, "gelu", device="cuda", head_name="value_head", seed=42)
            val.ensure_grad_tail(nn.stats_tail_floats(D) + n)
            reps.append((pol, val, nn.Adam(pol.params(), 5e-5, net=pol), nn.Adam(val.params(), 3e-4, net=val)))
            trs.append(nn.CPpoTrainer(*reps[-1], T * E, E, torch.device("cuda"), all_reduce=group.fn))
        data = []
        for r in range(W):
            data.append(dict(states=torch.randn(T * E, D, generator=g).clamp(-5, 5).cuda(), last=torch.randn(E, D, generator=g).clamp(-5, 5).cuda(),
                             actions=(0.1 * torch.randn(T * E, A, generator=g)).cuda(), rewards=torch.rand(T, E, generator=g).cuda(),
                             masks=(torch.rand(T, E, generator=g) > 0.05).float().cuda(), exps=torch.ones(T * E, device="cuda"),
                             zf=torch.zeros(1 + 2 * D, device="cuda", dtype=torch.float64), zs=torch.zeros(1 + 2 * D, device="cuda", dtype=torch.float64),
                             losses=torch.zeros(2, device="cuda"), xin=torch.zeros(n, device="cuda"), xout=torch.zeros(n, device="cuda")))
        log_std = torch.full((A,), -2.3, device="cuda")

        def update(flag):
            def rank(r):
                d = data[r]
                trs[r].update(d["states"], d["last"], d["actions"], d["rewards"], d["masks"], d["exps"], log_std, T, E, 0.95, 0.95, 0.2, 10, 40.0, d["losses"],
                              zfilter=d["zf"], z_sync=d["zs"], comm=group.comm(r), world=W, extra_in=d["xin"] if flag else None, extra_out=d["xout"] if flag else None)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            group.run(rank)
            torch.cuda.synchronize()
            return time.perf_counter() - t0

        times = {False: [], True: []}
        update(False); update(True)                      # warm-up of both shapes
        for _ in range(a.reps):                          # alternated, so drift on a shared host hits both alike
            for flag in (False, True):
                times[flag].append(update(flag))
        for t in trs:
            t.close()
        del reps, trs, data
        torch.cuda.empty_cache()
        print(json.dumps(dict(world=W, T=T, envs_per_rank=E, clips=a.clips, payload_floats=n, payload_bytes=4 * n,
                              value_gradient_bytes=4 * nn.MLPNet.flat_layout([D, *hs, 1])[1],
                              update_s_loopback_flag_off=float(np.median(times[False])), update_s_loopback_flag_on=float(np.median(times[True])),
                              stage_plus_merge_ms=merge_ms, nccl_all_reduce="not measured (one GPU)")), flush=True)
    eng.close()


if __name__ == "__main__":
    main()
