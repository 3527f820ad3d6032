#!/usr/bin/env python
"""step_phase_cycles.py -- where k_env_step<float> spends its cycles, phase by phase, and whether each phase is latency- or issue-bound.

  python scripts/step_phase_cycles.py --out DIR [--steps 20] [--warmup 3] [--build-dir DIR] [--table-only]

Builds two variants of the library beside the production one (uhc_b200.build: -DUHC_PHASE_CLOCKS, and -DUHC_PHASE_CLOCKS -DUHC_NO_CTA_SYNC)
into --build-dir (default: a temporary directory; reused when up to date), then runs each library in a child process (the engine loads the
library UHC_B200_SO names) on the bench's rollout: the bench's clip, agent and seed, one uhc_rollout graph launch per control step.

  table   4096 envs (two waves of 132 x 16 warps): the cycles every warp spends in each phase of a control step (sim_core.h, PC_*),
          read with clock64() by the instrumented kernel, averaged over the warps and the timed steps; kin_rne and collide are also split
          into their sub-phases (PS_*)
  probe   132 x 16 envs (one CTA on every SM), only the envs with slot % 16 < k reset, k = 4, 8, 12, 16.  A warp whose env was never reset
          has an invalid record: it leaves the kernel at once and is not counted in the substep barrier, so k warps of each 16-warp CTA
          (k / 4 per SM sub-partition) do the work.  A phase whose per-warp cycles stay flat as k grows is bound by dependent latency;
          one whose cycles grow in proportion to k is bound by instruction issue or a shared pipe.
  nosync  the table and the k = 16 probe again with the substep alignment barriers compiled out
  production  the table's workload on the production library: kernel time only (it has no clocks)
  groups  the table's workload on production builds with other substep alignment: one 16-warp group per CTA (-DUHC_SYNC_GROUP=16) and no
          barriers (-DUHC_NO_CTA_SYNC), kernel time only, against the production library's two 8-warp groups

--table-only runs the table and the production library's kernel time only.
Writes DIR/step_phase_cycles.json and prints the phase table.  The card's name, power limit and SM clock are read in the same call.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
EPB, NSM, NSUB = 16, 132, 15
PHASES = ["load", "pd", "kin_rne", "collide", "smooth", "constraint_setup", "newton_aba", "newton_rows", "sync_substep", "sync_pd",
          "sync_smooth", "integrate", "epilogue"]      # the order of the PC_* enum in sim_core.h
SUBPHASES = ["kin_sincos", "kin_levels", "kin_inertia", "kin_subtree", "kin_project_force", "collide_broad", "collide_narrow",
             "collide_prefix"]                        # the order of the PS_* enum: the first five split kin_rne, the last three collide


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0].split(",")
        return dict(name=r[0].strip(), power_limit_w=float(r[1]), sm_mhz=float(r[2]), sm_max_mhz=float(r[3]))
    except Exception as e:      # the numbers are still measured; the card description is then missing
        return dict(error=str(e))


def worker(cfgs, steps, warmup, clocks):
    import numpy as np
    import torch
    from bench import make_clip
    from uhc_b200.agent import BatchedAgent, RolloutBuffer
    ex, shape = make_clip()
    out = []
    for E, k in cfgs:
        agent = BatchedAgent(E, [ex], [shape], device=0, seed=1)
        ids = np.array([i for i in range(E) if i % EPB < k], np.int32)
        agent.reset_envs(ids)
        L, h = agent.engine.lib, agent.engine.h
        cyc = torch.zeros(E, len(PHASES), dtype=torch.int64, device=agent.dev)
        sub = torch.zeros(E, len(SUBPHASES), dtype=torch.int64, device=agent.dev)
        if clocks:
            n = L.uhc_phase_clocks(h, C.c_void_p(cyc.data_ptr()))
            assert n == len(PHASES), "the library counts %d phases, this script names %d" % (n, len(PHASES))
            n = L.uhc_phase_subclocks(h, C.c_void_p(sub.data_ptr()))
            assert n == len(SUBPHASES), "the library counts %d sub-phases, this script names %d" % (n, len(SUBPHASES))
        buf = RolloutBuffer(1, E, agent.dev, agent.act_dim, agent.obs_dim)
        assert L.uhc_rollout_time_env_step(h, C.c_int(1)) == 0
        for _ in range(warmup):
            agent.rollout(buf, 1, 0)
        torch.cuda.synchronize()
        cyc.zero_()
        sub.zero_()
        kms, ms = [], C.c_float(0)
        for _ in range(steps):
            agent.rollout(buf, 1, 0)
            torch.cuda.synchronize()
            assert L.uhc_rollout_env_step_ms(h, C.c_int(0), C.byref(ms)) == 0
            kms.append(ms.value)
        clk = card()
        st = agent.engine.get_states(ids)
        r = dict(envs=E, k=k, working_warps=int(len(ids)), steps=steps, kernel_ms_median=float(np.median(kms)), kernel_ms=kms, card_after=clk,
                 newton_iters_mean=float(st["newton_iters"].mean()), contacts_max_mean=float(st["ncon"].mean()))
        if clocks:
            c = cyc.cpu().numpy()[ids].astype(np.float64) / steps          # per working warp and control step
            r["cycles_per_warp_step"] = {p: float(c[:, i].mean()) for i, p in enumerate(PHASES)}
            r["cycles_per_warp_step_total"] = float(c.sum(1).mean())
            c = sub.cpu().numpy()[ids].astype(np.float64) / steps
            r["subphase_cycles_per_warp_step"] = {p: float(c[:, i].mean()) for i, p in enumerate(SUBPHASES)}
        out.append(r)
        agent.engine.close()
        del agent
        torch.cuda.empty_cache()
    return out


def run_variant(so, cfgs, steps, warmup, clocks):
    env = dict(os.environ, UHC_B200_SO=so)
    with tempfile.NamedTemporaryFile("r", suffix=".json") as f:
        subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", json.dumps(dict(cfgs=cfgs, steps=steps, warmup=warmup, clocks=clocks, out=f.name))],
                       env=env, check=True, cwd=ROOT)
        return json.load(open(f.name))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory of step_phase_cycles.json (required)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--build-dir", default=None, help="where the instrumented libraries are built (default: a temporary directory)")
    ap.add_argument("--table-only", action="store_true", help="the 4096-env table and the production kernel time only")
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        w = json.loads(a.worker)
        json.dump(worker([tuple(c) for c in w["cfgs"]], w["steps"], w["warmup"], w["clocks"]), open(w["out"], "w"))
        return
    if not a.out:
        ap.error("--out DIR is required")
    from uhc_b200 import build
    tmp = None
    bdir = a.build_dir
    if bdir is None:
        tmp = tempfile.TemporaryDirectory()
        bdir = tmp.name
    libs = {}
    variants = (("clocks", ["UHC_PHASE_CLOCKS"]), ("clocks_nosync", ["UHC_PHASE_CLOCKS", "UHC_NO_CTA_SYNC"]),
                ("sync16", ["UHC_SYNC_GROUP=16"]), ("nosync", ["UHC_NO_CTA_SYNC"]))
    for name, defs in variants[:1] if a.table_only else variants:
        os.makedirs(os.path.join(bdir, name), exist_ok=True)
        libs[name] = build.build(so=os.path.join(bdir, name, "libuhc_b200.so"), defines=defs)
    prod = build.build()
    full, wave = 4096, NSM * EPB
    res = dict(card_before=card(), steps=a.steps, warmup=a.warmup, phases=PHASES, substeps_per_step=NSUB,
               cycles_note="clock64() cycles per working warp and control step, summed over the step's 15 substeps (divide by 15 for a substep)")
    if a.table_only:
        res["table"] = run_variant(libs["clocks"], [(full, EPB)], a.steps, a.warmup, True)[0]
        res["production"] = run_variant(prod, [(full, EPB)], a.steps, a.warmup, False)
    else:
        res["table"], *res["probe"] = run_variant(libs["clocks"], [(full, EPB)] + [(wave, k) for k in (4, 8, 12, 16)], a.steps, a.warmup, True)
        res["nosync"] = run_variant(libs["clocks_nosync"], [(full, EPB), (wave, EPB)], a.steps, a.warmup, True)
        res["production"] = run_variant(prod, [(full, EPB), (wave, EPB)], a.steps, a.warmup, False)
        res["groups"] = {name: run_variant(libs[name], [(full, EPB)], a.steps, a.warmup, False)[0] for name in ("sync16", "nosync")}
    res["card_after"] = card()
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "step_phase_cycles.json"), "w") as f:
        json.dump(res, f, indent=1)
    t = res["table"]["cycles_per_warp_step"]
    tot = sum(t.values())
    print("card: %s" % res["card_before"])
    sub = res["table"]["subphase_cycles_per_warp_step"]
    print("sub-phases (cycles per warp and control step, 4096 envs):")
    for p in SUBPHASES:
        print("  %-18s %12.0f" % (p, sub[p]))
    print("  kin_rne = %.0f, its sub-phases %.0f; collide = %.0f, its sub-phases %.0f" % (
        t["kin_rne"], sum(sub[p] for p in SUBPHASES[:5]), t["collide"], sum(sub[p] for p in SUBPHASES[5:])))
    if a.table_only:
        for p in PHASES:
            print("%-18s %12.0f %6.1f%%" % (p, t[p], 100 * t[p] / tot))
        print("kernel ms: instrumented %.3f, production %.3f" % (res["table"]["kernel_ms_median"], res["production"][0]["kernel_ms_median"]))
        if tmp:
            tmp.cleanup()
        return
    print("%-18s %12s %7s | probe cycles/warp/step at k = 4 8 12 16 (132 x 16 envs) | nosync" % ("phase", "cyc/warp/st", "share"))
    for p in PHASES:
        pr = " ".join("%10.0f" % r["cycles_per_warp_step"][p] for r in res["probe"])
        print("%-18s %12.0f %6.1f%% | %s | %10.0f" % (p, t[p], 100 * t[p] / tot, pr, res["nosync"][0]["cycles_per_warp_step"][p]))
    print("kernel ms: instrumented %.3f, production %.3f, production one wave %.3f, no alignment barriers %.3f" % (
        res["table"]["kernel_ms_median"], res["production"][0]["kernel_ms_median"], res["production"][1]["kernel_ms_median"], res["nosync"][0]["kernel_ms_median"]))
    print("probe kernel ms at k = 4 8 12 16:", " ".join("%.3f" % r["kernel_ms_median"] for r in res["probe"]))
    print("kernel ms at 4096 envs: two 8-warp groups %.3f, one 16-warp group %.3f, no barriers %.3f" % (
        res["production"][0]["kernel_ms_median"], res["groups"]["sync16"]["kernel_ms_median"], res["groups"]["nosync"]["kernel_ms_median"]))
    if tmp:
        tmp.cleanup()


if __name__ == "__main__":
    main()
