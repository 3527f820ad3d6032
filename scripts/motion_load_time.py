"""Time getting a motion dataset into the engine, host path against device path, on one GPU.

  host    motion_lib.make_expert per clip (numpy / scipy, fp64) + Engine.load_clips: wall time and peak RSS growth
  device  Engine.load_motions (uhc_load_motions): wall time to a device synchronise, and its kernel / row-copy time from CUDA events

N synthetic SMPL frames (seeded; clips of --clip-len frames, AMASS-like sinusoidal joint angles and a slow root walk).  Prints the card
name and power limit, both figures and whether the two tables agree (values not bit-identical, largest difference in fp32 ulps), then
one JSON line.  Usage: python scripts/motion_load_time.py [--frames 1000000] [--clip-len 300] [--chunk-frames 0]
"""
import argparse
import ctypes as C
import json
import os
import resource
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def synthetic_smpl(nframes, clip_len, seed):
    rng = np.random.default_rng(seed)
    lens = [clip_len] * (nframes // clip_len)
    rest = nframes - sum(lens)
    if rest >= 2 or not lens:
        lens.append(rest)
    else:
        lens[-1] += rest
    clips = []
    for T in lens:
        t = np.arange(T)[:, None] / 30.0
        pose = (rng.uniform(0, 0.25, 72) * np.sin(2 * np.pi * rng.uniform(0.2, 1.0, 72) * t + rng.uniform(0, 6.28, 72)))
        pose[:, :3] = 1.2092 + 0.1 * np.sin(t * rng.uniform(0.1, 0.5, 3))
        trans = np.concatenate([0.3 * t, 0.1 * np.sin(t), 0.7 + 0.02 * np.sin(3 * t)], 1)
        clips.append({"pose_aa": pose, "trans": trans})
    return clips


def rss_mb():
    return resource.getrusage(resource.RUSAGE_SELF).ru_maxrss / 1024.0


def power_limit():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        return r.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def compare(dev, host, nclips):
    """values of the device-built table that differ from the host-built one, the largest difference in fp32 ulps and absolute"""
    nbad, ulps, absd = 0, 0.0, 0.0
    for c in range(nclips):
        n = int(dev.clip_len[c])
        a, b = np.zeros((n, 576)), np.zeros((n, 576))
        for eng, out in ((dev, a), (host, b)):
            assert eng.lib.uhc_get_clip_frames(eng.h, c, 0, n, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
        nbad += int((a != b).sum())
        absd = max(absd, float(np.abs(a - b).max()))
        if dev.precision == 32:
            ulps = max(ulps, float((np.abs(a - b) / np.spacing(np.abs(b).astype(np.float32))).max()))
    return nbad, ulps, absd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1_000_000)
    ap.add_argument("--clip-len", type=int, default=300)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--chunk-frames", type=int, default=0)
    ap.add_argument("--precision", type=int, default=32, choices=(32, 64))
    a = ap.parse_args()
    import torch
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    clips = synthetic_smpl(a.frames, a.clip_len, a.seed)
    shapes = np.zeros((len(clips), 17))
    dev, host = Engine(64, precision=a.precision), Engine(64, precision=a.precision)
    torch.cuda.synchronize()
    rss0 = rss_mb()
    # device path: the raw rows only
    t0 = time.perf_counter()
    ms = ML.MotionSet(clips)
    t1 = time.perf_counter()
    dev.load_motions(ms, shapes, chunk_frames=a.chunk_frames)
    torch.cuda.synchronize()
    t2 = time.perf_counter()
    ev = dev.load_motions_time
    rss1 = rss_mb()
    # host path: today's expert tables
    t3 = time.perf_counter()
    experts = [ML.make_expert(c["pose_aa"], c["trans"]) for c in clips]
    t4 = time.perf_counter()
    host.load_clips(experts, shapes)
    torch.cuda.synchronize()
    t5 = time.perf_counter()
    rss2 = rss_mb()
    del experts
    nbad, ulps, absd = compare(dev, host, len(clips))
    nval = a.frames * 576
    res = dict(card=torch.cuda.get_device_name(0), power_limit=power_limit(), frames=a.frames, clips=len(clips), precision=a.precision,
               host_make_expert_s=round(t4 - t3, 3), host_load_clips_s=round(t5 - t4, 3), host_total_s=round(t5 - t3, 3),
               host_peak_rss_growth_mb=round(rss2 - rss1, 1), host_us_per_frame=round((t5 - t3) / a.frames * 1e6, 2),
               device_motionset_s=round(t1 - t0, 3), device_load_motions_s=round(t2 - t1, 3), device_kernel_ms=round(ev["kernel_ms"], 2),
               device_copy_ms=round(ev["copy_ms"], 2), device_peak_rss_growth_mb=round(rss1 - rss0, 1),
               device_us_per_frame=round((t2 - t1) / a.frames * 1e6, 3), input_bytes_per_frame=ms.rows.shape[1] * 8,
               tables_values=nval, tables_values_not_identical=nbad, tables_max_abs_diff=absd, tables_max_fp32_ulps=ulps if a.precision == 32 else None)
    print(f"{res['card']}, power limit {res['power_limit']}: {a.frames} frames in {len(clips)} clips, fp{a.precision} engine")
    print(f"  host    make_expert {res['host_make_expert_s']:.2f} s + load_clips {res['host_load_clips_s']:.2f} s = {res['host_us_per_frame']:.1f} us/frame, "
          f"peak RSS +{res['host_peak_rss_growth_mb']:.0f} MB")
    print(f"  device  load_motions {res['device_load_motions_s'] * 1e3:.1f} ms to synchronise ({res['device_us_per_frame']:.3f} us/frame): kernels "
          f"{res['device_kernel_ms']:.1f} ms, row copies {res['device_copy_ms']:.1f} ms; MotionSet {res['device_motionset_s']:.2f} s, "
          f"peak RSS +{res['device_peak_rss_growth_mb']:.0f} MB")
    print(f"  tables  {nbad} of {nval} values not bit-identical, max |diff| {absd:.3g}" + (f", max {ulps:.0f} fp32 ulp" if a.precision == 32 else ""))
    print(json.dumps(res))
    dev.close(); host.close()


if __name__ == "__main__":
    main()
