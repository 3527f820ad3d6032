"""Seeded per-state corpus of the env step and its references (TEST INFRASTRUCTURE, a plain helper module).

A case is (qpos, qvel, action, clip, start), every number rounded to fp32 before any engine sees it: uhc_env_reset takes its qpos / qvel
override as float, so the oracle, the host emulation and both CUDA builds start from the same bits.  Each case is reset onto that state and
stepped ONCE (one 30 Hz control step = 15 substeps), so the comparison measures the step's own error, not the amplification of a trajectory.

Regimes (contact counts are the oracle's at the reset state):
  airborne     0 contacts, tumbling with large angular velocities
  standing     feet on the floor
  crouching    root low and tilted: 9 .. 32 contacts
  leaning      leaning far forward close to the floor: 33 .. 40 contacts (the second 32-contact chunk of the wrench prefix sums)
  saturating   standing, with joint targets far off (torques at torque_lim), meta-PD gains clipped at 0 and at 10, large root wrenches
  episode_end  the clip's last step (the `end` flag) and poses displaced past body_diff_thresh (the `fail` flag)
Engine-wide variants: tightened joint ranges ("jnt_range"), the explicit residual force ("explicit", 315-wide actions) and two body shapes
mixed in one batch ("shapes").  Cases whose oracle contact count exceeds the kernel's 40 are dropped and counted.
"""
import functools
import os

import numpy as np

from oracle import oracle as O

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
GOLDEN = os.path.join(ROOT, "tests", "golden")

REGIMES = ("airborne", "standing", "crouching", "leaning", "saturating", "episode_end")
VARIANTS = ("base", "jnt_range", "explicit", "shapes")
BANDS = ((0, 0), (1, 8), (9, 32), (33, 40))          # contact-count bands: none, feet, many, the second 32-contact chunk
MAXCON = 40
# states per regime in the base corpus, and the least number of them each regime must put in a contact band (band index -> count)
N_PER_REGIME = 80
MIN_BAND = {"airborne": {0: 60}, "standing": {1: 30, 2: 10}, "crouching": {2: 50}, "leaning": {2: 10, 3: 25},
            "saturating": {1: 30, 2: 8}, "episode_end": {1: 40}}
N_VARIANT = 48
JNT_RANGE = np.tile(np.array([[-0.4, 0.5]]), (69, 1))
KEYS = ("qpos", "qvel", "xpos", "bquat", "obs", "reward", "cinfo", "fail", "end", "torque", "ncon0", "ncon", "iters")


def f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def band_of(n):
    for i, (lo, hi) in enumerate(BANDS):
        if lo <= n <= hi:
            return i
    return len(BANDS)


def _qmul(a, b):
    return np.array([a[0] * b[0] - a[1:] @ b[1:], *(a[0] * b[1:] + b[0] * a[1:] + np.cross(a[1:], b[1:]))])


def _axis_angle(v):
    ang = np.linalg.norm(v) + 1e-300
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * v / ang])


_BASE = np.array([0.7071068, 0.7071068, 0.0, 0.0])      # the upright root orientation of the Z-up world


def _expert(tag):
    z = np.load(os.path.join(GOLDEN, f"expert_{tag}.npz"))
    ex = {k: z[k] for k in z.files}
    return ex, np.concatenate([ex["beta"][0], [ex["gender"][0]]])


class Setup:
    """One engine configuration: its clips, body models and the matching oracle models."""

    def __init__(self, name):
        from uhc_b200 import motion_lib
        from uhc_b200.model import HumanoidModel
        self.name = name
        sway, so = _expert("sway")
        self.clips, self.shapes, self.clip_models = [sway], [so], None
        self.engine_kw, self.emu_kw, self.explicit = {}, {}, False
        hm = HumanoidModel()
        self.models = [hm]                                                   # body model of variant v (HumanoidModel)
        self.oracle_models = [O.Model()]
        if name == "jnt_range":
            self.models = [HumanoidModel(jnt_range=JNT_RANGE)]
            self.oracle_models = [O.Model(tables={"jnt_range": JNT_RANGE})]
        elif name == "explicit":
            self.explicit = True
            self.engine_kw = dict(rfc_mode="explicit")
            import ctypes
            self.emu_kw = dict(rfc_mode=1, vf_slot=(ctypes.c_int * 24)(*hm.vf_slot()))
        elif name == "shapes":
            z = np.load(os.path.join(GOLDEN, "expert_sway.npz"))
            pose = np.concatenate([z["pose_aa"][:, :66], np.zeros((len(z["pose_aa"]), 6))], 1)
            hm1 = HumanoidModel(scale=np.random.RandomState(4).uniform(0.85, 1.15, 24))
            self.models = [hm, hm1]
            self.clips = [motion_lib.make_expert(pose, z["trans"], m) for m in self.models]
            self.shapes = [so, so]
            self.clip_models = [0, 1]
            self.oracle_models = [O.Model(), O.Model(tables=dict(body_offset=hm1.offset, body_mass=hm1.mass, body_ipos=hm1.ipos,
                                                                 body_inertia=hm1.inertia, body_invweight0=np.stack([hm1.invw, np.zeros(24)], 1),
                                                                 hull_vert=hm1.hull))]
        elif name != "base":
            raise ValueError(name)
        self.act_dim = 69 + (216 if self.explicit else 6) + 30
        self.lens = np.array([len(c["qpos"]) for c in self.clips])

    def variant_of_clip(self, clip):
        return 0 if self.clip_models is None else self.clip_models[clip]

    def engine(self, E, precision, **kw):
        from uhc_b200.engine import Engine
        if self.clip_models is None:
            eng = Engine(E, model=self.models[0], precision=precision, **self.engine_kw, **kw)
            eng.load_clips(self.clips, self.shapes)
        else:
            eng = Engine(E, self.models[0], precision=precision, variants=self.models, **self.engine_kw, **kw)
            eng.load_clips(self.clips, self.shapes, clip_models=self.clip_models)
        return eng


@functools.lru_cache(maxsize=None)
def setup(name):
    return Setup(name)


# ---- the states
def _action(rng, s, scale=0.1):
    a = rng.normal(0, scale, s.act_dim)
    if s.explicit:
        a[69:69 + 216] = rng.normal(0, 0.05, 216)         # per body: contact point (m), force and torque (x rfc_scale)
    else:
        a[69:75] *= 0.3
    return a


def _case(s, rng, regime):
    """one state of a regime on Setup s: (qpos, qvel, action, clip, start) before rounding"""
    clip = int(rng.integers(0, len(s.clips))) if s.clip_models is not None else 0
    L = int(s.lens[clip])
    start = int(rng.integers(0, L - 3))
    ex = s.clips[clip]
    q, v = ex["qpos"][start].copy(), ex["qvel"][start].copy()
    a = _action(rng, s)
    if regime == "airborne":
        q[:2] += rng.normal(0, 0.3, 2)
        q[2] = rng.uniform(2.5, 3.5)
        u = rng.normal(size=4)
        q[3:7] = u / np.linalg.norm(u)
        q[7:] = rng.uniform(-0.8, 0.8, 69)
        v = np.concatenate([rng.normal(0, 1.0, 3), rng.normal(0, 8.0, 3), rng.normal(0, 3.0, 69)])
    elif regime in ("standing", "saturating"):
        q[2] -= rng.uniform(0.03, 0.05)                          # the clip's own root height leaves the feet 1 .. 3 cm above the floor
        q[7:] += rng.normal(0, 0.03, 69)
        v = v + rng.normal(0, 0.2, 75)
        if regime == "saturating":
            sg = rng.choice([-1.0, 1.0], 69)
            a[:69] = sg * rng.uniform(0.3, 0.8, 69)              # targets far off: the PD torques clip at torque_lim
            if s.explicit:
                a[69:69 + 216] = rng.normal(0, 0.5, 216)
            else:
                a[69:75] = rng.choice([-1.0, 1.0], 6) * rng.uniform(1.5, 3.0, 6)     # x rfc_scale 100 -> clipped at rfc_lim 100
            off = s.act_dim - 30
            a[off:] = rng.choice([-1.5, 9.5], 30)               # meta-PD scales 1 + a clip at 0 and at 10
    elif regime == "crouching":
        q[2] = rng.uniform(0.3, 0.6)
        q[3:7] = _qmul(_axis_angle(rng.normal(size=3) * rng.uniform(0.2, 0.8)), _BASE)
        q[7:] = rng.uniform(-0.6, 0.6, 69)
        v = rng.normal(0, 0.5, 75)
    elif regime == "leaning":
        q[:2] = ex["qpos"][start, :2]
        q[2] = 0.16 + rng.uniform(-0.01, 0.01)
        a2 = np.deg2rad(40.0 + rng.uniform(-2, 2)) / 2
        q[3:7] = [np.cos(a2), 0, np.sin(a2), 0]
        q[7:] = rng.normal(0, 0.02, 69)
        v = rng.normal(0, 0.2, 75)
    elif regime == "episode_end":
        q[2] -= rng.uniform(0.03, 0.05)
        q[7:] += rng.normal(0, 0.03, 69)
        v = v + rng.normal(0, 0.1, 75)
        if rng.uniform() < 0.5:
            start = L - 2                                        # one step left: cur_t = 1 = len - 1 sets `end`
            q, v = ex["qpos"][start].copy(), ex["qvel"][start].copy()
            q[2] -= 0.04
        else:
            q[:2] += rng.choice([-1.0, 1.0], 2) * rng.uniform(0.5, 0.8, 2)     # the mean body-position error is past 0.5 m: `fail`
    else:
        raise ValueError(regime)
    q[3:7] /= np.linalg.norm(q[3:7])
    return dict(qpos=f32(q), qvel=f32(v), action=f32(a), clip=clip, start=start, regime=regime)


def _with_jnt_range(case, rng):
    """the tightened-range variant: several upper-body joints past their limits"""
    q = case["qpos"].copy()
    idx = rng.choice(np.arange(24, 69), 6, replace=False)
    q[7 + idx] = rng.choice([-0.55, 0.65], 6) + rng.normal(0, 0.02, 6)
    case["qpos"] = f32(q)
    return case


def corpus(variant="base"):
    """the kept cases of a Setup (a tuple of dicts) and the number dropped for more than 40 oracle contacts"""
    cases, ref, dropped = _corpus(variant)
    return cases, dropped


def oracle_results(variant="base"):
    return _corpus(variant)[1]


@functools.lru_cache(maxsize=None)
def _corpus(variant, seed=0):
    s = setup(variant)
    rng = np.random.default_rng(1000 * VARIANTS.index(variant) + seed)
    regimes = REGIMES
    n = N_PER_REGIME if variant == "base" else N_VARIANT // len(regimes)
    cases, dropped = [], 0
    for r in regimes:
        for _ in range(n):
            c = _case(s, rng, r)
            if variant == "jnt_range" and r in ("airborne", "standing", "crouching", "saturating"):
                c = _with_jnt_range(c, rng)
            cases.append(c)
    ref = run_oracle(variant, cases)
    keep = (ref["ncon0"] <= MAXCON) & (ref["ncon"] <= MAXCON)
    return tuple(c for c, k in zip(cases, keep) if k), {k: x[keep] for k, x in ref.items()}, int((~keep).sum())


def coverage(variant="base"):
    """counts of (regime, band) plus the flag / clip / limit coverage of the kept cases, from the oracle's results"""
    cases, dropped = corpus(variant)
    ref = oracle_results(variant)
    s = setup(variant)
    counts = {}
    for c, n0 in zip(cases, ref["ncon0"]):
        counts[(c["regime"], band_of(int(n0)))] = counts.get((c["regime"], band_of(int(n0))), 0) + 1
    tl = np.stack([m.torque_lim for m in s.models])
    torque_clipped = np.array([np.isclose(np.abs(t), tl[s.variant_of_clip(c["clip"])]).any() for c, t in zip(cases, ref["torque"])])
    lim_active = np.array([((c["qpos"][7:] < s.models[0].jnt_range[:, 0]) | (c["qpos"][7:] > s.models[0].jnt_range[:, 1])).any() for c in cases])
    return dict(counts=counts, dropped=dropped, n=len(cases), fail=int(ref["fail"].sum()), end=int(ref["end"].sum()),
                alive=int((~ref["fail"] & ~ref["end"]).sum()), torque_clipped=int(torque_clipped.sum()), limit_active=int(lim_active.sum()))


# ---- the references
def _slice(ex, start):
    return {k: ex[k][start:] for k in ("qpos", "qvel", "wbpos", "wbquat", "bquat", "bangvel", "ee_wpos", "com")}


def run_oracle(variant, cases):
    """oracle.Env (fp64, dense algorithms): reset(q, v) on the clip from `start`, then step(a)"""
    s = setup(variant)
    envs = {}
    out = {k: [] for k in KEYS}
    for c in cases:
        v = s.variant_of_clip(c["clip"])
        if v not in envs:
            envs[v] = O.Env(s.oracle_models[v], _slice(s.clips[c["clip"]], 0), s.shapes[c["clip"]])
            if s.explicit:
                envs[v].set_rfc_mode(True)
        oe = envs[v]
        oe.load_expert(_slice(s.clips[c["clip"]], c["start"]), s.shapes[c["clip"]])
        oe.reset(c["qpos"], c["qvel"])
        out["ncon0"].append(oe.d.ncon)
        obs, r, done, info = oe.step(c["action"])
        out["qpos"].append(oe.d.qpos.copy()); out["qvel"].append(oe.d.qvel.copy()); out["xpos"].append(oe.d.xpos.copy())
        out["bquat"].append(oe.bquat.copy()); out["obs"].append(obs); out["reward"].append(r); out["cinfo"].append(info["c_info"])
        out["fail"].append(info["fail"]); out["end"].append(info["end"]); out["torque"].append(oe.torque.copy())
        out["ncon"].append(oe.d.ncon); out["iters"].append(oe.d.newton_iters)
    return {k: np.array(v) for k, v in out.items()}


@functools.lru_cache(maxsize=None)
def emu_results(variant="base", precision=64):
    """the kernel source compiled for the host (tests/emu), one case at a time.  ncon = the largest contact count of the 15 substeps and
    iters = the Newton iterations summed over them (the step kernel's istate); ncon0 = the reset's contact count."""
    from tests.emu.emu import Emu
    s = setup(variant)
    emus = {}
    out = {k: [] for k in KEYS}
    for c in corpus(variant)[0]:
        v = s.variant_of_clip(c["clip"])
        if v not in emus:
            emus[v] = Emu(precision, model=s.models[v], **s.emu_kw)
            emus[v].load_clips(s.clips, s.shapes)
        e = emus[v]
        e.reset(clip=c["clip"], start=c["start"], qpos=c["qpos"], qvel=c["qvel"])
        out["ncon0"].append(e.state()[1][7])
        obs, r, done, info = e.step(c["action"])
        st, ist = e.state()
        out["qpos"].append(st[0:76]); out["qvel"].append(st[76:151]); out["xpos"].append(st[996:1068]); out["bquat"].append(st[1236:1332])
        out["obs"].append(obs); out["reward"].append(r); out["cinfo"].append(info["c_info"]); out["fail"].append(info["fail"])
        out["end"].append(info["end"]); out["torque"].append(info["torque"]); out["ncon"].append(ist[7]); out["iters"].append(ist[6])
    return {k: np.array(v) for k, v in out.items()}


def run_engine(eng, cases, slots=None, torque=True, reset_ids=None):
    """reset every case into its slot of a live engine (one uhc_env_reset with the fp32 overrides), then ONE uhc_env_step of the whole batch.
    Slots without a case keep whatever record they had (never-reset envs are invalid records the kernel skips).  Returns the outputs of the
    case slots (dict of arrays in case order) plus the raw per-env outputs under "_all"."""
    import torch
    slots = np.arange(len(cases), dtype=np.int32) if slots is None else np.asarray(slots, np.int32)
    q = np.stack([c["qpos"] for c in cases]); v = np.stack([c["qvel"] for c in cases])
    clip = np.array([c["clip"] for c in cases], np.int32); start = np.array([c["start"] for c in cases], np.int32)
    eng.reset(slots, clip=clip, start=start, qpos=q, qvel=v)
    st0 = eng.get_states(slots)
    act = np.zeros((eng.E, eng.act_dim), np.float32)
    act[slots] = np.stack([c["action"] for c in cases]).astype(np.float32)
    tq = torch.zeros(eng.E, 15, 69, device="cuda") if torque else None
    obs, rew, ci, fail, end, pct = eng.step(torch.tensor(act, device="cuda"), torque_out=tq)
    torch.cuda.synchronize()
    st = eng.get_states(slots)
    sel = lambda t: t.cpu().numpy()[slots]
    out = dict(qpos=st["qpos"], qvel=st["qvel"], xpos=st["xpos"].reshape(len(slots), 72), bquat=st["bquat"], obs=sel(obs).astype(np.float64),
               reward=sel(rew).astype(np.float64), cinfo=sel(ci).astype(np.float64), fail=sel(fail).astype(bool), end=sel(end).astype(bool),
               torque=sel(tq).astype(np.float64) if torque else None, ncon0=st0["ncon"], ncon=st["ncon"], iters=st["newton_iters"], flags=st["flags"])
    return out


def err(a, b):
    """per-case max |a - b| over every axis but the first"""
    d = np.abs(np.asarray(a, np.float64) - np.asarray(b, np.float64))
    return d.reshape(len(d), -1).max(1)


def quantiles(e):
    return np.array([np.median(e), np.quantile(e, 0.99), e.max()])
