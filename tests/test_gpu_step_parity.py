"""GPU: the env-step kernel one control step at a time, per state, against the fp64 oracle and the host emulation of the same source, on the
seeded corpus of tests/step_corpus.py; and placement invariance of the step kernel, bit for bit.

A trajectory test has to allow for the round-off that contact make / break events amplify over many steps.  One step from a fixed state does
not, so these bounds are 10^3 .. 10^7 tighter than the trajectory tests of tests/test_gpu_env.py.  Every bound is 3x or more the worst error
measured on an H100 80GB HBM3 (700 W power limit), which is given beside it."""
import functools

import numpy as np
import pytest

from tests import step_corpus as S

pytestmark = pytest.mark.gpu

# fp64 kernel against the oracle, max over each variant's corpus (measured worst on the H100 in the comment)
FP64_BOUND = dict(qpos=1e-10,      # 1.7e-11
                  qvel=2e-8,       # 4.2e-9
                  xpos=3e-12,      # 4.1e-13
                  bquat=6e-11)     # 8.4e-12
# obs, reward, c_info and torques leave the kernel as fp32: |Δ| / max(1, |oracle|), half an fp32 ulp (6e-8) on top of the fp64 error
OUT_REL = 2.5e-7                   # 5.9e-8 (obs), 3.0e-8 (reward, c_info, torque)
# fp32 product kernel, 4096 envs in one launch
# contact-free states, absolute max|Δqpos|, max|Δqvel|: 1.35e-6, 1.30e-4 measured.  The emulation gives 1.27e-6, 9.8e-5 compiled without multiply-add
# contraction and 1.27e-4 in qvel with it (g++ -mfma -ffp-contract=fast): the GPU's larger qvel error is the contraction nvcc applies
FP32_FREE_Q, FP32_FREE_V = 5e-6, 4e-4
FP32_TORQUE0 = 1e-2                         # the first substep's torques, every state: 2.7e-3 measured, of torque_lim 500
# Contact states are compared per regime with the fp32 emulation on the same states: the GPU's median, 99th percentile and max within FP32_FACTOR of the
# emulation's, plus a round-off floor.  Measured GPU / emulation ratios: at most 1.1 (median; 2.1 for the airborne qvel, 2.3e-5 against 1.1e-5, inside the
# floor), 1.3 (p99) and 1.3 (max).  In the saturating regime (meta-PD gains at 10, torques at their limits) the fp32 error is round-off of the fp32
# arithmetic itself: the emulation's worst qvel error is 7.2 rad/s, and 2.8 with multiply-add contraction, while a 1-ulp change of the input pose moves the
# oracle by 4.5e-4.  There the fp32 comparison cannot see a fault below ~1 rad/s; the fp64 test covers that regime.
FP32_FACTOR = 4.0
# The Newton loop also ends when a step's line-search derivative is within 1e-6 of its slope and no row changes state (newton_advance: the step was
# exact), a test newton_tol does not enter.  In fp32 it sits at round-off, so multiply-add contraction moves the exit by an iteration on some states:
# compiled with -mfma -ffp-contract=fast, the emulation's Newton total differs from its plain build on 27 of the 462 states (by up to 4).  On the GPU it
# differs from the plain emulation's on 28 (by 1, or 3), and those states are compared separately.  Their worst qvel error is 0.31 rad/s; the crouching
# state with 0.114 rad/s (81 against 82 iterations) diverges from the emulation in its last substep's torque (1.6 N m) after one earlier exit.
FP32_EXIT_FLIPS = 70                        # distinct states whose Newton total differs from the emulation's (28 measured)
FP32_EXIT_FLIP_ITERS = 4                    # by at most (3 measured; 4 between the contracted and plain emulation)
FP32_EXIT_FLIP_QVEL = 1.0                   # their qvel error against the oracle (0.31 measured)
FP32_FLOOR_Q, FP32_FLOOR_V = 2e-6, 1e-4     # ... plus an fp32 round-off floor for regimes whose median error is itself round-off


@pytest.fixture(autouse=True)
def _identity_slots(monkeypatch):
    monkeypatch.delenv("UHC_SORT_ENVS", raising=False)     # env id = warp slot: the placement is what the test sets


def _tiled(n, E, seed):
    """case index per slot: the corpus tiled over E slots under a seeded permutation"""
    return np.random.default_rng(seed).permutation(np.arange(E) % n)


def _run(variant, precision, idx, E=None, only=None, cur=False):
    """one launch: case idx[j] in slot j (slots listed in `only` when given; the other envs are never reset)"""
    cases, _ = S.corpus(variant)
    s = S.setup(variant)
    E = len(idx) if E is None else E
    eng = s.engine(E, precision)
    if cur:
        eng.curriculum_enable(max_freq=50)
    slots = np.arange(len(idx), dtype=np.int32) if only is None else np.asarray(only, np.int32)
    out = S.run_engine(eng, [cases[i] for i in idx], slots=slots)
    eng.close()
    return out


@functools.lru_cache(maxsize=None)
def _fp64(variant):
    n = len(S.corpus(variant)[0])
    return _run(variant, 64, np.arange(n))


@functools.lru_cache(maxsize=None)
def _fp32_4096(cur=False):
    idx = _tiled(len(S.corpus("base")[0]), 4096, 0)
    return idx, _run("base", 32, idx, cur=cur)


def fp64_errors(variant):
    g, ref = _fp64(variant), S.oracle_results(variant)
    e = {k: S.err(g[k], ref[k]).max() for k in FP64_BOUND}
    for k in ("obs", "reward", "cinfo", "torque"):
        e[k + "_rel"] = (np.abs(g[k] - ref[k]) / np.maximum(1.0, np.abs(ref[k]))).max()
    return e


@pytest.mark.parametrize("variant", S.VARIANTS)
def test_fp64_kernel_per_state_matches_oracle(variant):
    """fp64 build (2 warps per CTA), one step per state against the oracle: every output, torques at every substep, flags, contact counts."""
    g, ref, em = _fp64(variant), S.oracle_results(variant), S.emu_results(variant, 64)
    e = fp64_errors(variant)
    for k, b in FP64_BOUND.items():
        assert e[k] < b, (k, e[k], b)
    for k in ("obs", "reward", "cinfo", "torque"):
        assert e[k + "_rel"] < OUT_REL, (k, e[k + "_rel"])
    for k in ("fail", "end", "ncon0"):
        assert np.array_equal(g[k], ref[k]), k
    assert np.array_equal(g["ncon"], em["ncon"]) and not g["flags"].any()        # the largest contact count of the 15 substeps, no overflow
    # the Newton iteration totals of the 15 substeps equal the emulation's on every state (no residual of the corpus sits at the tolerance)
    assert np.array_equal(g["iters"], em["iters"]), np.flatnonzero(g["iters"] != em["iters"])


def _q(e):
    return S.quantiles(e)


def fp32_report(idx, g):
    """per regime: GPU and emulation error quantiles (median, p99, max) of qpos / qvel against the oracle, on the same states (those whose Newton
    iteration total equals the emulation's); the states whose total differs, separately"""
    cases, _ = S.corpus("base")
    ref, em = S.oracle_results("base"), S.emu_results("base", 32)
    reg = np.array([cases[i]["regime"] for i in idx])
    flip = g["iters"] != em["iters"][idx]
    rep = {"flips": sorted(set(int(i) for i in idx[flip])), "flip_iters": np.abs(g["iters"] - em["iters"][idx])[flip].tolist(),
           "flip_qvel": float(S.err(g["qvel"][flip], ref["qvel"][idx[flip]]).max()) if flip.any() else 0.0}
    for r in S.REGIMES:
        m = (reg == r) & ~flip
        ii = idx[m]
        rep[r] = {k: (_q(S.err(g[k][m], ref[k][ii])), _q(S.err(em[k][ii], ref[k][ii]))) for k in ("qpos", "qvel")}
    free = g["ncon"] == 0
    rep["free"] = (S.err(g["qpos"][free], ref["qpos"][idx[free]]).max(), S.err(g["qvel"][free], ref["qvel"][idx[free]]).max(), int(free.sum()))
    rep["torque0"] = S.err(g["torque"][:, 0], ref["torque"][idx, 0]).max()
    return rep


def _check_fp32(idx, g):
    ref = S.oracle_results("base")
    rep = fp32_report(idx, g)
    q, v, nfree = rep["free"]
    assert nfree >= 500 and q < FP32_FREE_Q and v < FP32_FREE_V, rep["free"]
    assert rep["torque0"] < FP32_TORQUE0, rep["torque0"]
    for r in S.REGIMES:
        for k, floor in (("qpos", FP32_FLOOR_Q), ("qvel", FP32_FLOOR_V)):
            gq, eq = rep[r][k]
            assert (gq <= FP32_FACTOR * eq + floor).all(), (r, k, gq, eq)
    assert len(rep["flips"]) <= FP32_EXIT_FLIPS and max(rep["flip_iters"], default=0) <= FP32_EXIT_FLIP_ITERS and rep["flip_qvel"] < FP32_EXIT_FLIP_QVEL, rep["flips"]
    for k in ("fail", "end", "ncon0"):
        assert np.array_equal(g[k], ref[k][idx]), k
    assert not g["flags"].any()


def test_fp32_kernel_4096_envs_per_state_against_oracle_and_emulation():
    """The product build as it runs: 4096 envs, 256 full 16-warp CTAs in two waves, one launch; every slot holds a state of the corpus.
    A kernel-only defect shows up as an error distribution the emulation of the same source does not have."""
    _check_fp32(*_fp32_4096())


def test_fp32_curriculum_kernel_per_state():
    """k_env_step<float, 16, true>, the instantiation launched while the device curriculum is enabled, through the same comparison"""
    _check_fp32(*_fp32_4096(cur=True))


# ---- placement invariance
PKEYS = ("qpos", "qvel", "xpos", "bquat", "obs", "reward", "cinfo", "fail", "end", "torque", "ncon0", "ncon", "iters", "flags")


def _placements(precision):
    """(case index per slot, outputs) of launches that put the same states into different slots, neighbours and grid shapes"""
    cases, _ = S.corpus("base")
    n = len(cases)
    reg = np.array([c["regime"] for c in cases])
    probes = np.array([np.flatnonzero(reg == r)[0] for r in S.REGIMES])
    epb = 16 if precision == 32 else 2
    E = 4096 if precision == 32 else 2113
    # first / last warp of each alignment group, a CTA in the middle of the first wave, the first and a later CTA of the second wave, the last slot
    spots = [0, 7, 8, 15, 64 * 16 + 3, 64 * 16 + 12, 131 * 16 + 15, 132 * 16, 200 * 16 + 9, E - 1] if precision == 32 else \
            [0, 1, 500 * 2, 500 * 2 + 1, 1055 * 2, 1055 * 2 + 1, E - 1]
    runs = []

    def tiled_with_probes(E, seed, at, rot):
        idx = _tiled(n, E, seed)
        for j, s in enumerate(at):
            idx[s] = probes[(j + rot) % len(probes)]
        return idx

    if precision == 32:
        runs.append(_fp32_4096())
    else:
        idx = tiled_with_probes(E, 0, spots, 0)
        runs.append((idx, _run("base", 64, idx)))
    idx = tiled_with_probes(E, 1, spots, 1)                       # other neighbours, probes shifted to other slots
    runs.append((idx, _run("base", precision, idx)))
    idx = probes[np.arange(len(spots)) % len(probes)]             # only the probes are reset: every other record is invalid and skips the barrier count
    runs.append((idx, _run("base", precision, idx, E=E, only=spots)))
    for Ep in (17, 2113, 4095):                                   # a partial last CTA
        at = [Ep - 1, Ep - 2, Ep - 1 - epb, 0]
        idx = tiled_with_probes(Ep, Ep, at, Ep)
        runs.append((idx, _run("base", precision, idx)))
    return probes, runs


@pytest.mark.parametrize("precision", [32, 64])
def test_placement_does_not_change_a_single_bit(precision):
    """The same state gives the same bits in any slot: first, middle or last warp of a CTA and of either alignment group, the first or the second
    wave, the partial last CTA of E = 17, 2113 and 4095, next to other regimes and next to never-reset records.  No warp may read another env's
    data, so a difference is cross-talk: a shared-memory overlap, an overlay's lifetime, a barrier or staging."""
    probes, runs = _placements(precision)
    idx = np.concatenate([i for i, _ in runs])
    first = {}
    for j, c in enumerate(idx):
        first.setdefault(int(c), j)
    ref_rows = np.array([first[int(c)] for c in idx])
    seen = np.bincount(idx, minlength=int(idx.max()) + 1)
    assert (seen[probes] >= len(runs)).all()
    for k in PKEYS:
        a = np.concatenate([o[k] for _, o in runs])
        same = np.array([np.array_equal(a[j], a[ref_rows[j]]) for j in range(len(a))])
        assert same.all(), (k, np.flatnonzero(~same)[:10], idx[~same][:10])
