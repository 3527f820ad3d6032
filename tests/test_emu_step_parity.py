"""CPU: the env step's kernel source (host emulation, tests/emu) against the fp64 oracle, one control step per state, on the seeded corpus of
tests/step_corpus.py.  fp64 pins the algorithm; fp32 pins the error that the kernel source's own fp32 arithmetic makes, regime by regime, so
the GPU test that compares the CUDA kernel's error distribution against it (tests/test_gpu_step_parity.py) rests on numbers checked here.
Each bound is 3x or more the worst value measured (x86-64, g++ -O2 -ffp-contract=off), given beside it."""
import numpy as np
import pytest

from tests import step_corpus as S

# fp64: max |emu - oracle| over every variant's corpus (measured worst in the comment)
FP64_BOUND = dict(qpos=1e-10,      # 3.6e-11
                  qvel=2e-8,       # 6.7e-9
                  xpos=3e-12,      # 6.9e-13
                  bquat=6e-11,     # 1.8e-11
                  obs=2e-8,        # 6.7e-9 (the joint velocities of the observation)
                  reward=2e-12,    # 5.2e-13
                  cinfo=4e-12,     # 1.2e-12
                  torque=1.2e-7)   # 3.7e-8 of torque_lim 500, over all 15 substeps
# fp32: per regime of the base corpus, (median, 99th percentile, max) of max|Δqpos| and max|Δqvel| after one step, measured
EMU32_MEASURED = {
    "airborne": ((2.9e-7, 9.5e-7, 1.27e-6), (1.1e-5, 8.0e-5, 9.8e-5)),
    "standing": ((1.07e-6, 7.16e-6, 8.06e-6), (3.1e-5, 3.08e-4, 4.66e-4)),
    "crouching": ((3.07e-5, 6.28e-4, 1.26e-3), (4.5e-4, 1.10e-2, 1.30e-2)),
    "leaning": ((2.10e-5, 3.92e-4, 4.28e-4), (2.13e-4, 4.29e-3, 4.54e-3)),
    # meta-PD gains at 10, torques at their limits: round-off of the fp32 arithmetic (2.8 rad/s worst with multiply-add contraction, while a 1-ulp change
    # of the input pose moves the oracle by 4.5e-4), so the fp32 pins are blind below ~1 rad/s here; test_emu_fp64_one_step_matches_oracle covers it
    "saturating": ((3.09e-4, 5.73e-3, 9.06e-3), (2.28e-2, 2.12, 7.21)),
    "episode_end": ((1.54e-6, 5.43e-6, 5.71e-6), (3.8e-5, 1.68e-4, 3.01e-4)),
}
# fp32, the engine-wide variants (few states per regime): the worst max|Δqpos|, max|Δqvel| over the corpus, measured
EMU32_VARIANT_MEASURED = {"jnt_range": (1.37e-3, 0.774), "explicit": (2.69e-2, 2.50), "shapes": (2.64e-3, 0.653)}
# fp32, the first substep's torque (from the state as given, before any fp32 error has been integrated): 4.2e-3 measured, of torque_lim 500
EMU32_TORQUE0_BOUND = 1.5e-2


def _regimes(variant):
    return np.array([c["regime"] for c in S.corpus(variant)[0]])


@pytest.mark.parametrize("variant", S.VARIANTS)
def test_corpus_covers_every_regime_band_and_flag(variant):
    """The corpus asserts its own coverage: each regime's contact band, torque clipping, joint-limit rows, clip ends and failures."""
    cov = S.coverage(variant)
    counts = cov["counts"]
    per_regime = S.N_PER_REGIME if variant == "base" else S.N_VARIANT // len(S.REGIMES)
    for r in S.REGIMES:
        assert sum(v for (rr, _), v in counts.items() if rr == r) >= per_regime * 3 // 4, (r, counts)
    if variant == "base":
        for r, need in S.MIN_BAND.items():
            for band, n in need.items():
                assert counts.get((r, band), 0) >= n, (r, S.BANDS[band], counts)
    else:
        for band in range(len(S.BANDS)):             # every band, in every variant
            assert sum(v for (_, b), v in counts.items() if b == band) >= 3, (variant, S.BANDS[band], counts)
    assert cov["torque_clipped"] >= 1 and cov["fail"] >= 1 and cov["end"] >= 1 and cov["alive"] >= 10, cov
    if variant == "jnt_range":
        assert cov["limit_active"] >= 20, cov
    # more than 40 contacts is the kernel's overflow path (flagged, tested elsewhere): such states are dropped, and they stay few
    assert cov["dropped"] <= cov["n"] // 10, cov


@pytest.mark.parametrize("variant", S.VARIANTS)
def test_emu_fp64_one_step_matches_oracle(variant):
    ref, em = S.oracle_results(variant), S.emu_results(variant, 64)
    for k, b in FP64_BOUND.items():
        e = S.err(em[k], ref[k]).max()
        assert e < b, (k, e, b)
    for k in ("fail", "end", "ncon0"):
        assert np.array_equal(em[k], ref[k]), k


def test_emu_fp32_error_quantiles_per_regime():
    """The fp32 error of the kernel source after one step, per regime: median, 99th percentile and max within 3x of what was measured.
    A change to the fp32 arithmetic of sim_core.h / env_step.h that moves these is a change the GPU bounds depend on."""
    ref, em = S.oracle_results("base"), S.emu_results("base", 32)
    reg = _regimes("base")
    for r, (mq, mv) in EMU32_MEASURED.items():
        m = reg == r
        q = S.quantiles(S.err(em["qpos"][m], ref["qpos"][m]))
        v = S.quantiles(S.err(em["qvel"][m], ref["qvel"][m]))
        assert (q <= 3 * np.array(mq)).all() and (v <= 3 * np.array(mv)).all(), (r, q, v)
    for k in ("fail", "end", "ncon0"):
        assert np.array_equal(em[k], ref[k]), k
    assert S.err(em["torque"][:, 0], ref["torque"][:, 0]).max() < EMU32_TORQUE0_BOUND


@pytest.mark.parametrize("variant", ["jnt_range", "explicit", "shapes"])
def test_emu_fp32_error_engine_variants(variant):
    ref, em = S.oracle_results(variant), S.emu_results(variant, 32)
    mq, mv = EMU32_VARIANT_MEASURED[variant]
    assert S.err(em["qpos"], ref["qpos"]).max() <= 3 * mq and S.err(em["qvel"], ref["qvel"]).max() <= 3 * mv
    assert S.err(em["torque"][:, 0], ref["torque"][:, 0]).max() < EMU32_TORQUE0_BOUND
    for k in ("fail", "end", "ncon0"):
        assert np.array_equal(em[k], ref[k]), k


def test_fp32_contact_error_is_in_the_constraint_solve():
    """Attribution of the fp32 contact-state error: at one state, fp32 forward dynamics of the kernel source against the oracle, split by stage.
    The bias C (kinematics + RNE) stays at fp32 round-off; the error of qacc comes from the contact solve (Newton on the soft-constraint cost),
    and it is larger the more contacts there are."""
    from oracle import oracle as O
    from tests.emu.emu import Emu
    om, d = O.Model(), O.Data()
    e = Emu(32)
    cases, _ = S.corpus("base")
    reg = _regimes("base")
    rel_c, rel_free, rel_con = [], [], []
    for i in np.flatnonzero((reg == "airborne") | (reg == "crouching") | (reg == "leaning"))[::4]:
        c = cases[i]
        d.qpos[:], d.qvel[:], d.ctrl[:] = c["qpos"], c["qvel"], 0
        d.qfrc_applied[:] = 0
        d.qacc_warm[:] = 0
        O.forward(om, d)
        r = e.forward(c["qpos"], c["qvel"])
        rel_c.append(np.abs(r["C"] - d.C).max() / max(1.0, np.abs(d.C).max()))
        ea = np.abs(r["qacc"] - d.qacc).max() / max(1.0, np.abs(d.qacc).max())
        (rel_free if d.ncon == 0 else rel_con).append(ea)
    # measured: C 2.1e-6 of max|C|; qacc without contacts 1.1e-5 (median 4.4e-6), with 9 .. 40 contacts 7.6e-3 (median 1.4e-3) of max|qacc|
    assert max(rel_c) < 7e-6                            # fp32 round-off of the smooth dynamics
    assert max(rel_free) < 4e-5 and len(rel_free) >= 10  # the unconstrained articulated-body solve
    assert np.median(rel_con) > 30 * np.median(rel_free) and max(rel_con) < 2.5e-2 and len(rel_con) >= 20
