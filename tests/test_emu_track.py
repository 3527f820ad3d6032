"""CPU: the tracker's per-env code compiled for the host (tests/emu/track_emu.cpp).

Streaming: a clip pushed frame by frame through a window of H rows, rebased whenever the window is full, yields the rows of the whole
clip -- bit for bit the rows of motion_core.h's whole-clip emulation, and within 1e-12 of uhc_b200/motion_lib.py's table -- both at the
window index the step reads as its target (cur_t + 1) and at the one fail_safe re-seats on (cur_t).

Observation: for the states of tests/step_corpus.py, the observation rebuilt from the stored state record equals, bit for bit, the one the
emulated step wrote for the same state, for obs v1, v2, v5 and v6, with and without the shape vector."""
import numpy as np
import pytest

from tests import step_corpus as S
from tests.emu import motion_emu, track_emu
from tests.test_emu_motion import adversarial_clip, golden, host_table, smpl_clip
from uhc_b200 import motion_lib as ML
from uhc_b200.model import HumanoidModel

TOL = 1e-12
pytestmark = pytest.mark.filterwarnings("ignore:Gimbal lock")


def _check_stream(clip, H, models=None, variant=0):
    ms = ML.MotionSet([clip])
    nxt, cur, nreb = track_emu.stream_clip(ms.kind, ms.pose_dim, ms.rows, H, models, variant)
    whole = motion_emu.motion_table(ms, models, [variant])
    assert np.array_equal(nxt, whole), "streamed rows differ from the whole-clip rows"
    assert np.array_equal(cur, whole[:-1]), "a rebase moved the wrong rows"
    want = host_table([clip], models, [variant])
    assert np.abs(nxt - want).max() <= TOL
    # the reset leaves rows 0, 1 in the window; frame k is pushed when rows 0 .. k - 1 are held, so the first rebase comes with frame H
    assert (nreb > 0) == (len(ms.rows) > H)
    return nreb


@pytest.mark.parametrize("H", [3, 4, 64])
@pytest.mark.parametrize("tag", ["sway", "kick"])
def test_golden_clips_streamed(tag, H):
    z = golden(tag)
    n = _check_stream({"pose_aa": z["pose_aa"], "trans": z["trans"]}, H)
    n += _check_stream({"qpos": z["qpos"]}, H)
    assert n > 0 or H == 64


@pytest.mark.parametrize("H", [3, 4, 64])
def test_seeded_clips_streamed(H):
    rng = np.random.default_rng(21)
    for T in (2, 3, 5, 70):
        _check_stream({"qpos": ML.synthetic_clip(T, rng)["qpos"]}, H)
        _check_stream(smpl_clip(T, rng), H)
    pose_h = {"pose_aa": rng.normal(0, 0.4, (41, 156)), "trans": rng.normal(0, 0.3, (41, 3))}     # SMPL-H: hands read as zero
    _check_stream(pose_h, H)
    _check_stream(adversarial_clip(), H)


def test_shape_variants_streamed():
    rng = np.random.default_rng(11)
    models = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.85, 1.15, 24))]
    for H in (3, 4, 64):
        _check_stream(smpl_clip(30, rng), H, models, 1)
        _check_stream({"qpos": ML.synthetic_clip(25, rng)["qpos"]}, H, models, 1)


OBS_CASES = [(64, dict(obs_v=2)), (64, dict(obs_v=2, no_shape=1)), (64, dict(obs_v=1)), (64, dict(obs_v=5)), (64, dict(obs_v=5, no_shape=1)),
             (64, dict(obs_v=6)), (64, dict(obs_v=6, no_shape=1)), (32, dict(obs_v=2)), (32, dict(obs_v=6))]


@pytest.mark.parametrize("precision,cfg", OBS_CASES, ids=[f"fp{p}-" + "-".join(f"{k}{v}" for k, v in c.items()) for p, c in OBS_CASES])
def test_obs_from_stored_record_equals_step_obs(precision, cfg):
    s = S.setup("base")
    e = track_emu.TrackEmu(precision, model=s.models[0], **cfg)
    e.load_clips(s.clips, s.shapes)
    cases = S.corpus("base")[0][::3]
    regimes = set()
    for c in cases:
        obs_reset = e.reset(clip=c["clip"], start=c["start"], qpos=c["qpos"], qvel=c["qvel"])
        assert np.array_equal(e.track_obs(), obs_reset), "reset observation"
        obs, r, done, info = e.step(c["action"])
        assert np.array_equal(e.track_obs(), obs), ("step observation", c["regime"])
        regimes.add(c["regime"])
    assert regimes == set(S.REGIMES)
