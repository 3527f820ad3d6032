"""GPU: subject bodies built on the device (include/uhc_subject.h) against the fp64 restatement tests/subject_ref.py, the same bits alone and
in a batch, the refused arguments; clips on their own subject's body evaluated bit for bit as on an engine holding that body alone; one
subject variant stepped against the fp64 oracle; and subject_bodies through AgentCopycat.  The SMPL files are licence-gated, so the models
are synthetic: the neutral humanoid's hulls as an SMPL mesh (tests/subject_ref.py uniform_scale_model) and two perturbed genders."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.subject_ref import gendered, subject_body, uniform_scale_model

pytestmark = pytest.mark.gpu
REL, ABS_M = 1e-12, 1e-14


@pytest.fixture(scope="module")
def setup():
    from uhc_b200.model import HumanoidModel
    from uhc_b200.subject_body import SubjectBasis
    hm = HumanoidModel()
    n = uniform_scale_model()
    models = (n, gendered(n, 1), gendered(n, 2))
    return hm, models, SubjectBasis.from_models(hm, *models)


def random_subjects(n, seed):
    rng = np.random.RandomState(seed)
    b = rng.uniform(-2.0, 2.0, (n, 10))
    b[:, 0] = rng.uniform(-0.25, 0.25, n)                 # direction 0 of the synthetic model scales the whole body by 1 + beta_0
    return b, rng.randint(0, 3, n).astype(np.int32)


def test_device_matches_the_restatement(setup):
    hm, models, basis = setup
    betas, genders = random_subjects(24, 1)
    genders[:3] = [0, 1, 2]
    bf, hull, maps = basis.bodies(betas, genders)
    for r in range(len(genders)):
        rb, rh, rm = subject_body(hm, models[0], models[genders[r]], betas[r])
        assert np.abs(maps[r] - rm).max() < REL
        assert np.abs(hull[r] - rh).max() < ABS_M + REL * np.abs(rh).max()
        scale = np.abs(rb).max(0) + 1e-300
        assert np.all(np.abs(bf[r] - rb) <= 10 * REL * scale + (np.arange(20) < 3) * ABS_M), (r, np.abs(bf[r] - rb).max(0) / scale)
        assert np.all(np.abs(bf[r, :, 13] - rb[:, 13]) <= 1e-10 * rb[:, 13])
    from tests.emu.subject_emu import subject_body as emu
    for r in range(3):
        eb, eh, em = emu(basis, betas[r], genders[r])
        assert np.abs(bf[r] - eb).max() <= 1e-12 * np.abs(eb).max() and np.array_equal(hull[r], eh) and np.array_equal(maps[r], em)


def test_zero_beta_neutral_is_the_shipped_body(setup):
    hm, _, basis = setup
    bf, hull, maps = basis.bodies(np.zeros((2, 10)), np.zeros(2, np.int32))
    cols = [c for c in range(20) if c != 13]
    assert np.array_equal(bf[0][:, cols], hm.body_f[:, cols]) and np.array_equal(hull[0], hm.hull)
    assert np.all(np.abs(bf[0][:, 13] - hm.body_f[:, 13]) <= 1e-12 * hm.body_f[:, 13])


def test_same_bits_alone_and_in_a_batch(setup):
    _, _, basis = setup
    betas, genders = random_subjects(10000, 2)
    bf, hull, maps = basis.bodies(betas, genders)
    for r in (0, 1, 255, 4095, 4096, 9999):
        b1, h1, m1 = basis.bodies(betas[r:r + 1], genders[r:r + 1])
        assert np.array_equal(b1[0], bf[r]) and np.array_equal(h1[0], hull[r]) and np.array_equal(m1[0], maps[r])


def test_refused_arguments_leave_the_process_usable(setup):
    from uhc_b200.engine import load_library
    hm, _, basis = setup
    lib = load_library()
    base, st = hm.host_struct(), basis.struct()
    d = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_double))
    ip = lambda a: None if a is None else a.ctypes.data_as(C.POINTER(C.c_int))
    bf, hull, mp = np.zeros((2, 24, 20)), np.zeros((2, len(hm.hull), 3)), np.zeros((2, 24, 12))

    def call(n=2, b=np.zeros((2, 10)), g=np.zeros(2, np.int32), bs=st, out=bf):
        return lib.uhc_subject_bodies(C.c_int(0), C.byref(base), None if bs is None else C.byref(bs), C.c_int(n), d(b), ip(g), d(out), d(hull), d(mp))
    nan = np.zeros((2, 10))
    nan[1, 3] = np.inf
    assert call(n=-1) == -2 and call(b=None) == -2 and call(g=None) == -2 and call(bs=None) == -2 and call(out=None) == -2
    assert call(g=np.array([0, 3], np.int32)) == -2 and call(g=np.array([-1, 0], np.int32)) == -2 and call(b=nan) == -2
    from uhc_b200.subject_body import SubjectBasis
    only = SubjectBasis.from_models(hm, setup[1][0]).struct()
    assert call(bs=only, g=np.array([0, 1], np.int32)) == -2 and b"has no model" in lib.uhc_last_error()
    inv = np.zeros((2, 10))
    inv[1, 0] = -1.5                                       # scale -0.5: every body inverted
    assert call(b=inv) == -2 and b"det A" in lib.uhc_last_error() and not bf.any()
    cols = [c for c in range(20) if c != 13]                   # invweight0 is recomputed (within 1e-12, test above)
    assert call(n=0) == 0 and call() == 0 and np.array_equal(bf[0][:, cols], hm.body_f[:, cols])


def _subject_agent(variants, clips, shapes, clip_models, E):
    from uhc_b200.agent import BatchedAgent
    return BatchedAgent(E, clips, shapes, seed=3, policy_hsize=(128, 64), value_hsize=(128, 64), model=variants[0],
                        variants=variants if len(variants) > 1 else None, clip_models=clip_models, auto_reset=False, t_min=5, t_max=-1)


def test_clips_on_their_own_subject_are_the_single_body_engine(setup):
    """N clips, each on its own subject: evaluate() gives every clip the bits an engine whose only model is that subject gives it"""
    from uhc_b200 import motion_lib
    _, _, basis = setup
    z = np.load(os.path.join(os.path.dirname(__file__), "golden", "expert_sway.npz"))
    pose = np.concatenate([z["pose_aa"][:, :66], np.zeros((len(z["pose_aa"]), 6))], 1)
    N = 16
    betas, genders = random_subjects(N, 3)
    variants, idx = basis.build(betas, genders)
    assert len(variants) == N + 1 and np.array_equal(idx, np.arange(1, N + 1))
    clips = [motion_lib.make_expert(pose, z["trans"], variants[v]) for v in idx]
    shapes = [np.concatenate([b, np.zeros(6), [g]]) for b, g in zip(betas, genders)]
    multi = _subject_agent(variants, clips, shapes, idx, N)
    res = multi.evaluate(np.arange(N), fail_safe=False, record_states=True)
    multi.engine.close()
    for c in range(N):
        solo = _subject_agent([variants[idx[c]]], [clips[c]], [shapes[c]], None, N)
        r1 = solo.evaluate([0], fail_safe=False, record_states=True)[0]
        solo.engine.close()
        for k in ("frames", "states"):
            assert np.array_equal(res[c][k], r1[k]), (c, k)
        assert res[c]["last_t"] == r1["last_t"] and res[c]["reward_sum"] == r1["reward_sum"] and res[c]["fail_any"] == r1["fail_any"]


def test_one_subject_against_the_oracle(setup):
    """fp64 kernel, one control step per state on a subject's body, against the oracle given that body's tables (test_gpu_step_parity's bounds)"""
    from oracle import oracle as O
    from tests import step_corpus as S
    from tests.test_gpu_step_parity import FP64_BOUND, OUT_REL
    from uhc_b200 import motion_lib
    _, _, basis = setup
    betas, genders = random_subjects(1, 4)
    genders[:] = 2
    variants, _ = basis.build(betas, genders)
    hm, sb = variants
    s = S.Setup("base")
    z = np.load(os.path.join(S.GOLDEN, "expert_sway.npz"))
    pose = np.concatenate([z["pose_aa"][:, :66], np.zeros((len(z["pose_aa"]), 6))], 1)
    so = np.concatenate([betas[0], np.zeros(6), [2.0]])
    s.models, s.clip_models, s.shapes = [hm, sb], [0, 1], [so, so]
    s.clips = [motion_lib.make_expert(pose, z["trans"], m) for m in s.models]
    s.lens = np.array([len(c["qpos"]) for c in s.clips])
    ora = O.Model(tables=dict(body_offset=sb.offset, body_mass=sb.mass, body_ipos=sb.ipos, body_inertia=sb.inertia,
                              body_invweight0=np.stack([sb.invw, np.zeros(24)], 1), hull_vert=sb.hull))
    rng = np.random.default_rng(5)
    cases = []
    while len(cases) < 40:
        c = S._case(s, rng, ("standing", "crouching", "airborne")[len(cases) % 3])     # "leaning" is placed for the neutral body's geometry
        if c["clip"] == 1:
            cases.append(c)
    env = O.Env(ora, S._slice(s.clips[1], 0), so)
    ref = {k: [] for k in ("qpos", "qvel", "xpos", "reward", "fail", "ncon")}
    for c in cases:
        env.load_expert(S._slice(s.clips[1], c["start"]), so)
        env.reset(c["qpos"], c["qvel"])
        _, r, _, info = env.step(c["action"])
        ref["qpos"].append(env.d.qpos.copy()); ref["qvel"].append(env.d.qvel.copy()); ref["xpos"].append(env.d.xpos.copy())
        ref["reward"].append(r); ref["fail"].append(info["fail"]); ref["ncon"].append(env.d.ncon)
    assert max(ref["ncon"]) > 0                               # contact states are among them
    eng = s.engine(len(cases), 64)
    g = S.run_engine(eng, cases)
    eng.close()
    for k in ("qpos", "qvel", "xpos"):
        e = S.err(g[k], np.array(ref[k])).max()
        assert e < FP64_BOUND[k], (k, e)
    assert (np.abs(g["reward"] - np.array(ref["reward"])) / np.maximum(1.0, np.abs(ref["reward"]))).max() < OUT_REL
    assert np.array_equal(g["fail"], np.array(ref["fail"])) and not g["flags"].any()


def _write_models(root):
    n = uniform_scale_model()
    n["shapedirs"][:, :, 0] *= 0.05                        # beta_0 = 1: 5 % larger, as SMPL's first component is a few cm of height
    os.makedirs(root / "data" / "smpl", exist_ok=True)
    for name, m in zip(("NEUTRAL", "MALE", "FEMALE"), (n, gendered(n, 1), gendered(n, 2))):
        kt = np.stack([np.where(m["parents"] < 0, 4294967295, m["parents"]), np.arange(24)]).astype(np.int64)
        np.savez(root / "data" / "smpl" / f"SMPL_{name}.npz", kintree_table=kt, **{k: v for k, v in m.items() if k != "parents"})


def test_subject_bodies_through_the_dropin(tmp_path, monkeypatch):
    import torch
    from tests.test_gpu_dropin import _cfg
    from uhc.agents import agent_dict
    from uhc_b200 import motion_lib
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    dev = torch.device("cuda", index=0)
    try:
        cfg = _cfg(tmp_path, monkeypatch)
        cfg.cfg_dict["subject_bodies"] = True
        cfg.data_specs["expert_tables"] = "host"
        with pytest.raises(AssertionError, match="subject_bodies.*expert_tables"):
            agent_dict[cfg.agent_name](cfg, torch.float64, dev, training=True, checkpoint_epoch=0)
        cfg.data_specs["expert_tables"] = "device"
        with pytest.raises(FileNotFoundError, match="SMPL_NEUTRAL"):
            agent_dict[cfg.agent_name](cfg, torch.float64, dev, training=True, checkpoint_epoch=0)
        _write_models(tmp_path)
        agent = agent_dict[cfg.agent_name](cfg, torch.float64, dev, training=True, checkpoint_epoch=0)
        eng, loader = agent.agent.engine, agent.data_loader
        shapes = np.asarray(loader.shapes)
        assert len(set(shapes[:, 16].astype(int))) == 3 and len(eng.variants) == len(shapes) + 1
        assert np.array_equal(eng.clip_models, np.arange(1, len(shapes) + 1))
        # the expert tables come from each clip's own body: frame 0 root height as the host FK of that variant gives it
        for c in range(len(shapes)):
            rows = loader.motions.rows[int(np.sum(loader.motions.lens[:c])):][:int(loader.motions.lens[c])]
            ex = motion_lib.qpos_fk(motion_lib.smpl_to_qpos(rows[:, :72], rows[:, 72:75], eng.variants[c + 1]), eng.variants[c + 1])
            got = eng.clip_frames(c)
            assert np.abs(got["qpos"][:, 2] - ex["qpos"][:, 2]).max() < 1e-6 and np.abs(got["wbpos"] - ex["wbpos"]).max() < 1e-5
        heights = [eng.clip_frames(c)["qpos"][0, 2] for c in range(len(shapes))]
        assert len(set(np.round(heights, 6))) == len(shapes)           # the subjects stand at different heights
        info = agent.optimize_policy(0)
        assert np.isfinite(info["log"]["avg_reward"])
        name = loader.name
        out = {}
        for on_device in (True, False):
            cfg.cfg_dict["eval_on_device"] = on_device
            out[on_device] = agent.eval_policy(epoch=1)[0][f"coverage_{name}"]
            assert 0.0 <= out[on_device]["mean_coverage"] <= 1.0
        assert out[True]["all_coverage"] == out[False]["all_coverage"]
        mot = agent.export_motion(epoch=1, dump=False)
        assert all(len(r["pose_aa"]) == len(r["pred"]) for r in mot[name].values())
        agent.render_motion(epoch=1, out_dir=str(tmp_path / "video"), size=(64, 36), video="mjpeg")
        assert len(os.listdir(tmp_path / "video")) == len(shapes)
        eng.close()
    finally:
        torch.set_default_dtype(old)
