"""GPU: run-time subjects of the tracker (include/uhc_track.h uhc_track_subjects_enable / uhc_track_set_subjects, Tracker.set_subjects).

- a slot holds uhc_subject_bodies' bodies: fp64 tables bit for bit, engine-precision tables rounded as uhc_engine_create rounds them;
- a tracker whose envs get their subjects at run time is, bit for bit, a tracker on an engine created with those subjects as shape variants
  (state, reward, fail, observation, SMPL and floor rows), for qpos and SMPL streams, with and without fail_safe;
- one env swapped to a new subject mid-session: the others are untouched, the swapped env is a fresh tracker that had that subject from its
  reset, and no track graph is captured for it;
- refused calls leave every table and trajectory as before;
- an evaluation before and after the tables move gives the same results.
The SMPL files are licence-gated, so the models are synthetic (tests/subject_ref.py), as in tests/test_gpu_subject.py."""
import ctypes as C

import numpy as np
import pytest

from tests.subject_ref import gendered, uniform_scale_model
from tests.test_gpu_track import TRACK_KW, Run, _clips, _raw

pytestmark = [pytest.mark.gpu, pytest.mark.filterwarnings("ignore:Gimbal lock")]


@pytest.fixture(scope="module")
def basis():
    from uhc_b200.model import HumanoidModel
    from uhc_b200.subject_body import SubjectBasis
    n = uniform_scale_model()
    return SubjectBasis.from_models(HumanoidModel(), n, gendered(n, 1), gendered(n, 2))


def _subjects(n, seed):
    """shape rows [n][17]: beta 16 (the first 10 shape the body), gender; every gender present"""
    rng = np.random.RandomState(seed)
    s = np.zeros((n, 17))
    s[:, :16] = rng.uniform(-1.5, 1.5, (n, 16))
    s[:, 0] = rng.uniform(-0.2, 0.2, n)                   # direction 0 of the synthetic model scales the whole body by 1 + beta_0
    s[:, 16] = np.arange(n) % 3
    return s


def _stream(E, T, kind, seed):
    from uhc_b200 import motion_lib as ML
    ms = ML.MotionSet(_clips(np.random.default_rng(seed), [T] * E, kind))
    return ms, np.stack([_raw(ms, c) for c in range(E)])              # [E][T][row width]


def _engines(basis, shapes, precision=32, **kw):
    """A: created with the subjects as variants; B: neutral, the same subjects given at run time"""
    from uhc_b200.engine import Engine
    cfg = dict(TRACK_KW, **kw)
    variants, idx = basis.build(shapes[:, :10], shapes[:, 16].astype(np.int32))
    a = Engine(len(shapes), model=variants[0], precision=precision, variants=variants, **cfg)
    b = Engine(len(shapes), model=basis.humanoid, precision=precision, **cfg)
    b.track_subjects_enable(basis)
    return a, b, idx


def test_slots_hold_the_builders_bodies(basis):
    shapes = _subjects(6, 1)
    bf, hull, _ = basis.bodies(shapes[:, :10], shapes[:, 16].astype(np.int32))
    for precision in (32, 64):
        from uhc_b200.engine import Engine
        eng = Engine(6, model=basis.humanoid, precision=precision, **TRACK_KW)
        eng.track_subjects_enable(basis)
        eng.track_begin(4, "qpos")
        s0 = eng.track_subject_tables(2)                     # a slot starts as variant 0
        cast = (lambda x: x.astype(np.float32).astype(np.float64)) if precision == 32 else (lambda x: x)
        assert np.array_equal(s0["body_f"], cast(basis.humanoid.body_f)) and np.array_equal(s0["hull64"], basis.humanoid.hull)
        eng.track_set_subjects([4, 1, 3], shapes[[4, 1, 3]])
        for env in range(6):
            s = eng.track_subject_tables(env)
            r = env if env in (1, 3, 4) else None
            want_bf = bf[r] if r is not None else basis.humanoid.body_f
            want_hull = hull[r] if r is not None else basis.humanoid.hull
            assert np.array_equal(s["body_f"], cast(want_bf)) and np.array_equal(s["hull"], cast(want_hull)), (precision, env)
            assert np.array_equal(s["fk_body"], want_bf[:, :6]) and np.array_equal(s["hull64"], want_hull), (precision, env)
        eng.close()


@pytest.mark.parametrize("kind", ["qpos", "smpl"])
@pytest.mark.parametrize("fail_safe", [True, False])
def test_run_time_subjects_equal_creation_time_variants(basis, kind, fail_safe):
    t = _torch()
    E, T, H = 64, 62, 6
    shapes = _subjects(E, 2)
    a, b, idx = _engines(basis, shapes)
    ms, raw = _stream(E, T, kind, 3)
    a.track_begin(H, kind, ms.pose_dim, fk_models=idx, shapes=shapes)
    b.track_begin(H, kind, ms.pose_dim)
    b.track_set_subjects(np.arange(E), shapes)
    runs = [Run(e, fail_safe=fail_safe) for e in (a, b)]
    f01 = t.tensor(raw[:, :2], device="cuda").contiguous()
    for e in (a, b):
        e.track_reset(np.arange(E), f01)
    for k in range(60):
        nxt = None if k == 0 else t.tensor(raw[:, k + 1], device="cuda").contiguous()
        out = []
        for e, run in zip((a, b), runs):
            obs = e.track_obs().cpu().numpy()
            state, rew, fail = run.step(nxt)
            pose, trans = e.track_smpl(state)
            out.append((obs, state.cpu().numpy(), rew.cpu().numpy(), fail.cpu().numpy(), pose.cpu().numpy(), trans.cpu().numpy(),
                        e.track_floor(state).cpu().numpy()))
        for name, x, y in zip(("obs", "state", "reward", "fail", "pose", "trans", "floor"), *out):
            assert np.array_equal(x, y), (k, name)
    assert b.counters == a.counters
    a.close()
    b.close()


def _torch():
    import torch
    return torch


def _frames(t, x):
    return t.tensor(np.ascontiguousarray(x), device="cuda")


def test_swap_one_env_mid_session(basis):
    t = _torch()
    from uhc_b200.engine import Engine
    E, T, k, s0 = 16, 70, 5, 25
    shapes = _subjects(E + 1, 4)
    new = shapes[E]                                     # env k's second subject
    _, raw = _stream(E + 1, T, "qpos", 5)
    g = raw[E]                                          # env k's second stream

    def engine(rows):
        e = Engine(E, model=basis.humanoid, **TRACK_KW)
        e.track_subjects_enable(basis)
        e.track_begin(6, "qpos")
        e.track_set_subjects(np.arange(E), rows)
        return e, Run(e)
    (x, rx), (y, ry) = engine(shapes[:E]), engine(shapes[:E])
    for e in (x, y):
        e.track_reset(np.arange(E), _frames(t, raw[:E, :2]))
    for j in range(s0):
        nxt = None if j == 0 else _frames(t, raw[:E, j + 1])
        rx.step(nxt)
        ry.step(nxt)
    graphs = x.track_graph_count
    x.track_set_subjects([k], new[None])
    x.track_reset([k], _frames(t, g[None, :2]))
    assert x.track_graph_count == graphs == 2
    z_rows = shapes[:E].copy()
    z_rows[k] = new
    z, rz = engine(z_rows)
    z0 = raw[:E, s0:s0 + 2].copy()
    z0[k] = g[:2]
    z.track_reset(np.arange(E), _frames(t, z0))
    mask = np.ones(E, np.int32)
    mask[k] = 0
    for j in range(s0, T - 2):
        nxt = raw[:E, j + 1].copy()
        if j > s0:
            nxt[k] = g[j - s0 + 1]
        m = _frames(t, mask) if j == s0 else None
        sx, wx, fx = (a.cpu().numpy() for a in rx.step(_frames(t, nxt), m))
        sy, wy, fy = (a.cpu().numpy() for a in ry.step(_frames(t, raw[:E, j + 1]), m))
        others = np.arange(E) != k
        assert np.array_equal(sx[others], sy[others]) and np.array_equal(wx[others], wy[others]) and np.array_equal(fx[others], fy[others]), j
        zn = raw[:E, j + 1].copy()
        zn[k] = g[j - s0 + 1]
        sz, wz, fz = (a.cpu().numpy() for a in rz.step(None if j == s0 else _frames(t, zn)))
        assert np.array_equal(sx[k], sz[k]) and wx[k] == wz[k] and fx[k] == fz[k], j
    assert x.track_graph_count == y.track_graph_count == 3     # one more for the masked step, in both: the swap itself captured nothing
    assert z.track_graph_count == 2
    for e in (x, y, z):
        e.close()


def test_refusals_leave_tables_and_trajectories(basis):
    t = _torch()
    from uhc_b200.engine import Engine
    from uhc_b200.subject_body import SubjectBasis
    E, T = 8, 40
    shapes = _subjects(E, 6)
    _, raw = _stream(E, T, "qpos", 7)

    def engine():
        e = Engine(E, model=basis.humanoid, **TRACK_KW)
        e.track_subjects_enable(basis)
        e.track_begin(6, "qpos")
        e.track_set_subjects(np.arange(E), shapes)
        e.track_reset(np.arange(E), _frames(t, raw[:, :2]))
        return e, Run(e)
    (x, rx), (y, ry) = engine(), engine()
    for j in range(10):
        nxt = None if j == 0 else _frames(t, raw[:, j + 1])
        rx.step(nxt)
        ry.step(nxt)
    tables = [x.track_subject_tables(e) for e in range(E)]
    L, h = x.lib, x.h
    keep = []

    def call(ids, rows, eng=x):
        ids, rows = np.ascontiguousarray(ids, np.int32), np.ascontiguousarray(rows, np.float64)
        keep.append((ids, rows))
        return eng.lib.uhc_track_set_subjects(eng.h, C.c_int(len(ids)), ids.ctypes.data_as(C.POINTER(C.c_int)),
                                              rows.ctypes.data_as(C.POINTER(C.c_double)), None)
    ok = shapes[:2]
    nan, bad_g, frac_g, inv = ok.copy(), ok.copy(), ok.copy(), ok.copy()
    nan[1, 3] = np.nan
    bad_g[0, 16] = 3
    frac_g[1, 16] = 0.5
    inv[1, 0], inv[1, 16] = -1.5, 0                     # neutral at scale -0.5: every body inverted
    err = lambda: L.uhc_last_error().decode()
    assert call([0, E], ok) == -2 and call([-1, 0], ok) == -2 and call([2, 2], ok) == -2
    assert call([0, 1], nan) == -2 and "non-finite" in err()
    assert call([0, 1], bad_g) == -2 and call([0, 1], frac_g) == -2
    assert call([3, 4], inv) == -2 and "det A" in err()
    assert L.uhc_track_set_subjects(h, C.c_int(0), None, None, None) == -2
    only = Engine(E, model=basis.humanoid, **TRACK_KW)           # a basis without the male model
    only.track_subjects_enable(SubjectBasis.from_models(basis.humanoid, uniform_scale_model()))
    only.track_begin(6, "qpos")
    assert call([0, 1], ok, only) == -2 and "no basis" in err()
    only.close()
    plain = Engine(E, model=basis.humanoid, **TRACK_KW)          # not enabled
    plain.track_begin(6, "qpos")
    assert call([0, 1], ok, plain) == -2 and "not enabled" in err()
    plain.track_end()
    assert call([0, 1], ok, plain) == -2 and "not tracking" in err()
    assert plain.lib.uhc_track_subjects_enable(plain.h, None) == -2
    plain.close()
    assert L.uhc_track_subjects_enable(h, C.byref(basis.struct())) == -2 and "tracking is active" in err()
    for e in range(E):
        now = x.track_subject_tables(e)
        assert all(np.array_equal(now[n], tables[e][n]) for n in now), e
    for j in range(10, T - 2):
        sx, wx, fx = (a.cpu().numpy() for a in rx.step(_frames(t, raw[:, j + 1])))
        sy, wy, fy = (a.cpu().numpy() for a in ry.step(_frames(t, raw[:, j + 1])))
        assert np.array_equal(sx, sy) and np.array_equal(wx, wy) and np.array_equal(fx, fy), j
    x.close()
    y.close()


def test_evaluation_after_the_tables_move(basis):
    from uhc_b200 import motion_lib as ML
    from uhc_b200.engine import Engine
    rng = np.random.default_rng(8)
    E = 6
    ms = ML.MotionSet(_clips(rng, [30, 24, 28, 20], "qpos"))
    eng = Engine(E, model=basis.humanoid, **TRACK_KW)
    eng.load_motions(ms)
    run = Run(eng, fail_safe=True)
    ev = lambda: eng.eval_run(np.arange(4), run.pol, run.log_std, run.zf.stats, run.zf.clip, True, window=7, record_states=True, floor=True)
    before = ev()
    assert eng.eval_graph_count == 1
    eng.track_subjects_enable(basis)
    after = ev()
    assert eng.eval_graph_count == 1                    # the graph over the old tables was dropped, not kept beside the new one
    for k in ("frames", "states", "floor", "nframes", "last_t", "fail_any", "reward_sum"):
        assert np.array_equal(before[k], after[k]), k
    eng.close()
