"""GPU: SMPL linear blend skinning on the device (include/uhc_mesh.h) against the fp64 restatement tests/smpl_ref.py, its floor reduction
against the reference's formulas, determinism, bad arguments, and full_eval through AgentCopycat.  The SMPL model files are licence-gated,
so the models are synthetic: one built from this project's neutral humanoid (its hull vertices at rest in SMPL's y-up frame, the rest
joints, weights on the owning body and its parent, shape and pose blends at SMPL-like magnitudes), and small random ones."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.smpl_ref import floor_rows, smpl_forward
from tests.test_smpl_model import PARENTS

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-5


def humanoid_model(seed=0):
    from uhc_b200 import model as M
    hm = M.HumanoidModel()
    gpos = np.load(M.ASSET)["body_gpos"].astype(np.float64)
    order = [hm.body_names.index(n) for n in hm.SMPL_BONE_ORDER]             # SMPL joint -> body
    inv = {b: j for j, b in enumerate(order)}
    parents = np.array([-1] + [inv[int(hm.parent[order[j]])] for j in range(1, 24)], np.int32)
    to_smpl = lambda x: np.stack([x[..., 0], x[..., 2], -x[..., 1]], -1)       # z-up world -> SMPL's y-up
    J = to_smpl(gpos[order])
    vt, owner = [], []
    for j, b in enumerate(order):
        v = hm.hull[hm.hull_adr[b]:hm.hull_adr[b] + hm.hull_num[b]] + gpos[b]
        vt.append(to_smpl(v)); owner += [j] * len(v)
    vt, owner = np.concatenate(vt), np.array(owner)
    V = len(vt)
    reg = np.zeros((24, V))
    for j in range(24):                                                        # min-norm weights of the body's vertices with sum 1 that give J
        idx = np.nonzero(owner == j)[0]
        A = np.vstack([vt[idx].T, np.ones(len(idx))])
        reg[j, idx] = np.linalg.lstsq(A, np.append(J[j], 1.0), rcond=None)[0]
    w = np.zeros((V, 24))
    w[np.arange(V), owner] = 0.7
    w[np.arange(V)[owner > 0], parents[owner[owner > 0]]] += 0.3
    w[owner == 0, 0] = 1.0
    rng = np.random.RandomState(seed)
    return dict(v_template=vt, shapedirs=rng.normal(0, 0.004, (V, 3, 10)), posedirs=rng.normal(0, 0.003, (V, 3, 207)), J_regressor=reg,
                weights=w, parents=parents)


def random_model(V, seed=0):
    rng = np.random.RandomState(seed)
    w = rng.rand(V, 24) * (rng.rand(V, 24) < 0.15)
    w[np.arange(V), rng.randint(0, 24, V)] += 1.0
    w /= w.sum(1, keepdims=True)
    return dict(v_template=rng.normal(0, 0.4, (V, 3)), shapedirs=rng.normal(0, 0.01, (V, 3, 10)), posedirs=rng.normal(0, 0.01, (V, 3, 207)),
                J_regressor=rng.dirichlet(np.ones(V), 24), weights=w, parents=np.array(PARENTS, np.int32))


def random_poses(n, rng, scale=0.6):
    pose = rng.normal(0, scale, (n, 72))
    ax = rng.normal(size=(n, 24, 3))
    ax /= np.linalg.norm(ax, axis=2, keepdims=True)
    k = n // 4
    pose[:k] = (ax[:k] * rng.choice([0.0, 1e-9, 1e-4, np.pi - 1e-6, np.pi], (k, 24, 1))).reshape(k, 72)   # angles near 0 and pi
    trans = rng.normal(0, 1.0, (n, 3))
    return pose, trans


@pytest.fixture(scope="module")
def eng():
    from uhc_b200.engine import Engine
    e = Engine(8)
    yield e
    e.close()


def _mesh(e, model, pose, trans, betas, bidx):
    e.mesh_init(model)
    v, j = e.smpl_mesh(pose, trans, betas, bidx)
    return v.cpu().numpy(), j.cpu().numpy()


def _against_ref(model, pose, trans, betas, bidx, v, j):
    b = betas[np.zeros(len(pose), int) if bidx is None else bidx]
    rv, rj = smpl_forward(model, pose, trans, b)
    assert np.abs(v - rv).max() < TOL and np.abs(j - rj).max() < TOL
    return rv


def test_golden_clips_through_qpos_to_smpl(eng):
    m = humanoid_model()
    for clip in ("expert_sway.npz", "expert_kick.npz"):
        q = np.load(os.path.join(GOLDEN, clip))["qpos"]
        pose, trans = eng.qpos_to_smpl(q)
        betas = np.random.RandomState(1).uniform(-3, 3, (2, 10))
        bidx = np.arange(len(q), dtype=np.int32) % 2
        eng.mesh_init(m)
        v, j = eng.smpl_mesh(pose, trans, betas, bidx)
        _against_ref(m, pose.cpu().numpy(), trans.cpu().numpy(), betas, bidx, v.cpu().numpy(), j.cpu().numpy())
        vq, jq = eng.qpos_mesh(q, betas, bidx)                                # the chained convenience gives the same bits
        assert np.array_equal(vq.cpu().numpy(), v.cpu().numpy()) and np.array_equal(jq.cpu().numpy(), j.cpu().numpy())


@pytest.mark.parametrize("V,n", [(1, 0), (1, 1), (33, 7), (33, 41), (6890, 5), (1199, 33)])
def test_random_models_and_poses(eng, V, n):
    m = random_model(V, seed=V) if V != 1199 else humanoid_model()
    rng = np.random.RandomState(n)
    pose, trans = random_poses(n, rng)
    betas = rng.uniform(-3, 3, (3, 10))
    bidx = rng.randint(0, 3, n).astype(np.int32)
    v, j = _mesh(eng, m, pose, trans, betas, bidx)
    assert v.shape == (n, V, 3) and v.dtype == np.float32 and j.shape == (n, 24, 3)
    if n:
        _against_ref(m, pose, trans, betas, bidx, v, j)


def test_more_rows_than_a_grid_dimension(eng):
    m = random_model(1, seed=5)
    n = 70001
    rng = np.random.RandomState(6)
    pose, trans = random_poses(n, rng)
    betas = rng.uniform(-3, 3, (2, 10))
    bidx = rng.randint(0, 2, n).astype(np.int32)
    v, j = _mesh(eng, m, pose, trans, betas, bidx)
    _against_ref(m, pose, trans, betas, bidx, v, j)
    fl = eng.smpl_floor(pose, trans, betas, bidx).cpu().numpy()
    want = floor_rows(v)
    assert np.abs(fl - want).max() < 1e-9 and np.array_equal(fl[:, 4], want[:, 4])


def _floor_case(eng, n=301, seed=7):
    m = humanoid_model()
    rng = np.random.RandomState(seed)
    pose, trans = random_poses(n, rng, scale=0.3)
    pose[:, :3] = [np.pi / 2, 0, 0]                                           # upright in the z-up world, as qpos_to_smpl writes it
    betas = rng.uniform(-3, 3, (2, 10))
    bidx = (np.arange(n) // 50 % 2).astype(np.int32)
    trans = np.cumsum(rng.normal(0, 0.01, (n, 3)), 0)                        # drifting, and the lowest vertex within a few cm of the floor
    trans[:, 2] = -smpl_forward(m, pose, np.zeros((n, 3)), betas[bidx])[0][:, :, 2].min(1) + rng.normal(0, 0.01, n)
    first = np.zeros(n, np.int32)
    first[[0, 77, 150]] = 1
    return m, pose, trans, betas, bidx, first


def test_floor_rows(eng):
    m, pose, trans, betas, bidx, first = _floor_case(eng)
    v, _ = _mesh(eng, m, pose, trans, betas, bidx)
    fl = eng.smpl_floor(pose, trans, betas, bidx, first).cpu().numpy()
    want = floor_rows(v, first)
    assert (want[:, 4] > 0).any() and (want[:, 2] > 0).any()                  # the case has vertices below the floor and skating
    assert np.abs(fl - want).max() < 1e-9 and np.array_equal(fl[:, 4], want[:, 4])
    rv, _ = smpl_forward(m, pose, trans, betas[bidx])                         # against the fp64 mesh where no vertex is near the floor
    ref = floor_rows(rv, first)
    near = np.abs(rv[:, :, 2]).min(1) < 2e-5
    prev_near = np.concatenate([[False], near[:-1]])
    ok = ~near & ~prev_near
    assert ok.sum() > len(ok) // 2 and np.abs(fl[ok, :4] - ref[ok, :4]).max() < 0.02 and np.array_equal(fl[ok, 4], ref[ok, 4])
    one = eng.smpl_floor(pose, trans, betas, bidx).cpu().numpy()              # first = None: one clip
    assert np.abs(one - floor_rows(v)).max() < 1e-9


def test_bit_identical_alone_and_in_a_batch(eng):
    m = random_model(6890, seed=11)
    eng.mesh_init(m)
    rng = np.random.RandomState(12)
    n = 10000
    pose, trans = random_poses(n, rng)
    trans[:, 2] = rng.normal(0, 0.2, n)
    betas = rng.uniform(-3, 3, (4, 10))
    bidx = rng.randint(0, 4, n).astype(np.int32)
    first = (rng.rand(n) < 0.05).astype(np.int32)
    va, ja = eng.smpl_mesh(pose, trans, betas, bidx)
    vb, jb = eng.smpl_mesh(pose, trans, betas, bidx)
    fa = eng.smpl_floor(pose, trans, betas, bidx, first).cpu().numpy()
    fb = eng.smpl_floor(pose, trans, betas, bidx, first).cpu().numpy()
    assert np.array_equal(va.cpu().numpy(), vb.cpu().numpy()) and np.array_equal(ja.cpu().numpy(), jb.cpu().numpy()) and np.array_equal(fa, fb)
    va, ja = va.cpu().numpy(), ja.cpu().numpy()
    for r in (0, 1, 15, 16, 17, 4999, n - 1):
        b = np.array([bidx[r]], np.int32)
        v1, j1 = eng.smpl_mesh(pose[r:r + 1], trans[r:r + 1], betas, b)
        assert np.array_equal(v1.cpu().numpy()[0], va[r]) and np.array_equal(j1.cpu().numpy()[0], ja[r])
        lo = max(r - 1, 0)                                                    # the row with its predecessor only
        f2 = eng.smpl_floor(pose[lo:r + 1], trans[lo:r + 1], betas, bidx[lo:r + 1], np.array([1, first[r]][-(r + 1 - lo):], np.int32)).cpu().numpy()
        assert np.array_equal(f2[-1], fa[r])


def test_bad_arguments_leave_the_engine_usable(eng):
    lib = eng.lib
    m = random_model(33, seed=3)
    eng.mesh_init(m)
    t = eng.torch
    d = lambda *s: t.zeros(*s, dtype=t.float64, device="cuda")
    pose, trans, betas = d(4, 72), d(4, 3), d(2, 10)
    vo = t.zeros(4, 33, 3, dtype=t.float32, device="cuda")
    fo = d(4, 5)
    p = lambda x: C.c_void_p(x.data_ptr() if x is not None else None)
    idx = lambda *v: t.tensor(v, dtype=t.int32, device="cuda")

    def mesh(n=4, ps=pose, tr=trans, nb=2, bt=betas, bi=None, e=eng.h):
        return lib.uhc_smpl_mesh(e, C.c_long(n), p(ps), p(tr), C.c_int(nb), p(bt), p(bi), p(vo), None, None)

    def floor(n=4, out=fo, bi=None):
        return lib.uhc_smpl_floor(eng.h, C.c_long(n), p(pose), p(trans), C.c_int(2), p(betas), p(bi), None, p(out), None)
    assert mesh(n=-1) == -2 and mesh(ps=None) == -2 and mesh(tr=None) == -2 and mesh(bt=None) == -2 and mesh(nb=0) == -2 and mesh(e=None) == -2
    assert mesh(bi=idx(0, 1, 2, 0)) == -2 and mesh(bi=idx(0, -1, 0, 0)) == -2 and floor(bi=idx(0, 0, 0, 2)) == -2 and floor(out=None) == -2
    bad = dict(m, parents=np.array([-1] + [5] * 23, np.int32))
    with pytest.raises(ValueError):
        eng.mesh_init(bad)                                                    # refused: the model loaded before stays
    assert mesh() == 0 and floor() == 0 and mesh(n=0) == 0
    v, _ = eng.smpl_mesh(pose, trans, betas, idx(0, 1, 1, 0))
    assert np.abs(v.cpu().numpy() - m["v_template"][None]).max() < TOL
    from uhc_b200.engine import Engine
    other = Engine(2)
    try:
        assert lib.uhc_smpl_mesh(other.h, C.c_long(4), p(pose), p(trans), C.c_int(2), p(betas), None, p(vo), None, None) == -2   # no model
    finally:
        other.close()


def test_full_eval_through_the_dropin(tmp_path, monkeypatch):
    """eval_policy with full_eval: pentration / skate from the mesh, the same on the host loop and the device evaluation, equal to the
    restatement over the dumped qpos; the dump carries vertices and joints.  Without the model file it names the path it looked for."""
    import joblib
    import torch
    from tests.test_gpu_dropin import _cfg
    from uhc.agents import agent_dict
    old = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)
    try:
        cfg = _cfg(tmp_path, monkeypatch)
        cfg.cfg_dict.update(full_eval=True, eval_dump_motion=True)
        agent = agent_dict[cfg.agent_name](cfg, torch.float64, torch.device("cuda", index=0), training=True, checkpoint_epoch=0)
        with pytest.raises(FileNotFoundError, match=os.path.join("data", "smpl")):
            agent.eval_policy(epoch=0)
        m = humanoid_model()
        os.makedirs(tmp_path / "data" / "smpl")
        kt = np.stack([np.where(m["parents"] < 0, 4294967295, m["parents"]), np.arange(24)]).astype(np.int64)
        np.savez(tmp_path / "data" / "smpl" / "SMPL_NEUTRAL.npz", kintree_table=kt, **{k: v for k, v in m.items() if k != "parents"})
        name = agent.data_loader.name
        out = {}
        for on_device in (True, False):
            cfg.cfg_dict["eval_on_device"] = on_device
            out[on_device] = agent.eval_policy(epoch=int(on_device), dump=True)[0][f"coverage_{name}"]
            for k in ("pentration", "skate", "pentration_gt", "skate_gt"):
                assert np.isfinite(out[on_device][k]) and out[on_device][k] >= 0, k
        for k in ("pentration", "skate", "pentration_gt", "skate_gt"):
            assert out[True][k] == out[False][k], k
        res = joblib.load(os.path.join(cfg.output_dir, f"1_{name}_coverage_full.pkl"))
        eng = agent.agent.engine
        for key, r in res.items():
            T = len(r["pred"])
            assert r["pred_vertices"].shape == (T, len(m["v_template"]), 3) and r["pred_vertices"].dtype == np.float32
            assert r["gt_vertices"].shape == r["pred_vertices"].shape and r["pred_joints"].shape == (T, 24, 3) and r["gt_joints"].shape == (T, 24, 3)
            c = agent.data_loader.data_keys.index(key)
            beta = np.asarray(agent.data_loader.shapes[c], np.float64)[:10]          # has_shape: true in this config
            assert np.abs(beta).max() > 0
            for who in ("pred", "gt"):
                pose, trans = eng.qpos_to_smpl(r[who], None if eng.clip_models is None else int(eng.clip_models[c]))
                rv, rj = smpl_forward(m, pose.cpu().numpy(), trans.cpu().numpy(), np.repeat(beta[None], T, 0))
                assert np.abs(r[who + "_vertices"] - rv).max() < TOL and np.abs(r[who + "_joints"] - rj).max() < TOL
                fr = floor_rows(r[who + "_vertices"])
                sfx = "" if who == "pred" else "_gt"
                assert abs(r["pentration" + sfx] - fr[:, 1].mean()) < 1e-9 and abs(r["skate" + sfx] - (fr[1:, 2].mean() if T > 1 else 0.0)) < 1e-9
        cfg.cfg_dict["eval_floor_metrics"] = True
        with pytest.raises(ValueError, match="full_eval.*eval_floor_metrics"):
            agent.eval_policy(epoch=2)
        eng.close()
    finally:
        torch.set_default_dtype(old)
