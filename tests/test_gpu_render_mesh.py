"""GPU: the mesh renderer (include/uhc_render.h uhc_render_mesh) -- rgb, depth and label against the host emulation bit for bit, a frame
alone against a batch, render_smpl against its parts, bad arguments and output bounds, BatchedAgent.render_motion(body="mesh") against
render_smpl, and the drop-in's mesh videos.  The meshes are synthetic (tests/mesh_scenes.py): a real SMPL file is licence-gated."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.emu import render_emu, render_mesh_emu
from tests.mesh_scenes import hull_mesh, pose_verts, smpl_sized_model
from tests.test_gpu_render import _agent_clips, _qpos
from uhc_b200.render_mesh import build_tables

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def setup():
    from uhc_b200.engine import Engine, UhcRenderMesh
    v, f, owner, w = hull_mesh()
    e = Engine(4)
    tb = build_tables(f, w, v)                                      # the triangulated hulls' topology, uploaded through the C ABI
    e._rmesh = UhcRenderMesh.of(tb, len(v))
    assert e.lib.uhc_render_mesh_init(e.h, C.byref(e._rmesh)) == 0
    yield e, tb, v, owner
    e.close()


def _scene(v, owner, n, seed):
    P = np.zeros((n, 2, 24, 12), np.float32)
    P[:, 0], P[:, 1] = render_emu.pose(_qpos(n, seed)), render_emu.pose(_qpos(n, seed + 100))
    X = pose_verts(P, v, owner)
    return P, X


CASES = [((1, 1), 1, True, dict(fovy=2.0, lookat=(0.0, 0.0, 0.6), distance=3.0)),
         ((17, 9), 3, False, dict()),
         ((17, 9), 1024, True, dict(focus=True, shift_expert=1.0)),
         ((320, 180), 3, True, dict(focus=True, shift_expert=1.0, distance=3.5)),
         ((320, 180), 3, False, dict(azimuth=120.0, elevation=-20.0)),
         ((320, 180), 3, True, dict(hide_expert=True, shift_expert=0.7)),
         ((320, 180), 3, True, dict(hide_im=True, shift_expert=0.7)),
         ((640, 360), 1, True, dict(shift_expert=1.0, distance=3.0))]


@pytest.mark.parametrize("case", range(len(CASES)))
def test_mesh_equals_emulation_bit_for_bit(setup, case):
    import torch
    eng, tb, v, owner = setup
    size, n, ghost, cam = CASES[case]
    P, X = _scene(v, owner, n, case)
    root = P[:, 0, 0, 9:12].copy()
    xs = torch.tensor(X[:, 0], device="cuda")
    gs = torch.tensor(X[:, 1], device="cuda") if ghost else None
    rgb, dep, lab = eng.render_mesh(xs, gs, torch.tensor(root, device="cuda"), cam, size, depth=True, label=True)
    torch.cuda.synchronize()
    erg, edp, elb = render_mesh_emu.render_mesh(tb, X[:, 0], size, cam, X[:, 1] if ghost else None, root)
    assert np.array_equal(rgb.cpu().numpy(), erg)
    assert np.array_equal(dep.cpu().numpy().view(np.uint32), edp.view(np.uint32))
    assert np.array_equal(lab.cpu().numpy(), elb)
    if size != (1, 1):
        assert (elb >= 2).any() and (elb == 1).any()
    if n == 1024:                                                   # a frame alone gives the bits it has inside the batch
        for i in (0, 517, 1023):
            one = eng.render_mesh(xs[i:i + 1].contiguous(), gs[i:i + 1].contiguous(), torch.tensor(root[i:i + 1], device="cuda"), cam, size,
                                  depth=True, label=True)
            for a, b in zip(one, (rgb, dep, lab)):
                assert torch.equal(a[0], b[i])


def test_outputs_stay_in_bounds_and_bad_arguments(setup):
    """canary bytes around every output stay untouched; refused calls return -2 and write nothing"""
    import torch
    from uhc_b200.engine import Engine, make_camera
    eng, tb, v, owner = setup
    W, H, n, G = 33, 17, 4, 4096
    P, X = _scene(v, owner, n, 3)
    V = len(v)
    xs, gs = torch.tensor(X[:, 0], device="cuda"), torch.tensor(X[:, 1], device="cuda")
    root = torch.tensor(P[:, 0, 0, 9:12].copy(), device="cuda")
    npx = n * H * W
    rgb = torch.full((npx * 3 + 2 * G,), 0xA5, dtype=torch.uint8, device="cuda")
    lab = torch.full((npx + 2 * G,), 0x5A, dtype=torch.uint8, device="cuda")
    dep = torch.full((npx + 2 * G,), -7.0, dtype=torch.float32, device="cuda")
    p = lambda x: C.c_void_p(x.data_ptr())
    good = make_camera(dict(shift_expert=1.0, focus=True))

    def call(cam=good, W=W, H=H, n=n, verts=xs, ghost=gs, root=root, nvert=V, out=rgb, e=eng):
        return e.lib.uhc_render_mesh(e.h, C.byref(cam) if cam is not None else None, C.c_int(W), C.c_int(H), C.c_long(n),
                                     p(verts) if verts is not None else None, p(ghost) if ghost is not None else None,
                                     p(root) if root is not None else None, C.c_int(nvert),
                                     C.c_void_p(out.data_ptr() + G) if out is not None else None, C.c_void_p(dep.data_ptr() + 4 * G),
                                     C.c_void_p(lab.data_ptr() + G), e._stream())

    bad_cams = []
    for k, val in (("distance", 0.0), ("fovy", 180.0), ("azimuth", float("nan"))):
        c = make_camera()
        setattr(c, k, val)
        bad_cams.append(c)
    rcs = [call(cam=None), call(W=0), call(H=16385), call(n=-1), call(verts=None), call(out=None), call(root=None), call(nvert=V - 1)]
    rcs += [call(cam=c) for c in bad_cams]
    e2 = Engine(2)
    rcs.append(call(e=e2))                                          # no uhc_render_mesh_init
    e2.close()
    assert rcs == [-2] * len(rcs)
    torch.cuda.synchronize()
    for buf, fill in ((rgb, 0xA5), (lab, 0x5A), (dep, -7.0)):
        assert (buf == fill).all(), "a refused call wrote its output"
    assert call() == 0
    torch.cuda.synchronize()
    for buf, fill, m in ((rgb, 0xA5, npx * 3), (lab, 0x5A, npx), (dep, -7.0, npx)):
        assert (buf[:G] == fill).all() and (buf[G + m:] == fill).all()
        assert not (buf[G:G + m] == fill).all()
    assert call(root=None, cam=make_camera()) == 0                  # the root is needed only with focus


def test_init_refusals_keep_the_previous_tables(setup):
    eng, tb, v, owner = setup
    from uhc_b200.engine import UhcRenderMesh
    V = len(v)
    bad = dict(tb, face=np.where(np.arange(tb["face"].size).reshape(-1, 3) == 5, V, tb["face"]).astype(np.int32))
    assert eng.lib.uhc_render_mesh_init(eng.h, C.byref(UhcRenderMesh.of(bad, V))) == -2
    # 4096 one-face leaves: their boxes for two humanoids do not fit the trace's shared memory
    F = 4096
    big = dict(face=np.zeros((F, 3), np.int32) + np.arange(3, dtype=np.int32), face_body=np.zeros(F, np.int32),
               leaf_first=np.arange(F + 1, dtype=np.int32), body_leaf=np.array([0] + [F] * 24, np.int32))
    assert eng.lib.uhc_render_mesh_init(eng.h, C.byref(UhcRenderMesh.of(big, V))) == -2
    test_mesh_equals_emulation_bit_for_bit(setup, 1)                # the previous tables still draw


def _smpl_engine(variants=None):
    from uhc_b200.engine import Engine
    m = smpl_sized_model()
    e = Engine(4, model=variants[0] if variants else None, variants=variants)
    e.mesh_init(m)
    e.render_mesh_init(m)
    return e, m


def test_render_smpl_is_its_parts_bit_for_bit():
    """render_smpl = render_mesh(smpl_mesh(qpos_to_smpl(...))) on an SMPL-sized model (6890 vertices) with two betas rows; the focus root is
    the hull renderer's"""
    import torch
    e, m = _smpl_engine()
    n = 6
    qa, qb = _qpos(n, 40), _qpos(n, 41)
    betas = np.random.default_rng(3).normal(0, 1.0, (2, 10))
    bidx = np.array([0, 1, 1, 0, 1, 0], np.int32)
    cam = dict(focus=True, shift_expert=1.0, distance=3.5)
    e.render(qa, qb, camera=cam, size=(16, 9))                      # the hull renderer's upload leaves the mesh tables in place
    a = e.render_smpl(qa, qb, betas, bidx, camera=cam, size=(160, 90), depth=True, label=True)
    pa, ta = e.qpos_to_smpl(qa)
    pb, tb_ = e.qpos_to_smpl(qb)
    va = e.smpl_mesh(pa, ta, betas, bidx, joints=False)[0]
    vb = e.smpl_mesh(pb, tb_, betas, bidx, joints=False)[0]
    root = torch.tensor(qa[:, :3], dtype=torch.float32, device="cuda")
    assert torch.equal(root, e.render_pose(qa)[:, 0, 0, 9:12])      # framed exactly like the hull frame of the same qpos
    b = e.render_mesh(va, vb, root, cam, (160, 90), depth=True, label=True)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    assert (a[2] >= 2).any() and (a[2] >= 26).any()
    e.close()


def test_render_motion_mesh_equals_render_smpl_and_ignores_chunking():
    from uhc_b200.agent import BatchedAgent
    from uhc_b200.model import HumanoidModel
    rng = np.random.default_rng(3)
    variants = [HumanoidModel(), HumanoidModel(scale=rng.uniform(0.9, 1.1, 24))]
    clips = _agent_clips()
    ag = BatchedAgent(4, clips, [np.zeros(17)] * len(clips), policy_hsize=(128, 64), value_hsize=(64,), seed=2, body_diff_thresh=0.2,
                      auto_reset=False, model=variants[0], variants=variants, clip_models=[0, 1, 1, 0, 1])
    m = smpl_sized_model()
    ag.engine.mesh_init(m)
    ag.engine.render_mesh_init(m)
    order = [3, 0, 4]
    betas = rng.normal(0, 1.0, (3, 10))
    size, cam = (80, 45), dict(focus=True, shift_expert=1.0)
    a = ag.render_motion(order, True, size, cam, body="mesh", betas=betas)
    got = {}
    per = 80 * 45 * 3 + 2 * 6890 * 12
    ag.render_motion(order, True, size, cam, max_bytes=3 * per, body="mesh", betas=betas, writer=lambda i, ch: got.__setitem__(i, [c for c in ch]))
    for i, (c, x) in enumerate(zip(order, a)):
        nf = len(x["pred"])
        assert all(len(ch) <= 3 for ch in got[i]) and np.array_equal(np.concatenate(got[i]), x["frames"])
        want = ag.engine.render_smpl(x["pred"], x["gt"], betas[i], variants=int(ag.engine.clip_models[c]), camera=cam, size=size)[0]
        assert np.array_equal(x["frames"], want.cpu().numpy()) and x["frames"].shape == (nf, 45, 80, 3)
    hull = ag.render_motion(order[:1], True, size, cam)[0]["frames"]
    assert not np.array_equal(hull, a[0]["frames"])                 # the default stays the hulls
    ag.engine.close()


def test_dropin_mesh_videos(tmp_path, monkeypatch):
    """AgentCopycat.render_motion(body="mesh") from a working directory holding data/smpl/SMPL_NEUTRAL.npz writes decodable mp4 and mjpeg
    files under the usual names; without the model it names the path, without faces the key"""
    import cv2
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, test_clips=2)
    ld = agent.test_data_loaders[0]
    with pytest.raises(FileNotFoundError, match=os.path.join("data", "smpl")):
        agent.render_motion(epoch=1, loaders=[ld], out_dir=str(tmp_path / "x"), size=(96, 54), body="mesh")
    m = smpl_sized_model()
    os.makedirs(tmp_path / "data" / "smpl")
    kt = np.stack([np.where(m["parents"] < 0, 4294967295, m["parents"]), np.arange(24)]).astype(np.int64)
    arrays = {k: x for k, x in m.items() if k not in ("parents", "faces")}
    np.savez(tmp_path / "data" / "smpl" / "SMPL_NEUTRAL.npz", kintree_table=kt, **arrays)
    with pytest.raises(ValueError, match="key f"):
        agent.render_motion(epoch=1, loaders=[ld], out_dir=str(tmp_path / "x"), size=(96, 54), body="mesh")
    np.savez(tmp_path / "data" / "smpl" / "SMPL_NEUTRAL.npz", kintree_table=kt, f=m["faces"], **arrays)
    agent._mesh_ready = False
    ev = agent.export_motion(epoch=0, dump=False)[ld.name]
    for video, ext in (("mp4", "mp4"), ("mjpeg", "avi")):
        out = agent.render_motion(epoch=7, loaders=[ld], out_dir=str(tmp_path / video), size=(96, 54), video=video, body="mesh")[ld.name]
        for key, path in out.items():
            assert os.path.basename(path) == f"{key}_{cfg.id}_7_0.{ext}"
            cap = cv2.VideoCapture(path)
            k = 0
            while True:
                ok, fr = cap.read()
                if not ok:
                    break
                assert fr.shape == (54, 96, 3)
                k += 1
            cap.release()
            assert k == len(ev[key]["pred"])
    agent.agent.engine.close()


def test_seam_rays_on_the_device(setup):
    """tests/test_render_mesh_ref.py's rays through leaf seams on the flat-leaved cube, on the GPU: the emulation's bits, stopping at the
    surface"""
    import torch
    from tests.mesh_scenes import cube_mesh, seam_rays
    from uhc_b200.engine import Engine, UhcRenderMesh
    cv, cf, cowner, cw = cube_mesh()
    ctb = build_tables(cf, cw, cv)
    e = Engine(2)
    m = UhcRenderMesh.of(ctb, len(cv))
    assert e.lib.uhc_render_mesh_init(e.h, C.byref(m)) == 0
    verts = torch.tensor(cv[None], device="cuda")
    for p, cam in seam_rays(ctb, cv, cowner, n_edges=150, n_verts=100):
        rgb, dep, lab = e.render_mesh(verts, camera=cam, size=(1, 1), depth=True, label=True)
        erg, edp, elb = render_mesh_emu.render_mesh(ctb, cv[None], (1, 1), cam)
        assert np.array_equal(rgb.cpu().numpy(), erg) and np.array_equal(dep.cpu().numpy().view(np.uint32), edp.view(np.uint32))
        assert np.array_equal(lab.cpu().numpy(), elb) and elb[0, 0, 0] >= 2 and edp[0, 0, 0] <= 1.5 + 1e-4
    e.close()


def test_a_smaller_model_on_another_engine_leaves_the_staging_limit(setup):
    """the trace's shared-memory limit is per function: an engine whose tables need more than 48 KB of staging still draws after another
    engine uploads a small model"""
    import torch
    from uhc_b200.engine import Engine, UhcRenderMesh
    eng, tb, v, owner = setup
    lf, bl = tb["leaf_first"], tb["body_leaf"]
    F = len(tb["face"])
    one = dict(tb, leaf_first=np.arange(F + 1, dtype=np.int32), body_leaf=lf[bl].astype(np.int32))   # every face a leaf: ~120 KB of staging
    big = Engine(2)
    mb = UhcRenderMesh.of(one, len(v))
    assert big.lib.uhc_render_mesh_init(big.h, C.byref(mb)) == 0
    P, X = _scene(v, owner, 2, 7)
    cam = dict(shift_expert=1.0)
    want = render_mesh_emu.render_mesh(one, X[:, 0], (64, 36), cam, X[:, 1])
    small = Engine(2)
    ms = UhcRenderMesh.of(tb, len(v))
    assert small.lib.uhc_render_mesh_init(small.h, C.byref(ms)) == 0
    got = big.render_mesh(torch.tensor(X[:, 0], device="cuda"), torch.tensor(X[:, 1], device="cuda"), camera=cam, size=(64, 36), depth=True, label=True)
    for a, b in zip(got, want):
        assert np.array_equal(a.cpu().numpy().view(np.uint8), b.view(np.uint8))
    small.close()
    big.close()


def test_render_motion_refuses_betas_of_another_length():
    from uhc_b200.agent import BatchedAgent
    clips = _agent_clips()
    ag = BatchedAgent(4, clips, [np.zeros(17)] * len(clips), policy_hsize=(128, 64), value_hsize=(64,), seed=2, auto_reset=False)
    m = smpl_sized_model()
    ag.engine.mesh_init(m)
    ag.engine.render_mesh_init(m)
    for rows in (2, 4):
        with pytest.raises(ValueError, match="betas"):
            ag.render_motion([0, 1, 2], True, (16, 9), body="mesh", betas=np.zeros((rows, 10)))
    ag.engine.close()
