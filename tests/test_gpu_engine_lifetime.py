"""GPU: an engine owns what its subsystems attach to it (uhc_b200/csrc/engine_slots.h).

- uhc_engine_destroy alone frees the evaluation, tracker, rollout, renderers, SMPL mesh, floor hulls and JPEG encoder of an engine: an
  engine created right after it, very likely at the same address, starts with none of them;
- the uhc_*_release calls and uhc_track_end stay optional and repeatable, and a later init attaches afresh."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.mesh_scenes import smpl_sized_model
from tests.test_gpu_track import _policy, _zfilter

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
E = 32
KW = dict(trail_steps=1)          # a cfg the tracker can run
SMPL_NVERT = 6890
RELEASES = ("uhc_eval_release", "uhc_track_end", "uhc_render_release", "uhc_video_release", "uhc_floor_release", "uhc_mesh_release",
            "uhc_rollout_release")


def _clip():
    """the golden clip and its shape row, as smoke() loads them"""
    z = np.load(os.path.join(ROOT, "tests", "golden", "expert_sway.npz"))
    ex = {k: z[k] for k in z.files}
    return ex, np.concatenate([ex["beta"][0], [ex["gender"][0]]])


def _assert_bare(lib, h, nvert):
    """h has no evaluation or tracker graphs, renderer, floor hulls, SMPL model or mesh tables.  Each call has n = 0 and null buffers with
    every other argument valid (default camera, 64 x 36 pixels, precision 32, pitch 76, one beta row), so a refusal can only come from the
    missing state, and nothing is launched whatever the engine holds"""
    from uhc_b200.engine import make_camera
    cam = make_camera()
    assert lib.uhc_eval_graph_count(h) == 0
    assert lib.uhc_track_graph_count(h) == 0
    calls = (("no hull planes", lambda: lib.uhc_render_bodies(h, C.byref(cam), 64, 36, C.c_long(0), None, 1, None, None, None, None, None)),
             ("no hull vertices", lambda: lib.uhc_floor_qpos(h, None, 32, C.c_long(0), C.c_long(76), None, None, None, None)),
             ("no SMPL model", lambda: lib.uhc_smpl_mesh(h, C.c_long(0), None, None, 1, None, None, None, None, None)),
             ("no mesh tables", lambda: lib.uhc_render_mesh(h, C.byref(cam), 64, 36, C.c_long(0), None, None, None, nvert, None, None, None, None)))
    for why, call in calls:
        rc = call()
        err = lib.uhc_last_error().decode()
        assert rc == -2 and why in err, (why, rc, err)


def test_engine_destroy_alone_tears_an_engine_down():
    import torch
    from uhc_b200.engine import Engine, make_cfg
    from uhc_b200.model import HumanoidModel
    ex, so = _clip()
    a = Engine(E, precision=32, **KW)
    lib = a.lib
    a.load_clips([ex], [so])
    _, pol = _policy("gauss", 1, a.obs_dim, a.act_dim)
    zf = _zfilter(a.obs_dim)
    log_std = torch.full((a.act_dim,), -2.3, device="cuda")
    a.eval_run([0], pol, log_std, zf.stats, zf.clip)                 # the evaluation's and the rollout's contexts
    a.track_begin(window=8, kind="qpos")
    q = torch.tensor(np.ascontiguousarray(ex["qpos"][:2], np.float64), device="cuda")
    a.track_reset(np.arange(E), q[None].expand(E, 2, 76).contiguous())
    state = torch.zeros(E, 223, device="cuda")
    rew, fail = torch.zeros(E, device="cuda"), torch.zeros(E, device="cuda", dtype=torch.int32)
    a.track_step(None, None, pol, log_std, zf.stats, zf.clip, True, state, rew, fail)
    rgb = a.render(ex["qpos"][:1], size=(64, 36))[0]
    a.floor_qpos(ex["qpos"][:1])
    m = smpl_sized_model()
    a.mesh_init(m)
    a.render_mesh_init(m)
    a.encode_jpeg(rgb)
    torch.cuda.synchronize()
    assert a.eval_graph_count > 0 and a.track_graph_count > 0

    # B's structs are built before A goes, with A's arguments, so nothing allocates in between
    mb = HumanoidModel()
    ms, cfg = mb.host_struct(None), make_cfg(32, **KW)
    ha = a.h.value
    lib.uhc_engine_destroy(a.h)                                       # no release call before it
    a.h = None
    hb = C.c_void_p()
    assert lib.uhc_engine_create(C.byref(ms), C.byref(cfg), C.c_int(E), C.c_int(0), C.c_int(32), C.byref(hb)) == 0
    print(f"engine A {ha:#x}, engine B {hb.value:#x}: {'same' if ha == hb.value else 'different'} address")
    try:
        _assert_bare(lib, hb, len(m["v_template"]))
    finally:
        lib.uhc_engine_destroy(hb)


def test_release_calls_stay_optional_and_repeatable():
    from uhc_b200.engine import Engine
    ex, _ = _clip()
    e = Engine(E, precision=32, **KW)
    rgb0 = e.render(ex["qpos"][:1], size=(64, 36))[0]
    e.floor_qpos(ex["qpos"][:1])
    for _ in range(2):
        for f in RELEASES:
            getattr(e.lib, f)(e.h)
    _assert_bare(e.lib, e.h, SMPL_NVERT)
    assert e.lib.uhc_render_init(e.h, C.byref(e._rhulls)) == 0     # a later init attaches afresh
    rgb1 = e.render(ex["qpos"][:1], size=(64, 36))[0]
    assert e.torch.equal(rgb0, rgb1)
    e.close()
