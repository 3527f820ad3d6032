"""GPU: the JPEG encoder (include/uhc_video.h) -- the device's bytes against the host emulation byte for byte (synthetic and rendered frames, every
size and quality of the CPU tests, n = 1, 3 and 1024, one and several scratch passes), the packed output in a poisoned allocation, bad arguments
and a short buffer, BatchedAgent.render_motion(encode="jpeg") against Engine.encode_jpeg, and the drop-in's Motion-JPEG files."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.emu import video_emu as V
from tests.test_emu_video import QUALITIES, SIZES
from tests.test_jpeg_ref import frames

pytestmark = pytest.mark.gpu

# PSNR of the decoded frames of render_motion(encode="jpeg") at q = 90 against the rendered RGB, held with margin under the 35.6 dB the host
# emulation gives on rendered 160 x 90 frames of the two humanoids
PSNR_MIN_DB = 30.0


@pytest.fixture(scope="module")
def eng():
    from uhc_b200.engine import Engine
    e = Engine(4)
    yield e
    e.close()


def _synthetic(size, n, seed=0):
    W, H = size
    smooth, noise = frames(W, H, seed)
    out = np.stack([np.roll(smooth, 5 * k, 1) for k in range(n)])
    if n > 1 and W * H <= 700000:
        out[1] = noise
    return out


def _device(eng, rgb, q):
    import torch
    data, offs = eng.encode_jpeg(torch.as_tensor(rgb, device="cuda"), q)
    return data.cpu().numpy(), offs.cpu().numpy()


def _equal(eng, rgb, q):
    d, o = _device(eng, rgb, q)
    e, eo = V.encode(rgb, q)
    assert np.array_equal(o, eo) and np.array_equal(d, e)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("q", QUALITIES)
def test_device_bytes_equal_emulation(eng, size, q):
    _equal(eng, _synthetic(size, 3 if size[0] * size[1] < 100000 else 1), q)


def test_n1024_and_several_passes(eng):
    _equal(eng, _synthetic((33, 31), 1024, 1), 90)
    _equal(eng, _synthetic((1920, 1080), 20, 2), 75)        # 16 frames of 1080p per 256 MiB pass: two passes


@pytest.mark.parametrize("ghost", [False, True])
def test_rendered_frames_equal_emulation(eng, ghost):
    from tests.test_gpu_render import _qpos
    for size in ((17, 9), (640, 360)):
        rgb = eng.render(_qpos(5, 1), _qpos(5, 2) if ghost else None, camera=dict(focus=True, shift_expert=1.0), size=size)[0].cpu().numpy()
        for q in (50, 90):
            _equal(eng, rgb, q)


def _call(eng, rgb, n, W, H, q, out, cap, offs, total):
    import torch
    p = lambda t: C.c_void_p(t.data_ptr() if t is not None else None)
    rc = eng.lib.uhc_jpeg_encode(eng.h, p(rgb), C.c_long(n), C.c_int(W), C.c_int(H), C.c_int(q), p(out), C.c_size_t(cap), p(offs), total,
                                 eng._stream())
    torch.cuda.synchronize()
    return rc


def test_packed_output_in_poisoned_allocation_and_refusals(eng):
    import torch
    rgb_h = _synthetic((65, 47), 5, 3)
    rgb = torch.as_tensor(rgb_h, device="cuda")
    want, wo = V.encode(rgb_h, 90)
    total = C.c_size_t(12345)
    out = torch.full((len(want) + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
    offs = torch.full((6,), -7, dtype=torch.int64, device="cuda")
    assert _call(eng, rgb, 5, 65, 47, 90, out, out.numel(), offs, C.byref(total)) == 0
    o = out.cpu().numpy()
    assert total.value == len(want) and np.array_equal(offs.cpu().numpy(), wo)
    assert np.array_equal(o[:len(want)], want) and (o[len(want):] == 0xA5).all()
    # -3: the size it needs, nothing written
    out.fill_(0x5A); offs.fill_(-7)
    total.value = 0
    assert _call(eng, rgb, 5, 65, 47, 90, out, len(want) - 1, offs, C.byref(total)) == -3
    assert total.value == len(want) and (out.cpu().numpy() == 0x5A).all() and (offs.cpu().numpy() == -7).all()
    assert "out_cap" in eng.lib.uhc_last_error().decode()
    # -2: nothing launched, nothing written
    bad = [(5, 0, 47, 90), (5, 65, 16385, 90), (5, 65, 47, 0), (5, 65, 47, 101), (-1, 65, 47, 90)]
    for n, W, H, q in bad:
        total.value = 99
        assert _call(eng, rgb, n, W, H, q, out, out.numel(), offs, C.byref(total)) == -2
        assert total.value == 99
    assert _call(eng, None, 5, 65, 47, 90, out, out.numel(), offs, C.byref(total)) == -2
    assert _call(eng, rgb, 5, 65, 47, 90, None, out.numel(), offs, C.byref(total)) == -2
    assert _call(eng, rgb, 5, 65, 47, 90, out, out.numel(), None, C.byref(total)) == -2
    assert _call(eng, rgb, 5, 65, 47, 90, out, out.numel(), offs, None) == -2
    assert (out.cpu().numpy() == 0x5A).all() and (offs.cpu().numpy() == -7).all()
    with pytest.raises(ValueError, match="^uhc_jpeg_encode: .*quality"):
        eng.encode_jpeg(rgb, 0)
    # a tight buffer over several passes is sized first: -3 writes nothing there either
    big = torch.as_tensor(_synthetic((1920, 1080), 17, 4), device="cuda")
    d, _ = eng.encode_jpeg(big, 90)
    out2 = torch.full((d.numel() - 1,), 0x33, dtype=torch.uint8, device="cuda")
    offs2 = torch.full((18,), -7, dtype=torch.int64, device="cuda")
    assert _call(eng, big, 17, 1920, 1080, 90, out2, out2.numel(), offs2, C.byref(total)) == -3
    assert total.value == d.numel() and (out2.cpu().numpy() == 0x33).all() and (offs2.cpu().numpy() == -7).all()
    assert eng.lib.uhc_jpeg_encode(eng.h, None, C.c_long(0), C.c_int(8), C.c_int(8), C.c_int(90), None, C.c_size_t(0), None, None, None) == 0


def test_multi_pass_calls_write_each_frame_once_at_any_capacity(eng):
    """20 frames of 1080p take two passes: written straight into out_dev when out_cap holds n worst-case frames, and through the staging
    buffer when it may not (the exact total, and the total with slack)"""
    import torch
    rgb_h = _synthetic((1920, 1080), 20, 5)
    want, wo = V.encode(rgb_h, 90)
    rgb = torch.as_tensor(rgb_h, device="cuda")
    eng.lib.uhc_jpeg_bound.restype = C.c_size_t
    bound = int(eng.lib.uhc_jpeg_bound(C.c_int(1920), C.c_int(1080)))
    assert bound == V.bound(1920, 1080)
    total = C.c_size_t(0)
    for cap in (20 * bound, len(want), len(want) + 4096):
        out = torch.full((cap,), 0xA5, dtype=torch.uint8, device="cuda")
        offs = torch.full((21,), -7, dtype=torch.int64, device="cuda")
        assert _call(eng, rgb, 20, 1920, 1080, 90, out, cap, offs, C.byref(total)) == 0
        o = out.cpu().numpy()
        assert total.value == len(want) and np.array_equal(offs.cpu().numpy(), wo) and np.array_equal(o[:len(want)], want)
        assert (o[len(want):] == 0xA5).all()
        del out


def test_render_motion_time_split():
    """render_times: the encoder's seconds in encoding only, the writer's in writer only (an encoder and a writer slowed by 0.1 s a call)"""
    import time
    from uhc_b200.agent import BatchedAgent
    from tests.test_gpu_render import _agent_clips
    clips = _agent_clips()
    ag = BatchedAgent(4, clips, [np.zeros(17)] * len(clips), policy_hsize=(128, 64), value_hsize=(64,), seed=2, body_diff_thresh=0.2,
                      auto_reset=False)
    order = [3, 0, 4, 1, 2]
    ag.render_motion(order[:1], True, (160, 90), None, encode="jpeg")                # warm-up: planes, scratch
    enc = ag.engine.encode_jpeg
    calls = []

    def slow(rgb, quality=90):
        calls.append(1)
        time.sleep(0.1)
        return enc(rgb, quality)

    ag.engine.encode_jpeg = slow
    ag.render_motion(order, True, (160, 90), None, encode="jpeg", writer=lambda i, ch: (list(ch), time.sleep(0.1)))
    t = ag.render_times
    assert len(calls) == len(order)
    assert 0.1 * len(calls) <= t["encoding"] < 0.1 * len(calls) + 0.25
    assert t["rendering"] < 0.25
    assert 0.1 * len(order) <= t["writer"] < 0.1 * len(order) + 0.25
    ag.engine.close()


def test_render_motion_jpeg_equals_encode_of_rgb_and_ignores_chunking():
    import cv2
    import torch
    from uhc_b200.agent import BatchedAgent
    from tests.test_gpu_render import _agent_clips
    clips = _agent_clips()
    ag = BatchedAgent(4, clips, [np.zeros(17)] * len(clips), policy_hsize=(128, 64), value_hsize=(64,), seed=2, body_diff_thresh=0.2,
                      auto_reset=False)
    order = [3, 0, 4, 1, 2]
    size, cam = (160, 90), dict(focus=True, shift_expert=1.0)
    a = ag.render_motion(order, True, size, cam)
    j = ag.render_motion(order, True, size, cam, encode="jpeg")
    assert set(ag.render_times) == {"evaluation", "rendering", "copy", "writer", "encoding"}
    got = {}
    ag.render_motion(order, True, size, cam, max_bytes=3 * 160 * 90 * 3, encode="jpeg", writer=lambda i, ch: got.__setitem__(i, [c for c in ch]))
    worst = np.inf
    for i, (x, y) in enumerate(zip(a, j)):
        d, o = ag.engine.encode_jpeg(torch.as_tensor(x["frames"], device="cuda"), 90)
        d, o = d.cpu().numpy(), o.cpu().numpy()
        want = [d[o[k]:o[k + 1]].tobytes() for k in range(len(o) - 1)]
        assert y["frames"] == want
        assert all(len(ch) <= 3 for ch in got[i]) and [f for ch in got[i] for f in ch] == want
        for f, rgb in zip(want, x["frames"]):
            dec = cv2.cvtColor(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB).astype(np.float64)
            worst = min(worst, 10 * np.log10(255.0 ** 2 / ((dec - rgb) ** 2).mean()))
    print(f"render_motion jpeg q=90 at 160x90: worst PSNR {worst:.2f} dB")
    assert worst >= PSNR_MIN_DB
    ag.engine.close()


def test_dropin_writes_one_mjpeg_avi_per_clip(tmp_path, monkeypatch):
    import cv2
    from tests.test_gpu_eval import _agent
    agent, cfg = _agent(tmp_path, monkeypatch, test_clips=4)
    eng = agent.agent.engine
    ld = agent.test_data_loaders[0]
    mp4 = agent.render_motion(epoch=3, loaders=[ld], out_dir=str(tmp_path / "a"), size=(96, 54))[ld.name]
    mp4b = agent.render_motion(epoch=3, loaders=[ld], out_dir=str(tmp_path / "b"), size=(96, 54), video="mp4")[ld.name]
    avi = agent.render_motion(epoch=3, loaders=[ld], out_dir=str(tmp_path / "c"), size=(96, 54), video="mjpeg")[ld.name]
    assert sorted(avi) == sorted(ld.data_keys)
    for key, path in avi.items():
        assert os.path.basename(path) == f"{key}_{cfg.id}_3_0.avi"
        assert open(mp4[key], "rb").read() == open(mp4b[key], "rb").read()
        cap = cv2.VideoCapture(mp4[key])
        n_mp4 = int(cap.get(cv2.CAP_PROP_FRAME_COUNT))
        cap.release()
        cap = cv2.VideoCapture(path)
        assert cap.get(cv2.CAP_PROP_FPS) == 30.0
        k = 0
        while True:
            ok, fr = cap.read()
            if not ok:
                break
            assert fr.shape == (54, 96, 3)
            k += 1
        cap.release()
        assert k == n_mp4 > 0
    eng.close()
