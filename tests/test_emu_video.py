"""CPU: the JPEG encoder's per-block arithmetic (uhc_b200/csrc/video_core.h), compiled into the host emulation, against the independent fp64
statement of tests/jpeg_ref.py; the marker structure and the size bound of its files; and the Motion-JPEG AVI writer (uhc_b200/video.py)."""
import io
import os

import numpy as np
import pytest

from tests import jpeg_ref as R
from tests.emu import video_emu as V
from tests.test_jpeg_ref import frames

# |X / 2^17 - F| of the integer DCT, in coefficient units, stated with a 3x margin over what test_dct_error_bound measures (0.284 on the
# sign patterns of the basis functions, 0.018 mean over random blocks)
DCT_BOUND = 0.875
SIZES = [(1, 1), (8, 8), (16, 16), (17, 9), (33, 31), (640, 360), (1920, 1080)]
QUALITIES = [1, 50, 90, 100]


def adversarial_blocks():
    rng = np.random.default_rng(1)
    b = [rng.integers(-128, 128, (20000, 8, 8)), np.where(rng.random((2000, 8, 8)) < 0.5, -128, 127), np.full((1, 8, 8), -128), np.full((1, 8, 8), 127)]
    k = np.arange(8)
    for u in range(8):
        for v in range(8):
            c = np.outer(np.cos((2 * k + 1) * u * np.pi / 16), np.cos((2 * k + 1) * v * np.pi / 16))
            b += [np.where(c >= 0, 127, -128)[None], np.where(c >= 0, -128, 127)[None]]
    return np.concatenate(b)


def test_dct_error_bound():
    b = adversarial_blocks()
    err = np.abs(V.fdct(b) / 2.0 ** 17 - R.dct(b)).max()
    assert 3 * err <= DCT_BOUND, err


def _frame(size, seed=0):
    """a smooth frame with a sharp box; at small sizes uniform noise as well"""
    W, H = size
    smooth, noise = frames(W, H, seed)
    return [smooth] if W * H > 100000 else [smooth, noise]


def _qz(q):
    """quantiser per block of an MCU in zigzag order [6][64]"""
    t = V.quant(q).reshape(2, 64)[:, R.ZZ]
    assert np.array_equal(V.quant(q), R.quant_tables(q))
    return np.stack([t[0]] * 4 + [t[1]] * 2)


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("q", QUALITIES)
def test_coefficients_equal_fp64_reference_off_rounding_boundaries(size, q):
    Q = _qz(q)
    for img in _frame(size):
        emu = V.coefs(img[None], q)[0].astype(np.int64)
        ref, r = R.coefs(img, q)
        # every value a DCT within DCT_BOUND of the fp64 one can round to
        rnd = lambda x: np.clip(np.sign(x) * np.floor(np.abs(x) + 0.5), -1023, 1023)
        lo, hi = rnd(r - DCT_BOUND / Q), rnd(r + DCT_BOUND / Q)
        assert ((emu >= lo) & (emu <= hi)).all()
        assert np.abs(emu - ref).max() <= 1


def _entropy(f):
    """the entropy-coded part of a file: (the bytes between SOS and EOI, DRI's interval, mcu columns)"""
    sos = f.index(b"\xff\xda")
    dri = f.index(b"\xff\xdd")
    return f[sos + 2 + int.from_bytes(f[sos + 2:sos + 4], "big"):], int.from_bytes(f[dri + 4:dri + 6], "big")


@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("q", QUALITIES)
def test_bytes_equal_reference_huffman_coding_and_decode(size, q):
    import cv2
    from PIL import Image
    W, H = size
    imgs = _frame(size)
    data, offs = V.encode(np.stack(imgs), q)
    c = V.coefs(np.stack(imgs), q)
    assert offs[0] == 0 and offs[-1] == len(data)
    for i, img in enumerate(imgs):
        f = data[offs[i]:offs[i + 1]].tobytes()
        assert f == R.file_from_coefs(c[i], W, H, q)
        assert len(f) <= V.bound(W, H)
        # markers: every 0xFF in the entropy data is stuffed, or an RST in cyclic order, and the last is EOI; DRI = one MCU row
        ent, dri = _entropy(f)
        assert dri == (W + 15) // 16
        pos = [k for k in range(len(ent) - 1) if ent[k] == 0xFF]
        marks = [ent[k + 1] for k in pos if ent[k + 1] != 0]
        assert marks == [0xD0 + (r & 7) for r in range((H + 15) // 16 - 1)] + [0xD9] and ent.endswith(b"\xff\xd9")
        a = cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR)
        b = np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))
        assert a.shape == b.shape == (H, W, 3)


@pytest.mark.parametrize("size", [(1, 1), (8, 8), (17, 9), (33, 31), (640, 360)])
def test_bound_holds_on_adversarial_frames(size):
    W, H = size
    rng = np.random.default_rng(3)
    y, x = np.mgrid[0:H, 0:W]
    checker = np.where(((x + y) % 2 == 0)[..., None], 255, 0).astype(np.uint8).repeat(3, -1)
    colour_checker = np.where(((x + y) % 2 == 0)[..., None], [255, 0, 255], [0, 255, 0]).astype(np.uint8)
    cases = [rng.integers(0, 256, (H, W, 3), dtype=np.uint8), checker, colour_checker, np.zeros((H, W, 3), np.uint8), np.full((H, W, 3), 255, np.uint8)]
    for q in (100, 90, 1):
        data, offs = V.encode(np.stack(cases), q)
        assert (np.diff(offs) <= V.bound(W, H)).all()


def test_flat_colours_stay_in_sample_range():
    """the eight corners of the RGB cube as flat frames at q = 100: every sample is BT.601's fp64 value within one level and inside 0 .. 255,
    so its DC is 8 (sample - 128) clamped to +-1023, at most 1016 (pure blue's Cb and pure red's Cr are 255, not 256)"""
    for rgb in np.array(np.meshgrid([0, 255], [0, 255], [0, 255], indexing="ij")).reshape(3, -1).T:
        r, g, b = (float(x) for x in rgb)
        want = np.clip(np.round([0.299 * r + 0.587 * g + 0.114 * b, 128 - 0.168736 * r - 0.331264 * g + 0.5 * b,
                                 128 + 0.5 * r - 0.418688 * g - 0.081312 * b]), 0, 255)
        dc = V.coefs(np.broadcast_to(rgb.astype(np.uint8), (1, 16, 16, 3)), 100)[0, 0, 0, :, 0].astype(int)
        got = np.array([dc[0], dc[4], dc[5]])
        lo, hi = (np.clip(8 * (np.clip(want + d, 0, 255) - 128), -1023, 1023) for d in (-1, 1))
        assert (got >= lo).all() and (got <= hi).all(), (rgb, got, want)
        assert (dc[:4] == dc[0]).all()


def test_bound_against_worst_case_blocks():
    """the Huffman coding of the longest blocks baseline allows (every AC at +-1023, the DC differences at +-2046, the magnitude bits chosen so
    that most bytes are 0xFF) fits uhc_jpeg_bound, and fills more than half of it: the bound is not off by a factor"""
    W, H = 64, 32
    mx, my = W // 16, H // 16
    c = np.full((my, mx, 6, 64), 1023, np.int64)
    c[..., 0] = np.where(np.arange(mx) % 2 == 0, 1023, -1023)[None, :, None]
    data = R.file_from_coefs(c, W, H, 100)
    assert len(data) <= V.bound(W, H)
    assert len(data) > 0.5 * V.bound(W, H), (len(data), V.bound(W, H))
    # the block bound itself: the largest DC code + 11 magnitude bits, then 63 of the largest AC codes + 10 bits (the EOB never follows 63
    # coefficients, and a block with an EOB has fewer AC codes)
    lens = lambda spec: [len(v) for v in R.huff_codes(spec).values()]
    worst = max(lens(R.DC_LUM) + lens(R.DC_CHR)) + 11 + max(63 * (max(lens(s)) + 10) for s in (R.AC_LUM, R.AC_CHR))
    seg = (mx * 6 * worst + 7) // 8 + 1
    assert V.bound(W, H) >= len(R.header(W, H, 100)) + my * (2 * seg + 2) + 2
    assert V.bound(W, H) <= len(R.header(W, H, 100)) + my * (2 * (seg + mx * 6 * 16 // 8 + 1) + 2) + 2


def test_avi_writer_reads_back(tmp_path):
    import cv2
    from uhc_b200.video import write_mjpeg_avi
    rng = np.random.default_rng(4)
    W, H = 72, 40
    base, _ = frames(W, H)
    imgs = np.stack([np.roll(base, 3 * k, 1) for k in range(7)])
    imgs[2] = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)        # one large frame (odd sizes pad the chunk)
    data, offs = V.encode(imgs, 90)
    jpegs = [data[offs[i]:offs[i + 1]].tobytes() for i in range(len(imgs))]
    path = str(tmp_path / "a.avi")
    assert write_mjpeg_avi(path, iter(jpegs), W, H) == len(jpegs)
    cap = cv2.VideoCapture(path)
    assert (cap.get(cv2.CAP_PROP_FRAME_COUNT), cap.get(cv2.CAP_PROP_FPS)) == (len(jpegs), 30.0)
    assert (cap.get(cv2.CAP_PROP_FRAME_WIDTH), cap.get(cv2.CAP_PROP_FRAME_HEIGHT)) == (W, H)
    k = 0
    while True:
        ok, fr = cap.read()
        if not ok:
            break
        assert fr.shape == (H, W, 3)
        k += 1
    cap.release()
    assert k == len(jpegs)
    # the stream's packets are the JPEG files byte for byte, so every frame is cv2.imdecode of its JPEG
    cap = cv2.VideoCapture(path, cv2.CAP_FFMPEG)
    assert cap.set(cv2.CAP_PROP_FORMAT, -1)
    for j in jpegs:
        ok, pkt = cap.read()
        assert ok and pkt.tobytes() == j
        assert np.array_equal(cv2.imdecode(pkt.reshape(-1), cv2.IMREAD_COLOR), cv2.imdecode(np.frombuffer(j, np.uint8), cv2.IMREAD_COLOR))
    cap.release()


def test_avi_writer_refuses_past_classic_riff_limit(tmp_path, monkeypatch):
    from uhc_b200 import video
    monkeypatch.setattr(video, "RIFF_LIMIT", 20000)
    path = str(tmp_path / "big.avi")
    with pytest.raises(ValueError, match="1 GiB"):
        video.write_mjpeg_avi(path, (bytes(3000) for _ in range(10)), 16, 16)
    assert not os.path.exists(path)
    assert video.write_mjpeg_avi(path, (bytes(3000) for _ in range(5)), 16, 16) == 5
