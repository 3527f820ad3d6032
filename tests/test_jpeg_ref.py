"""CPU: the independent JPEG statement of tests/jpeg_ref.py writes files that OpenCV and PIL decode to the frame it encoded."""
import io

import numpy as np
import pytest

from tests import jpeg_ref as R


def frames(W, H, seed=0):
    """a smooth colour gradient with a sharp-edged box, and uniform noise"""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:H, 0:W]
    g = np.stack([x * 255 // max(W - 1, 1), y * 255 // max(H - 1, 1), (x + y) * 127 // max(W + H - 2, 1)], -1).astype(np.uint8)
    g[H // 4:H // 2 + 1, W // 4:W // 2 + 1] = (250, 20, 20)
    return g, rng.integers(0, 256, (H, W, 3), dtype=np.uint8)


def test_tables_are_annex_k():
    assert [len(s[1]) for s in (R.DC_LUM, R.DC_CHR, R.AC_LUM, R.AC_CHR)] == [sum(s[0]) for s in (R.DC_LUM, R.DC_CHR, R.AC_LUM, R.AC_CHR)] == [12, 12, 162, 162]
    assert np.array_equal(R.quant_tables(50)[0], R.LUM) and np.array_equal(R.quant_tables(50)[1], R.CHR)
    assert R.quant_tables(100).max() == 1 and R.quant_tables(1).max() == 255 and R.quant_tables(1).min() == 255
    assert sorted(R.ZZ) == list(range(64))


@pytest.mark.parametrize("size", [(1, 1), (8, 8), (17, 9), (33, 31), (96, 54)])
@pytest.mark.parametrize("q", [1, 50, 90, 100])
def test_reference_files_decode_with_opencv_and_pil(size, q):
    import cv2
    from PIL import Image
    W, H = size
    smooth, noise = frames(W, H)
    for img in (smooth, noise):
        f = R.encode(img, q)
        a = cv2.cvtColor(cv2.imdecode(np.frombuffer(f, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)
        b = np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))
        assert a.shape == b.shape == (H, W, 3)
        if img is smooth and q >= 90 and min(W, H) >= 31:
            # a decoder of our own files sees the frame we encoded: luma-weighted error within a few levels at high quality
            for d in (a, b):
                assert np.abs(d.astype(int) - img).mean() < 4.0
