"""Motion-JPEG AVI files from JPEG frames (Engine.encode_jpeg's): a classic RIFF AVI with one MJPG video stream and an idx1 index."""
import os
import struct

RIFF_LIMIT = 1 << 30      # a classic (AVI 1.0) RIFF file stays under 1 GiB; readers take larger files only as OpenDML, which this is not


def _chunk(fourcc, payload):
    return fourcc + struct.pack("<I", len(payload)) + payload + (b"\0" if len(payload) & 1 else b"")


def _list(kind, payload):
    return b"LIST" + struct.pack("<I", len(payload) + 4) + kind + payload


def _headers(W, H, fps, frames, max_frame):
    avih = struct.pack("<10I4I", round(1e6 / fps), 0, 0, 0x10, frames, 0, 1, max_frame, W, H, 0, 0, 0, 0)       # 0x10: AVIF_HASINDEX
    strh = b"vidsMJPG" + struct.pack("<IHHIIIIIIiI4h", 0, 0, 0, 0, 1, fps, 0, frames, max_frame, -1, 0, 0, 0, W, H)
    strf = struct.pack("<IiiHH4sIiiII", 40, W, H, 1, 24, b"MJPG", W * H * 3, 0, 0, 0, 0)
    return _list(b"hdrl", _chunk(b"avih", avih) + _list(b"strl", _chunk(b"strh", strh) + _chunk(b"strf", strf)))


def write_mjpeg_avi(path, jpegs, W, H, fps=30):
    """writes the JPEG files `jpegs` (an iterable of bytes, consumed one at a time) as the frames of a W x H Motion-JPEG AVI at fps frames
    per second (an integer).  Raises ValueError, and leaves no file, when the AVI would exceed the 1 GiB of a classic RIFF file.  Returns the
    number of frames."""
    fps = int(fps)
    if fps < 1 or not (1 <= W <= 65535 and 1 <= H <= 65535):
        raise ValueError("write_mjpeg_avi: fps must be >= 1 and W, H in 1 .. 65535")
    head = len(_headers(W, H, fps, 0, 0))
    index, pos, max_frame = [], 4, 0                   # offsets in idx1 count from the 'movi' fourcc
    try:
        with open(path, "wb") as f:
            f.write(b"\0" * (12 + head + 12))               # RIFF, hdrl and the movi LIST header, written when the sizes are known
            for jpg in jpegs:
                jpg = bytes(jpg)
                c = _chunk(b"00dc", jpg)
                if 12 + head + 8 + pos + len(c) + 8 + 16 * (len(index) + 1) > RIFF_LIMIT:
                    raise ValueError(f"write_mjpeg_avi: {path} would exceed the 1 GiB of a classic RIFF AVI after {len(index)} frames")
                f.write(c)
                index.append(struct.pack("<4sIII", b"00dc", 0x10, pos, len(jpg)))        # 0x10: AVIIF_KEYFRAME
                pos += len(c)
                max_frame = max(max_frame, len(jpg))
            f.write(_chunk(b"idx1", b"".join(index)))
            total = f.tell()
            f.seek(0)
            f.write(b"RIFF" + struct.pack("<I", total - 8) + b"AVI " + _headers(W, H, fps, len(index), max_frame))
            f.write(b"LIST" + struct.pack("<I", pos) + b"movi")
    except BaseException:
        if os.path.exists(path):
            os.remove(path)
        raise
    return len(index)
