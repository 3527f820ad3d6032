"""Import-compatible shim (scripts/eval_uhc.py:34).  Rendering is outside the accelerated hot path."""
import itertools

import numpy as np


def write_frames_to_video(frames, out_file_name="output.mp4", frame_rate=30, add_text=None, text_color=(255, 255, 255)):
    """frames: a sequence or an iterator of RGB images [H][W][3] (an iterator is consumed one frame at a time)"""
    try:
        import cv2
    except ImportError as e:  # pragma: no cover
        raise RuntimeError("write_frames_to_video needs OpenCV") from e
    it = iter(frames)
    first = next(it, None)
    if first is None:
        raise IndexError("write_frames_to_video: no frames")
    h, w = np.asarray(first).shape[:2]
    wr = cv2.VideoWriter(out_file_name, cv2.VideoWriter_fourcc(*"mp4v"), frame_rate, (w, h))
    for f in itertools.chain([first], it):
        wr.write(np.asarray(f)[..., ::-1].astype(np.uint8))
    wr.release()
