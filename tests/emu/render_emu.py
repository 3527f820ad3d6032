"""ctypes wrapper of the host build of the renderer's pose pass and pixel path, uhc_b200/csrc/render_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from uhc_b200.engine import make_camera
from uhc_b200.model import HumanoidModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_render_emu.so")


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    inc = os.path.join(_HERE, "..", "..", "include")
    srcs = [os.path.join(_HERE, "render_emu.cpp"), os.path.join(csrc, "render_core.h"), os.path.join(csrc, "motion_core.h"),
            os.path.join(inc, "uhc_b200.h"), os.path.join(inc, "uhc_render.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _p(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def pose(qpos, variants=None, variant=None, fk=False):
    """qpos [n][>= 76] (fp64) -> pose rows [n][24][12] fp32 through the kernel's per-frame code; with fk also (wpos [n][24][3], wq [n][24][4])
    in fp64 before rounding.  variants: HumanoidModel shape variants (default: the base model), variant: index per frame (default 0)."""
    lib = C.CDLL(build())
    q = np.ascontiguousarray(qpos, np.float64)
    n, pitch = q.shape
    models = variants or [HumanoidModel()]
    body_f = np.ascontiguousarray(np.concatenate([m.body_f for m in models]))
    v = None if variant is None else np.ascontiguousarray(np.broadcast_to(np.asarray(variant, np.int32), (n,)))
    m0 = models[0]
    par, ee = np.ascontiguousarray(m0.parent, np.int32), np.ascontiguousarray(m0.ee, np.int32)
    out = np.zeros((n, 24, 12), np.float32)
    wp, wq = (np.zeros((n, 24, 3)), np.zeros((n, 24, 4))) if fk else (None, None)
    lib.emu_render_pose(C.c_long(n), _p(q), C.c_long(pitch), _p(body_f), C.c_int(len(models)), _p(v, C.c_int), _p(par, C.c_int), _p(ee, C.c_int),
                        _p(out, C.c_float), _p(wp), _p(wq))
    return (out, wp, wq) if fk else out


def render_bodies(pose_table, size, camera=None, humanoids=None, variants=None, variant=None):
    """pose_table [n][2][24][12] fp32 -> (rgb [n][H][W][3] uint8, depth [n][H][W] fp32, label [n][H][W] uint8), uhc_render_bodies on the host.
    humanoids: 1 | 2 (default: 2)."""
    lib = C.CDLL(build())
    P = np.ascontiguousarray(pose_table, np.float32)
    n = P.shape[0]
    W, H = size
    models = variants or [HumanoidModel()]
    h = models[0].render_struct(models)
    keep = models[0]._rkeep
    v = None if variant is None else np.ascontiguousarray(np.broadcast_to(np.asarray(variant, np.int32), (n,)))
    rgb, depth, label = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32), np.zeros((n, H, W), np.uint8)
    cam = make_camera(camera)
    lib.emu_render_bodies(C.byref(cam), C.c_int(W), C.c_int(H), C.c_long(n), _p(P, C.c_float), C.c_int(2 if humanoids is None else humanoids),
                          _p(v, C.c_int), _p(keep["plane"]), C.c_int(h.nplane), _p(keep["adr"], C.c_int), _p(keep["num"], C.c_int), _p(keep["sphere"]),
                          _p(rgb, C.c_ubyte), _p(depth, C.c_float), _p(label, C.c_ubyte))
    return rgb, depth, label
