"""ctypes wrapper of the host build of the floor measurements' per-frame code, uhc_b200/csrc/floor_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from uhc_b200.model import HumanoidModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_floor_emu.so")


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    srcs = [os.path.join(_HERE, "floor_emu.cpp"), os.path.join(csrc, "floor_core.h"), os.path.join(csrc, "render_core.h"),
            os.path.join(csrc, "motion_core.h"), os.path.join(_HERE, "..", "..", "include", "uhc_b200.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _p(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def _model_args(models):
    m0 = models[0]
    keep = [np.ascontiguousarray(m0.parent, np.int32), np.ascontiguousarray(m0.ee, np.int32),
            np.ascontiguousarray(np.concatenate([m.body_f for m in models])), np.ascontiguousarray(np.stack([m.hull for m in models]), np.float64),
            np.ascontiguousarray(m0.hull_adr, np.int32), np.ascontiguousarray(m0.hull_num, np.int32)]
    args = (_p(keep[0], C.c_int), _p(keep[1], C.c_int), _p(keep[2]), C.c_int(len(models)), _p(keep[3]), C.c_int(len(m0.hull)), _p(keep[4], C.c_int),
            _p(keep[5], C.c_int))
    return args, keep


def floor_qpos(qpos, variants=None, variant=None, first=None):
    """qpos [n][>= 76] -> rows [n][5] through the kernel's per-frame code.  variants: HumanoidModel shape variants (default: the base model),
    variant: index per row (default: 0), first: per row, 1 = no previous frame (default: the rows are one clip)."""
    lib = C.CDLL(build())
    q = np.ascontiguousarray(qpos, np.float64)
    n, pitch = q.shape
    args, keep = _model_args(variants or [HumanoidModel()])
    v = None if variant is None else np.ascontiguousarray(np.broadcast_to(np.asarray(variant, np.int32), (n,)))
    f = None if first is None else np.ascontiguousarray(np.broadcast_to(np.asarray(first, np.int32), (n,)))
    out = np.zeros((n, 5))
    lib.emu_floor_qpos(C.c_long(n), _p(q), C.c_long(pitch), _p(v, C.c_int), _p(f, C.c_int), *args, _p(out))
    return out


class EmuFloor:
    """stands in for uhc_b200.engine.Engine where MotionSet.floor_audit needs one: motion_floor through the kernel's per-frame code"""

    def __init__(self, variants=None):
        self.model = (variants or [HumanoidModel()])[0]
        self.variants = variants

    def motion_floor(self, motions, fk_models=None, chunk_frames=0):
        lib = C.CDLL(build())
        args, keep = _model_args(self.variants or [self.model])
        lens = np.ascontiguousarray(motions.lens, np.int32)
        rows = np.ascontiguousarray(motions.rows, np.float64)
        fk = None if fk_models is None else np.ascontiguousarray(fk_models, np.int32)
        n = int(lens.sum())
        out, feet = np.zeros((n, 5)), np.zeros((n, 4))
        lib.emu_motion_floor(C.c_int(len(lens)), _p(lens, C.c_int), C.c_int(motions.kind), C.c_int(motions.pose_dim), _p(rows), _p(fk, C.c_int), *args,
                             _p(out), _p(feet))
        return out, feet
