"""ctypes wrapper of the host build of the device motion library's per-frame code, uhc_b200/csrc/motion_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from uhc_b200.model import HumanoidModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_motion_emu.so")
EX_SIZE = 576


def build():
    srcs = [os.path.join(_HERE, "motion_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "motion_core.h"),
            os.path.join(_HERE, "..", "..", "include", "uhc_b200.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _p(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def motion_table(motions, variants=None, fk_models=None):
    """expert table [frames][576] of a uhc_b200.motion_lib.MotionSet, built on the CPU by the motion kernel's per-frame code.
    variants: HumanoidModel shape variants (default: the base model), fk_models: variant per clip (default: variant 0)."""
    lib = C.CDLL(build())
    models = variants or [HumanoidModel()]
    m0 = models[0]
    body_f = np.ascontiguousarray(np.concatenate([m.body_f for m in models]))
    lens = np.ascontiguousarray(motions.lens, np.int32)
    fk = None if fk_models is None else np.ascontiguousarray(fk_models, np.int32)
    rows = np.ascontiguousarray(motions.rows, np.float64)
    out = np.zeros((int(lens.sum()), EX_SIZE))
    lib.emu_motion_table(C.c_int(len(lens)), _p(lens, C.c_int), C.c_int(motions.kind), C.c_int(motions.pose_dim), _p(rows),
                         _p(np.ascontiguousarray(m0.parent, np.int32), C.c_int), _p(np.ascontiguousarray(m0.ee, np.int32), C.c_int),
                         _p(body_f), C.c_int(len(models)), _p(fk, C.c_int), _p(out))
    return out
