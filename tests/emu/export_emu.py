"""ctypes wrapper of the host build of the device SMPL export's per-frame code, uhc_b200/csrc/smpl_export_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from uhc_b200.model import HumanoidModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_export_emu.so")


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    srcs = [os.path.join(_HERE, "export_emu.cpp"), os.path.join(csrc, "smpl_export_core.h"), os.path.join(csrc, "motion_core.h"),
            os.path.join(_HERE, "..", "..", "include", "uhc_b200.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def qpos_to_smpl(qpos, variants=None, variant=None):
    """qpos [n][>= 76] -> (pose [n][72], trans [n][3]) through the kernel's per-frame code.  variants: HumanoidModel shape variants (default:
    the base model), variant: index per frame (default: 0)."""
    lib = C.CDLL(build())
    q = np.ascontiguousarray(qpos, np.float64)
    n, pitch = q.shape
    models = variants or [HumanoidModel()]
    body_f = np.ascontiguousarray(np.concatenate([m.body_f for m in models]))
    v = None if variant is None else np.ascontiguousarray(np.broadcast_to(np.asarray(variant, np.int32), (n,)))
    out = np.zeros((n, 75))
    p = lambda a, t=C.c_double: None if a is None else a.ctypes.data_as(C.POINTER(t))
    lib.emu_qpos_to_smpl(C.c_long(n), p(q), C.c_long(pitch), p(body_f), C.c_int(len(models)), p(v, C.c_int), p(out))
    return out[:, :72], out[:, 72:]
