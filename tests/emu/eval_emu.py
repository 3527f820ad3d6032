"""ctypes wrapper of the host build of the evaluation kernel's per-frame metrics, uhc_b200/csrc/eval_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_eval_emu.so")


def build():
    srcs = [os.path.join(_HERE, "eval_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "eval_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def eval_frames(pred, gt, pred_jpos, gt_jpos):
    """[T][6] per-frame values of eval_core.h for one episode (qpos [T][76], joint positions [T][72])"""
    lib = C.CDLL(build())
    a = [np.ascontiguousarray(x, np.float64) for x in (pred, gt, np.reshape(pred_jpos, (len(pred), 72)), np.reshape(gt_jpos, (len(gt), 72)))]
    out = np.zeros((len(pred), 6))
    p = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))
    lib.emu_eval_frames(C.c_int(len(pred)), p(a[0]), p(a[1]), p(a[2]), p(a[3]), p(out))
    return out
