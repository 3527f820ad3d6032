"""ctypes wrapper of the host build of the global curriculum's payload rules, uhc_b200/csrc/curriculum_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_curriculum_global_emu.so")


def build():
    srcs = [os.path.join(_HERE, "curriculum_global_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "curriculum_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _lib():
    return C.CDLL(build())


_i = lambda x: x.ctypes.data_as(C.POINTER(C.c_int))
_f = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))


def stage(clip_log, pct_log, start_log):
    """k_cur_stage on the host: n log entries -> [n][3] fp32 (clip, percent, start)"""
    c, p, s = (np.ascontiguousarray(x, t).reshape(-1) for x, t in ((clip_log, np.int32), (pct_log, np.float32), (start_log, np.int32)))
    out = np.zeros((len(c), 3), np.float32)
    _lib().emu_cur_stage(len(c), _i(c), _f(p), _i(s), _f(out))
    return out


def unpack(summed):
    """k_cur_unpack on the host: [n][3] fp32 -> (clip, percent, start) logs"""
    x = np.ascontiguousarray(summed, np.float32).reshape(-1, 3)
    n = len(x)
    c, p, s = np.zeros(n, np.int32), np.zeros(n, np.float32), np.zeros(n, np.int32)
    _lib().emu_cur_unpack(n, _f(x), _i(c), _f(p), _i(s))
    return c, p, s


def stage_exact(num_clips, longest_clip):
    """stage_exact: True when every clip index and start frame of such a table is exact in fp32"""
    return bool(_lib().emu_cur_stage_exact(C.c_longlong(num_clips), C.c_longlong(longest_clip)))
