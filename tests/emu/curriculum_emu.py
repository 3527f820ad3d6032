"""ctypes wrapper of the host build of the device curriculum's rules, uhc_b200/csrc/curriculum_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_curriculum_emu.so")


def build():
    srcs = [os.path.join(_HERE, "curriculum_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "curriculum_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _lib():
    L = C.CDLL(build())
    L.emu_pairwise_sum.restype = C.c_double
    return L


_i = lambda x: x.ctypes.data_as(C.POINTER(C.c_int))
_f = lambda x: x.ctypes.data_as(C.POINTER(C.c_float))
_d = lambda x: x.ctypes.data_as(C.POINTER(C.c_double))


class Rings:
    """the per-clip rings of C clips x M slots, as the device holds them"""

    def __init__(self, C, M=50):
        self.C, self.M = C, M
        self.meta = np.zeros(2 * C, np.int32)
        self.pct = np.zeros(C * M, np.float32)
        self.start = np.zeros(C * M, np.int32)

    def append(self, clip_log, pct_log, start_log):
        c, p, s = (np.ascontiguousarray(x, t).reshape(-1) for x, t in ((clip_log, np.int32), (pct_log, np.float32), (start_log, np.int32)))
        _lib().emu_cur_append(self.C, self.M, _i(self.meta), _f(self.pct), _i(self.start), len(c), _i(c), _f(p), _i(s))

    def history(self, c):
        """[(percent, start), ...] of clip c, oldest first"""
        head, n = self.meta[2 * c], self.meta[2 * c + 1]
        return [(float(self.pct[c * self.M + (head - n + k) % self.M]), int(self.start[c * self.M + (head - n + k) % self.M])) for k in range(n)]

    def set(self, hist):
        """hist: one list of (percent, start) per clip, oldest first"""
        self.meta[:] = 0
        for c, h in enumerate(hist):
            h = list(h)[-self.M:]
            for k, (p, s) in enumerate(h):
                self.pct[c * self.M + k], self.start[c * self.M + k] = p, s
            self.meta[2 * c], self.meta[2 * c + 1] = len(h) % self.M, len(h)

    def weights(self, temp, freq, t_max=-1, clip_len=None):
        w, cdf = np.zeros(self.C, np.float32), np.zeros(self.C, np.float32)
        cl = np.ascontiguousarray(np.zeros(self.C) if clip_len is None else clip_len, np.int32)
        _lib().emu_cur_weights(self.C, self.M, _i(self.meta), _f(self.pct), C.c_double(temp), C.c_double(freq), int(t_max), _i(cl), _f(w), _f(cdf))
        return w, cdf

    def start_law(self, c, L, t_min, prec_freq):
        pmf = np.zeros(L)
        _lib().emu_cur_start_law(self.M, _i(self.meta), _f(self.pct), _i(self.start), int(c), int(L), int(t_min), C.c_double(prec_freq), _d(pmf))
        return pmf


def pairwise_sum(a):
    a = np.ascontiguousarray(a, np.float64)
    return _lib().emu_pairwise_sum(_d(a), len(a))
