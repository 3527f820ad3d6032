"""ctypes wrapper of the host build of the grouped GEMM's row-tile schedule, uhc_b200/csrc/group_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_group_emu.so")


def build():
    srcs = [os.path.join(_HERE, "group_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "group_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", _SO, srcs[0]])
    return _SO


def group_tiles(row0, rows, M):
    """(code, tiles) of group_core.h's plan: tiles = [(group, first row, end row)] per tile, or None when the plan is refused (code -2)"""
    lib = C.CDLL(build())
    r0, rs = np.ascontiguousarray(row0, np.int32), np.ascontiguousarray(rows, np.int32)
    cap = int(np.sum((np.maximum(rs, 0) + 127) // 128)) + 1
    nt = C.c_int(0)
    g, f, e = (np.zeros(cap, np.int32) for _ in range(3))
    p = lambda x: x.ctypes.data_as(C.POINTER(C.c_int))
    rc = lib.emu_group_tiles(C.c_int(len(rs)), p(r0), p(rs), C.c_int(int(M)), C.c_int(cap), C.byref(nt), p(g), p(f), p(e))
    if rc:
        return rc, None
    return 0, list(zip(g[:nt.value].tolist(), f[:nt.value].tolist(), e[:nt.value].tolist()))
