"""ctypes wrapper of the host build of the mesh renderer's refit and pixel path, uhc_b200/csrc/render_mesh_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from uhc_b200.engine import UhcRenderMesh, make_camera

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_render_mesh_emu.so")


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    inc = os.path.join(_HERE, "..", "..", "include")
    srcs = [os.path.join(_HERE, "render_mesh_emu.cpp"), os.path.join(csrc, "render_mesh_core.h"), os.path.join(csrc, "render_core.h"),
            os.path.join(csrc, "motion_core.h"), os.path.join(inc, "uhc_b200.h"), os.path.join(inc, "uhc_render.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _p(a, t):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def check(tables, nvert):
    """uhc_render_mesh_init's table checks on the host: (0 | -2, reason)"""
    lib = C.CDLL(build())
    why = C.create_string_buffer(256)
    rc = lib.emu_render_mesh_check(C.byref(UhcRenderMesh.of(tables, nvert)), why, C.c_int(256))
    return rc, why.value.decode()


def render_mesh(tables, verts, size, camera=None, ghost=None, root=None, boxes=False):
    """verts / ghost [n][V][3] fp32 -> (rgb [n][H][W][3] uint8, depth [n][H][W] fp32, label [n][H][W] uint8) as uhc_render_mesh draws them;
    root [n][3] (needed with focus).  With boxes also the refitted boxes [n][48 + 2 nleaf][6]."""
    lib = C.CDLL(build())
    v = np.ascontiguousarray(verts, np.float32)
    n, V = v.shape[:2]
    g = None if ghost is None else np.ascontiguousarray(ghost, np.float32)
    r = None if root is None else np.ascontiguousarray(root, np.float32)
    W, H = size
    m = UhcRenderMesh.of(tables, V)
    rgb, depth, label = np.zeros((n, H, W, 3), np.uint8), np.zeros((n, H, W), np.float32), np.zeros((n, H, W), np.uint8)
    bx = np.zeros((n, 48 + 2 * m.nleaf, 6), np.float32) if boxes else None
    cam = make_camera(camera)
    lib.emu_render_mesh(C.byref(cam), C.c_int(W), C.c_int(H), C.c_long(n), _p(v, C.c_float), _p(g, C.c_float), _p(r, C.c_float), C.byref(m),
                        _p(rgb, C.c_ubyte), _p(depth, C.c_float), _p(label, C.c_ubyte), _p(bx, C.c_float))
    return (rgb, depth, label, bx) if boxes else (rgb, depth, label)
