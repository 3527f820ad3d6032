"""ctypes wrapper of the host build of the JPEG encoder's per-block arithmetic, uhc_b200/csrc/video_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_video_emu.so")


def build():
    srcs = [os.path.join(_HERE, "video_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "video_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-o", _SO, srcs[0]])
    return _SO


def _lib():
    lib = C.CDLL(build())
    lib.emu_jpeg_bound.restype = C.c_size_t
    lib.emu_jpeg_encode.restype = C.c_size_t
    return lib


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def bound(W, H):
    """the worst-case bytes of one W x H frame (uhc_jpeg_bound)"""
    return int(_lib().emu_jpeg_bound(C.c_int(W), C.c_int(H)))


def fdct(blocks):
    """level-shifted blocks [n][8][8] int -> X = 2^17 F [n][8][8] int32 (the kernel's integer DCT)"""
    s = np.ascontiguousarray(blocks, np.int32).reshape(-1, 64)
    X = np.zeros_like(s)
    _lib().emu_jpeg_fdct(C.c_long(len(s)), _p(s, C.c_int), _p(X, C.c_int))
    return X.reshape(-1, 8, 8)


def quant(quality):
    """the quantisation tables [2][8][8] (luminance, chrominance; natural order) of a quality"""
    q = np.zeros((2, 64), np.int32)
    _lib().emu_jpeg_quant(C.c_int(quality), _p(q, C.c_int))
    return q.reshape(2, 8, 8)


def coefs(rgb, quality):
    """frames [n][H][W][3] uint8 -> quantised coefficients [n][mcu rows][mcu cols][6][64] int16, zigzag order"""
    f = np.ascontiguousarray(rgb, np.uint8)
    n, H, W = f.shape[:3]
    out = np.zeros((n, (H + 15) // 16, (W + 15) // 16, 6, 64), np.int16)
    _lib().emu_jpeg_coefs(_p(f, C.c_ubyte), C.c_long(n), C.c_int(W), C.c_int(H), C.c_int(quality), _p(out, C.c_short))
    return out


def encode(rgb, quality):
    """frames [n][H][W][3] uint8 -> (packed bytes uint8, offsets [n + 1]) as uhc_jpeg_encode packs them"""
    f = np.ascontiguousarray(rgb, np.uint8)
    n, H, W = f.shape[:3]
    lib = _lib()
    total = lib.emu_jpeg_encode(_p(f, C.c_ubyte), C.c_long(n), C.c_int(W), C.c_int(H), C.c_int(quality), None, C.c_size_t(0), None)
    out, offs = np.zeros(max(total, 1), np.uint8), np.zeros(n + 1, np.uint64)
    lib.emu_jpeg_encode(_p(f, C.c_ubyte), C.c_long(n), C.c_int(W), C.c_int(H), C.c_int(quality), _p(out, C.c_ubyte), C.c_size_t(total),
                        _p(offs, C.c_size_t))
    return out[:total], offs.astype(np.int64)
