"""ctypes wrapper of the host build of the subject body builder's per-item code, uhc_b200/csrc/subject_core.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_subject_emu.so")


def build():
    srcs = [os.path.join(_HERE, "subject_emu.cpp"), os.path.join(_HERE, "..", "..", "uhc_b200", "csrc", "subject_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def subject_body(basis, beta, gender):
    """one subject through the kernel's per-item code: (body_f [24][20], hull [nvert][3], maps [24][3][4]) from a
    uhc_b200.subject_body.SubjectBasis.  ValueError naming the body when a map inverts it."""
    lib = C.CDLL(build())
    hm = basis.humanoid
    d = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    i = lambda a: a.ctypes.data_as(C.POINTER(C.c_int))
    keep = dict(mb=np.ascontiguousarray(basis.map[gender], np.float64), ob=np.ascontiguousarray(basis.offset[gender], np.float64),
                beta=np.ascontiguousarray(np.asarray(beta, np.float64)[:10]), bf0=np.ascontiguousarray(hm.body_f), hull0=np.ascontiguousarray(hm.hull),
                adr=np.ascontiguousarray(hm.hull_adr, np.int32), num=np.ascontiguousarray(hm.hull_num, np.int32),
                par=np.ascontiguousarray(hm.parent, np.int32), sub=np.ascontiguousarray(hm.body_sub_end, np.int32), df=np.ascontiguousarray(hm.dof_f))
    bf, hull, mp = np.zeros((24, 20)), np.zeros((len(hm.hull), 3)), np.zeros((24, 3, 4))
    k = keep
    rc = lib.emu_subject_body(d(k["mb"]), d(k["ob"]), d(k["beta"]), d(k["bf0"]), d(k["hull0"]), C.c_int(len(hm.hull)), i(k["adr"]), i(k["num"]),
                              i(k["par"]), i(k["sub"]), d(k["df"]), d(bf), d(hull), d(mp))
    if rc:
        raise ValueError(f"the map of body {rc - 1} inverts it (det A <= 0)")
    return bf, hull, mp
