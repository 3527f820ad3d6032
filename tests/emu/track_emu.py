"""ctypes wrapper of the host build of the tracker's per-env code, uhc_b200/csrc/track_core.h and track_obs.h (TEST INFRASTRUCTURE)."""
import ctypes as C
import os
import subprocess

import numpy as np

from tests.emu import emu
from uhc_b200.model import HumanoidModel

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libuhc_track_emu.so")
EX_SIZE = 576


def build():
    csrc = os.path.join(_HERE, "..", "..", "uhc_b200", "csrc")
    srcs = [os.path.join(_HERE, "track_emu.cpp"), os.path.join(_HERE, "emu.cpp")] + [os.path.join(csrc, h) for h in (
        "track_core.h", "track_obs.h", "motion_core.h", "env_step.h", "sim_core.h", "curriculum_core.h")]
    if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-ffp-contract=off", "-o", _SO, srcs[0]])
    return _SO


def _p(a, t=C.c_double):
    return None if a is None else a.ctypes.data_as(C.POINTER(t))


def stream_clip(kind, pose_dim, rows, H, variants=None, variant=0):
    """one clip's raw rows streamed through a window of H rows: (rows read at cur_t + 1 after each push [T][576], rows read at cur_t before
    each push [T - 1][576], number of rebases)"""
    lib = C.CDLL(build())
    models = variants or [HumanoidModel()]
    m0 = models[0]
    body_f = np.ascontiguousarray(np.concatenate([m.body_f for m in models]))
    rows = np.ascontiguousarray(rows, np.float64)
    T = len(rows)
    nxt, cur = np.zeros((T, EX_SIZE)), np.zeros((T - 1, EX_SIZE))
    nreb = lib.emu_track_stream(C.c_int(kind), C.c_int(pose_dim), _p(rows), C.c_int(T), C.c_int(H), _p(np.ascontiguousarray(m0.parent, np.int32), C.c_int),
                                _p(np.ascontiguousarray(m0.ee, np.int32), C.c_int), _p(body_f), C.c_int(len(models)), C.c_int(variant), _p(nxt), _p(cur))
    assert nreb >= 0, "a push was dropped"
    return nxt, cur, nreb


class TrackEmu(emu.Emu):
    """the env-step emulation (tests/emu/emu.py Emu) built together with the tracker's observation pass"""

    def __init__(self, precision=64, num_envs=1, model=None, **cfg):
        self.lib = C.CDLL(build())
        self.lib.emu_create.restype = C.c_void_p
        self.prec = precision
        self.model = model or HumanoidModel()
        self._ms = self.model.host_struct()
        self._cfg = emu.default_cfg(precision, **cfg)
        blk = 640 if self._cfg.no_shape else 657
        self.obs_dim = 784 if self._cfg.obs_v == 1 else blk
        if self._cfg.obs_v in (5, 6):
            self.obs_dim = (636 if self._cfg.obs_v == 5 else 384) + (0 if self._cfg.no_shape else 17)
        self.h = C.c_void_p(self.lib.emu_create(C.byref(self._ms), C.byref(self._cfg), C.c_int(num_envs), C.c_int(precision)))

    def track_obs(self, env=0):
        obs = np.zeros(self.obs_dim)
        self.lib.emu_track_obs(self.h, self.prec, env, _p(obs))
        return obs
