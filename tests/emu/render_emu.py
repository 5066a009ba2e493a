"""ctypes wrapper of the host build of the renderer source (tests only; see render_emu.cpp)."""
import ctypes
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
LIB = os.path.join(HERE, "_build", "librender_emu.so")
CSRC = os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc")


def build():
    srcs = [os.path.join(HERE, "render_emu.cpp")] + [os.path.join(CSRC, f) for f in ("render_core.h", "sim_core.h", "model_pack.h")]
    if not os.path.exists(LIB) or any(os.path.getmtime(s) > os.path.getmtime(LIB) for s in srcs):
        os.makedirs(os.path.dirname(LIB), exist_ok=True)
        # no contraction: the device build (-fmad=false) then does the same arithmetic
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-ffp-contract=off", "-o", LIB, srcs[0]])
    return LIB


class RenderEmu:
    def __init__(self, flat, precision=64):
        self.lib = ctypes.CDLL(build())
        self.lib.render_emu_create.restype = ctypes.c_void_p
        flat = np.ascontiguousarray(flat, dtype=np.float64)
        self.h = ctypes.c_void_p(self.lib.render_emu_create(flat.ctypes.data_as(ctypes.c_void_p), len(flat), precision))
        assert self.h.value, "render_emu_create failed"
        self.prec = precision
        self.dt = np.float64 if precision == 64 else np.float32
        self.nl = 1 + 2 * (int(flat[0]) % 100)

    @staticmethod
    def _p(a):
        return a.ctypes.data_as(ctypes.c_void_p)

    def fk(self, qpos):
        q = np.ascontiguousarray(qpos, dtype=self.dt)
        xpos, xmat = np.zeros((self.nl, 3), np.float32), np.zeros((self.nl, 3, 3), np.float32)
        self.lib.render_emu_fk(self.h, self.prec, self._p(q), self._p(xpos), self._p(xmat))
        return xpos, xmat

    def image(self, sr, si, width, height, cam, only_box=-1, nbox=64):
        """One record -> (rgb [H, W, 3] uint8, scene boxes [nbox, 15]: centre, rotation, half sizes)."""
        sr = np.ascontiguousarray(sr, dtype=self.dt)
        si = np.ascontiguousarray(si, dtype=np.int32)
        c7 = np.ascontiguousarray(cam, dtype=np.float64)
        rgb = np.zeros((height, width, 3), np.uint8)
        boxes = np.zeros((nbox, 15), np.float32)
        self.lib.render_emu_image(self.h, self.prec, self._p(sr), self._p(si), width, height, self._p(c7), int(only_box), self._p(rgb),
                                  self._p(boxes))
        return rgb, boxes
