"""ctypes wrappers of sim_emu_variants.cpp / render_emu_variants.cpp (tests only): emu.Emu and render_emu.RenderEmu for every
variant of the step kernel (csrc/sim_core.h LHW_FOR_EACH_VARIANT), h1_walk included."""
import ctypes
import os
import subprocess

import numpy as np

import emu
import render_emu

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(os.path.dirname(HERE)), "learninghumanoidwalking_b200", "csrc")
HEADERS = [os.path.join(CSRC, f) for f in ("sim_core.h", "model_pack.h", "render_core.h")]


def _build(src, base, lib, flags):
    srcs = [os.path.join(HERE, src), os.path.join(HERE, base)] + HEADERS
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        os.makedirs(os.path.dirname(lib), exist_ok=True)
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17"] + flags + ["-o", lib, srcs[0]])
    return lib


class _Lib:
    """The library with its entry points renamed from `old*` to `new*`, so that the base classes' calls reach them."""

    def __init__(self, path, old, new):
        self._lib, self._old, self._new = ctypes.CDLL(path), old, new

    def __getattr__(self, name):
        return getattr(self._lib, self._new + name[len(self._old):] if name.startswith(self._old) else name)


class Emu(emu.Emu):
    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = os.path.join(HERE, "_build", "libsim_emu_variants" + "".join("." + d.replace("=", "_") for d in emu.DEFINES) + ".so")
        self.lib = _Lib(_build("sim_emu_variants.cpp", "sim_emu.cpp", lib, ["-D" + d for d in emu.DEFINES]), "emu_", "emuv_")
        self.lib.emu_create.restype = ctypes.c_void_p
        flat = np.ascontiguousarray(flat, dtype=np.float64)
        self.h = ctypes.c_void_p(self.lib.emu_create(flat.ctypes.data_as(ctypes.c_void_p), len(flat), precision))
        assert self.h.value, "emu_create failed"
        self.prec, self.n, self.seed, self.first_id = precision, n, seed, first_id
        self.dt = np.float64 if precision == 64 else np.float32
        self.nr = self.lib.emu_state_words(self.h)
        self.nobs = self.lib.emu_obs_dim(self.h)
        self.nu = 2 * (int(flat[0]) % 100)
        self.nq, self.nv = 7 + self.nu, 6 + self.nu
        self.sr = np.zeros((n, self.nr), dtype=self.dt)
        self.si = np.zeros((n, emu.NSTATE_I), dtype=np.int32)


class RenderEmu(render_emu.RenderEmu):
    def __init__(self, flat, precision=64):
        # no contraction: the device build (-fmad=false) then does the same arithmetic
        lib = _build("render_emu_variants.cpp", "render_emu.cpp", os.path.join(HERE, "_build", "librender_emu_variants.so"),
                     ["-ffp-contract=off"])
        self.lib = _Lib(lib, "render_emu_", "render_emuv_")
        self.lib.render_emu_create.restype = ctypes.c_void_p
        flat = np.ascontiguousarray(flat, dtype=np.float64)
        self.h = ctypes.c_void_p(self.lib.render_emu_create(flat.ctypes.data_as(ctypes.c_void_p), len(flat), precision))
        assert self.h.value, "render_emu_create failed"
        self.prec = precision
        self.dt = np.float64 if precision == 64 else np.float32
        self.nl = 1 + 2 * (int(flat[0]) % 100)
