"""One physics substep of the step kernel at crafted states, for the tests (tests/test_gpu_substep_edges.py on the device,
tests/test_substep_harness.py on the host): builds and ctypes wrappers of the device harness tests/dev/substep_dev.cu and of its
host twin tests/dev/substep_emu.cpp, the crafted cases, the mapping of a case onto a kernel record and onto an oracle env, and
the comparison with the float64 oracle (oracle/) with the bounds each quantity is held to.

A case is a list of seeded states of one variant.  Each state holds qpos, qvel, ctrl and what the variant adds (per-env H1
parameters and wrenches, stepping-stone / terrace poses and the task mode).  Every case names the branch it is for, and
`reached` asserts from the kernel's Work record that the branch was taken: a case that stops reaching its branch fails.

delta: the margin by which a crafted quantity sits on one side of a threshold.  1e-9 at fp64; at fp32 1e-4 in the quantity's
unit (m, rad, rad/s), so every threshold decision is the same in the fp32 kernel and in the float64 oracle."""
import ctypes
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
import solver_pieces as SP  # noqa: E402  (the content-hashed build cache and the package's nvcc flags)

CSRC = os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc")
DEV_SRC = os.path.join(HERE, "substep_dev.cu")
EMU_SRC = os.path.join(HERE, "substep_emu.cpp")
RECORD_H = os.path.join(HERE, "substep_record.h")
DEV_DEPS = [DEV_SRC, RECORD_H] + [os.path.join(CSRC, f) for f in ("sim_core.h", "sim_kernels.cu", "render_kernels.cu", "model_pack.h", "render_core.h")] + \
    [os.path.join(ROOT, "include", "lhw_b200.h")]

NAMES = {6: "jvrc_walk", 5: "h1", 106: "jvrc_step", 206: "jvrc_walk_terrain", 305: "h1_walk"}
CODE = {v: k for k, v in NAMES.items()}
NJ = {6: 6, 5: 5, 106: 6, 206: 6, 305: 5}
CPF = {6: 4, 5: 6, 106: 8, 206: 8, 305: 6}
RFOOT = {6: 0, 106: 0, 206: 0, 5: 1, 305: 1}             # the chain that ends in the right foot
SLABS = {6: False, 5: False, 106: True, 206: True, 305: False}
PERENV = {6: False, 5: True, 106: False, 206: False, 305: True}
WARPS = {(64, 6): 8, (64, 5): 7, (64, 106): 7, (64, 206): 7, (64, 305): 7}   # the product's lock-step warps per block
NSTATE_I = 8
FIELDS = ["size", "qpos", "qvel", "qacc_warm", "qacc", "qfs", "act_force", "M", "ncon", "ncorner", "nside", "cmul", "cn", "cpos",
          "xcd", "lside", "grf", "cz_min", "foot_vel", "root_vlin", "status", "nfloor", "iters_total", "flim", "fjar"]
DELTA = {64: 1e-9, 32: 1e-4}


def product_warps(prec, code):
    return WARPS.get((prec, code), 14)


# ---------------------------------------------------------------- builds
def nvcc_command(out):
    # render_kernels.cu: its own translation unit, as in the product, for the render_launch that sim_kernels.cu calls
    return SP.nvcc_command(out)[:-1] + ["-Xcompiler", "-fvisibility=hidden", DEV_SRC, os.path.join(CSRC, "render_kernels.cu")]


def build_device():
    return SP._compiled("libsubstep_dev", DEV_DEPS, nvcc_command)


def build_emu():
    return SP._compiled("libsubstep_emu", [EMU_SRC, RECORD_H] + DEV_DEPS[2:],
                        lambda out: ["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", out, EMU_SRC])


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class Harness:
    """Substeps of one model at one precision: device=True loads substep_dev.cu (dev_*), else substep_emu.cpp (emu_*)."""

    def __init__(self, flat, prec, device):
        self.device, self.prec = device, prec
        self.code = int(flat[0])
        self.lib = L = ctypes.CDLL(build_device() if device else build_emu())
        pre = "dev_" if device else "emu_"
        self._create, self._destroy = getattr(L, pre + "substep_create"), getattr(L, pre + "substep_destroy")
        self._run, self._layout = getattr(L, pre + "substeps"), getattr(L, pre + "substep_layout")
        self._create.restype = ctypes.c_void_p
        self._destroy.argtypes = [ctypes.c_void_p]
        self.flat = np.ascontiguousarray(flat, np.float64)
        self.h = ctypes.c_void_p(self._create(_p(self.flat), len(self.flat), prec))
        if device:
            L.dev_substep_error.restype = ctypes.c_char_p
        assert self.h.value, "creating the substep harness failed" + (f": {L.dev_substep_error().decode()}" if device else "")
        o = np.zeros(len(FIELDS), np.int64)
        assert self._layout(self.code, prec, _p(o)) == 0
        self.layout = dict(zip(FIELDS, (int(x) for x in o)))
        self.dt = np.float64 if prec == 64 else np.float32

    def close(self):
        if self.h.value:
            self._destroy(self.h)
            self.h = ctypes.c_void_p(0)

    def run(self, sr, si, ctrl, nsub, n_warps=1):
        """nsub substeps of the records sr [n, NSTATE_R], si [n, 8] with ctrl [n, 2 NJ] held -> (sr, si, Work bytes [n, size])."""
        sr = np.ascontiguousarray(sr, self.dt).copy()
        si = np.ascontiguousarray(si, np.int32).copy()
        ctrl = np.ascontiguousarray(ctrl, self.dt)
        n = sr.shape[0]
        work = np.zeros((n, self.layout["size"]), np.uint8)
        extra = [ctypes.c_int(n_warps)] if self.device else []
        rc = self._run(self.h, ctypes.c_int(n), *extra, ctypes.c_int(nsub), _p(sr), _p(si), _p(ctrl), _p(work))
        assert rc == 0, rc
        return sr, si, work

    def fields(self, wb):
        """The named Work fields of one record's bytes."""
        nj = NJ[self.code]
        nv, nu, ncon = 6 + 2 * nj, 2 * nj, 2 * CPF[self.code]
        nst = SLABS[self.code]
        R, I = self.dt, np.int32

        def get(name, dtype, count):
            o = self.layout[name]
            return wb[o:o + np.dtype(dtype).itemsize * count].view(dtype).copy()
        aw = 36 + 12 * nj + 2 * nj * nj
        f = dict(qpos=get("qpos", R, nv + 1), qvel=get("qvel", R, nv), qacc=get("qacc", R, nv), qfs=get("qfs", R, nv),
                 act_force=get("act_force", R, nu), M=get("M", R, aw).astype(np.float64), ncon=get("ncon", I, 2),
                 ncorner=get("ncorner", I, 2), nside=get("nside", I, 2), lside=get("lside", I, nu), grf=get("grf", R, 2),
                 cz_min=get("cz_min", R, 1)[0], foot_vel=get("foot_vel", R, 6).reshape(2, 3), root_vlin=get("root_vlin", R, 3),
                 status=int(get("status", I, 1)[0]), nfloor=int(get("nfloor", I, 1)[0]), iters=int(get("iters_total", I, 1)[0]))
        f["cpos"] = get("cpos", R, ncon * (5 if nst else 3)).reshape(ncon, 5 if nst else 3)[:, :3]
        f["cmul"] = get("cmul", R, 16) if nst else None
        f["xcd"] = get("xcd", R, ncon) if nst else None
        f["cn"] = get("cn", R, 2 * ncon).reshape(ncon, 2) if nst else None
        if PERENV[self.code]:
            f["flim"], f["fjar"] = get("flim", R, nu), get("fjar", R, nu)
        # o (the root position of the last substep's pre-integration state) sits 3 reals before xr in Work; read it through qpos
        # of the oracle instead (see compare)
        return f


# ---------------------------------------------------------------- models and the oracle
_MODELS = {}


def model(name):
    """(mj, the kernel's flat model at tolerance 1e-14, the oracle) of a variant, cached."""
    if name not in _MODELS:
        from learninghumanoidwalking_b200.model import load_model, pack_model
        mj = load_model(name)
        if name == "h1_walk":
            sys.path.insert(0, os.path.join(ROOT, "tests"))
            from h1_walk_oracle import H1WalkOracle
            o = H1WalkOracle(tolerance=1e-14)
        else:
            from oracle.oracle import Oracle
            o = Oracle(name, tolerance=1e-14)
        _MODELS[name] = (mj, pack_model(mj, tolerance=1e-14), o)
    return _MODELS[name]


def flat_at(name, tolerance):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model(name), tolerance=tolerance)


def joint_table(mj):
    """Per hinge dof: (range lo, range hi, limited, damping) of the model."""
    js = [lk["joint"] for lk in mj["links"][1:]]
    return (np.array([j["range"][0] for j in js]), np.array([j["range"][1] for j in js]),
            np.array([j.get("limited", True) for j in js]), np.array([j.get("damping", 0.0) for j in js]))


# ---------------------------------------------------------------- kinematics of the contact geometry (numpy, float64)
def foot_points(mj, q):
    """World positions of each foot's candidate points, [2 (chain), k, 3]: the 8 box corners (index bits: x, y, z sign) of a box
    foot, the sphere centres lowered by the radius of a sphere foot."""
    from tools.compile_model import kinematics
    xpos, xmat = kinematics(mj, q)
    nj = (len(mj["links"]) - 1) // 2
    out = []
    for ch in range(2):
        lk = (ch + 1) * nj
        g = [g for g in mj["geoms"] if g["link"] == lk][0]
        R, p0 = np.array(xmat[lk]), np.array(xpos[lk])
        if g["type"] == "box":
            size, gpos = np.array(g["size"]), np.array(g["pos"])
            pts = [p0 + R @ (gpos + np.array([(1 if i & 1 else -1) * size[0], (1 if i & 2 else -1) * size[1],
                                              (1 if i & 4 else -1) * size[2]])) for i in range(8)]
        else:
            pts = [p0 + R @ np.array(c) - np.array([0, 0, g["radius"]]) for c in g["points"]]
        out.append(np.array(pts))
    return out


def quat(ang):
    n = np.linalg.norm(ang)
    return np.array([1.0, 0, 0, 0]) if n == 0 else np.concatenate([[np.cos(n / 2)], np.sin(n / 2) * np.asarray(ang) / n])


# ---------------------------------------------------------------- a state: kernel record and oracle env
class State(dict):
    """q, v, ctrl; optional: seq [20, 4] and mode (slab variants), params (PERENV: the oracle's P fields and xfrc)."""


def record(code, prec, st):
    """The kernel's state record (sr, si) of a State."""
    nj = NJ[code]
    nq, nv, nu = 7 + 2 * nj, 6 + 2 * nj, 2 * nj
    base = nq + 2 * nv + 5 * nu + 4
    nparam = (1 + 2 * nj) * 4 + 6 + 2 * nu + 15 if PERENV[code] else (85 if SLABS[code] else 0)
    sr = np.zeros(base + nparam)
    sr[:nq], sr[nq:nq + nv] = st["q"], st["v"]
    sr[nq + 2 * nv:nq + 2 * nv + nu] = st["q"][7:]          # act_len, act_vel: what the last substep left
    sr[nq + 2 * nv + nu:nq + 2 * nv + 2 * nu] = st["v"][6:]
    si = np.zeros(NSTATE_I, np.int32)
    if SLABS[code]:
        sr[base:base + 80] = st["seq"].reshape(-1)
        sr[base + 80:base + 85] = [1, 0, 0, 0, 0]
        si[1] = st.get("mode", 1)
    if PERENV[code]:
        P, nl = st["params"], 1 + 2 * nj
        o = base
        sr[o:o + nl] = P["P_mass"][:nl]; o += nl
        sr[o:o + 3 * nl] = P["P_com"][:3 * nl]; o += 3 * nl
        I0 = P["P_inertia"][:9].reshape(3, 3)
        sr[o:o + 6] = [I0[0, 0], I0[1, 1], I0[2, 2], I0[0, 1], I0[0, 2], I0[1, 2]]; o += 6
        sr[o:o + nu] = P["P_damping"][6:6 + nu]; o += nu
        sr[o:o + nu] = P["P_frictionloss"][6:6 + nu]; o += nu
        sr[o:o + 3] = P["P_pel_com"]; o += 3
        sr[o:o + 12] = P["xfrc"]
    if prec == 32:
        sr = sr.astype(np.float32)
    return sr, si


def oracle_env(o, code, st, seed=0):
    """A fresh oracle env holding the State (rounded as given: pass the fp32-rounded State for fp32 comparisons)."""
    envs = o.make_envs(1, seed=seed)
    if PERENV[code]:
        o.reset(envs)
    pad = lambda a, n: np.concatenate([a, np.zeros(n - len(a))])
    o.set_field(envs, 0, "qpos", pad(np.asarray(st["q"], np.float64), 19))
    o.set_field(envs, 0, "qvel", pad(np.asarray(st["v"], np.float64), 18))
    o.set_field(envs, 0, "qacc_warm", np.zeros(18))
    if SLABS[code]:
        o.set_field(envs, 0, "seq", st["seq"].reshape(-1))
        o.set_field(envs, 0, "seq_len", 1)
        o.set_field(envs, 0, "t1", 0)
        o.set_field(envs, 0, "t2", 0)
        o.set_field(envs, 0, "mode", st.get("mode", 1))
    if PERENV[code]:
        for k, a in st["params"].items():
            o.set_field(envs, 0, k, a)
    return envs


def rounded(code, prec, st):
    """The State as the kernel holds it at the precision (fp32: every real rounded to float)."""
    if prec == 64:
        return st
    r = lambda a: np.asarray(a, np.float64).astype(np.float32).astype(np.float64)
    out = State(st)
    for k in ("q", "v", "ctrl", "seq"):
        if k in st:
            out[k] = r(st[k])
    if "params" in st:
        P = dict(st["params"])
        for k in ("P_mass", "P_com", "P_inertia", "P_damping", "P_frictionloss", "P_pel_com", "xfrc"):
            P[k] = r(P[k])
        out["params"] = P
    return out


# ---------------------------------------------------------------- the crafted cases
def _nominal(mj):
    q = np.array(mj["cfg"]["nominal_qpos"], np.float64)
    return q


def _lift_to(mj, q, ch, k, target):
    """Shift the root height so that the k-th lowest candidate point of chain ch sits at height `target`."""
    z = np.sort(foot_points(mj, q)[ch][:, 2])
    q = q.copy()
    q[2] += target - z[k]
    return q


def _params_at_edges(o, mj, rng, code, hi):
    """The oracle's per-env parameters after a seeded reset (the root composite as drawn), with every other link's mass at
    0.95 / 1.05 of the model's, its CoM offset by -0.01 / +0.01 m on each axis, every joint's damping at 0.02 / 2 and friction
    loss at 0 / 2 (the ends of env_randomize's ranges), and non-zero wrenches on the pelvis and the torso."""
    envs = o.make_envs(1, seed=int(rng.integers(1 << 30)))
    o.reset(envs)
    P = {k: o.field(envs, 0, k) for k in ("P_mass", "P_com", "P_inertia", "P_damping", "P_frictionloss", "P_pel_com", "P_pel_mass")}
    nl = len(mj["links"])
    nu = nl - 1
    sgn = (1 if hi else -1)
    for b in range(1, nl):
        P["P_mass"][b] = mj["links"][b]["mass"] * (1 + 0.05 * sgn)
        P["P_com"][3 * b:3 * b + 3] = np.array(mj["links"][b]["com"]) + 0.01 * sgn * np.array([1, -1, 1])
    P["P_damping"][6:6 + nu] = 2.0 if hi else 0.02
    P["P_frictionloss"][6:6 + nu] = 2.0 if hi else 0.0
    P["xfrc"] = np.concatenate([rng.uniform(-20, 20, 3), rng.uniform(-5, 5, 3), rng.uniform(-20, 20, 3), rng.uniform(-5, 5, 3)])
    del P["P_pel_mass"]
    return P


def _base(name, rng, prec, z=None):
    mj, _, o = model(name)
    code = CODE[name]
    q = _nominal(mj)
    q[3:7] = quat(rng.normal(size=3) * 0.01)
    q[7:] += rng.uniform(-0.02, 0.02, len(q) - 7)
    if z is not None:
        q[2] = z
    v = rng.normal(size=len(q) - 1) * 0.2
    st = State(q=q, v=v, ctrl=rng.uniform(-20, 20, len(q) - 7))
    if SLABS[code]:
        st["seq"] = np.tile([0.0, 0.0, -1.0, 0.0], (20, 1))
        st["mode"] = 1
    if PERENV[code]:
        st["params"] = _params_at_edges(o, mj, rng, code, bool(rng.integers(2)))
    return mj, o, code, st


def case_free_flight(name, prec, rng, n=3):
    """No contact: the robot 2 m up, the root spinning at about 10 rad/s and joint velocities of several rad/s (Coriolis terms
    dominate)."""
    out = []
    for _ in range(n):
        mj, o, code, st = _base(name, rng, prec, z=2.0)
        st["v"][3:6] = rng.normal(size=3) * 6
        st["v"][6:] = rng.uniform(-6, 6, len(st["v"]) - 6)
        st["v"][:3] = rng.normal(size=3)
        out.append(st)
    return out


def case_contact_count(name, prec, rng, k):
    """Flat stance on the floor with the k lowest candidate points of the right foot in contact: the k-th lowest exactly at -delta;
    the right ankle's roll or pitch is solved (brentq) so that the (k+1)-th lowest sits at +delta, where one ankle angle can bring
    it there (otherwise it stays above by its own gap, asserted >= delta); the left foot lifted clear."""
    from scipy.optimize import brentq
    d = DELTA[prec]
    out = []
    for trial in range(2):
        mj, o, code, st = _base(name, rng, prec)
        q = st["q"]
        rch, lch = RFOOT[code], 1 - RFOOT[code]
        nj = NJ[code]
        q[7 + lch * nj + 3] += 0.6             # left knee / hip pitch: the left foot a few cm up
        q[7 + lch * nj + 2] -= 0.3
        zs = lambda qq: np.sort(foot_points(mj, qq)[rch][:, 2])
        if k < len(zs(q)):
            for dof in (7 + rch * nj + nj - 1 - trial, 7 + rch * nj + nj - 2 + trial):   # ankle roll / pitch, in turn
                def gap(a, dof=dof):
                    qq = q.copy()
                    qq[dof] = a
                    z = zs(qq)
                    return z[k] - z[k - 1] - 2 * d
                grid = q[dof] + np.linspace(-0.03, 0.03, 61)
                g = [gap(a) for a in grid]
                roots = [(grid[i], grid[i + 1]) for i in range(60) if g[i] * g[i + 1] < 0]
                if roots:
                    lo, hi = min(roots, key=lambda r: abs(r[0] - q[dof]))
                    q[dof] = brentq(gap, lo, hi, xtol=1e-15, rtol=1e-15)
                    break
        z = zs(q)
        q[2] -= z[k - 1] + d                      # the k-th lowest at -delta
        z = zs(q)
        assert abs(z[k - 1] + d) <= 1e-3 * d + 1e-15 and (k == len(z) or z[k] >= d * (1 - 1e-3)), (z[:k + 1], d)
        st["q"] = q
        st["v"] *= 0.25
        out.append(st)
    return out


def case_deep(name, prec, rng):
    """Deep penetration of a pitched box foot, its centre 4 mm under the floor: the four candidates mjc_PlaneBox keeps are two bottom
    and two TOP corners, interleaved in corner-index order.  (A box never has more than four corners on the plane side of its
    centre: the sign of each corner's offset flips with the corner opposite it, so four candidates is the most the rule allows,
    and the slots are never short.)"""
    out = []
    for pitch in (0.35, -0.35):
        mj, o, code, st = _base(name, rng, prec)
        q = st["q"]
        nj = NJ[code]
        rch = RFOOT[code]
        q[7 + rch * nj + nj - 2] += pitch    # ankle pitch
        lch = 1 - rch
        q[7 + lch * nj + 3] += 0.4
        pts = foot_points(mj, q)[rch]
        ctr = pts.mean(axis=0)
        q[2] -= ctr[2] + 0.004                # the box centre 4 mm under the floor
        pts = foot_points(mj, q)[rch]
        cand = [i for i in range(8) if pts[i, 2] < -1e-3 and pts[i, 2] <= pts.mean(axis=0)[2]]
        assert len(cand) == 4 and min(cand) < 4 <= max(cand), cand   # bottom and top corners among them, each >= 1 mm in
        st["q"] = q
        st["v"] *= 0.1
        out.append(st)
    return out


def case_limits(name, prec, rng, which):
    """Joint limits in free flight: 'lo' every limited joint at range_lo - delta moving further in, 'hi' at range_hi + delta,
    'inside' at delta inside either end moving out, 'mixed' alternating (every limit active at once)."""
    d = DELTA[prec]
    mj, o, code, st = _base(name, rng, prec, z=2.0)
    lo, hi, lim, _ = joint_table(mj)
    nu = len(lo)
    q, v = st["q"], st["v"]
    for u in range(nu):
        side = {"lo": 0, "hi": 1, "inside": u % 2, "mixed": u % 2}[which]
        if which == "inside":
            q[7 + u] = lo[u] + d if side == 0 else hi[u] - d
            v[6 + u] = -0.5 if side == 0 else 0.5      # moving towards the limit
        else:
            q[7 + u] = lo[u] - d if side == 0 else hi[u] + d
            v[6 + u] = (-0.5 if side == 0 else 0.5) * (1 if u % 3 else -1)   # into and out of the limit
    st["lim"] = lim
    return [st]


def case_floss(name, prec, rng):
    """H1 friction loss in free flight, every joint at once: joint velocity exactly 0, inside the quadratic zone, saturated.  No
    actuation and a resting root, so the joint accelerations are small and the row residual is set by the velocity."""
    mj, o, code, st = _base(name, rng, prec, z=2.0)
    st["ctrl"][:] = 0
    st["v"][:6] = 0
    st["params"]["P_frictionloss"][6:] = np.where(np.arange(len(st["params"]["P_frictionloss"]) - 6) < len(st["q"]) - 7, 2.0, 0.0)
    nu = len(st["q"]) - 7
    v = st["v"]
    for u in range(nu):
        v[6 + u] = [0.0, 1e-3, -1e-3, 2.0, -2.0][u % 5]
    return [st]


def _slab_under(mj, q, ch, top, dx=0.0, dy=0.0, yaw=0.0):
    """A slab whose top face is at height `top`, centred under chain ch's sole (plus dx, dy), yawed."""
    pts = foot_points(mj, q)[ch][:4]
    c = pts.mean(axis=0)
    return [c[0] + dx, c[1] + dy, top, yaw]


def case_step(name, prec, rng, kind):
    """Stepping stones (jvrc_step; terraces for jvrc_walk_terrain): 'centred' a slab under each foot in FORWARD mode (no floor),
    'overhang' the slab edge across the sole (sole-edge x slab-boundary crossings), 'riser' the toes inside a slab 0.1 m higher
    (a corner behind a riser), 'coplanar' the floor and two or three slabs at one height (multiplicity 2 and 3), 'full' both feet
    across slab boundaries with every crossing slot used (16 slots)."""
    mj, o, code, st = _base(name, rng, prec)
    q = st["q"]
    st["v"] *= 0.25
    seq = st["seq"]
    hx = mj["stepping"]["slab_half"][0] if "stepping" in mj else mj["terrain"]["strip_half"][0]
    rz = lambda ch: np.sort(foot_points(mj, q)[ch][:4, 2])
    if kind == "centred":
        st["mode"] = 4
        for ch in range(2):
            z = rz(ch)
            seq[ch] = _slab_under(mj, q, ch, z[-1] + 0.002, yaw=0.05 * (ch - 0.5))
    elif kind == "overhang":
        st["mode"] = 4
        for ch in range(2):
            z = rz(ch)
            seq[ch] = _slab_under(mj, q, ch, z[-1] + 0.002, dx=hx - 0.03 * (1 + ch), yaw=0.3 * (ch - 0.5))
    elif kind == "riser":
        st["mode"] = 1
        q[2] -= min(rz(0)[0], rz(1)[0]) + 0.002           # standing on the floor
        toe = max(foot_points(mj, q)[ch][:4, 0].max() for ch in range(2))
        yaw = rng.uniform(-0.1, 0.1)
        face = toe - 0.008
        seq[0] = [face + hx * np.cos(yaw), q[1] + hx * np.sin(yaw), 0.1, yaw]
    elif kind == "coplanar":
        st["mode"] = 1
        q[2] -= min(rz(0)[0], rz(1)[0]) + 0.0005
        seq[0] = [q[0] + 0.12, 0.0, 0.0, 0.05]
        seq[1] = [q[0] + 0.12, 0.2 * (2 * rng.integers(2) - 1), 0.0, -0.05]
        seq[2] = [q[0] + 0.05, 0.0, 0.0, 0.6]
    elif kind == "full":
        st["mode"] = 4
        for ch in range(2):
            z = rz(ch)
            c = _slab_under(mj, q, ch, z[-1] + 0.003)
            seq[2 * ch] = [c[0] + hx - 0.04, c[1] + 0.02, c[2], 0.4]
            seq[2 * ch + 1] = [c[0] - hx + 0.05, c[1] - 0.01, c[2], -0.3]
    elif kind == "terraces":
        st["mode"] = 1
        for ch in range(2):
            z = rz(ch)
            c = _slab_under(mj, q, ch, z[-1] + 0.002)
            seq[2 * ch] = [c[0] + hx - 0.02, c[1], c[2], 0.1]
            seq[2 * ch + 1] = [c[0] - hx + 0.03, c[1], c[2] - 0.004, -0.1]
    st["q"] = q
    return [st]


def cases(name, prec):
    """(case id, states, branch check) of a variant.  The branch check takes the list of (State, Work fields) after one substep
    and asserts the branch the case is for."""
    rng = np.random.default_rng([CODE[name], prec])
    code = CODE[name]
    out = [("free_flight", case_free_flight(name, prec, rng), lambda r: all(f["ncon"].sum() == 0 for _, f in r))]
    if not SLABS[code]:
        counts = (1, 2, 4) if code in (6,) else (1, 2, 3, 6)
        for k in counts:
            out.append((f"contacts_{k}", case_contact_count(name, prec, rng, k),
                        lambda r, k=k: all(f["ncon"][RFOOT[code]] == k and f["ncon"][1 - RFOOT[code]] == 0 for _, f in r)))
    if code == 6:
        out.append(("deep", case_deep(name, prec, rng), lambda r: all(f["ncon"][RFOOT[code]] == CPF[code] for _, f in r)))
    for which in ("lo", "hi", "inside", "mixed"):
        def chk(r, which=which):
            for st, f in r:
                lim = st["lim"]
                if which == "inside":
                    assert (f["lside"] == 0).all(), f["lside"]
                else:
                    want = np.where(lim, {"lo": 1, "hi": -1}.get(which, 0), 0)
                    if which == "mixed":
                        want = np.where(lim, np.where(np.arange(len(lim)) % 2 == 0, 1, -1), 0)
                    assert (f["lside"] == want).all(), (f["lside"], want)
            return True
        out.append((f"limits_{which}", case_limits(name, prec, rng, which), chk))
    if PERENV[code]:
        def floss_chk(r):
            for st, f in r:
                # after the solve fjar holds each row's residual J a - aref at the solution: inside (-flim, flim) the row is in
                # its quadratic zone, outside it is saturated
                # rows by their velocity class: every row at exactly 0 rad/s ends in the quadratic zone, every row at 2 rad/s
                # saturated, and rows at 1e-3 rad/s in the zone (the coupling of the fast joints may push one out)
                fj, fl, vj = f["fjar"], f["flim"], np.asarray(st["v"][6:])
                assert (vj == 0).any() and (np.abs(vj) == 2).any(), vj
                assert (np.abs(fj[vj == 0]) < fl[vj == 0]).all(), (fj, fl, vj)
                small = np.isclose(np.abs(vj), 1e-3)
                assert (np.abs(fj[small]) < fl[small]).any(), (fj, fl, vj)
                assert (np.abs(fj[np.abs(vj) == 2]) > fl[np.abs(vj) == 2]).all(), (fj, fl, vj)
            return True
        out.append(("friction_loss", case_floss(name, prec, rng), floss_chk))
    if code == 106:
        out += [
            ("slab_centred", case_step(name, prec, rng, "centred"),
             lambda r: all(f["ncorner"].min() == 4 and f["nfloor"] == 0 for _, f in r)),
            ("slab_overhang", case_step(name, prec, rng, "overhang"),
             lambda r: all((f["ncon"] > f["ncorner"]).all() and f["nside"].sum() == 0 for _, f in r)),
            ("riser", case_step(name, prec, rng, "riser"), lambda r: all(f["nside"].sum() > 0 for _, f in r)),
            ("coplanar", case_step(name, prec, rng, "coplanar"),
             lambda r: all(np.abs(f["cmul"]).max() >= 2 for _, f in r)),
            ("full_16_slots", case_step(name, prec, rng, "full"), lambda r: all((f["ncon"] == CPF[code]).all() for _, f in r)),
        ]
    if code == 206:
        out.append(("terraces", case_step(name, prec, rng, "terraces"),
                    lambda r: all((f["ncon"] > f["ncorner"]).any() and f["ncorner"].sum() > 0 for _, f in r)))
    return out


# ---------------------------------------------------------------- the comparison with the oracle
BOUNDS = {64: dict(qpos=1e-11, qvel=1e-10, qacc=1e-7, act_force=1e-12, grf=1e-7, cz=1e-11, vel=1e-10, cpos=1e-11, M=1e-12, qfs=1e-9),
          32: dict(qpos=1e-4, qvel=1e-4, qacc=1e-4, act_force=1e-5, grf=1e-3, cz=1e-5, vel=1e-4, cpos=1e-5, M=1e-5, qfs=1e-4)}


def _rel(err, ref):
    return float(np.max(np.abs(err) / np.maximum(1.0, np.abs(ref)))) if np.size(err) else 0.0


def oracle_run(name, st, nsub):
    """The oracle from State st: nsub mj_steps with ctrl held.  Returns the fields after the last one and the contacts, M and
    qfrc_smooth of the last step's pre-integration state."""
    mj, _, o = model(name)
    code = CODE[name]
    envs = oracle_env(o, code, st)
    nv = 6 + 2 * NJ[code]
    ctrl = np.zeros(12)
    ctrl[:len(st["ctrl"])] = st["ctrl"]
    for s in range(nsub):
        if s == nsub - 1:
            q0, v0 = o.field(envs, 0, "qpos")[:nv + 1].copy(), o.field(envs, 0, "qvel")[:nv].copy()
            con = o.contacts(envs, 0)
        o.mj_step(envs, 0, ctrl)
    g = lambda k: o.field(envs, 0, k)
    out = dict(qpos=g("qpos")[:nv + 1], qvel=g("qvel")[:nv], qacc=g("qacc")[:nv], act_force=g("act_force")[:nv - 6],
               grf=np.array([g("rfoot_grf")[0], g("lfoot_grf")[0]]), cz_min=g("contact_z_min")[0],
               foot_vel=np.stack([g("rfoot_vel"), g("lfoot_vel")]), root_vlin=g("root_vlin"), ncon=int(g("ncon")[0]),
               status=int(g("status")[0]), q0=q0, v0=v0, con=con)
    if not PERENV[code]:
        _, _, _, damp = joint_table(mj)
        out["M"] = o.mass_matrix(q0)[:nv, :nv]
        out["qfs"] = -o.bias(q0, v0)[:nv] - np.concatenate([np.zeros(6), damp * v0[6:]]) + np.concatenate([np.zeros(6), st["ctrl"]])
    return out


def compare(name, prec, st, f, ref, nsub):
    """Hold the kernel's Work fields f (after nsub substeps from State st) to the oracle's ref; returns the largest error-to-bound
    ratio per quantity (<= 1 passes) after asserting each."""
    code = CODE[name]
    B = BOUNDS[prec]
    nj = NJ[code]
    nv = 6 + 2 * nj
    r = {}
    r["qpos"] = np.max(np.abs(f["qpos"] - ref["qpos"])) / B["qpos"]
    r["qvel"] = np.max(np.abs(f["qvel"] - ref["qvel"])) / B["qvel"]
    if prec == 32:   # DESIGN §2's one-step bound, relative
        r["qpos"] = _rel(f["qpos"] - ref["qpos"], ref["qpos"]) / B["qpos"]
        r["qvel"] = _rel(f["qvel"] - ref["qvel"], ref["qvel"]) / B["qvel"]
    # qacc against max(1, max |ref|): the Newton solve stops on the norm of its gradient, so its error is a share of the whole
    # vector's scale, not of each component's
    r["qacc"] = float(np.max(np.abs(f["qacc"] - ref["qacc"]))) / max(1.0, float(np.max(np.abs(ref["qacc"])))) / B["qacc"]
    r["act_force"] = _rel(f["act_force"] - ref["act_force"], ref["act_force"]) / B["act_force"]
    rf = RFOOT[code]
    kgrf = np.array([f["grf"][rf], f["grf"][1 - rf]])
    kvel = np.stack([f["foot_vel"][rf], f["foot_vel"][1 - rf]])
    r["grf"] = _rel(kgrf - ref["grf"], ref["grf"]) / B["grf"]
    r["foot_vel"] = _rel(kvel - ref["foot_vel"], ref["foot_vel"]) / B["vel"]
    r["root_vlin"] = _rel(f["root_vlin"] - ref["root_vlin"], ref["root_vlin"]) / B["vel"]
    if f["nfloor"] > 0:
        r["cz_min"] = abs(f["cz_min"] - ref["cz_min"]) / B["cz"]
    assert f["status"] == 0 and ref["status"] == 0, (f["status"], ref["status"])
    # contact points per foot: the oracle's list with coplanar duplicates merged (one contact per supporting surface there), against
    # the kernel's slots (positions relative to o, the root position of the pre-integration state); the count of distinct points
    # must be equal and every slot must sit on one of them.  The multiplicities themselves are the coplanar case's branch check
    pos, dist, foot, kind = ref["con"]
    o_root = ref["q0"][:3]
    worst = 0.0
    for ch in range(2):
        sel = foot == ch      # the oracle's foot index is the chain
        opts = pos[sel] if sel.any() else np.zeros((0, 3))
        if SLABS[code] and len(opts):   # coplanar surfaces: one contact each at one point (H1's two coincident spheres stay two)
            opts = np.unique(np.round(opts, 12), axis=0)
        kp = f["cpos"][ch * CPF[code]:ch * CPF[code] + int(f["ncon"][ch])] + o_root
        assert len(kp) == len(opts), (name, "contacts of chain", ch, len(kp), len(opts))
        for p in kp:
            worst = max(worst, np.min(np.max(np.abs(opts - p), axis=1)) / B["cpos"])
    r["cpos"] = worst
    if "M" in ref:
        from solver_pieces import dense_from_lower, arrow_mask
        Md = dense_from_lower(nj, f["M"])
        r["M"] = _rel((Md - ref["M"])[arrow_mask(nj)], ref["M"][arrow_mask(nj)]) / B["M"]
        r["qfs"] = _rel(f["qfs"] - ref["qfs"], ref["qfs"]) / B["qfs"]
    r = {k: float(x) for k, x in r.items()}
    bad = {k: x for k, x in r.items() if not x <= 1}
    assert not bad, (name, prec, nsub, bad)
    return r


# ---------------------------------------------------------------- one case end to end (the host and device tests share it)
def twin_flat(name, prec):
    """The kernel's model: solver tolerance 1e-14 at fp64 (as the oracle), the trainer's default 1e-6 at fp32."""
    return model(name)[1] if prec == 64 else flat_at(name, 1e-6)


def case_ids(name):
    return [cid for cid, _, _ in cases(name, 64)]


def case_states(name, prec, cid):
    (states, chk), = [(s, c) for i, s, c in cases(name, prec) if i == cid]
    code = CODE[name]
    return [rounded(code, prec, s) for s in states], chk


def records(code, prec, states):
    recs = [record(code, prec, s) for s in states]
    return np.stack([r[0] for r in recs]), np.stack([r[1] for r in recs]), np.stack([s["ctrl"] for s in states])


def run_case(H, name, prec, cid, n_warps=1):
    """Case cid through the harness H after 1 and frame_skip substeps: its branch check, then every state against the oracle
    started from the same (at fp32: fp32-rounded) state.  Returns the largest error-to-bound ratios as text."""
    code = CODE[name]
    states, chk = case_states(name, prec, cid)
    sr, si, ctrl = records(code, prec, states)
    worst = {}
    for nsub in (1, int(model(name)[0]["cfg"]["frame_skip"])):
        _, _, work = H.run(sr, si, ctrl, nsub, n_warps)
        fs = [H.fields(w) for w in work]
        if nsub == 1:
            assert chk(list(zip(states, fs))), f"{name} {cid}: the case no longer reaches its branch"
        for s, f in zip(states, fs):
            for k, x in compare(name, prec, s, f, oracle_run(name, s, nsub), nsub).items():
                worst[k] = max(worst.get(k, 0.0), x)
    return " ".join(f"{k} {v:.2g}" for k, v in worst.items())


# ---------------------------------------------------------------- one control step of the shipped kernel at the crafted states
SEED = 13


def control_step_states(name, prec):
    """Every crafted state of a variant, one per env, with a seeded action each."""
    states = [s for cid in case_ids(name) for s in case_states(name, prec, cid)[0]]
    rng = np.random.default_rng([CODE[name], prec, 7])
    acts = rng.normal(size=(len(states), 2 * NJ[CODE[name]])) * 0.3
    if prec == 32:
        acts = acts.astype(np.float32).astype(np.float64)
    return states, acts


def oracle_control_step(name, states, acts, max_traj_len=400):
    """orc_step (through the oracle's batched step, auto-reset on) of every state from a fresh episode: no previous action, event
    counter 0, phase 0, env i of seed SEED.  -> obs, reward, done, qpos, qvel after the step."""
    mj, _, o = model(name)
    code = CODE[name]
    n = len(states)
    envs = o.make_envs(n, seed=SEED, first_id=0)
    o.batch_reset(envs, n)
    pad = lambda a, k: np.concatenate([np.asarray(a, np.float64), np.zeros(k - len(a))])
    for i, st in enumerate(states):
        nq = len(st["q"])
        o.set_field(envs, i, "qpos", pad(st["q"], 19))
        o.set_field(envs, i, "qvel", pad(st["v"], 18))
        for k in ("qacc_warm", "prev_prediction", "prev_action", "prev_torque", "act_force"):
            o.set_field(envs, i, k, np.zeros(len(o.field(envs, i, k))))
        o.set_field(envs, i, "act_len", pad(st["q"][7:], 12))
        o.set_field(envs, i, "act_vel", pad(st["v"][6:], 12))
        o.set_field(envs, i, "mode_ref", np.zeros(3))
        for k, val in (("have_prev", 0), ("phase", 0), ("traj_len", 0), ("ep_len", 0), ("rng_ctr", 0), ("status", 0)):
            o.set_field(envs, i, k, val)
        o.set_field(envs, i, "ep_rew", 0.0)
        o.set_field(envs, i, "mode", st.get("mode", 1) if SLABS[code] else 0)
        if SLABS[code]:
            o.set_field(envs, i, "seq", st["seq"].reshape(-1))
            for k, val in (("seq_len", 1), ("t1", 0), ("t2", 0), ("target_reached", 0), ("target_reached_frames", 0)):
                o.set_field(envs, i, k, val)
        if PERENV[code]:
            for k, a in st["params"].items():
                o.set_field(envs, i, k, a)
    obs, _, _, rew, done, _ = o.batch_step(envs, n, np.ascontiguousarray(acts), max_traj_len=max_traj_len)
    nv = 6 + 2 * NJ[code]
    q = np.stack([o.field(envs, i, "qpos")[:nv + 1] for i in range(n)])
    v = np.stack([o.field(envs, i, "qvel")[:nv] for i in range(n)])
    return obs, rew, done, q, v


def kernel_records(name, prec, states):
    """The crafted states as the env's records at the start of an episode (the event counter and phase 0, no previous action)."""
    code = CODE[name]
    sr, si, _ = records(code, prec, states)
    si[:, 1] = [s.get("mode", 1) if SLABS[code] else 0 for s in states]
    return sr, si
