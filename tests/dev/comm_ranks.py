"""The fused gradient exchange at world sizes above one on one GPU, for the tests (tests/test_gpu_exchange_ranks.py on the device,
tests/test_exchange_harness.py on the host): builds of the device harness tests/dev/comm_dev.cu and of the product's
comm_kernels.cu alone (to compare their SASS), a ctypes + torch wrapper of W stand-in ranks, and the float32 / float64
references each step is held to.

The reduction the kernels specify: starting from +0.0f, add g_0 ... g_{W-1} in rank order in float32, then multiply by
(1.0f / W).  Every rank computes exactly that, so replicas never drift."""
import ctypes
import os
import re
import subprocess

import numpy as np

from solver_pieces import ROOT, _compiled

HERE = os.path.dirname(os.path.abspath(__file__))
COMM_SRC = os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", "comm_kernels.cu")
HEADER = os.path.join(ROOT, "include", "lhw_b200.h")
DEV_SRC = os.path.join(HERE, "comm_dev.cu")

MAX_WORLD = 16
WORLDS = [1, 2, 3, 4, 5, 8, 16]           # 3 and 5: 1 / W is inexact in float32; 16 is MAX_WORLD
U32 = 2.0 ** -24
PAD = 37                                   # sentinel floats after n_total in param / m / v
SENTINEL = np.uint32(0x7FC0DEAD)           # a NaN payload no kernel produces
SPIN_LIMIT = 2 ** 16                       # polls before a wait of the stand-in ranks gives up
ST_EPOCH, ST_ERROR, ST_TICKET, ST_STEP = range(4)
D = 2.0 ** -7                              # desired_kl, as tests/test_gpu_adaptive_lr.py: 2 D and D / 2 exact in float32
# non-default hyper-parameters (the learner's are lr 3e-4, betas (0.9, 0.999), eps 1e-5, max_norm 0.05)
HP = dict(lr=7e-4, b1=0.85, b2=0.995, eps=3e-6, max_norm=0.7)
PARAM_LR = 1e-4                            # parameter allowance |dp| <= ulp32(p) + PARAM_LR lr (DESIGN.md §2)
MOMENT_BOUND = 2e-5                        # moments, ||d||_2 / ||ref||_2 per network (DESIGN.md §2)
KERNELS = ["exchange_reduce_kernelILb0E", "exchange_reduce_kernelILb1E", "clip_adam_pair_kernelILb0E",
           "clip_adam_pair_kernelILb1E", "exchange_finish_kernel"]


# ---------------------------------------------------------------- builds and SASS
def nvcc_command(out, src, extra=()):
    """The package's nvcc flags (learninghumanoidwalking_b200/build.py) without the ptxas report, then `extra`."""
    from learninghumanoidwalking_b200 import build as B
    flags = " ".join(B.NVCC_FLAGS).replace("-Xptxas -v", "").split()
    return [os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")] + flags + list(extra) + ["-shared", "-o", out, src]


def build_harness():
    return _compiled("libcomm_dev", [DEV_SRC, COMM_SRC, HEADER],
                     lambda out: nvcc_command(out, DEV_SRC, ["-Xcompiler", "-fvisibility=hidden"]))


def build_product():
    """comm_kernels.cu alone with the package's flags: the machine code liblhw_b200.so carries for the exchange."""
    return _compiled("libcomm_product", [COMM_SRC, HEADER], lambda out: nvcc_command(out, COMM_SRC))


def cuobjdump():
    return os.path.join(os.path.dirname(os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")), "cuobjdump")


def sass_functions(lib):
    """{kernel name without its anonymous-namespace prefix: SASS lines}.  The prefix (nvcc derives it from the source path, as
    build.py:_sass_md5 notes) and the dump's `identifier =` line are the only things that tell two builds of one source apart."""
    sass = subprocess.run([cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    out, name = {}, None
    for line in sass.splitlines():
        if line.startswith("identifier ="):
            continue
        line = re.sub(r"\d+_GLOBAL__N__[0-9a-f]+_\d+_\w+?_cu_[0-9a-f]{8}", "_GLOBAL__N_", line)
        m = re.search(r"Function : (\S+)", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name is not None and line.strip():
            out[name].append(line.strip())
    return out


# ---------------------------------------------------------------- sizes
def network_sizes():
    """{case: (n_total, n_actor)} of the learner's flat buffer: Gaussian_FF_Actor then FF_V at each environment's dimensions."""
    from learninghumanoidwalking_b200.rl.imitation import ENV_DIMS
    from learninghumanoidwalking_b200.rl.policies.actor import Gaussian_FF_Actor
    from learninghumanoidwalking_b200.rl.policies.critic import FF_V
    out = {}
    for env, learn_std in (("jvrc_walk", False), ("jvrc_step", False), ("h1", False), ("jvrc_walk", True)):
        o, a = ENV_DIMS[env]
        na = sum(p.numel() for p in Gaussian_FF_Actor(o, a, learn_std=learn_std).parameters())
        nc = sum(p.numel() for p in FF_V(o).parameters())
        out[env + ("_learn_std" if learn_std else "")] = (na + nc, na)
    return out


def grid_cap_size(n_sm):
    """One float4 past K1's resident-grid cap (8 blocks of 1024 floats per SM) plus a 3-float tail: every thread of K1 takes
    two grid-stride iterations or more."""
    return 8 * n_sm * 1024 + 7


def actor_splits(n, boundary=None):
    """n_actor at 0, 1, a multiple of 4, 4k + 1 and 4k + 3 (inside a float4), inside the scalar tail after the last full float4
    when it has two floats or more, n, and the networks' own boundary."""
    n4 = n // 4
    cand = [0, 1, 4 * (n4 // 2), 4 * (n4 // 2) + 1, 4 * (n4 // 2) + 3, 4 * n4 + 1 if n % 4 >= 2 else None, n, boundary]
    out = []
    for a in cand:
        if a is not None and 0 <= a <= n and a not in out:
            out.append(a)
    return out


# ---------------------------------------------------------------- references
def f32(x):
    return np.float32(x)


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def reduce_f32(gs):
    """gs [W, n] float32 -> the specified float32 average (module docstring)."""
    s = np.zeros(gs.shape[1], np.float32)
    for g in gs:
        s = s + g
    return s * (f32(1) / f32(len(gs)))


def reduce_bound(gs):
    """|reduce_f32 - float64 mean| <= (W + 1) u32 sum_r |g_r| / W: W - 1 roundings of the sum, 1 / W and the product."""
    W = len(gs)
    return (W + 1) * U32 * np.abs(gs.astype(np.float64)).sum(0) / W


def norms64(reduced, n_actor):
    r = reduced.astype(np.float64)
    return float(np.sqrt(np.sum(r[:n_actor] ** 2))), float(np.sqrt(np.sum(r[n_actor:] ** 2)))


def clip_coef(t, max_norm):
    """min(1, max_norm / (t + 1e-6f)) in float32 (torch.nn.utils.clip_grad_norm_ on float32 tensors)."""
    c = f32(max_norm) / (f32(t) + f32(1e-6))
    return f32(1) if c > 1 else c


def ulp32(x):
    x = np.abs(np.asarray(x, np.float64))
    return np.where(x > 0, 2.0 ** (np.floor(np.log2(np.maximum(x, 1e-38))) - 23), 2.0 ** -149)


def adam64(p, m, v, reduced, coef_a, coef_c, n_actor, t, hp):
    """One clip + Adam step in float64 from float32 state, with the float32 hyper-parameters the kernels take, widened."""
    g = reduced.astype(np.float64)
    g[:n_actor] *= float(coef_a)
    g[n_actor:] *= float(coef_c)
    lr, b1, b2, eps = (float(f32(hp[k])) for k in ("lr", "b1", "b2", "eps"))
    m = b1 * m.astype(np.float64) + (1 - b1) * g
    v = b2 * v.astype(np.float64) + (1 - b2) * g * g
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    p = p.astype(np.float64) - lr / bc1 * m / (np.sqrt(v) / np.sqrt(bc2) + eps)
    return p, m, v


def scaled_grads(rng, W, n, n_actor, clipped, max_norm):
    """Per-rank float32 gradients whose float64 average has norm 3 max_norm on each network marked clipped and 0.3 max_norm on
    the others.  From 8 floats on, a few elements are -0.0 on every rank: the specified sum starts at +0.0f and gives +0.0."""
    g = rng.standard_normal((W, n))
    if n >= 8:
        g[:, rng.choice(n, 3, replace=False)] = -0.0
    mean = g.mean(0)
    for (lo, hi), c in zip(((0, n_actor), (n_actor, n)), clipped):
        nrm = np.linalg.norm(mean[lo:hi])
        if nrm > 0:
            g[:, lo:hi] *= (3.0 if c else 0.3) * max_norm / nrm
    return g.astype(np.float32)


# ---------------------------------------------------------------- the adaptive rate: per-rank KL sets
def kl_cases(W, seed=0):
    """[(name, float32 KLs of the W ranks, expected move of the rate)] with distinct KLs where W allows."""
    from learninghumanoidwalking_b200.rl.schedule import adapt_lr, rank_mean_kl
    rng = np.random.default_rng(seed + W)
    off = np.arange(W) - (W - 1) / 2
    cases = [("on_2D", 2 * D + off * 2.0 ** -12, "same"),             # mean exactly 2 D: not above it
             ("on_D/2", D / 2 + off * 2.0 ** -16, "same"),            # mean exactly D / 2: not below it
             ("above_2D", rng.uniform(2.5 * D, 4 * D, W), "down"),
             ("below_D/2", rng.uniform(D / 8, D / 3, W), "up")]
    nan = rng.uniform(D / 8, D / 3, W)
    nan[W // 2] = np.nan                                              # would raise the rate without the NaN
    cases.append(("nan_on_one_rank", nan, "same"))
    if W >= 4:
        # rank order: 1 + e = 1, 1 - 1 = 0, 0 + e = e > 0 -> raised; reversed: e - 1 = -1, -1 + e = -1, -1 + 1 = 0 -> unchanged
        cases.append(("order", np.array([1.0, 2.0 ** -60, -1.0, 2.0 ** -60] + [0.0] * (W - 4)), "up"))
    out = []
    for name, kls, move in cases:
        kls = np.asarray(kls, np.float32)
        lr0 = 3e-4
        new = adapt_lr(lr0, rank_mean_kl(kls), D)
        assert (new < lr0, new > lr0, new == lr0) == (move == "down", move == "up", move == "same"), (name, W, new)
        out.append((name, kls, move))
    return out


# ---------------------------------------------------------------- W stand-in ranks on one device
class _CudaArray:
    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3, "strides": None}


def _lib():
    L = ctypes.CDLL(build_harness())
    vp, ll, f, d, i = ctypes.c_void_p, ctypes.c_longlong, ctypes.c_float, ctypes.c_double, ctypes.c_int
    sig = {"cx_create": (i, [vp, ll, i, i]), "cx_destroy": (None, [vp, i]), "cx_pointers": (None, [vp, vp]),
           "cx_set_spin_limit": (None, [vp, ll]), "cx_preset_later_peers": (i, [vp, vp]),
           "cx_step": (i, [vp, vp, vp, vp, ll, ll, f, f, f, f, f, vp]),
           "cx_step_adaptive": (i, [vp, vp, vp, vp, ll, ll, vp, vp, d, f, f, f, f, vp]),
           "cx_status": (i, [vp, vp, vp, vp, vp]), "cx_last_error": (ctypes.c_char_p, [])}
    for name, (res, args) in sig.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = res, args
    return L


class Ranks:
    """W comm records of n floats on the current device, wired to each other.  Per rank: torch views of its grad, flags (int32:
    MAX_WORLD flag words, then the KL words), reduced, coef, state (int32) and lr (float64), and its own param / m / v of
    n + PAD floats (sentinels after n)."""
    _L = None

    def __init__(self, n, world, p0):
        import torch
        if Ranks._L is None:
            Ranks._L = _lib()
        self.n, self.world = n, world
        self._c = (ctypes.c_void_p * world)()
        dev = torch.cuda.current_device()
        if self._L.cx_create(self._c, n, world, dev):
            raise RuntimeError(self._L.cx_last_error().decode())
        for r in range(world):
            # no wait spins here; a protocol slip should end in an error word after milliseconds, not the default minute
            self.set_spin_limit(r, SPIN_LIMIT)
        self._keep, self.grad, self.flags, self.reduced, self.coef, self.state, self.lr = [], [], [], [], [], [], []
        for r in range(world):
            o = (ctypes.c_ulonglong * 8)()
            self._L.cx_pointers(self._c[r], o)
            for dst, ptr, cnt, ts in ((self.grad, o[0], o[6], "<f4"), (self.flags, o[1], o[7], "<i4"), (self.reduced, o[2], o[6], "<f4"),
                                      (self.coef, o[3], 4, "<f4"), (self.state, o[4], 4, "<i4"), (self.lr, o[5], 1, "<f8")):
                a = _CudaArray(ptr, cnt, ts)
                self._keep.append(a)
                dst.append(torch.as_tensor(a, device=dev))
            # the padding of `reduced` after n holds sentinels: nothing may write there
            self.reduced[r][n:].view(torch.int32).fill_(int(SENTINEL.view(np.int32)))
        tail = np.full(PAD, SENTINEL).view(np.float32)
        init = (np.concatenate([p0, tail]), np.concatenate([np.zeros(n, np.float32), tail]))
        self.p = [torch.tensor(init[0], device=dev) for _ in range(world)]
        self.m = [torch.tensor(init[1], device=dev) for _ in range(world)]
        self.v = [torch.tensor(init[1], device=dev) for _ in range(world)]

    def close(self):
        if self._c is not None:
            import torch
            torch.cuda.synchronize()
            self._L.cx_destroy(self._c, self.world)
            self._c = None

    def set_spin_limit(self, r, polls):
        self._L.cx_set_spin_limit(self._c[r], polls)

    def set_grads(self, gs):
        import torch
        for r in range(self.world):
            self.grad[r][:self.n].copy_(torch.from_numpy(gs[r]))

    def set_kl_words(self, kls):
        """Each rank's KL into its KL word (a later rank writes its own only in its K1, after an earlier rank has read it)."""
        import torch
        for r in range(self.world):
            self.flags[r][MAX_WORLD:MAX_WORLD + 1].view(torch.float32).fill_(float(kls[r]))

    def step(self, r, n_actor, hp, kl=None, preset=True):
        """Rank r's three launches on the current stream, after the flag words of the later ranks are preset (preset=False
        leaves them as they are); kl: this rank's [1] float32 KL tensor -> the adaptive instantiation at desired_kl D."""
        import torch
        st = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
        c = self._c[r]
        if preset and self._L.cx_preset_later_peers(c, st):
            raise RuntimeError(self._L.cx_last_error().decode())
        ptrs = [self.p[r].data_ptr(), self.m[r].data_ptr(), self.v[r].data_ptr()]
        if kl is None:
            rc = self._L.cx_step(c, *ptrs, n_actor, self.n, hp["lr"], hp["b1"], hp["b2"], hp["eps"], hp["max_norm"], st)
        else:
            rc = self._L.cx_step_adaptive(c, *ptrs, n_actor, self.n, kl.data_ptr(), self.lr[r].data_ptr(), D, hp["b1"], hp["b2"],
                                          hp["eps"], hp["max_norm"], st)
        if rc:
            raise RuntimeError(self._L.cx_last_error().decode())

    def status(self, r):
        """(return code, error word, Adam steps, norms, message)."""
        import torch
        err, steps, norms = ctypes.c_int(0), ctypes.c_int(0), (ctypes.c_float * 2)()
        rc = self._L.cx_status(self._c[r], ctypes.byref(err), ctypes.byref(steps), norms,
                               ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
        return rc, err.value, steps.value, (norms[0], norms[1]), self._L.cx_last_error().decode() if rc else ""

    def host(self, r):
        """Rank r's buffers on the host: param, m, v (with their sentinel tails), reduced (with its padding), coef, state, flags."""
        return {k: getattr(self, k)[r].cpu().numpy() for k in ("p", "m", "v", "reduced", "coef", "state", "flags")}
