"""The Newton solver pieces of sim_core.h for the tests (tests/test_gpu_solver_pieces.py on the device, tests/test_solver_harness.py
on the host): builds and ctypes wrappers of the device harness tests/dev/solver_dev.cu and of its host twin tests/dev/solver_emu.cpp,
random inputs, and the numpy float64 references with the error bounds each piece is held to.

Arrow words: a symmetric [root | chain0 | chain1] matrix as sim_core.h's Arrow record stores it, r (6 x 6), x (2 x 6 x nj: root
rows, chain columns), c (2 x nj x nj).  The pieces read and write only the lower triangles of r and c."""
import ctypes
import hashlib
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
BUILD_DIR = os.path.join(HERE, "_build")
SIM_CORE = os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", "sim_core.h")
RECORD_H = os.path.join(HERE, "solver_record.h")
DEV_SRC = os.path.join(HERE, "solver_dev.cu")
EMU_SRC = os.path.join(HERE, "solver_emu.cpp")

VARIANTS = [(6, 0), (5, 0), (6, 1), (6, 2), (5, 3)]      # (nj, tk) of LHW_FOR_EACH_VARIANT
CPF = {(6, 0): 4, (5, 0): 6, (6, 1): 8, (6, 2): 8, (5, 3): 6}
FLOSS = {v: v[0] == 5 for v in VARIANTS}                # the H1 variants carry dof friction-loss rows
U = {64: 2.0 ** -53, 32: 2.0 ** -24}                     # unit roundoff

# Relative error of the reciprocal square root that scales each pivot (sim_core.h m_rsqrt), device build.
#   fp64: a float seed, rsqrt.approx.ftz.f32 (PTX ISA: at most 2^-22.9 relative) of the operand rounded to float (2^-25 more),
#         then one Newton step in double, which squares it: 1.5 e^2, plus a few roundings of the step.
#   fp32: rsqrtf, at most 2 ulp (CUDA Programming Guide, single-precision intrinsics), 2^-22 relative.
# The host emulation's 1 / sqrt is two correctly rounded operations, well inside both.
RSQRT = {64: 1.5 * (2.0 ** -22.9 + 2.0 ** -25) ** 2 + 4 * U[64], 32: 2.0 ** -22}


def code(v):
    return v[0] + 100 * v[1]


def nwords(nj):
    return 36 + 12 * nj + 2 * nj * nj


def solve_eta(prec, n):
    """Componentwise backward error of the arrow Cholesky solve in units of |H||x|: (3n + 1) u, Higham's bound for a Cholesky
    factorisation followed by two triangular solves (Accuracy and Stability of Numerical Algorithms, Thm. 10.4), plus 2 RSQRT.
    A pivot scale with relative error d is used both for the column below the pivot and in the back substitution, so L L' = H
    still holds for every off-diagonal entry; the diagonal entry k moves by 2 d times the pivot, which is at most H_kk."""
    return (3 * n + 1) * U[prec] + 2 * RSQRT[prec]


# ---------------------------------------------------------------- builds (once per source content)
def _compiled(name, sources, cmd):
    h = hashlib.sha256(" ".join(cmd("")).encode())
    for s in sources:
        h.update(open(s, "rb").read())
    lib = os.path.join(BUILD_DIR, f"{name}.{h.hexdigest()[:16]}.so")
    if not os.path.exists(lib):
        os.makedirs(BUILD_DIR, exist_ok=True)
        tmp = f"{lib}.{os.getpid()}.tmp"
        r = subprocess.run(cmd(tmp), capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"building {name} failed:\n{r.stdout}{r.stderr}")
        os.replace(tmp, lib)
    return lib


def nvcc_command(out):
    """The package's nvcc flags (learninghumanoidwalking_b200/build.py) without the ptxas report."""
    from learninghumanoidwalking_b200 import build as B
    flags, i = [], 0
    while i < len(B.NVCC_FLAGS):
        if B.NVCC_FLAGS[i:i + 2] == ["-Xptxas", "-v"]:
            i += 2
            continue
        flags.append(B.NVCC_FLAGS[i])
        i += 1
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return [nvcc] + flags + ["-shared", "-o", out, DEV_SRC]


def build_device():
    return _compiled("libsolver_dev", [DEV_SRC, RECORD_H, SIM_CORE], nvcc_command)


def build_emu():
    return _compiled("libsolver_emu", [EMU_SRC, RECORD_H, SIM_CORE],
                     lambda out: ["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", out, EMU_SRC])


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


class Pieces:
    """The entry points of one build: device=True loads solver_dev.cu (dev_*), else solver_emu.cpp (emu_*; no mma_lanes)."""

    def __init__(self, device):
        self.device = device
        self.lib = ctypes.CDLL(build_device() if device else build_emu())
        if device:
            self._lanes, self._hessian = self.lib.dev_mma_lanes, self.lib.dev_hessian
            self._arrow, self._layout = self.lib.dev_arrow_solve, self.lib.dev_layout
        else:
            self._lanes, self._hessian = None, self.lib.emu_hessian
            self._arrow, self._layout = self.lib.arrow_emu_solve, self.lib.emu_layout
        for f in filter(None, (self._lanes, self._hessian, self._arrow, self._layout)):
            f.restype = ctypes.c_int

    def _n(self, n, n_warps):   # the problem count, then (device only) the warps per block
        return [ctypes.c_int(n)] + ([ctypes.c_int(n_warps)] if self.device else [])

    def layout(self, v, prec):
        o = np.zeros(10, np.int64)
        assert self._layout(code(v), prec, _p(o)) == 0
        k = ["size", "H", "H_bytes", "hdinv", "hdinv_bytes", "sdir", "sdir_bytes", "status", "T", "T_bytes"]
        return dict(zip(k, (int(x) for x in o)))

    def mma_lanes(self, ks, a, b, c):
        d = np.zeros((32, 2))
        a, b, c = (np.ascontiguousarray(x, np.float64) for x in (a, b, c))
        assert self._lanes(ks, _p(a), _p(b), _p(c), _p(d)) == 0
        return d

    def hessian(self, v, inp, n_warps=1):
        """inp: hessian_inputs() of n problems stacked on a leading axis.  -> H words, T [n, 2, NA, 6], records before / after."""
        nj = v[0]
        n = inp["S"].shape[0]
        a = {k: np.ascontiguousarray(x, np.int32 if k in ("ncon", "lside") else np.float64) for k, x in inp.items()}
        H, T = np.zeros((n, nwords(nj))), np.zeros((n, 2, 6 + nj, 6))
        size = self.layout(v, 64)["size"]
        rin, rout = np.zeros((n, size), np.uint8), np.zeros((n, size), np.uint8)
        args = [a[k] for k in ("S", "Af", "ncon", "M", "lside", "ljar", "lD", "fjar", "flim", "fD")]
        rc = self._hessian(code(v), *self._n(n, n_warps), *map(_p, args), _p(H), _p(T), _p(rin), _p(rout))
        assert rc == 0, rc
        return H, T, rin, rout

    def arrow(self, v, prec, Hw, b, status=None, n_warps=1):
        """arrow_factor_solve of n problems: Hw [n, words], b [n, NV] (rounded to the precision on the way in).
        -> factor words, hdinv, x, status, records before / after."""
        Hw, b = np.ascontiguousarray(Hw, np.float64), np.ascontiguousarray(b, np.float64)
        n, nv = b.shape
        status = np.zeros(n, np.int32) if status is None else np.ascontiguousarray(status, np.int32)
        F, hd, x, st = np.zeros_like(Hw), np.zeros((n, nv)), np.zeros((n, nv)), np.zeros(n, np.int32)
        size = self.layout(v, prec)["size"]
        rin, rout = np.zeros((n, size), np.uint8), np.zeros((n, size), np.uint8)
        rc = self._arrow(code(v), prec, *self._n(n, n_warps), _p(Hw), _p(b), _p(status), _p(F), _p(hd), _p(x), _p(st),
                         _p(rin), _p(rout))
        assert rc == 0, rc
        return F, hd, x, st, rin, rout


def written_mask(lay, regions):
    """Bytes of one record that a piece may write: the named regions of layout()."""
    m = np.zeros(lay["size"], bool)
    for r in regions:
        nb = 4 if r == "status" else lay[r + "_bytes"]
        m[lay[r]:lay[r] + nb] = True
    return m


# ---------------------------------------------------------------- arrow-packed matrices
def arrow_words(nj, dense):
    r = dense[:6, :6]
    x = np.stack([dense[:6, 6 + ch * nj:6 + (ch + 1) * nj] for ch in range(2)])
    c = np.stack([dense[6 + ch * nj:6 + (ch + 1) * nj, 6 + ch * nj:6 + (ch + 1) * nj] for ch in range(2)])
    return np.concatenate([r.ravel(), x.ravel(), c.ravel()])


def arrow_blocks(nj, words):
    r = words[:36].reshape(6, 6)
    x = words[36:36 + 12 * nj].reshape(2, 6, nj)
    c = words[36 + 12 * nj:].reshape(2, nj, nj)
    return r, x, c


def dense_from_lower(nj, words):
    """The symmetric matrix the pieces see in arrow words: lower triangles of r and c, all of x."""
    r, x, c = arrow_blocks(nj, words)
    nv = 6 + 2 * nj
    D = np.zeros((nv, nv))
    D[:6, :6] = np.tril(r) + np.tril(r, -1).T
    for ch in range(2):
        s = slice(6 + ch * nj, 6 + (ch + 1) * nj)
        D[:6, s] = x[ch]
        D[s, :6] = x[ch].T
        D[s, s] = np.tril(c[ch]) + np.tril(c[ch], -1).T
    return D


def arrow_mask(nj):
    """The arrow pattern of a dense matrix: True where entries are stored (the chain0-chain1 coupling is structurally zero)."""
    nv = 6 + 2 * nj
    m = np.ones((nv, nv), bool)
    m[6:6 + nj, 6 + nj:] = False
    m[6 + nj:, 6:6 + nj] = False
    return m


def random_arrow_spd(nj, kappa, rng, prec=64):
    """A random symmetric positive definite matrix with the arrow pattern and 2-norm condition number kappa, rounded to the
    precision (returned in float64, with the condition number of the rounded matrix).  kappa = 1: a multiple of the identity."""
    nv = 6 + 2 * nj
    if kappa == 1:
        Hd = rng.uniform(0.5, 2.0) * np.eye(nv)
    else:
        G = rng.normal(size=(nv, nv))
        A = np.where(arrow_mask(nj), (G + G.T) / 2, 0.0)
        lam = np.linalg.eigvalsh(A)
        s = (lam[-1] - kappa * lam[0]) / (kappa - 1)    # (lam_max + s) / (lam_min + s) = kappa
        Hd = A + s * np.eye(nv)
    if prec == 32:
        Hd = Hd.astype(np.float32).astype(np.float64)
    lam = np.linalg.eigvalsh(Hd)
    assert lam[0] > 0
    return Hd, lam[-1] / lam[0]


ORDER = lambda nj: list(range(6, 6 + 2 * nj)) + list(range(6))   # the kernel's elimination order: chain 0, chain 1, root


def factor_reference(nj, Hd):
    """numpy's Cholesky of Hd in the kernel's elimination order, as the kernel stores it: strict lower triangles of the chain
    blocks (c) and of the root block (r), the coupling X_c = B_c L_c^-T (x), the diagonal of the root block's Schur complement
    C - sum_c X_c X_c' (what the kernel leaves on r's diagonal), and hdinv = 1 / diag(L) in the global dof order."""
    p = ORDER(nj)
    L = np.linalg.cholesky(Hd[np.ix_(p, p)])
    c = np.stack([L[ch * nj:(ch + 1) * nj, ch * nj:(ch + 1) * nj] for ch in range(2)])
    x = np.stack([L[2 * nj:, ch * nj:(ch + 1) * nj] for ch in range(2)])
    LC = L[2 * nj:, 2 * nj:]
    hdinv = np.zeros(6 + 2 * nj)
    hdinv[p] = 1.0 / np.diag(L)
    return dict(c=c, x=x, r=LC, schur_diag=(LC ** 2).sum(axis=1), hdinv=hdinv, L=L)


def residual(Hd, x, b):
    """H x - b and |H| |x| in extended precision (np.longdouble), so that the residual of an fp64 solution is not lost in the
    rounding of its own evaluation."""
    Hl, xl = Hd.astype(np.longdouble), x.astype(np.longdouble)
    return (Hl @ xl - b.astype(np.longdouble)).astype(np.float64), (np.abs(Hl) @ np.abs(xl)).astype(np.float64)


# ---------------------------------------------------------------- the Newton Hessian
def hessian_inputs(v, ncon, rng, spd=False):
    """One problem for newton_hessian_f64: random S, Af (general 6 x 6, or symmetric positive semidefinite with spd=True) and an
    arrow-SPD M; the limit rows cover inactive rows and active rows with ljar < 0, = 0 and > 0, the friction-loss rows
    (variants with FLOSS) residuals inside, outside and exactly at -flim and +flim."""
    nj = v[0]
    nv, nu = 6 + 2 * nj, 2 * nj
    S = rng.normal(size=(nv, 6))
    if spd:
        Af = np.stack([(lambda g: g @ g.T)(rng.normal(size=(6, 6))) for _ in range(2)])
    else:
        Af = rng.normal(size=(2, 6, 6))
    G = rng.normal(size=(nv, nv))
    Md = np.where(arrow_mask(nj), G @ G.T + nv * np.eye(nv), 0.0)
    # limit rows: (side, sign of ljar); ljar = 0 exactly is not active (strict ljar < 0)
    lcases = [(0, -1), (0, 1), (1, -1), (-1, -1), (1, 1), (-1, 1), (1, 0), (-1, 0)]
    lc = [lcases[i] for i in rng.permutation(np.resize(np.arange(len(lcases)), nu))]
    lside = np.array([s for s, _ in lc], np.int32)
    ljar = np.array([g * rng.uniform(0.1, 2.0) for _, g in lc])
    flim = rng.uniform(0.2, 1.5, size=nu)
    # friction-loss residual: inside, outside below / above, exactly at -flim / +flim (strict inequality: no D there)
    fk = rng.permutation(np.resize(np.arange(5), nu))
    fjar = np.choose(fk, [flim * rng.uniform(-0.95, 0.95, size=nu), -flim * rng.uniform(1.05, 2, size=nu),
                          flim * rng.uniform(1.05, 2, size=nu), -flim, flim])
    return dict(S=S, Af=Af, ncon=np.array(ncon, np.int32), M=arrow_words(nj, Md), lside=lside, ljar=ljar,
                lD=rng.uniform(1, 2, size=nu), fjar=fjar, flim=flim, fD=rng.uniform(1, 2, size=nu))


def stack(problems):
    return {k: np.stack([p[k] for p in problems]) for k in problems[0]}


def hessian_reference(v, inp):
    """Dense H = M + sum_f S_f' Af_f S_f + the diagonal D of the active limit and friction-loss rows, T_f = (Af_f S_f)', in
    extended precision; and the elementwise bounds |H - H_ref| <= 16 u (sum_f |S_f|' |Af_f| |S_f| + |M| + D),
    |T_f - T_ref| <= 16 u |Af_f| |S_f|.  16 u covers the 6-term sums of T_f followed by the tiles' sums of up to 12 products and C,
    each rounding once per term at worst; the largest ratio measured on the device is about 0.2."""
    nj = v[0]
    nv, na, nu = 6 + 2 * nj, 6 + nj, 2 * nj
    ld = np.longdouble
    S, Af = inp["S"].astype(ld), inp["Af"].astype(ld)
    Md = dense_from_lower(nj, inp["M"]).astype(ld)
    H, mag = Md.copy(), np.abs(Md)
    T, Tb = np.zeros((2, na, 6)), np.zeros((2, na, 6))
    for f in range(2):
        if not inp["ncon"][f]:
            continue
        dofs = list(range(6)) + [6 + f * nj + j for j in range(nj)]
        Sf = S[dofs].T
        Tf = Af[f] @ Sf
        T[f] = Tf.T.astype(np.float64)
        Tb[f] = (np.abs(Af[f]) @ np.abs(Sf)).T.astype(np.float64)
        H[np.ix_(dofs, dofs)] += Sf.T @ Tf
        mag[np.ix_(dofs, dofs)] += np.abs(Sf.T) @ np.abs(Af[f]) @ np.abs(Sf)
    for j in range(nu):
        d = 6 + j
        if inp["lside"][j] and inp["ljar"][j] < 0:
            H[d, d] += ld(inp["lD"][j])
            mag[d, d] += ld(inp["lD"][j])
        if FLOSS[v] and -inp["flim"][j] < inp["fjar"][j] < inp["flim"][j]:
            H[d, d] += ld(inp["fD"][j])
            mag[d, d] += ld(inp["fD"][j])
    u = U[64]
    return H.astype(np.float64), 16 * u * mag.astype(np.float64), T, 16 * u * Tb


def lower_words_mask(nj):
    """Arrow words the Hessian writes: lower triangles of r and c, all of x."""
    r = np.tril(np.ones((6, 6), bool))
    c = np.stack([np.tril(np.ones((nj, nj), bool))] * 2)
    return np.concatenate([r.ravel(), np.ones(12 * nj, bool), c.ravel()])


# ---------------------------------------------------------------- checks shared by the host and device tests
# Each returns the largest ratio of error to bound per quantity (<= 1 passes) after asserting it; the tests print them.
STATUS_PREFILL = 0b1101   # bits of the status word other than the pivot-failure bit (2): they must survive a solve


def _ratio(err, bound):
    """max err / bound; where the bound is 0 the error must be exactly 0."""
    err, bound = np.abs(err), np.broadcast_to(bound, np.shape(err))
    assert np.isfinite(err).all(), "non-finite result"
    assert (err[bound == 0] == 0).all(), "inexact where the result must be exact"
    return float(np.max(err[bound > 0] / bound[bound > 0], initial=0.0))


def check_untouched(rin, rout, mask, what):
    for p in range(rin.shape[0]):
        bad = np.nonzero((rin[p] != rout[p]) & ~mask)[0]
        assert bad.size == 0, f"{what}: problem {p} wrote record bytes outside its outputs, first at byte {bad[:8]}"


def check_hessian(P, v, ncon, seed, n=3):
    """newton_hessian_f64 on n random problems against hessian_reference: H's lower triangles and X, T, the 1e300 sentinel in the
    upper triangles, every other record byte unchanged."""
    nj = v[0]
    rng = np.random.default_rng(seed)
    inp = stack([hessian_inputs(v, ncon, rng) for _ in range(n)])
    H, T, rin, rout = P.hessian(v, inp)
    low = lower_words_mask(nj)
    rh = rt = 0.0
    for p in range(n):
        Href, Hb, Tref, Tb = hessian_reference(v, {k: x[p] for k, x in inp.items()})
        rh = max(rh, _ratio((H[p] - arrow_words(nj, Href))[low], arrow_words(nj, Hb)[low]))
        rt = max(rt, _ratio(T[p] - Tref, Tb))
        assert (H[p][~low] == 1e300).all(), "an upper-triangle entry of H.r / H.c was written"
    assert rh <= 1 and rt <= 1, (rh, rt)
    check_untouched(rin, rout, written_mask(P.layout(v, 64), ["H", "T"]), "newton_hessian_f64")
    return dict(H=rh, T=rt)


def arrow_problems(v, prec, kappa, seed, n=4):
    """n random arrow-SPD problems at condition number kappa: dense matrices, their words, right-hand sides, true condition numbers."""
    nj = v[0]
    rng = np.random.default_rng(seed)
    mats = [random_arrow_spd(nj, kappa, rng, prec) for _ in range(n)]
    b = rng.normal(size=(n, 6 + 2 * nj))
    if prec == 32:
        b = b.astype(np.float32).astype(np.float64)
    return [m for m, _ in mats], np.stack([arrow_words(nj, m) for m, _ in mats]), b, [k for _, k in mats]


def check_arrow(P, v, prec, kappa, seed, n=4):
    """arrow_factor_solve on n random arrow-SPD problems.  Held to:
    backward error  ||H x - b||_inf <= eta ||H| |x||_inf                            (eta = solve_eta: independent of kappa)
    forward error   ||x - x_np||_inf <= 2 kappa_inf eta ||x_np||_inf                (x - x_true = H^-1 (H x - b); 2: numpy's own error)
    factor entries  |L - L_np| <= eta kappa_2 ||L||_2, hdinv to the same over L_kk^2 (first-order perturbation of the Cholesky factor)
    Schur diagonal  |r_kk - (C - sum_c X_c X_c')_kk| <= 2 eta kappa_2 ||H||_2
    and the words the factorisation must not write (upper triangles, the chain diagonals) unchanged, status = its prefill."""
    nj, nv = v[0], 6 + 2 * v[0]
    mats, W, b, kap = arrow_problems(v, prec, kappa, seed, n)
    st = np.full(n, STATUS_PREFILL, np.int32)
    F, hd, x, st_out, rin, rout = P.arrow(v, prec, W, b, st)
    eta = solve_eta(prec, nv)
    out = dict(backward=0.0, forward=0.0, factor=0.0, hdinv=0.0, schur=0.0)
    tri6, trinj = np.tril_indices(6, -1), np.tril_indices(nj, -1)
    for p in range(n):
        Hd = mats[p]
        res, mag = residual(Hd, x[p], b[p])
        out["backward"] = max(out["backward"], _ratio(np.max(np.abs(res)), eta * np.max(mag)))
        xr = np.linalg.solve(Hd, b[p])
        kinf = np.linalg.norm(Hd, np.inf) * np.linalg.norm(np.linalg.inv(Hd), np.inf)
        out["forward"] = max(out["forward"], _ratio(np.max(np.abs(x[p] - xr)), 2 * kinf * eta * np.max(np.abs(xr))))
        ref = factor_reference(nj, Hd)
        nH = np.linalg.norm(Hd, 2)
        fb = eta * kap[p] * np.sqrt(nH)
        r, xx, c = arrow_blocks(nj, F[p])
        r0, _, c0 = arrow_blocks(nj, W[p])
        e = [r[tri6] - ref["r"][tri6], (xx - ref["x"]).ravel()] + [c[ch][trinj] - ref["c"][ch][trinj] for ch in range(2)]
        out["factor"] = max(out["factor"], _ratio(np.concatenate(e), fb))
        out["hdinv"] = max(out["hdinv"], _ratio(hd[p] - ref["hdinv"], fb * ref["hdinv"] ** 2))
        out["schur"] = max(out["schur"], _ratio(np.diag(r) - ref["schur_diag"], 2 * eta * kap[p] * nH))
        up6, upnj = np.triu_indices(6, 1), np.triu_indices(nj)   # chain blocks: the diagonal is never stored either
        assert (r[up6] == r0[up6]).all(), "an upper-triangle entry of the root block was written"
        for ch in range(2):
            assert (c[ch][upnj] == c0[ch][upnj]).all(), f"an upper-triangle or diagonal entry of chain block {ch} was written"
    assert (st_out == STATUS_PREFILL).all(), st_out
    assert all(q <= 1 for q in out.values()), out
    check_untouched(rin, rout, written_mask(P.layout(v, prec), ["H", "hdinv", "sdir", "status"]), "arrow_factor_solve")
    return out


PIVOT_FAULTS = ["chain_negative", "chain_zero", "root_negative", "nan_chain", "nan_coupling", "spd"]


def check_pivot_failure(P, v, prec, fault, seed=5):
    """A pivot that is not positive (chain or root row), or a NaN in the chain block or the coupling, sets status bit 2; the bits
    already in status survive (OR), and an SPD matrix leaves bit 2 clear."""
    nj = v[0]
    mats, _, b, _ = arrow_problems(v, prec, 1e2, seed, n=1)
    Hd = mats[0].copy()
    if fault == "chain_negative":
        Hd[6 + nj + 2, 6 + nj + 2] = -1.0          # chain 1, third column
    elif fault == "chain_zero":
        Hd[6, 6] = 0.0                             # chain 0, first pivot exactly 0
    elif fault == "root_negative":
        Hd[3, 3] = -1.0
    elif fault == "nan_chain":
        Hd[6 + 3, 6 + 1] = Hd[6 + 1, 6 + 3] = np.nan
    elif fault == "nan_coupling":
        Hd[2, 6 + nj + 1] = Hd[6 + nj + 1, 2] = np.nan
    W = arrow_words(nj, Hd)[None]
    st = np.full(1, STATUS_PREFILL, np.int32)
    _, _, _, st_out, _, _ = P.arrow(v, prec, W, b, st)
    want = STATUS_PREFILL if fault == "spd" else STATUS_PREFILL | 2
    assert st_out[0] == want, (fault, st_out[0], want)


def check_newton_direction(P, v, ncon, seed, n=3):
    """The Newton direction as the step kernel makes it: H from newton_hessian_f64 (symmetric positive semidefinite Af), solved by
    arrow_factor_solve, against numpy's solve of the dense reference H.  x - x_ref = H^-1 ((H x - b) + (H - H_dev) x), so
    ||x - x_ref||_inf <= 2 ||H^-1||_inf (eta ||H| |x||_inf + ||B_H |x|||_inf), B_H the Hessian's elementwise bound (2: numpy)."""
    nj, nv = v[0], 6 + 2 * v[0]
    rng = np.random.default_rng(seed)
    inp = stack([hessian_inputs(v, ncon, rng, spd=True) for _ in range(n)])
    H, _, _, _ = P.hessian(v, inp)
    b = rng.normal(size=(n, nv))
    _, _, x, st, _, _ = P.arrow(v, 64, H, b)
    assert (st == 0).all()
    worst = 0.0
    for p in range(n):
        Href, Hb, _, _ = hessian_reference(v, {k: q[p] for k, q in inp.items()})
        Href, Hb = (Href + Href.T) / 2, np.maximum(Hb, Hb.T)
        xr = np.linalg.solve(Href, b[p])
        bound = 2 * np.linalg.norm(np.linalg.inv(Href), np.inf) * (
            solve_eta(64, nv) * np.max(np.abs(Href) @ np.abs(xr)) + np.max(Hb @ np.abs(xr)))
        worst = max(worst, _ratio(np.max(np.abs(x[p] - xr)), bound))
    assert worst <= 1, worst
    return worst
