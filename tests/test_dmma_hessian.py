"""The fp64 tensor-core pieces of the step kernel source on the host (tests/emu/dmma_emu.cpp, sim_core.h with LHW_CPU_EMU) against
numpy: the warp_mma_f64 fragment layout and accumulation, the Newton Hessian newton_hessian_f64 assembles from S and Af."""
import ctypes
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "emu"))
import emu  # noqa: E402
import emu_variants  # noqa: E402


@pytest.fixture(scope="module")
def lib():
    path = os.path.join(HERE, "emu", "_build", "libdmma_emu" + "".join("." + d.replace("=", "_") for d in emu.DEFINES) + ".so")
    L = ctypes.CDLL(emu_variants._build("dmma_emu.cpp", "dmma_emu.cpp", path, ["-D" + d for d in emu.DEFINES]))
    L.dmma_emu_lanes.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 4
    L.dmma_emu_hessian.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 12
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


@pytest.mark.parametrize("ks", [1, 2, 3, 4])
def test_fragment_layout_and_accumulation_from_c(lib, ks):
    """Per-lane fragments in, per-lane D out: A_k[l >> 2][l & 3], B_k[l & 3][l >> 2], C / D[l >> 2][2 (l & 3) + i] (PTX ISA,
    mma.sync m8n8k4 .f64), D = C + sum_k A_k B_k."""
    rng = np.random.default_rng(ks)
    a, b, c = rng.normal(size=(32, ks)), rng.normal(size=(32, ks)), rng.normal(size=(32, 2))
    d = np.zeros((32, 2))
    assert lib.dmma_emu_lanes(ks, _p(a), _p(b), _p(c), _p(d)) == 0
    A, B, C = np.zeros((ks, 8, 4)), np.zeros((ks, 4, 8)), np.zeros((8, 8))
    for l in range(32):
        A[:, l >> 2, l & 3] = a[l]
        B[:, l & 3, l >> 2] = b[l]
        C[l >> 2, 2 * (l & 3):2 * (l & 3) + 2] = c[l]
    D = C + sum(A[k] @ B[k] for k in range(ks))
    want = np.array([[D[l >> 2, 2 * (l & 3) + i] for i in range(2)] for l in range(32)])
    np.testing.assert_allclose(d, want, rtol=1e-14, atol=1e-14)


def test_zero_padding_adds_nothing(lib):
    """A 6 x 6 block padded to 8 x 8 with zero k-columns: the product equals the unpadded one exactly where it is defined."""
    rng = np.random.default_rng(7)
    A6, B6 = rng.normal(size=(6, 6)), rng.normal(size=(6, 6))
    a, b = np.zeros((32, 2)), np.zeros((32, 2))
    for l in range(32):
        for k in range(2):
            q = (l & 3) + 4 * k
            a[l, k] = A6[l >> 2, q] if (l >> 2) < 6 and q < 6 else 0.0
            b[l, k] = B6[q, l >> 2] if (l >> 2) < 6 and q < 6 else 0.0
    d = np.zeros((32, 2))
    assert lib.dmma_emu_lanes(2, _p(a), _p(b), _p(np.zeros((32, 2))), _p(d)) == 0
    D = np.zeros((8, 8))
    for l in range(32):
        D[l >> 2, 2 * (l & 3):2 * (l & 3) + 2] = d[l]
    np.testing.assert_allclose(D[:6, :6], A6 @ B6, rtol=1e-13, atol=1e-13)
    assert (D[6:] == 0).all() and (D[:, 6:] == 0).all()


def _arrow_words(nj, dense):
    """Pack a dense symmetric [root | chain0 | chain1] matrix into sim_core.h's Arrow record (r, x, c)."""
    r = dense[:6, :6]
    x = np.stack([dense[:6, 6 + ch * nj:6 + (ch + 1) * nj] for ch in range(2)])
    c = np.stack([dense[6 + ch * nj:6 + (ch + 1) * nj, 6 + ch * nj:6 + (ch + 1) * nj] for ch in range(2)])
    return np.concatenate([r.ravel(), x.ravel(), c.ravel()])


def _arrow_blocks(nj, words):
    r = words[:36].reshape(6, 6)
    x = words[36:36 + 12 * nj].reshape(2, 6, nj)
    c = words[36 + 12 * nj:].reshape(2, nj, nj)
    return r, x, c


def _random_arrow_spd(nj, rng):
    nv = 6 + 2 * nj
    G = rng.normal(size=(nv, nv))
    Hd = G @ G.T + nv * np.eye(nv)
    Hd[6:6 + nj, 6 + nj:] = 0
    Hd[6 + nj:, 6:6 + nj] = 0
    return Hd


@pytest.mark.parametrize("nj", [6, 5])
@pytest.mark.parametrize("ncon", [(4, 3), (0, 2), (1, 0), (0, 0)])
def test_hessian_from_random_s_and_af_against_the_scalar_formula(lib, nj, ncon):
    """H = M + sum_f S_f' Af_f S_f (over feet with contacts) + the active limit rows' D on the chain diagonals (+ the
    friction-loss D inside the quadratic zone, H1), lower triangles of the arrow blocks; T_f = Af_f S_f (0 without contacts)."""
    rng = np.random.default_rng(100 * nj + 10 * ncon[0] + ncon[1])
    nv, na, nu = 6 + 2 * nj, 6 + nj, 2 * nj
    S = rng.normal(size=(nv, 6))
    Af = np.stack([(lambda g: g @ g.T)(rng.normal(size=(6, 6))) for _ in range(2)])
    Md = _random_arrow_spd(nj, rng)
    M = _arrow_words(nj, Md)
    lside = rng.integers(-1, 2, size=nu).astype(np.int32)
    ljar, lD = rng.normal(size=nu), rng.uniform(1, 2, size=nu)
    fjar, flim, fD = rng.normal(size=nu), rng.uniform(0.2, 1.5, size=nu), rng.uniform(1, 2, size=nu)
    H, T = np.zeros_like(M), np.zeros((2, na, 6))
    nc = np.array(ncon, np.int32)
    assert lib.dmma_emu_hessian(nj, _p(S), _p(Af), _p(nc), _p(M), _p(lside), _p(ljar), _p(lD), _p(fjar), _p(flim), _p(fD),
                                _p(H), _p(T)) == 0
    want = Md.copy()
    for f in range(2):
        dofs = list(range(6)) + [6 + f * nj + j for j in range(nj)]
        Sf = S[dofs].T                                    # 6 x NA
        Tf = Af[f] @ Sf if ncon[f] else np.zeros((6, na))
        np.testing.assert_allclose(T[f], Tf.T, rtol=1e-13, atol=1e-12)
        want[np.ix_(dofs, dofs)] += Sf.T @ Tf
    for j in range(nu):
        d = 6 + j
        if lside[j] and ljar[j] < 0:
            want[d, d] += lD[j]
        if nj == 5 and -flim[j] < fjar[j] < flim[j]:     # H1: friction-loss rows
            want[d, d] += fD[j]
    r, x, c = _arrow_blocks(nj, H)
    wr, wx, wc = _arrow_blocks(nj, _arrow_words(nj, want))
    low6, lownj = np.tril_indices(6), np.tril_indices(nj)
    np.testing.assert_allclose(r[low6], wr[low6], rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(x, wx, rtol=1e-12, atol=1e-12)
    for ch in range(2):
        np.testing.assert_allclose(c[ch][lownj], wc[ch][lownj], rtol=1e-12, atol=1e-12)

