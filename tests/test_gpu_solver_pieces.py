"""The Newton solver pieces of the step kernel, compiled for the device as the kernel compiles them (tests/dev/solver_dev.cu) and
launched on their own, against numpy float64 (tests/dev/solver_pieces.py has the references and the bounds): the fragment layout
of warp_mma_f64, newton_hessian_f64 for every variant, arrow_factor_solve for every variant at both precisions, its pivot-failure
status, the Newton direction the two make together, and launches of many warps per block.  A failure names the piece, the
variant and the quantity, where the end-to-end tests only see a trajectory move."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import solver_pieces as SP  # noqa: E402

pytestmark = pytest.mark.gpu

VARIANTS = SP.VARIANTS
IDS = [f"{nj}_{tk}" for nj, tk in VARIANTS]


@pytest.fixture(scope="module")
def dev():
    return SP.Pieces(device=True)


@pytest.fixture(scope="module")
def emu():
    return SP.Pieces(device=False)


def _tiles(ks, a, b, c):
    """Per-lane fragments -> A_k [8 x 4], B_k [4 x 8], C (PTX ISA, mma.sync m8n8k4 .f64)."""
    A, B, C = np.zeros((ks, 8, 4)), np.zeros((ks, 4, 8)), np.zeros((8, 8))
    for l in range(32):
        A[:, l >> 2, l & 3] = a[l]
        B[:, l & 3, l >> 2] = b[l]
        C[l >> 2, 2 * (l & 3):2 * (l & 3) + 2] = c[l]
    return A, B, C


@pytest.mark.parametrize("ks", [1, 2, 3, 4])
def test_fragment_layout_and_accumulation(dev, ks):
    rng = np.random.default_rng(ks)
    a, b, c = rng.normal(size=(32, ks)), rng.normal(size=(32, ks)), rng.normal(size=(32, 2))
    d = dev.mma_lanes(ks, a, b, c)
    A, B, C = _tiles(ks, a, b, c)
    D = C + sum(A[k] @ B[k] for k in range(ks))
    want = np.array([[D[l >> 2, 2 * (l & 3) + i] for i in range(2)] for l in range(32)])
    np.testing.assert_allclose(d, want, rtol=1e-14, atol=1e-14)


def test_zero_padding_adds_nothing(dev):
    """A 6 x 6 product padded to 8 x 8 with zero k-columns: exact zeros outside the 6 x 6 block, the product inside."""
    rng = np.random.default_rng(7)
    A6, B6 = rng.normal(size=(6, 6)), rng.normal(size=(6, 6))
    a, b = np.zeros((32, 2)), np.zeros((32, 2))
    for l in range(32):
        for k in range(2):
            q = (l & 3) + 4 * k
            a[l, k] = A6[l >> 2, q] if (l >> 2) < 6 and q < 6 else 0.0
            b[l, k] = B6[q, l >> 2] if (l >> 2) < 6 and q < 6 else 0.0
    d = dev.mma_lanes(2, a, b, np.zeros((32, 2)))
    D = np.zeros((8, 8))
    for l in range(32):
        D[l >> 2, 2 * (l & 3):2 * (l & 3) + 2] = d[l]
    np.testing.assert_allclose(D[:6, :6], A6 @ B6, rtol=1e-13, atol=1e-13)
    assert (D[6:] == 0).all() and (D[:, 6:] == 0).all()


NCON = {"none": lambda v: (0, 0), "right": lambda v: (0, 2), "left": lambda v: (3, 0), "full": lambda v: (SP.CPF[v], SP.CPF[v])}


@pytest.mark.parametrize("ncon", list(NCON))
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_hessian_every_variant(dev, emu, v, ncon):
    """H and T against the scalar formula (sentinel upper triangles, nothing else written), and the device build against the host
    emulation of the same source to the same bound."""
    nc = NCON[ncon](v)
    seed = 11 * v[0] + sum(nc)
    print(f"\n[ratio hessian] {v} ncon {nc}: {SP.check_hessian(dev, v, nc, seed)}")
    rng = np.random.default_rng(seed + 1)
    inp = SP.stack([SP.hessian_inputs(v, nc, rng) for _ in range(3)])
    Hd, Td, _, _ = dev.hessian(v, inp)
    He, Te, _, _ = emu.hessian(v, inp)
    low = SP.lower_words_mask(v[0])
    for p in range(3):
        Href, Hb, _, Tb = SP.hessian_reference(v, {k: x[p] for k, x in inp.items()})
        r = (SP._ratio((Hd[p] - He[p])[low], SP.arrow_words(v[0], Hb)[low]), SP._ratio(Td[p] - Te[p], Tb))
        print(f"[ratio hessian device vs host] {v} ncon {nc}: H {r[0]:.2e} T {r[1]:.2e}")
        assert max(r) <= 1, r


@pytest.mark.parametrize("prec,kappa", [(64, 1), (64, 1e4), (64, 1e8), (32, 1), (32, 1e2), (32, 1e4)])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_arrow_solve_against_numpy(dev, v, prec, kappa):
    out = SP.check_arrow(dev, v, prec, kappa, seed=int(kappa) % 997 + v[0], n=8)
    print(f"\n[ratio arrow] {v} fp{prec} kappa {kappa:g}: " + " ".join(f"{k} {q:.2e}" for k, q in out.items()))


@pytest.mark.parametrize("fault", SP.PIVOT_FAULTS)
@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_pivot_failure_sets_status(dev, v, prec, fault):
    SP.check_pivot_failure(dev, v, prec, fault)


@pytest.mark.parametrize("ncon", ["right", "full"])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_newton_direction(dev, v, ncon):
    nc = NCON[ncon](v)
    print(f"\n[ratio newton direction] {v} ncon {nc}: {SP.check_newton_direction(dev, v, nc, seed=v[0] + v[1] + nc[0]):.2e}")


@pytest.mark.parametrize("prec,n_warps", [(64, 8), (32, 14)])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_many_warps_per_block_match_one_warp(dev, v, prec, n_warps):
    """Several blocks of n_warps warps, the last one partly filled, each warp with its own problem: bit-identical to one warp per
    block, whole records included (arrow_factor_solve, and newton_hessian_f64 for fp64)."""
    n = 3 * n_warps - 2
    _, W, b, _ = SP.arrow_problems(v, prec, 1e4, seed=17 + v[0], n=n)
    st = np.arange(n, dtype=np.int32) << 3
    one, many = dev.arrow(v, prec, W, b, st), dev.arrow(v, prec, W, b, st, n_warps=n_warps)
    for x, y in zip(one, many):
        assert np.array_equal(x, y)
    if prec == 64:
        rng = np.random.default_rng(23)
        inp = SP.stack([SP.hessian_inputs(v, (SP.CPF[v], (p % 3) * 2), rng) for p in range(n)])
        for x, y in zip(dev.hessian(v, inp), dev.hessian(v, inp, n_warps=n_warps)):
            assert np.array_equal(x, y)
