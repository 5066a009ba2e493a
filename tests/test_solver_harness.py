"""The Newton solver pieces of the step kernel source without a GPU: the device harness (tests/dev/solver_dev.cu) cross-compiles for
sm_90a with the Hessian on the fp64 tensor cores, and the host emulation of arrow_factor_solve and newton_hessian_f64 (tests/dev/
solver_emu.cpp) passes the checks tests/test_gpu_solver_pieces.py holds the device build to (tests/dev/solver_pieces.py)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import solver_pieces as SP  # noqa: E402

VARIANTS = SP.VARIANTS
IDS = [f"{nj}_{tk}" for nj, tk in VARIANTS]


@pytest.fixture(scope="module")
def emu():
    return SP.Pieces(device=False)


def _cuobjdump():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")


def test_device_harness_cross_compiles_with_the_hessian_on_dmma():
    """Every fp64 Hessian instantiation has the 20 mma.sync m8n8k4 .f64 of newton_hessian_f64 (per foot 2 tiles x 2 k-steps for
    T_f, the root tile 4 k-steps, per chain the coupling and the chain tile 2 k-steps each), and warp_mma_f64<KS> has KS."""
    lib = SP.build_device()
    sass = subprocess.run([_cuobjdump(), "-sass", lib], capture_output=True, text=True, check=True).stdout
    count, fn = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            fn = m.group(1)
            count[fn] = 0
        elif fn and re.search(r"\bDMMA\b", line):
            count[fn] += 1
    for nj, tk in VARIANTS:
        (name,) = [f for f in count if f.startswith(f"_Z9k_hessianILi{nj}ELi{tk}E")]
        assert count[name] == 20, (name, count[name])
    for ks in (1, 2, 3, 4):
        (name,) = [f for f in count if f.startswith(f"_Z7k_lanesILi{ks}E")]
        assert count[name] == ks, (name, count[name])
    assert sum(f.startswith("_Z7k_arrow") for f in count) == 10   # 5 variants x 2 precisions


@pytest.mark.parametrize("prec,kappa", [(64, 1), (64, 1e4), (64, 1e8), (32, 1), (32, 1e2), (32, 1e4)])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_emu_arrow_solve_against_numpy(emu, v, prec, kappa):
    print(f"\n[emu arrow] {v} fp{prec} kappa {kappa:g}: " + " ".join(f"{k} {q:.2e}" for k, q in
                                                              SP.check_arrow(emu, v, prec, kappa, seed=int(kappa) % 997 + v[0]).items()))


@pytest.mark.parametrize("fault", SP.PIVOT_FAULTS)
@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_emu_pivot_failure_sets_status(emu, v, prec, fault):
    SP.check_pivot_failure(emu, v, prec, fault)


@pytest.mark.parametrize("ncon", ["none", "right", "left", "full"])
@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_emu_hessian_every_variant(emu, v, ncon):
    nc = {"none": (0, 0), "right": (0, 2), "left": (3, 0), "full": (SP.CPF[v], SP.CPF[v])}[ncon]
    print(f"\n[emu hessian] {v} ncon {nc}: {SP.check_hessian(emu, v, nc, seed=11 * v[0] + sum(nc))}")


@pytest.mark.parametrize("v", VARIANTS, ids=IDS)
def test_emu_newton_direction(emu, v):
    print(f"\n[emu newton direction] {v}: {SP.check_newton_direction(emu, v, (SP.CPF[v], 1), seed=v[0] + v[1])}")
