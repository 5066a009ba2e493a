"""One physics substep of the step kernel source without a GPU: the device harness (tests/dev/substep_dev.cu) cross-compiles for
sm_90a for every variant and precision, and its host twin (tests/dev/substep_emu.cpp) passes every crafted case
of tests/dev/substep_cases.py against the float64 oracle at both precisions, so the cases, the mapping onto the oracle and the
bounds are rehearsed before tests/test_gpu_substep_edges.py holds the device build to them."""
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import substep_cases as C  # noqa: E402

VARIANTS = list(C.NAMES.values())


def _cuobjdump():
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    return shutil.which("cuobjdump") or os.path.join(os.path.dirname(nvcc), "cuobjdump")


def test_device_harness_cross_compiles_for_every_variant_and_precision():
    """The harness builds for sm_90a with its substep kernel for all five variants at both precisions."""
    sass = subprocess.run([_cuobjdump(), "-sass", C.build_device()], capture_output=True, text=True, check=True).stdout
    names = set(re.findall(r"Function : (\S*substep_kernel\S*)", sass))
    assert len(names) == 10, sorted(names)
    assert "arch = sm_90a" in sass


@pytest.fixture(scope="module")
def twins():
    hs = {}
    yield lambda name, prec: hs.setdefault((name, prec), C.Harness(C.twin_flat(name, prec), prec, device=False))
    for h in hs.values():
        h.close()


CASES = [(name, cid) for name in VARIANTS for cid in C.case_ids(name)]


@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("name,cid", CASES, ids=[f"{n}-{c}" for n, c in CASES])
def test_host_twin_against_the_oracle(twins, name, cid, prec):
    """Every crafted case reaches its branch in the host build and agrees with the oracle after 1 and frame_skip substeps."""
    H = twins(name, prec)
    print(f"\n[emu {name} fp{prec} {cid}] " + C.run_case(H, name, prec, cid))
