"""Build liblhw_b200.so (hand-written sm_90a CUDA for the H100 + the C-ABI of include/lhw_b200.h) in-tree with nvcc.

The .so is git-ignored and built next to the package sources; there is no JIT and no fallback.
Every build leaves `build_record.json` next to the library: the nvcc command lines, the nvcc version, the sha256 of every
source / header that went in, the md5 of the library's SASS and where / when it was built.  `needs_build()` compares the
CONTENT hashes of the sources with that record (file times do not survive a copy to another machine); the profiling tools
(tools/make_ncu_counters.py) use the SASS md5 to tell whether a capture belongs to the built kernels.
"""
from __future__ import annotations

import hashlib
import re
import json
import os
import platform
import subprocess
import sys
import time

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "liblhw_b200.so")
TORCH_LIB = os.path.join(PKG, "liblhw_b200_torch.so")     # csrc/torch_ops.cpp: the same entry points as torch.ops.lhw.*
RECORD = os.path.join(PKG, "build_record.json")
SOURCES = ["sim_kernels.cu", "ppo_kernels.cu", "comm_kernels.cu", "wgrad_kernels.cu", "render_kernels.cu"]
HEADERS = ["sim_core.h", "model_pack.h", "render_core.h", os.path.join("..", "..", "include", "lhw_b200.h"), "torch_ops.cpp"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
# the renderer is built without FMA contraction, so that its images equal those of the host build of render_core.h
SOURCE_FLAGS = {"render_kernels.cu": ["-fmad=false"]}


def source_hashes() -> dict:
    out = {}
    for f in SOURCES + HEADERS:
        path = os.path.normpath(os.path.join(CSRC, f))
        out[os.path.relpath(path, os.path.dirname(PKG))] = hashlib.sha256(open(path, "rb").read()).hexdigest()
    return out


def step_kernel_sass_md5() -> str | None:
    """md5 of the device code (SASS) of the step / reset kernels as built: the key that ties an ncu capture to a build.  Host-side
    edits of sim_kernels.cu move it only when they change the order in which the host code first instantiates the kernels (the
    dump lists them in the reverse of that order); any change of the kernels moves it.  Read from the build record, None when
    there is no record."""
    rec = read_record()
    return rec.get("step_kernel_sass_md5") if rec else None


def read_record() -> dict | None:
    try:
        return json.load(open(RECORD))
    except Exception:
        return None


def needs_build() -> bool:
    if not os.path.exists(LIB) or not os.path.exists(TORCH_LIB):
        return True
    rec = read_record()
    return (rec is None or rec.get("sources") != source_hashes() or rec.get("flags") != NVCC_FLAGS
            or rec.get("source_flags") != SOURCE_FLAGS)


def _sass_md5(nvcc: str, target: str = LIB) -> str | None:
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    try:
        sass = subprocess.run([cuobjdump, "-sass", target], capture_output=True, timeout=600).stdout
        if not sass:
            return None
        # the dump names the source file ("identifier = <absolute path>") and nvcc derives the anonymous-namespace prefix of
        # every kernel symbol from that path: strip both, so that the same sources give the same md5 in any checkout directory
        sass = re.sub(rb"(?m)^identifier = .*$", b"", sass)
        sass = re.sub(rb"_GLOBAL__N__[0-9a-f]+_\d+_(\w+?)_cu_[0-9a-f]+", rb"_GLOBAL__N__\1_cu", sass)
        return hashlib.md5(sass).hexdigest()
    except Exception:
        return None


def build_torch_ops(verbose: bool = False) -> list:
    """csrc/torch_ops.cpp -> liblhw_b200_torch.so: TORCH_LIBRARY registrations (torch.ops.lhw.*) over the C-ABI library, plain g++
    against the torch headers of the running interpreter (no JIT cache: the .so stays in-tree next to the C-ABI library)."""
    import torch
    from torch.utils import cpp_extension as E
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    cuda_inc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "include")
    cmd = (["g++", "-O2", "-std=c++17", "-fPIC", "-shared", f"-D_GLIBCXX_USE_CXX11_ABI={int(torch._C._GLIBCXX_USE_CXX11_ABI)}"]
           + [f"-I{p}" for p in E.include_paths()] + [f"-I{cuda_inc}", os.path.join(CSRC, "torch_ops.cpp"), "-o", TORCH_LIB,
              f"-L{PKG}", "-llhw_b200", f"-L{tlib}", "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch",
              "-Wl,-rpath,$ORIGIN", f"-Wl,-rpath,{tlib}"])
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        print(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("g++ failed on torch_ops.cpp")
    return cmd


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs, procs, cmds = [], [], []
    os.makedirs(os.path.join(PKG, "build"), exist_ok=True)
    t0 = time.time()
    for src in SOURCES:
        obj = os.path.join(PKG, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        cmd = [nvcc] + NVCC_FLAGS + SOURCE_FLAGS.get(src, []) + ["-c", os.path.join(CSRC, src), "-o", obj]
        cmds.append(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            print(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        with open(os.path.join(PKG, "build", src + ".ptxas.log"), "w") as f:
            f.write(out)
    link = [nvcc] + NVCC_FLAGS[:2] + ["-shared", "-o", LIB] + objs + ["-lcudart"]
    subprocess.check_call(link)
    cmds.append(" ".join(link))
    cmds.append(" ".join(build_torch_ops(verbose)))
    ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout.strip().splitlines()
    json.dump(dict(library=os.path.basename(LIB), commands=cmds, flags=NVCC_FLAGS, source_flags=SOURCE_FLAGS, nvcc=ver[-2:] if ver else None,
                   sources=source_hashes(), sass_md5=_sass_md5(nvcc),
                   step_kernel_sass_md5=_sass_md5(nvcc, os.path.join(PKG, "build", "sim_kernels.o")),
                   library_sha256=hashlib.sha256(open(LIB, "rb").read()).hexdigest(), host=platform.node(),
                   built_at=time.strftime("%Y-%m-%dT%H:%M:%SZ", time.gmtime()), seconds=round(time.time() - t0, 1)),
              open(RECORD, "w"), indent=1)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
