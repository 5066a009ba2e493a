#!/usr/bin/env python3
"""A/B harness for candidate step-kernel variants (development tool; bench.py is the contract).

  python tools/ab_variants.py build            # here (nvcc cross-compiles): one library per variant under .../build/variants/
  python tools/ab_variants.py run [--quick]    # on an H100: parity subset + device-resident timing of every variant

A variant = compile-time flags of csrc/sim_core.h (-DLHW_X_<name>=1: rewrites that passed the CPU tier but have no H100 timing
yet) x run-time launch knobs (LHW_WARPS_PER_BLOCK).  Every timing runs in its own process (the knobs are read once, at
lhw_sim_create) with LHW_B200_LIB pointing at the variant's library; the baseline is the shipped library built the same way.
The table goes to stdout and gpurun_out/ab_variants.json.
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "learninghumanoidwalking_b200")
VDIR = os.path.join(PKG, "build", "variants")

# name -> -D flags.  Round 2 ran the four round-1 candidates (profiles/r02_ab_variants.md): CF / RSQ / GMODEL won (+6.5 % together)
# and are now simply the kernel; SPLITBAR and 4- / 5-warp blocks lost and were deleted.  New candidates go here.
BUILDS = {
    "base": [],
    # round 2, second batch (profiles/r02_ab_variants.md): "-DLHW_X_REGCAP=576 | 640 | 896" = 112 / 96 / 72 registers per thread of the
    # fp64 lock-step kernel (18 / 20 / 28 warps per SM) — measured, not adopted
    # warm starts of the Newton solve, screened with tools/newton_census.py (DESIGN.md §4.1): the extrapolated warm start won on
    # every workload and regime and is now the kernel; the active-set warm start (first Hessian from the previous solve's final
    # active set), alone or with it, raised the block maximum everywhere and was deleted before any GPU timing
    # the Newton Hessian (T_f, H) on the fp64 tensor cores is now the fp64 kernel (DESIGN.md §4.1); the root Schur complement as one
    # DMMA tile timed x1.012 on top of it but made ptxas spill in reset_kernel<double, 6, 0>, and was dropped
}
# (build, env knobs) timed on (model, precision, n_envs); runs with knobs only time the headline workload
RUNS = [
    ("base", {}),
]
WORKLOADS = [("jvrc_walk", 64, 4096), ("jvrc_walk", 64, 32768)]
PARITY = ["tests/test_gpu_parity.py", "tests/test_gpu_h1.py::test_h1_fp64_closed_loop_with_randomisation_and_resets",
          "tests/test_gpu_step.py::test_step_fp64_closed_loop_all_modes_with_resets"]


def lib_path(name):
    return os.path.join(VDIR, f"liblhw_b200.{name}.so")


def build():
    sys.path.insert(0, ROOT)
    from learninghumanoidwalking_b200 import build as B
    os.makedirs(VDIR, exist_ok=True)
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    flags = [f for f in B.NVCC_FLAGS if f not in ("-Xptxas", "-v")]
    shared = []
    for src in B.SOURCES:
        if src == "sim_kernels.cu":
            continue
        obj = os.path.join(VDIR, src.replace(".cu", ".o"))
        subprocess.check_call([nvcc] + flags + B.SOURCE_FLAGS.get(src, []) + ["-c", os.path.join(B.CSRC, src), "-o", obj])
        shared.append(obj)
    procs = []
    for name, defs in BUILDS.items():
        obj = os.path.join(VDIR, f"sim_kernels.{name}.o")
        procs.append((name, obj, subprocess.Popen([nvcc] + flags + defs + ["-c", os.path.join(B.CSRC, "sim_kernels.cu"), "-o", obj])))
    for name, obj, p in procs:
        if p.wait() != 0:
            raise SystemExit(f"nvcc failed on variant {name}")
        subprocess.check_call([nvcc, "-shared", "-o", lib_path(name), obj] + shared + ["-lcudart"])
        os.remove(obj)      # only the libraries travel to the GPU box
        print("built", lib_path(name))
    for obj in shared:
        os.remove(obj)


TIMER = r"""
import sys
sys.path.insert(0, %r)
from tools.quick_bench import run
model, prec, n = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
# candidates worth a few per cent need a quiet number: 200 timed steps, best of 3
best = max(run(n, prec, steps=200 if n <= 8192 else 60, warm=20, sigma=0.223, model=model)[1] for _ in range(3))
print("RESULT", best)
"""


def run(quick):
    out = []
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    parity_done = {}
    for name, knobs in RUNS:
        env = dict(os.environ, LHW_B200_LIB=lib_path(name), **knobs)
        if name not in parity_done:     # the variant's arithmetic against the oracle, through the C-ABI, before any timing of it
            try:    # a candidate that hangs must cost its own time-out, not the GPU box
                r = subprocess.run([sys.executable, "-m", "pytest", "-x", "-q", "-m", "gpu"] + PARITY, cwd=ROOT, timeout=900,
                                   env=dict(os.environ, LHW_B200_LIB=lib_path(name), **knobs), capture_output=True, text=True)
            except subprocess.TimeoutExpired:
                r = subprocess.CompletedProcess([], 124, "timed out", "")
            last = r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ""
            parity_done[name] = r.returncode == 0 and " passed" in last and "skipped" not in last    # skipped = no GPU = not checked
            print(f"[{name}] parity subset: {'passed' if parity_done[name] else 'FAILED'}  {r.stdout.strip().splitlines()[-1] if r.stdout.strip() else ''}", flush=True)
        # block-size knobs are sized for the fp64 headline kernel; the split barrier is timed on its fp32 twin too
        loads = WORKLOADS[:1] if quick else [w for w in WORKLOADS if not knobs or (
            w[0] == "jvrc_walk" and (w[1] == 64 or "LHW_WARPS_PER_BLOCK" not in knobs))]
        for model, prec, n in loads:
            if not parity_done[name]:
                continue
            try:
                r = subprocess.run([sys.executable, "-c", TIMER % ROOT, model, str(prec), str(n)], cwd=ROOT, env=env, capture_output=True,
                                   text=True, timeout=300)
            except subprocess.TimeoutExpired:
                r = subprocess.CompletedProcess([], 124, "", "timed out")
            val = next((float(l.split()[1]) for l in r.stdout.splitlines() if l.startswith("RESULT")), None)
            rec = dict(build=name, knobs=knobs, model=model, precision=prec, n_envs=n, env_steps_per_s=val, parity=parity_done[name])
            if val is None:
                rec["error"] = (r.stderr or r.stdout)[-300:]
            out.append(rec)
            print(f"{name:6s} {json.dumps(knobs):34s} {model:10s} fp{prec} N={n:<6d} {val / 1e6 if val else float('nan'):.3f} M env-steps/s", flush=True)
    json.dump(out, open(os.path.join(ROOT, "gpurun_out", "ab_variants.json"), "w"), indent=1)
    # summary: every run against the unflagged build with default knobs on the same workload
    base = {(r["model"], r["precision"], r["n_envs"]): r["env_steps_per_s"] for r in out if r["build"] == "base" and not r["knobs"]}
    print("\n--- relative to base (same workload) ---")
    for r in out:
        b = base.get((r["model"], r["precision"], r["n_envs"]))
        if b and r["env_steps_per_s"] and (r["build"] != "base" or r["knobs"]):
            print(f"{r['build']:6s} {json.dumps(r['knobs']):62s} {r['model']:10s} fp{r['precision']} N={r['n_envs']:<6d} x{r['env_steps_per_s'] / b:.3f}")


if __name__ == "__main__":
    if len(sys.argv) < 2 or sys.argv[1] not in ("build", "run"):
        raise SystemExit(__doc__)
    build() if sys.argv[1] == "build" else run("--quick" in sys.argv)
