#!/usr/bin/env python3
"""Newton-step census of the step kernel's contact solve, counted on the CPU emulation of the kernel source (tests/emu).

  python tools/newton_census.py                                   # shipped kernel, every workload x regime
  python tools/newton_census.py --defines "LHW_X_FOO=1"           # a candidate's compile-time flags (csrc/sim_core.h)
  python tools/newton_census.py --workloads jvrc_walk --regimes noise --envs 512 --preroll 150 --steps 40

fp64 at each model's shipped solver tolerance, bench.py's action regimes: noise = N(0, 0.223^2) open loop, zero = a = 0,
trained = tests/golden/trained_actor_jvrc_walk.pt in the loop + N(0, 0.05^2) (jvrc_walk only).  `--preroll` uncounted control
steps, then `--steps` counted ones.  Columns (a "solve" = one substep's Newton solve; these are counts, not times):
  0/1/2/3/>=4   share of the lock-step substeps' solves that take that many Newton steps
  mean          Newton steps per solve of one environment (lock-step substeps)
  env-step      Newton steps per control step, auto-reset settling substeps included (bench.py's newton_iters_per_env_step)
  block max     mean over lock-step substeps of the largest count among W consecutive environments, W = the shipped warps per
                block (8 fp64 jvrc_walk, 7 the others): the steps a lock-step block waits for at its per-substep barrier
  ls/step       line-search evaluations after the one at alpha = 0, per Newton step
The emulation runs the kernel's own arithmetic, so the counts are the GPU's up to the order of floating-point sums.
"""
import argparse
import hashlib
import multiprocessing as mp
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
WPB = {"jvrc_walk": 8, "h1": 7, "jvrc_step": 7, "jvrc_walk_terrain": 7}   # sim_kernels.cu: shipped fp64 warps per block
SIGMA = 0.223
TRAINED_ACTOR = os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")


def build(defines):
    """tools/newton_census.cpp (the emulation of tests/emu with the census hook) + -D flags -> a library in the temp directory,
    named by the hash of its sources and flags, so the tree stays as it is and a source edit always gives a fresh build."""
    srcs = [os.path.join(ROOT, "tools", "newton_census.cpp"), os.path.join(EMU, "sim_emu.cpp")] + [
        os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", f) for f in ("sim_core.h", "model_pack.h")]
    h = hashlib.sha256(defines.encode())
    for s in srcs:
        h.update(open(s, "rb").read())
    out_dir = os.path.join(tempfile.gettempdir(), f"lhw_newton_census_{os.getuid()}")
    lib = os.path.join(out_dir, f"census_{h.hexdigest()[:16]}.so")
    if not os.path.exists(lib):
        os.makedirs(out_dir, exist_ok=True)
        tmp = f"{lib}.{os.getpid()}.tmp"
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17"] + ["-D" + d for d in defines.split()] +
                              ["-o", tmp, srcs[0]])
        os.replace(tmp, lib)
    return lib


def census(job):
    workload, regime, defines, lib, n, preroll, steps, seed = job
    sys.path[:0] = [ROOT, EMU]
    import ctypes
    import emu
    from emu import Emu
    emu.build = lambda: lib     # the tests' wrapper over the census build of the same emulation
    from learninghumanoidwalking_b200.model import load_model, pack_model
    mj = load_model(workload)
    F = int(mj["cfg"]["frame_skip"])
    e = Emu(pack_model(mj), 64, n, seed=seed)
    take = e.lib.emu_census_take
    buf = np.zeros(3 * n * (F + 8), np.int32)
    rng = np.random.default_rng(seed)
    pol = None
    if regime == "trained":
        import torch
        from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
        install_reference_aliases()
        pol = torch.load(TRAINED_ACTOR, map_location="cpu", weights_only=False).eval()
    obs = e.reset()
    take(buf.ctypes.data_as(ctypes.c_void_p), len(buf) // 3)     # the reset's settling solves are not counted
    lock, per_env_step, ls, newton = [], [], 0, 0
    for k in range(preroll + steps):
        if regime == "zero":
            a = np.zeros((n, e.nu))
        elif regime == "noise":
            a = rng.standard_normal((n, e.nu)) * SIGMA
        else:
            import torch
            with torch.no_grad():
                a = pol(torch.from_numpy(obs).float()).double().numpy() + rng.standard_normal((n, e.nu)) * 0.05
        obs = e.step(a)[0]
        r = take(buf.ctypes.data_as(ctypes.c_void_p), len(buf) // 3)
        rec = buf[:3 * r].reshape(r, 3)
        if k < preroll:
            continue
        counts = np.zeros((n, F), np.int64)
        for i in range(n):      # an environment's solves: its F lock-step substeps, then the auto-reset's settling substeps if any
            mine = rec[rec[:, 0] == i]
            counts[i] = mine[:F, 1]
            per_env_step.append(int(mine[:, 1].sum()))
        lock.append(counts)
        ls += int(rec[:, 2].sum())
        newton += int(rec[:, 1].sum())
    lock = np.stack(lock)                                            # [steps, n, F]
    W = WPB[workload]
    nb = n // W
    bmax = lock[:, :nb * W].reshape(steps, nb, W, F).max(axis=2)
    flat = lock.ravel()
    hist = [float((flat == c).mean()) for c in range(4)] + [float((flat >= 4).mean())]
    return dict(workload=workload, regime=regime, defines=defines, hist=hist, mean=float(flat.mean()),
                env_step=float(np.mean(per_env_step)), block_max=float(bmax.mean()), W=W, ls_per_step=ls / max(newton, 1))


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workloads", default="jvrc_walk,h1,jvrc_step,jvrc_walk_terrain")
    ap.add_argument("--regimes", default="noise,zero,trained")
    ap.add_argument("--defines", action="append", default=None,
                    help="space-separated -D flags of one kernel variant; repeat to compare variants ('' = shipped)")
    ap.add_argument("--envs", type=int, default=512)
    ap.add_argument("--preroll", type=int, default=150)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--jobs", type=int, default=os.cpu_count())
    args = ap.parse_args()
    variants = args.defines if args.defines is not None else [""]
    libs = {d: build(d) for d in variants}      # each library once, before the workers load it
    jobs = [(w, r, d, libs[d], args.envs, args.preroll, args.steps, args.seed) for w in args.workloads.split(",")
            for r in args.regimes.split(",") if r != "trained" or w == "jvrc_walk" for d in variants]
    # one process per job: a process keeps the first emulation library it loads
    with mp.get_context("spawn").Pool(min(args.jobs, len(jobs)), maxtasksperchild=1) as pool:
        rows = pool.map(census, jobs, chunksize=1)
    print(f"fp64, shipped tolerance, {args.envs} envs, {args.preroll} pre-roll + {args.steps} counted control steps, seed {args.seed}\n")
    print("| workload | regime | kernel | 0 / 1 / 2 / 3 / >=4 Newton steps | mean | env-step | block max (W) | ls/step |")
    print("|---|---|---|---|---|---|---|---|")
    for r in rows:
        h = " / ".join(f"{100 * x:.1f} %" for x in r["hist"])
        print(f"| {r['workload']} | {r['regime']} | {r['defines'] or 'shipped'} | {h} | {r['mean']:.3f} | {r['env_step']:.1f} | "
              f"{r['block_max']:.3f} ({r['W']}) | {r['ls_per_step']:.2f} |", flush=True)


if __name__ == "__main__":
    main()
