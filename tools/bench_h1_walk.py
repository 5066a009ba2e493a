#!/usr/bin/env python3
"""Throughput of the h1_walk environment (the H1 robot with the WalkingTask, csrc/sim_core.h Cfg<5, 3>), device resident.

bench.py measures the four workloads it has always measured; this tool times h1_walk the same way: 4096 environments, actions
N(0, 0.223^2) drawn before the timed region, the 50 MB L2 flushed before every step outside the timed region, one CUDA event
pair around each `step` launch, env-steps/s = environments x steps / summed event time.  It does so at fp64 and fp32, and in the
same call runs `bench.py --workload h1` for comparison and prints the card's name and power limit next to the numbers.

    python tools/bench_h1_walk.py [--envs 4096] [--steps 200] [--warmup 20] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SIGMA = 0.223      # bench.py's exploration noise


def gpu_identity() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().split(",")
    return {"name": out[0].strip(), "power_limit_w": float(out[1])}


def time_steps(precision: int, n: int, steps: int, warmup: int, seed: int = 0) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    dev = torch.device("cuda", 0)
    env = BatchedHumanoidEnv(n, model="h1_walk", precision=precision, seed=seed, device=0)
    env.reset()
    g = torch.Generator(device=dev).manual_seed(seed)
    acts = torch.randn(warmup + steps, n, env.act_dim, device=dev, generator=g, dtype=env.dtype) * SIGMA
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for k in range(warmup):
        env.step(acts[k])
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda.synchronize()
    for k in range(steps):
        flush.fill_(k & 0xFF)
        ev[k][0].record()
        env.step(acts[warmup + k])
        ev[k][1].record()
    torch.cuda.synchronize()
    ms = [a.elapsed_time(b) for a, b in ev]
    ended = int(env.ended.sum().item())
    env.close()
    return {"precision": precision, "envs": n, "steps": steps, "env_steps_per_s": n * steps / (sum(ms) * 1e-3),
            "step_ms_median": sorted(ms)[len(ms) // 2], "ended_last_step": ended}


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--out-dir", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_h1_walk needs a CUDA device")
    res = {"gpu": gpu_identity(), "h1_walk": [time_steps(p, args.envs, args.steps, args.warmup) for p in (64, 32)]}
    with tempfile.TemporaryDirectory() as tmp:   # bench.py compiles nothing, but keeps whatever it writes out of the tree
        out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--workload", "h1", "--steps",
                              str(args.steps), "--warmup", str(args.warmup), "--no-train-iter", "--no-cpu-baseline"],
                             capture_output=True, text=True, cwd=tmp, timeout=1800)
    line = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    res["bench_h1"] = json.loads(line[-1]) if line else {"error": out.stderr[-2000:]}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W")
    for r in res["h1_walk"]:
        print(f"h1_walk fp{r['precision']}: {r['env_steps_per_s'] / 1e6:.3f} M env-steps/s ({r['envs']} envs, {r['steps']} steps, "
              f"median step {r['step_ms_median']:.3f} ms)")
    b = res["bench_h1"]
    print("bench.py --workload h1 (fp64):", {k: b[k] for k in ("metric", "value", "unit") if k in b} if "value" in b else b)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_h1_walk.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
