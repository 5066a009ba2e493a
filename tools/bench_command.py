#!/usr/bin/env python3
"""Cost of the command-tracking sweep (DESIGN.md §7.6).

1. The signed-velocity accumulate launch alone (BatchedHumanoidEnv.command_accumulate): 200 launches captured in one CUDA graph
   and replayed between one CUDA event pair, at 4096 envs, jvrc_walk fp32 and fp64.
2. The batched evaluation of the trained jvrc_walk actor (tests/golden) at 4096 envs, fp64: plain against the sweep
   forward:0,0.2,0.4 inplace:-0.4,0.4 standing, alternating, `--repeats` timed runs of each after one untimed run of each.  The
   sweep's per-cell table is printed once.
The card's name and power limit are read in the same call.

    python tools/bench_command.py [--repeats 2] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
CELLS = [("FORWARD", 0.0), ("FORWARD", 0.2), ("FORWARD", 0.4), ("INPLACE", -0.4), ("INPLACE", 0.4), ("STANDING", 0.0)]


def launch_us(precision: int, n: int = 4096, k: int = 200) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=precision, seed=0, device=0)
    env.reset()
    env.step(torch.zeros(n, env.act_dim, dtype=env.dtype, device=env.device), autoreset=False)
    acc = torch.zeros(n, env.command_words(), dtype=torch.float64, device=env.device)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        env.command_accumulate(acc)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(k):
                env.command_accumulate(acc)
        g.replay()
        torch.cuda.synchronize()
        a.record()
        g.replay()
        b.record()
    torch.cuda.synchronize()
    env.close()
    return a.elapsed_time(b) * 1e3 / k


def eval_s(policy, sweep: bool, n: int = 4096, show: bool = False) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import evaluation as ev
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=64, seed=0, device=0)
    command = None
    if sweep:
        mode, value = ev.command_grid(n, CELLS)
        command = (mode, ev.command_refs(mode, value))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = ev.rollout(env, policy, env.max_traj_len, command=command)
    acc = (out[0] if sweep else out).cpu().numpy()
    s = time.perf_counter() - t0
    if show:
        print(ev.format_command_table(ev.command_summary(acc, out[1].cpu().numpy(), mode, value, CELLS)), flush=True)
    env.close()
    return s


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_command needs a CUDA device")
    from bench_eval import actor_for, gpu_identity
    res = {"gpu": gpu_identity(), "launch_us": {}, "eval_s": {"plain": [], "sweep": []}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W", flush=True)
    for precision in (32, 64):
        res["launch_us"][f"jvrc_walk_fp{precision}"] = us = launch_us(precision)
        print(f"command accumulate launch jvrc_walk fp{precision} 4096 envs: {us:.2f} us replayed from a graph", flush=True)
    policy = actor_for("jvrc_walk")
    eval_s(policy, False), eval_s(policy, True, show=True)    # untimed
    for _ in range(args.repeats):
        for key in ("plain", "sweep"):
            res["eval_s"][key].append(eval_s(policy, key == "sweep"))
            print(f"eval 4096 envs jvrc_walk fp64 {key}: {res['eval_s'][key][-1]:.4f} s", flush=True)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_command.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
