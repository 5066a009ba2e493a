#!/usr/bin/env python3
"""Cost of the root-velocity pushes (DESIGN.md §7.5).

1. The random-push launch alone (BatchedHumanoidEnv._push_random at the default 15 s interval): 200 back-to-back launches
   between one CUDA event pair, at 4096 envs, jvrc_walk and h1, fp32 and fp64; issued one by one from Python (the host's cost
   per launch bounds this) and replayed from one captured graph (the device's cost, as in the rollout's graphs).
2. DeviceRolloutWorker.sample at 4096 envs x 400 steps, jvrc_walk fp32 (training's default), without and with `--push-vel 1`,
   alternating, `--repeats` timed runs of each after one untimed run of each.
3. The batched evaluation of the trained jvrc_walk actor (tests/golden) at 4096 envs, fp64: plain against a 4 x 8 push sweep,
   alternating the same way.
The card's name and power limit are read in the same call.

    python tools/bench_push.py [--repeats 2] [--out-dir DIR]
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


def launch_us(env_name: str, precision: int, n: int = 4096, k: int = 200) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(n, model=env_name, precision=precision, seed=0, device=0, push_vel=1.0)
    env.reset()
    env.step(torch.zeros(n, env.act_dim, dtype=env.dtype, device=env.device))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    env._push_random(0, n)
    torch.cuda.synchronize()
    a.record()
    for _ in range(k):
        env._push_random(0, n)
    b.record()
    torch.cuda.synchronize()
    issued = a.elapsed_time(b) * 1e3 / k
    # the same k launches captured in one CUDA graph, as the rollout worker replays them: no host overhead between them
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            for _ in range(k):
                env._push_random(0, n)
        g.replay()
        torch.cuda.synchronize()
        a.record()
        g.replay()
        b.record()
    torch.cuda.synchronize()
    env.close()
    return issued, a.elapsed_time(b) * 1e3 / k


def sample_s(push_vel: float, n: int = 4096, T: int = 400) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import DeviceRolloutWorker, FF_V, Gaussian_FF_Actor
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=32, seed=0, device=0, push_vel=push_vel)
    torch.manual_seed(0)
    pol, cri = Gaussian_FF_Actor(env.obs_dim, env.act_dim, init_std=0.223).cuda(), FF_V(env.obs_dim).cuda()
    pol.obs_mean = cri.obs_mean = torch.tensor(env.obs_mean, dtype=torch.float32, device="cuda")
    pol.obs_std = cri.obs_std = torch.tensor(env.obs_std, dtype=torch.float32, device="cuda")
    w = DeviceRolloutWorker(env, pol, cri, seed=0)
    w.sample(0.99, 0.95, T, 400)          # capture + warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    w.sample(0.99, 0.95, T, 400)
    torch.cuda.synchronize()
    s = time.perf_counter() - t0
    env.close()
    return s


def eval_s(policy, sweep: bool, n: int = 4096) -> tuple[float, float | None]:
    import numpy as np
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import evaluation as ev
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=64, seed=0, device=0)
    push = None
    if sweep:
        speed, deg = ev.push_grid(n, [0, 0.5, 1, 1.5], 8)
        push = (int(round(2.0 / env.dt)), ev.push_vectors(speed, deg))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    acc = ev.rollout(env, policy, env.max_traj_len, push=push).cpu().numpy()
    s = time.perf_counter() - t0
    env.close()
    fell = float((acc[:, ev.DONE] != 0).mean())
    return s, fell


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_push needs a CUDA device")
    from bench_eval import actor_for, gpu_identity
    res = {"gpu": gpu_identity(), "launch_us": {}, "sample_s": {"off": [], "on": []}, "eval_s": {"plain": [], "sweep": []}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W", flush=True)
    for env_name in ("jvrc_walk", "h1"):
        for precision in (32, 64):
            issued, replayed = launch_us(env_name, precision)
            res["launch_us"][f"{env_name}_fp{precision}"] = dict(host_issued=issued, graph_replayed=replayed)
            print(f"push launch {env_name} fp{precision} 4096 envs: {issued:.2f} us issued from the host, {replayed:.2f} us "
                  "replayed from a graph", flush=True)
    sample_s(0.0), sample_s(1.0)           # untimed
    for _ in range(args.repeats):
        for key, v in (("off", 0.0), ("on", 1.0)):
            res["sample_s"][key].append(sample_s(v))
            print(f"sample 4096 x 400 jvrc_walk fp32 push {key}: {res['sample_s'][key][-1]:.4f} s", flush=True)
    policy = actor_for("jvrc_walk")
    eval_s(policy, False), eval_s(policy, True)
    for _ in range(args.repeats):
        for key in ("plain", "sweep"):
            s, fell = eval_s(policy, key == "sweep")
            res["eval_s"][key].append(s)
            print(f"eval 4096 envs jvrc_walk fp64 {key}: {s:.4f} s (fell {fell:.4f})", flush=True)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_push.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
