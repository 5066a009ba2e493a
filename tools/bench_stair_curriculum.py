#!/usr/bin/env python3
"""Cost of the stair curriculum (DESIGN.md §7.8).

jvrc_step control steps at 4096 envs with autoreset, fp64 and fp32: the plain env against one with `stair_curriculum=0.15` (levels
spread over 0 .. 15), alternating, `--repeats` timed runs of each after an untimed warm-up; then one full PPO iteration (4096 envs x
400 steps, fp32, the training defaults) each way after one untimed iteration.  The card's name and power limit are read in the same
call.

    python tools/bench_stair_curriculum.py [--repeats 2] [--steps 300] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
STAIRS = 0.15


def make_env(precision: int, stairs: float, n: int = 4096):
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(n, model="jvrc_step", precision=precision, seed=0, device=0, stair_curriculum=stairs)
    if env.stair_level is not None:
        env.stair_level.copy_(torch.arange(n, device=env.device, dtype=torch.int32) % env.stair_levels)
    env.reset()
    return env


def steps_per_s(precision: int, stairs: float, steps: int) -> float:
    import torch
    env = make_env(precision, stairs)
    g = torch.Generator(device=env.device).manual_seed(0)
    acts = [(torch.randn(env.num_envs, env.act_dim, generator=g, device=env.device) * 0.3).to(env.dtype) for _ in range(8)]
    for k in range(20):
        env.step(acts[k % 8])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for k in range(steps):
        env.step(acts[k % 8])
    torch.cuda.synchronize()
    rate = env.num_envs * steps / (time.perf_counter() - t0)
    env.close()
    return rate


def train_iter_s(stairs: float) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(4096, model="jvrc_step", precision=32, seed=0, stair_curriculum=stairs)
    probe = base()
    r = probe.robot
    probe.close()
    env_fn = lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=4096 * 400 // 4800 * 64,
                           epochs=3, max_traj_len=400, num_procs=4096, max_grad_norm=0.5, mirror_coeff=0.4, eval_freq=10**9,
                           recurrent=False, imitate_coeff=0.0, std_dev=0.223, learn_std=False, logdir="/tmp/lhw_bench_stairs",
                           steps_per_env=400, eval_batches=0, tf32=False, eval_at_start=False)
    os.environ["LHW_TENSORBOARD"] = "0"
    ppo = PPO(env_fn, args, seed=0)
    ppo.train(None, 1, verbose=False)    # warm-up (graph capture)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    log = ppo.train(None, 1, verbose=False)
    torch.cuda.synchronize()
    return dict(iter_s=time.perf_counter() - t0, sample_s=log[-1]["sample_time"], optimize_s=log[-1]["optimize_time"])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_stair_curriculum needs a CUDA device")
    from bench_eval import gpu_identity
    res = {"gpu": gpu_identity(), "steps_per_s": {}, "train_iter": {"plain": [], "stairs": []}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W", flush=True)
    for prec in (64, 32):
        for key in ("plain", "stairs"):
            steps_per_s(prec, STAIRS if key == "stairs" else 0.0, 50)     # untimed
        for _ in range(args.repeats):
            for key in ("plain", "stairs"):
                v = steps_per_s(prec, STAIRS if key == "stairs" else 0.0, args.steps)
                res["steps_per_s"].setdefault(f"fp{prec}_{key}", []).append(v)
                print(f"jvrc_step 4096 envs fp{prec} {key}: {v / 1e6:.4f} M env-steps/s", flush=True)
    for key in ("plain", "stairs"):
        r = train_iter_s(STAIRS if key == "stairs" else 0.0)
        res["train_iter"][key].append(r)
        print(f"train_iter jvrc_step 4096 x 400 fp32 {key}: {r['iter_s']:.3f} s (sampling {r['sample_s']:.3f} s, "
              f"optimisation {r['optimize_s']:.3f} s)", flush=True)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_stair_curriculum.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
