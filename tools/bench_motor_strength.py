#!/usr/bin/env python3
"""Cost of the motor strengths (DESIGN.md §7.11).

1. Control steps at 4096 envs with autoreset, every variant at fp64 and fp32, alternating within each repeat: the plain env, the
   motor step kernel with every factor 1 (`set_motor_strength(1)`: no draw), and random strengths (`motor_strength=0.3`: the
   motor step kernel, then the draw), `--repeats` timed runs of each after an untimed warm-up.
2. The draw launch alone, 4096 envs, replayed 1000 times from one CUDA graph.
3. One full PPO iteration of jvrc_walk (4096 envs x 400 steps, fp32, the training defaults) plain and with `--motor-strength 0.3`,
   after one untimed iteration each: the whole iteration and its sampling.
4. bench.py's headline (`--gpus 1 --steps 20 --warmup 3`), run as it ships.

The card's name, power limit and SM clock are read in the same call.

    python tools/bench_motor_strength.py [--repeats 3] [--steps 300] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
MODES = ("plain", "unit", "random")


def gpu_identity() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                          "-i", "0"], capture_output=True, text=True, timeout=60).stdout.strip().split(",")
    return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_clock_mhz": float(out[2]), "max_sm_clock_mhz": float(out[3])}


def steps_per_s(name: str, precision: int, mode: str, steps: int) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(4096, model=name, precision=precision, seed=0, device=0,
                             motor_strength=0.3 if mode == "random" else 0.0)
    env.reset()
    if mode == "unit":
        env.set_motor_strength(torch.ones(env.num_envs))
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


def draw_us(replays: int = 1000) -> float:
    """Microseconds per draw launch of 4096 envs, replayed from a graph of one launch (CUDA events around the replays)."""
    import torch
    from learninghumanoidwalking_b200 import _lib
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(4096, model="jvrc_walk", precision=32, seed=0, device=0, motor_strength=0.3)
    env.reset()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _lib.ops().sim_draw_motor(env._h.value, env.state_i, 0, 0, env.ended, 0.3, env.motor_strength)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            _lib.ops().sim_draw_motor(env._h.value, env.state_i, 0, 0, env.ended, 0.3, env.motor_strength)
        for _ in range(50):
            g.replay()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(replays):
            g.replay()
        b.record()
    b.synchronize()
    env.close()
    return a.elapsed_time(b) * 1000 / replays


def train_iter_s(r_motor: float) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(4096, model="jvrc_walk", precision=32, seed=0, motor_strength=r_motor)
    probe = base()
    r = probe.robot
    probe.close()
    env_fn = lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=4096 * 400 // 4800 * 64,
                           epochs=3, max_traj_len=400, num_procs=4096, max_grad_norm=0.5, mirror_coeff=0.4, eval_freq=10**9,
                           recurrent=False, imitate_coeff=0.0, std_dev=0.223, learn_std=False,
                           logdir=tempfile.mkdtemp(prefix="lhw_bench_motor_"), steps_per_env=400, eval_batches=0, tf32=False,
                           eval_at_start=False)
    os.environ["LHW_TENSORBOARD"] = "0"
    ppo = PPO(env_fn, args, seed=0)
    ppo.train(None, 1, verbose=False)    # warm-up (graph capture)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    log = ppo.train(None, 1, verbose=False)
    torch.cuda.synchronize()
    return dict(iter_s=time.perf_counter() - t0, sample_s=log[-1]["sample_time"], optimize_s=log[-1]["optimize_time"])


def bench_headline() -> dict:
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", "20", "--warmup", "3"],
                         capture_output=True, text=True, cwd=ROOT, timeout=1800)
    lines = [x for x in out.stdout.splitlines() if x.startswith("{")]
    if out.returncode != 0 or not lines:
        raise SystemExit(f"bench.py failed ({out.returncode}): {out.stderr[-2000:]}")
    return json.loads(lines[-1])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_motor_strength needs a CUDA device")
    res = {"gpu": gpu_identity(), "steps_per_s": {}, "train_iter": {}}
    g = res["gpu"]
    print(f"{g['name']}, power limit {g['power_limit_w']:.0f} W, SM clock {g['sm_clock_mhz']:.0f} MHz (max {g['max_sm_clock_mhz']:.0f})",
          flush=True)
    for name in VARIANTS:
        for prec in (64, 32):
            for mode in MODES:
                steps_per_s(name, prec, mode, 30)     # untimed
            for _ in range(args.repeats):
                for mode in MODES:
                    v = steps_per_s(name, prec, mode, args.steps)
                    res["steps_per_s"].setdefault(f"{name}_fp{prec}_{mode}", []).append(v)
            print(f"{name} 4096 envs fp{prec}: " + ", ".join(
                f"{m} {' '.join(f'{v / 1e6:.4f}' for v in res['steps_per_s'][f'{name}_fp{prec}_{m}'])}" for m in MODES)
                + " M env-steps/s", flush=True)
    res["draw_us"] = draw_us()
    print(f"draw launch, 4096 envs, graph replay: {res['draw_us']:.2f} us", flush=True)
    for key, r_motor in (("plain", 0.0), ("random", 0.3), ("plain_again", 0.0)):
        r = train_iter_s(r_motor)
        res["train_iter"][key] = r
        print(f"train_iter jvrc_walk 4096 x 400 fp32 {key}: {r['iter_s']:.3f} s (sampling {r['sample_s']:.3f} s, "
              f"optimisation {r['optimize_s']:.3f} s)", flush=True)
    res["bench"] = bench_headline()
    print("bench.py:", json.dumps(res["bench"]), flush=True)
    res["gpu_after"] = gpu_identity()
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_motor_strength.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
