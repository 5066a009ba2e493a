#!/usr/bin/env python3
"""Cost and effect of the carried payloads (DESIGN.md §7.10).

1. Control steps at 4096 envs with autoreset, every variant at fp64 and fp32: the plain env against one with random payloads up to
   20 kg within 0.1 m (`payload_mass=20, payload_offset=0.1`: the payload step kernel, then the draw), alternating, `--repeats`
   timed runs of each after an untimed warm-up.  Beside each rate, the mean Newton iterations per env of the last step.
2. The draw launch alone, 4096 envs, replayed 1000 times from one CUDA graph.
3. One full PPO iteration of jvrc_walk (4096 envs x 400 steps, fp32, the training defaults) plain and with `--payload-mass 20`,
   after one untimed iteration each: the whole iteration and its sampling.
4. With `--study ITERS`: two jvrc_walk trainings of ITERS iterations with the same seed, plain and `--payload-mass 20`, each
   evaluated on 4096 envs across payloads 0, 5, 10, 15, 20 and 25 kg; the fall fraction and FORWARD tracking error of each cell.

The card's name and power limit are read in the same call.

    python tools/bench_payload.py [--repeats 2] [--steps 300] [--study 0] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
STUDY_MASSES = (0, 5, 10, 15, 20, 25)


def steps_per_s(name: str, precision: int, mass: float, steps: int) -> tuple[float, float]:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(4096, model=name, precision=precision, seed=0, device=0, payload_mass=mass,
                             payload_offset=0.1 if mass else 0.0)
    env.reset()
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
    iters = float(env.solver_iterations().double().mean())
    env.close()
    return rate, iters


def draw_us(replays: int = 1000) -> float:
    """Microseconds per draw launch of 4096 envs, replayed from a graph of one launch (CUDA events around the replays)."""
    import torch
    from learninghumanoidwalking_b200 import _lib
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(4096, model="jvrc_walk", precision=32, seed=0, device=0, payload_mass=20.0)
    env.reset()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        _lib.ops().sim_draw_payload(env._h.value, env.state_i, 0, 0, env.ended, 20.0, 0.1, env.payload)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            _lib.ops().sim_draw_payload(env._h.value, env.state_i, 0, 0, env.ended, 20.0, 0.1, env.payload)
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


def train_iter_s(mass: float) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(4096, model="jvrc_walk", precision=32, seed=0, payload_mass=mass)
    probe = base()
    r = probe.robot
    probe.close()
    env_fn = lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=4096 * 400 // 4800 * 64,
                           epochs=3, max_traj_len=400, num_procs=4096, max_grad_norm=0.5, mirror_coeff=0.4, eval_freq=10**9,
                           recurrent=False, imitate_coeff=0.0, std_dev=0.223, learn_std=False,
                           logdir=tempfile.mkdtemp(prefix="lhw_bench_payload_"), steps_per_env=400, eval_batches=0, tf32=False,
                           eval_at_start=False)
    os.environ["LHW_TENSORBOARD"] = "0"
    ppo = PPO(env_fn, args, seed=0)
    ppo.train(None, 1, verbose=False)    # warm-up (graph capture)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    log = ppo.train(None, 1, verbose=False)
    torch.cuda.synchronize()
    return dict(iter_s=time.perf_counter() - t0, sample_s=log[-1]["sample_time"], optimize_s=log[-1]["optimize_time"])


def study(iters: int, out: str) -> dict:
    """Plain and payload trainings of jvrc_walk with one seed, each evaluated across STUDY_MASSES on 4096 envs."""
    import run_experiment as rx
    res = {}
    for key, mass in (("plain", "0"), ("payload_20", "20")):
        logdir = os.path.join(out, "study", key)
        t0 = time.perf_counter()
        rx.main(["train", "--env", "jvrc_walk", "--payload-mass", mass, "--logdir", logdir, "--n-itr", str(iters), "--seed", "1",
                 "--eval-freq", str(max(1, iters // 2))])
        train_s = time.perf_counter() - t0
        report = os.path.join(out, f"study_{key}.json")
        rx.main(["eval", "--logdir", logdir, "--num-envs", "4096", "--payloads", ",".join(map(str, STUDY_MASSES)), "--report", report])
        cells = json.load(open(report))["summary"]["payload"]["cells"]
        res[key] = dict(train_s=train_s, cells=[dict(mass_kg=c["mass"], fall_fraction=c["fall_fraction"],
                                                     forward_vx_error=c["tracking"]["FORWARD"]["vx_error"]) for c in cells])
        for c in res[key]["cells"]:
            print(f"study {key} ({iters} iterations): eval payload {c['mass_kg']:4.0f} kg  fell {c['fall_fraction']:.4f}  "
                  f"FORWARD |v_fwd - vx| {c['forward_vx_error']}", flush=True)
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--study", type=int, default=0, help="iterations of each outcome-study training (0: no study)")
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_payload needs a CUDA device")
    from bench_eval import gpu_identity
    res = {"gpu": gpu_identity(), "steps_per_s": {}, "newton_iters": {}, "train_iter": {}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W", flush=True)
    for name in VARIANTS:
        for prec in (64, 32):
            for mass in (0.0, 20.0):
                steps_per_s(name, prec, mass, 30)     # untimed
            for _ in range(args.repeats):
                for key, mass in (("plain", 0.0), ("payload", 20.0)):
                    v, it = steps_per_s(name, prec, mass, args.steps)
                    res["steps_per_s"].setdefault(f"{name}_fp{prec}_{key}", []).append(v)
                    res["newton_iters"].setdefault(f"{name}_fp{prec}_{key}", []).append(it)
                    print(f"{name} 4096 envs fp{prec} {key}: {v / 1e6:.4f} M env-steps/s, {it:.2f} Newton iterations per env "
                          "in the last step", flush=True)
    res["draw_us"] = draw_us()
    print(f"draw launch, 4096 envs, graph replay: {res['draw_us']:.2f} us", flush=True)
    for key, mass in (("plain", 0.0), ("payload", 20.0)):
        r = train_iter_s(mass)
        res["train_iter"][key] = r
        print(f"train_iter jvrc_walk 4096 x 400 fp32 {key}: {r['iter_s']:.3f} s (sampling {r['sample_s']:.3f} s, "
              f"optimisation {r['optimize_s']:.3f} s)", flush=True)
    if args.study:
        res["study"] = study(args.study, args.out_dir or tempfile.mkdtemp(prefix="lhw_payload_study_"))
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_payload.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
