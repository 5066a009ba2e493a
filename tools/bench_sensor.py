#!/usr/bin/env python3
"""Cost of the sensor errors (DESIGN.md §7.12), and what a trained actor makes of them.

1. The sensor pass alone (`sensor_kernel`), 4096 envs after a step with autoreset and the draw, fp32 and fp64, every variant's
   row width, replayed 1000 times from one CUDA graph (CUDA events around the replays).
2. DeviceRolloutWorker.sample at 4096 envs x 400 steps, jvrc_walk, fp32 and fp64: plain against random sensor errors
   (`sensor_noise=1, sensor_bias=(0.05, 0.1, 0.02)`), alternating, `--repeats` timed samples of each after an untimed one.
3. One full PPO iteration of jvrc_walk (4096 envs x 400 steps, fp32, the training defaults) plain and with the sensor errors
   above, after one untimed iteration each: the whole iteration and its sampling.
4. bench.py's headline (`--gpus 1 --steps 20 --warmup 3`, sensor errors off), run as it ships.
5. The falls per cell of the trained jvrc_walk actor of tests/golden/ over a roll / pitch / encoder / noise sweep, 4096 envs, fp64.

The card's name, power limit and SM clock are read in the same call.

    python tools/bench_sensor.py [--repeats 2] [--out-dir DIR]
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
ON = dict(sensor_noise=1.0, sensor_bias=(0.05, 0.1, 0.02))
SWEEP = ["roll:-0.1,-0.05,0,0.05,0.1", "pitch:-0.1,-0.05,0.05,0.1", "encoder:-0.05,0.05,0.1", "noise:1,2,4"]


def gpu_identity() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits",
                          "-i", "0"], capture_output=True, text=True, timeout=60).stdout.strip().split(",")
    return {"name": out[0].strip(), "power_limit_w": float(out[1]), "sm_clock_mhz": float(out[2]), "max_sm_clock_mhz": float(out[3])}


def pass_us(name: str, precision: int, replays: int = 1000) -> float:
    """Microseconds per sensor pass of 4096 envs after a step (autoreset, every env ended: term_obs, draw and obs), replayed
    from a graph of one launch."""
    import torch
    from learninghumanoidwalking_b200 import _lib
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(4096, model=name, precision=precision, seed=0, device=0, **ON)
    env.reset()
    ended = torch.ones(env.num_envs, dtype=torch.int32, device=env.device)
    call = lambda: _lib.ops().sim_sense(env._h.value, env.state_i, 0, 0, ended, True, True, list(env.sensor_bias), env.sensor,
                                        env.obs, env.term_obs)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        call()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            call()
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


def sample_s(precision: int, on: bool, n: int = 4096, T: int = 400) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import DeviceRolloutWorker, FF_V, Gaussian_FF_Actor
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=precision, seed=0, device=0, **(ON if on else {}))
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


def train_iter_s(on: bool) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(4096, model="jvrc_walk", precision=32, seed=0, **(ON if on else {}))
    probe = base()
    r = probe.robot
    probe.close()
    env_fn = lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=4096 * 400 // 4800 * 64,
                           epochs=3, max_traj_len=400, num_procs=4096, max_grad_norm=0.5, mirror_coeff=0.4, eval_freq=10**9,
                           recurrent=False, imitate_coeff=0.0, std_dev=0.223, learn_std=False,
                           logdir=tempfile.mkdtemp(prefix="lhw_bench_sensor_"), steps_per_env=400, eval_batches=0, tf32=False,
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


def sweep_falls(n: int = 4096) -> list:
    """The trained jvrc_walk actor of tests/golden/ over SWEEP: per cell (kind, value, fall fraction, mean length)."""
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import evaluation as ev
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    policy = torch.load(os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt"), weights_only=False).cuda().eval()
    cells = [(kind, float(v)) for spec in SWEEP for kind, _, vs in [spec.partition(":")] for v in vs.split(",")]
    env = BatchedHumanoidEnv(n, model="jvrc_walk", precision=64, seed=0, device=0)
    cell, noise, bias = ev.sensor_grid(n, cells, env.act_dim)
    acc = ev.rollout(env, policy, env.max_traj_len, sensor=(noise, bias)).cpu().numpy()
    s = ev.sensor_summary(acc, cell, cells, env.model_name, env.reward_names)
    env.close()
    return [dict(kind=c["kind"], value=c["value"], n=c["n"], fall_fraction=c["fall_fraction"], mean_length=c["mean_length"])
            for c in s["cells"]]


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_sensor needs a CUDA device")
    res = {"gpu": gpu_identity(), "pass_us": {}, "sample_s": {}, "train_iter": {}}
    g = res["gpu"]
    print(f"{g['name']}, power limit {g['power_limit_w']:.0f} W, SM clock {g['sm_clock_mhz']:.0f} MHz (max {g['max_sm_clock_mhz']:.0f})",
          flush=True)
    for name in VARIANTS:
        for prec in (32, 64):
            res["pass_us"][f"{name}_fp{prec}"] = v = pass_us(name, prec)
            print(f"sensor pass {name} fp{prec}, 4096 envs, graph replay: {v:.2f} us", flush=True)
    for prec in (32, 64):
        sample_s(prec, False, T=40)          # untimed
        sample_s(prec, True, T=40)
        for _ in range(args.repeats):
            for on in (False, True):
                res["sample_s"].setdefault(f"fp{prec}_{'on' if on else 'plain'}", []).append(sample_s(prec, on))
        print(f"DeviceRolloutWorker.sample jvrc_walk 4096 x 400 fp{prec}: plain "
              + " ".join(f"{v:.3f}" for v in res["sample_s"][f"fp{prec}_plain"]) + " s, sensor errors "
              + " ".join(f"{v:.3f}" for v in res["sample_s"][f"fp{prec}_on"]) + " s", flush=True)
    for key, on in (("plain", False), ("on", True), ("plain_again", False)):
        r = train_iter_s(on)
        res["train_iter"][key] = r
        print(f"train_iter jvrc_walk 4096 x 400 fp32 {key}: {r['iter_s']:.3f} s (sampling {r['sample_s']:.3f} s, "
              f"optimisation {r['optimize_s']:.3f} s)", flush=True)
    res["bench"] = bench_headline()
    print("bench.py:", json.dumps(res["bench"]), flush=True)
    res["sweep"] = sweep_falls()
    for c in res["sweep"]:
        print(f"trained jvrc_walk actor, {c['kind']:>7s} {c['value']:6.3f}: fell {c['fall_fraction']:.3f} of {c['n']}, "
              f"mean length {c['mean_length']:.1f}", flush=True)
    res["gpu_after"] = gpu_identity()
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_sensor.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
