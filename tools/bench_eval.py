#!/usr/bin/env python3
"""Cost of the batched evaluation (`run_experiment.py eval --num-envs N`, rl/evaluation.py, DESIGN.md §7.4).

For jvrc_walk and h1, at fp64 and fp32, with N in {1, 1024, 4096}: one whole evaluation (reset, the eager first step, the graph
capture and max_traj_len - 1 replays of actor + step + accumulate, up to the copy of the accumulators to the host) timed with
CUDA events, as control steps per second and env-steps per second; then the accumulate launch alone, 200 launches between one
event pair.  jvrc_walk runs the trained actor of tests/golden (it walks); h1 runs an untrained actor of the same shape (its
robots fall early, and keep being simulated: autoreset is off).  Every configuration is run once untimed first.  The card's
name and power limit are printed in the same call.

    python tools/bench_eval.py [--horizon 400] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
TRAINED = os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")


def gpu_identity() -> dict:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         capture_output=True, text=True, timeout=60).stdout.strip().split(",")
    return {"name": out[0].strip(), "power_limit_w": float(out[1])}


def actor_for(env_name: str):
    import torch
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    from learninghumanoidwalking_b200.rl.policies.actor import Gaussian_FF_Actor
    install_reference_aliases()
    if env_name == "jvrc_walk":
        return torch.load(TRAINED, weights_only=False).cuda().eval()
    torch.manual_seed(0)
    return Gaussian_FF_Actor(35, 10).cuda().eval()


def time_eval(env_name: str, precision: int, n: int, horizon: int, policy) -> dict:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import evaluation
    res = {"env": env_name, "precision": precision, "envs": n, "horizon": horizon}
    for timed in (False, True):
        env = BatchedHumanoidEnv(n, model=env_name, precision=precision, seed=0, device=0, max_traj_len=horizon)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        acc = evaluation.rollout(env, policy, horizon).cpu()
        b.record()
        torch.cuda.synchronize()
        if timed:
            s = a.elapsed_time(b) * 1e-3
            res.update(eval_s=s, control_steps_per_s=horizon / s, env_steps_per_s=n * horizon / s,
                       fall_fraction=float((acc[:, evaluation.DONE] != 0).double().mean()))
            k = 200
            acc_dev = torch.zeros(n, evaluation.WORDS, dtype=torch.float64, device=env.device)
            env.eval_accumulate(acc_dev)
            torch.cuda.synchronize()
            a.record()
            for _ in range(k):
                env.eval_accumulate(acc_dev)
            b.record()
            torch.cuda.synchronize()
            res["accumulate_us"] = a.elapsed_time(b) * 1e3 / k
            res["accumulate_share_of_step"] = res["accumulate_us"] * 1e-6 / (s / horizon)
        env.close()
    return res


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--horizon", type=int, default=400, help="control steps per evaluation (the default --max-traj-len)")
    ap.add_argument("--out-dir", default=None, help="also write the results as JSON here")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval needs a CUDA device")
    res = {"gpu": gpu_identity(), "runs": []}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W")
    for env_name in ("jvrc_walk", "h1"):
        policy = actor_for(env_name)
        for precision in (64, 32):
            for n in (1, 1024, 4096):
                r = time_eval(env_name, precision, n, args.horizon, policy)
                res["runs"].append(r)
                print(f"{env_name:>9s} fp{precision} N={n:>4d}: evaluation {r['eval_s']:.3f} s = {r['control_steps_per_s']:.0f} control "
                      f"steps/s = {r['env_steps_per_s'] / 1e6:.3f} M env-steps/s (fell {r['fall_fraction']:.3f}); accumulate "
                      f"{r['accumulate_us']:.2f} us = {100 * r['accumulate_share_of_step']:.2f}% of a control step", flush=True)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_eval.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
