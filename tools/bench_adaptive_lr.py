#!/usr/bin/env python3
"""What `train --schedule adaptive` costs: optimiser-step and whole-iteration time, fixed rate vs KL-adaptive rate.

At the default flags of `run_experiment.py train` (jvrc_walk, 4096 environments x 400 steps, minibatches scaled to 225 optimiser
steps per iteration, mirror loss on, fp32 simulator) it trains runs of the same seed, alternating fixed / adaptive --rounds times
in one process.  The first --warmup iterations of a run are not timed (cuBLAS warm-up, the capture of the update graph); of the
timed ones, a CUDA event pair around every `_update_step` call (the replayed update graph: forwards, fused loss, backward, the
fused exchange with or without the rate update) gives the optimiser-step time, and an event pair around each iteration (sampling,
GAE, advantages, the 225 updates, and under the adaptive schedule the one read of the rate) the iteration time.  The card's name
and power limit are read in the same call.

    python tools/bench_adaptive_lr.py [--envs 4096] [--iters 3] [--warmup 2] [--rounds 2] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_h1_walk import gpu_identity  # noqa: E402


def time_run(model: str, kind: str, envs: int, iters: int, warmup: int, tmp: str) -> dict:
    import torch
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import PPO
    parser = argparse.ArgumentParser()
    for flag, kw in rx.TRAIN_FLAGS:
        parser.add_argument(flag, **kw)
    argv = ["--env", model, "--num-procs", str(envs), "--logdir", tmp, "--seed", "0", "--schedule", kind]
    args = parser.parse_args(argv)
    args.eval_at_start, args.eval_freq = False, 10 ** 9
    ppo = PPO(rx.make_env_fn(args, 0, 1, 0), args, seed=0)
    ev = []
    inner = ppo._update_step

    def timed_update(*a):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        out = inner(*a)
        e.record()
        ev.append((s, e))
        return out

    ppo._update_step = timed_update
    step_ms, iter_ms, n_updates = [], [], 0
    for itr in range(warmup + iters):
        ev.clear()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        ppo.train(None, itr + 1, verbose=False, start_itr=itr)
        e.record()
        torch.cuda.synchronize()
        if itr >= warmup:
            iter_ms.append(s.elapsed_time(e))
            step_ms += [a.elapsed_time(b) for a, b in ev]
            n_updates = len(ev)
    replayed = ppo._ug is not None
    lr = ppo._comm.get_lr() if kind == "adaptive" else ppo.lr
    ppo.env.close()
    if ppo._comm is not None:
        ppo._comm.close()
    step_ms.sort()
    return dict(env=model, schedule=kind, final_lr=lr, envs=envs, updates_per_iteration=n_updates, update_graph=replayed,
                optimiser_step_ms_median=round(step_ms[len(step_ms) // 2], 4),
                optimiser_step_ms_mean=round(sum(step_ms) / len(step_ms), 4),
                iteration_ms=[round(t, 1) for t in iter_ms])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2, help="fixed / adaptive pairs, alternating")
    ap.add_argument("--out-dir", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_adaptive_lr.py times the CUDA learner: it needs a GPU")
    os.environ["LHW_TENSORBOARD"] = "0"
    res = dict(gpu=gpu_identity(), runs=[])
    with tempfile.TemporaryDirectory() as tmp:
        for _ in range(a.rounds):
            for kind in ("fixed", "adaptive"):
                r = time_run("jvrc_walk", kind, a.envs, a.iters, a.warmup, tmp)
                print(json.dumps(r), flush=True)
                res["runs"].append(r)
    for kind in ("fixed", "adaptive"):
        runs = [r for r in res["runs"] if r["schedule"] == kind]
        steps = sorted(r["optimiser_step_ms_median"] for r in runs)
        iters = sorted(t for r in runs for t in r["iteration_ms"])
        res[kind] = dict(optimiser_step_ms_median_of_runs=steps[len(steps) // 2], iteration_ms_median=iters[len(iters) // 2])
    res["gpu_after"] = gpu_identity()
    print(json.dumps(res))
    if a.out_dir:
        os.makedirs(a.out_dir, exist_ok=True)
        with open(os.path.join(a.out_dir, "bench_adaptive_lr.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
