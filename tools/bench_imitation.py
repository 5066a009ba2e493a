#!/usr/bin/env python3
"""What `train --imitate` costs: optimiser-step and whole-iteration time with and without a teacher.

At the default flags of `run_experiment.py train` (4096 environments x 400 steps, minibatches scaled to 225 optimiser steps per
iteration, mirror loss on, fp32 simulator) it trains two pairs of runs of the same seed, each without and with a teacher:
  * jvrc_walk with a jvrc_walk teacher (tests/golden/trained_actor_jvrc_walk.pt, the identity projector);
  * h1_walk with an h1 teacher (a 35-input actor written here next to an experiment.pkl naming h1: the standing projector).
The first --warmup iterations are not timed (cuBLAS warm-up, the capture of the update graph); of the timed ones, a CUDA event
pair around every `_update_step` call (the replayed update graph: the policy, old-policy, critic and teacher forwards, the fused
loss, the backward passes and the fused clip + Adam) gives the optimiser-step time, and an event pair around each iteration (sampling,
GAE, advantages, the 225 gathers and updates) the iteration time.  The card's name and power limit are read in the same call.

    python tools/bench_imitation.py [--envs 4096] [--iters 3] [--warmup 2] [--out-dir DIR]
"""
from __future__ import annotations

import argparse
import json
import os
import pickle
import sys
import tempfile
from argparse import Namespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tools.bench_h1_walk import gpu_identity  # noqa: E402

JVRC_TEACHER = os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")


def h1_teacher(tmp: str) -> str:
    import torch
    from learninghumanoidwalking_b200.rl.policies import Gaussian_FF_Actor, export_module
    torch.manual_seed(0)
    path = os.path.join(tmp, "actor_0.pt")
    torch.save(export_module(Gaussian_FF_Actor(35, 10)), path)
    with open(os.path.join(tmp, "experiment.pkl"), "wb") as f:
        pickle.dump(Namespace(env="h1"), f)
    return path


def time_run(model: str, teacher: str | None, envs: int, iters: int, warmup: int, tmp: str) -> dict:
    import torch
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import PPO
    parser = argparse.ArgumentParser()
    for flag, kw in rx.TRAIN_FLAGS:
        parser.add_argument(flag, **kw)
    argv = ["--env", model, "--num-procs", str(envs), "--logdir", tmp, "--seed", "0"]
    if teacher:
        argv += ["--imitate", teacher, "--imitate-coeff", "1"]
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
    ppo.env.close()
    if ppo._comm is not None:
        ppo._comm.close()
    step_ms.sort()
    return dict(env=model, teacher=bool(teacher), envs=envs, updates_per_iteration=n_updates, update_graph=replayed,
                optimiser_step_ms_median=round(step_ms[len(step_ms) // 2], 4),
                optimiser_step_ms_mean=round(sum(step_ms) / len(step_ms), 4),
                iteration_ms=[round(t, 1) for t in iter_ms])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out-dir", default=None, help="also write the results as JSON here")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_imitation.py times the CUDA learner: it needs a GPU")
    os.environ["LHW_TENSORBOARD"] = "0"
    res = dict(gpu=gpu_identity(), runs=[])
    with tempfile.TemporaryDirectory() as tmp:
        h1 = h1_teacher(tmp)
        for model, teacher in (("jvrc_walk", None), ("jvrc_walk", JVRC_TEACHER), ("h1_walk", None), ("h1_walk", h1)):
            r = time_run(model, teacher, a.envs, a.iters, a.warmup, tmp)
            print(json.dumps(r), flush=True)
            res["runs"].append(r)
    res["gpu_after"] = gpu_identity()
    print(json.dumps(res))
    if a.out_dir:
        os.makedirs(a.out_dir, exist_ok=True)
        with open(os.path.join(a.out_dir, "bench_imitation.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
