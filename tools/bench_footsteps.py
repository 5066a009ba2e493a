#!/usr/bin/env python3
"""Cost of the footstep sweep (DESIGN.md §7.7).

The batched evaluation of a jvrc_step actor at 4096 envs, fp64: plain (one reset()) against the sweep forward:0,0.05,0.1,0.15
lateral:left,right backward curved standing (one reset_footsteps() in its place), alternating, `--repeats` timed runs of each after
one untimed run of each.  The sweep's per-cell table is printed once.  The actor is `--actor` (a saved actor.pt) or, without it, a
freshly initialised one.  The card's name and power limit are read in the same call.

    python tools/bench_footsteps.py [--actor PATH] [--repeats 2] [--out-dir DIR]
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
CELLS = [("FORWARD", 0.0), ("FORWARD", 0.05), ("FORWARD", 0.1), ("FORWARD", 0.15), ("LATERAL", 1.0), ("LATERAL", -1.0),
         ("BACKWARD", 0.0), ("CURVED", -1.0), ("STANDING", 0.0)]


def eval_s(policy, sweep: bool, n: int = 4096, show: bool = False) -> float:
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import evaluation as ev
    env = BatchedHumanoidEnv(n, model="jvrc_step", precision=64, seed=0, device=0)
    plans = ev.footstep_grid(n, CELLS) if sweep else None
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    acc = ev.rollout(env, policy, env.max_traj_len, footsteps=plans).cpu().numpy()
    s = time.perf_counter() - t0
    if show:
        print(ev.format_footstep_table(ev.footstep_summary(acc, *plans, CELLS)), flush=True)
    env.close()
    return s


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--actor", default=None, help="a saved jvrc_step actor (actor.pt); default: a freshly initialised one")
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--out-dir", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_footsteps needs a CUDA device")
    from bench_eval import gpu_identity
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    from learninghumanoidwalking_b200.rl.policies.actor import Gaussian_FF_Actor
    install_reference_aliases()
    if args.actor:
        policy = torch.load(args.actor, weights_only=False).cuda().eval()
    else:
        torch.manual_seed(0)
        policy = Gaussian_FF_Actor(39, 12).cuda().eval()
    res = {"gpu": gpu_identity(), "actor": args.actor, "eval_s": {"plain": [], "sweep": []}}
    print(f"{res['gpu']['name']}, power limit {res['gpu']['power_limit_w']:.0f} W; actor {args.actor or 'freshly initialised'}",
          flush=True)
    eval_s(policy, False), eval_s(policy, True, show=True)    # untimed
    for _ in range(args.repeats):
        for key in ("plain", "sweep"):
            res["eval_s"][key].append(eval_s(policy, key == "sweep"))
            print(f"eval 4096 envs jvrc_step fp64 {key}: {res['eval_s'][key][-1]:.4f} s", flush=True)
    if args.out_dir:
        os.makedirs(args.out_dir, exist_ok=True)
        json.dump(res, open(os.path.join(args.out_dir, "bench_footsteps.json"), "w"), indent=1)


if __name__ == "__main__":
    main()
