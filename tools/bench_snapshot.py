#!/usr/bin/env python3
"""Wall time to write and to restore a training snapshot (learninghumanoidwalking_b200/rl/snapshot.py), one GPU.

    python tools/bench_snapshot.py [--envs 4096] [--precision 64] [--model jvrc_walk] [--reps 3]

A PPO on `--envs` environments trains one short iteration, then writes its snapshot `--reps` times (device -> host copies,
torch.save, fsync, rename, latest.json, pruning) into a temporary directory; a second PPO built like the first (and past
make_optimizers) restores it `--reps` times (torch.load, validation, host -> device copies).  Prints one JSON line with the
median times, the bytes on disk and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import sys
import tempfile
import time
from functools import partial
from pathlib import Path
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--precision", type=int, default=64, choices=[32, 64])
    ap.add_argument("--model", default="jvrc_walk")
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import bench
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO, snapshot
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    os.environ.setdefault("LHW_TENSORBOARD", "0")
    base = partial(BatchedHumanoidEnv, args.envs, model=args.model, precision=args.precision, seed=0)
    probe = base()
    r = probe.robot
    probe.close()
    env_fn = base if not hasattr(r, "mirrored_obs") else partial(SymmetricEnv, base, mirrored_obs=r.mirrored_obs,
                                                                 mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    with tempfile.TemporaryDirectory(prefix="lhw_bench_snapshot_") as tmp:
        a = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=4096, epochs=1,
                            max_traj_len=400, num_procs=args.envs, max_grad_norm=0.5, mirror_coeff=0.4, eval_freq=10 ** 9,
                            eval_at_start=False, recurrent=False, imitate_coeff=0.0, std_dev=0.223, learn_std=False, logdir=tmp,
                            steps_per_env=16, env=args.model, precision=args.precision)
        ppo = PPO(env_fn, a, seed=0)
        ppo.train(None, 1, verbose=False)
        write_s = []
        for k in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            snapshot.write(ppo, k, 1.0)
            write_s.append(time.perf_counter() - t0)
        d = snapshot.snapshot_root(tmp) / f"itr_{args.reps - 1}"
        sizes = {p.name: p.stat().st_size for p in sorted(Path(d).iterdir())}
        ppo.env.close()
        if ppo._comm is not None:
            ppo._comm.close()
        del ppo
        ppo = PPO(env_fn, a, seed=1)
        ppo.make_optimizers()
        restore_s = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ppo.restore(tmp)          # ends in a device synchronise
            restore_s.append(time.perf_counter() - t0)
        ppo.env.close()
    print(json.dumps({"workload": f"{args.model} fp{args.precision}", "envs": args.envs, "reps": args.reps,
                      "write_s_median": statistics.median(write_s), "restore_s_median": statistics.median(restore_s),
                      "write_s": write_s, "restore_s": restore_s, "bytes": sizes, "gpu": bench.gpu_identity(0)}))


if __name__ == "__main__":
    main()
