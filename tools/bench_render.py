#!/usr/bin/env python3
"""Cost of the renderer (torch.ops.lhw.sim_render) on the GPU, timed with CUDA events:

  * frames/s for 1 environment at 640x480 and for 64 environments at 320x240 (one launch renders all of them);
  * control steps/s of `run_experiment.py eval` with and without --out-dir, on an actor trained for one iteration here.
    Each is the difference of an --ep-len 12 and an --ep-len 2 run (440 - 80 control steps), so that loading the actor and
    building the environment drop out; with --out-dir it includes the copy to the host and the mp4 encoding.

Prints the card name and power limit with the results, as one JSON line.

    python tools/bench_render.py [--iters 200]
"""
import argparse
import contextlib
import io
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                            text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def frames_per_s(n_envs, width, height, iters):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(n_envs, model="jvrc_walk", precision=32, seed=0)
    env.reset()
    ids = list(range(n_envs))
    for _ in range(10):
        env.render_rgb(ids, width, height)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        env.render_rgb(ids, width, height)
    b.record()
    torch.cuda.synchronize()
    ms = a.elapsed_time(b) / iters
    env.close()
    return dict(n_envs=n_envs, width=width, height=height, ms_per_call=round(ms, 4), frames_per_s=round(n_envs * 1000.0 / ms, 1))


def eval_steps_per_s(tmp):
    import run_experiment as rx
    logs = os.path.join(tmp, "logs")
    with contextlib.redirect_stdout(io.StringIO()):
        rx.main(["train", "--env", "jvrc_walk", "--logdir", logs, "--num-procs", "64", "--n-itr", "1", "--max-traj-len", "40",
                 "--minibatch-size", "256", "--epochs", "1", "--seed", "0"])
    out = {}
    for label, extra in (("without_out_dir", []), ("with_out_dir", ["--out-dir", os.path.join(tmp, "video")])):
        t = {}
        for ep_len in (2, 12, 2, 12):
            with contextlib.redirect_stdout(io.StringIO()):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                rx.main(["eval", "--logdir", logs, "--ep-len", str(ep_len)] + extra)
                torch.cuda.synchronize()
            t[ep_len] = time.perf_counter() - t0     # the second (warm) run of each length counts
        out[label] = round((12 - 2) / 0.025 / (t[12] - t[2]), 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_render.py needs a CUDA device")
    name, pl = card()
    res = dict(card=name, power_limit=pl, one_env_640x480=frames_per_s(1, 640, 480, args.iters),
               batch_64_envs_320x240=frames_per_s(64, 320, 240, args.iters))
    with tempfile.TemporaryDirectory() as tmp:
        res["eval_control_steps_per_s"] = eval_steps_per_s(tmp)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
