"""Batched evaluation of a saved actor (`run_experiment.py eval --num-envs N`, DESIGN.md §7.4).

N environments of one batch are reset once and stepped together with the deterministic actor and autoreset off for exactly
max_traj_len control steps: each environment's first episode is one sample.  After every step one launch
(BatchedHumanoidEnv.eval_accumulate, csrc/sim_core.h eval_accumulate_env) adds it to a per-env float64 accumulator record on the
device; the host reads the records once, at the end.  The control step (actor forward, step, accumulate) is captured as one
CUDA graph after an eager first step and replayed, as the rollout worker does.
"""
from __future__ import annotations

import json

import numpy as np
import torch

# the accumulator words of csrc/sim_core.h (EV_*), per env
LEN, RET, DONE, TERMS, TRACK, REACHED, SEQLEN, WORDS = 0, 1, 2, 3, 13, 25, 26, 27
MODES = ("STANDING", "INPLACE", "FORWARD")     # WalkingTask's modes, in the order of the kernel's mode word
TRACKED = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1")   # h1: its StandingTask, against zero references


@torch.no_grad()
def rollout(env, policy, steps: int, graph: bool = True) -> torch.Tensor:
    """Reset `env` once and run `steps` control steps of the deterministic `policy` with autoreset off; returns the
    [N, WORDS] float64 device accumulators.  graph=False runs every step eagerly (the same launches, in the same order)."""
    if env.eval_words() != WORDS:
        raise RuntimeError(f"the library's evaluation record has {env.eval_words()} words, this module knows {WORDS}")
    acc = torch.zeros(env.num_envs, WORDS, dtype=torch.float64, device=env.device)
    state = env.reset().float().clone()

    def body():
        a = policy(state, deterministic=True)
        obs, _, _, _ = env.step(a if env.dtype == torch.float32 else a.double(), autoreset=False)
        env.eval_accumulate(acc)
        state.copy_(obs.float())

    if not graph or steps <= 1:
        for _ in range(steps):
            body()
        return acc
    cur = torch.cuda.current_stream(env.device)
    s = torch.cuda.Stream(device=env.device)
    s.wait_stream(cur)
    with torch.cuda.stream(s):
        body()     # the first step, eagerly: it also warms up the actor's GEMMs before the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            body()     # capturing does not execute: the replays run steps 2..steps
        env.bind()
        for _ in range(steps - 1):
            g.replay()
    cur.wait_stream(s)
    return acc


def summarize(acc: np.ndarray, env_name: str, reward_names) -> dict:
    """The statistics of N first episodes from their accumulator records [N, WORDS] (host float64)."""
    n = acc.shape[0]
    length, ret, fell = acc[:, LEN], acc[:, RET], acc[:, DONE] != 0
    steps = length.sum()
    out = dict(num_envs=int(n), fall_fraction=float(fell.mean()),
               length=dict(mean=float(length.mean()), min=float(length.min()), p5=float(np.percentile(length, 5)),
                           median=float(np.median(length))),
               reward_terms={name: float(acc[:, TERMS + k].sum() / steps) for k, name in enumerate(reward_names)})
    out["return"] = dict(mean=float(ret.mean()), std=float(ret.std()))
    if env_name in TRACKED:
        tracking = {}
        for m, mode in enumerate(MODES[:1] if env_name == "h1" else MODES):
            t = acc[:, TRACK + 4 * m:TRACK + 4 * m + 4].sum(0)
            tracking[mode] = dict(steps=int(t[0]), vx_error=float(t[1] / t[0]) if t[0] else None,
                                  vy_error=float(t[2] / t[0]) if t[0] else None, yaw_rate_error=float(t[3] / t[0]) if t[0] else None)
        out["tracking"] = tracking
    if env_name == "jvrc_step":
        reached, seq_len = acc[:, REACHED], acc[:, SEQLEN]
        out["footsteps"] = dict(mean_reached=float(reached.mean()), mean_sequence_length=float(seq_len.mean()),
                                completed_fraction=float((reached >= seq_len - 1).mean()))
    return out


def per_env(acc: np.ndarray, env_name: str, reward_names) -> dict:
    """The accumulator records as named per-env lists (the report's `per_env`)."""
    out = {"length": acc[:, LEN].astype(int).tolist(), "return": acc[:, RET].tolist()}
    out.update(fell=(acc[:, DONE] != 0).tolist(),
               reward_term_sums={name: acc[:, TERMS + k].tolist() for k, name in enumerate(reward_names)})
    if env_name in TRACKED:
        out["tracking"] = {mode: dict(steps=acc[:, TRACK + 4 * m].astype(int).tolist(),
                                      vx_error_sum=acc[:, TRACK + 4 * m + 1].tolist(),
                                      vy_error_sum=acc[:, TRACK + 4 * m + 2].tolist(),
                                      yaw_rate_error_sum=acc[:, TRACK + 4 * m + 3].tolist())
                           for m, mode in enumerate(MODES[:1] if env_name == "h1" else MODES)}
    if env_name == "jvrc_step":
        out["footsteps"] = dict(reached=acc[:, REACHED].astype(int).tolist(), sequence_length=acc[:, SEQLEN].astype(int).tolist())
    return out


def format_table(s: dict, max_traj_len: int) -> str:
    L = s["length"]
    lines = [f"{s['num_envs']} environments, one episode each, horizon {max_traj_len} control steps",
             f"  fell before the horizon   {s['fall_fraction']:.4f}",
             f"  episode length            mean {L['mean']:.1f}  min {L['min']:.0f}  p5 {L['p5']:.1f}  median {L['median']:.1f}",
             f"  return                    mean {s['return']['mean']:.4f}  std {s['return']['std']:.4f}",
             "  per-step mean of each reward term:"]
    lines += [f"    {name:>20s} {v:.4f}" for name, v in s["reward_terms"].items()]
    if "tracking" in s:
        lines.append("  command tracking, mean per step:   steps   |v_fwd - vx_ref|  |v_lat - vy_ref|  |w_z - yaw_ref|")
        for mode, t in s["tracking"].items():
            f = lambda v: "-" if v is None else f"{v:.4f}"
            lines.append(f"    {mode:>30s} {t['steps']:>8d} {f(t['vx_error']):>17s} {f(t['vy_error']):>17s} {f(t['yaw_rate_error']):>16s}")
    if "footsteps" in s:
        fs = s["footsteps"]
        lines.append(f"  footsteps reached         mean {fs['mean_reached']:.2f} of {fs['mean_sequence_length']:.2f}; "
                     f"sequences completed {fs['completed_fraction']:.4f}")
    return "\n".join(lines)


def evaluate_batched(policy, env, out_report=None, meta: dict | None = None) -> dict:
    """Roll `policy` out on every environment of `env` for env.max_traj_len control steps, print the table and, with
    out_report, write the JSON report (meta + summary + per-env arrays).  Returns the report."""
    acc = rollout(env, policy, env.max_traj_len).cpu().numpy()
    summary = summarize(acc, env.model_name, env.reward_names)
    print(format_table(summary, env.max_traj_len))
    report = dict(meta or {}, env=env.model_name, precision=env.precision, seed=env.seed, num_envs=env.num_envs,
                  max_traj_len=env.max_traj_len, summary=summary, per_env=per_env(acc, env.model_name, env.reward_names))
    if out_report is not None:
        with open(out_report, "w") as f:
            json.dump(report, f, indent=1)
        print(f"Wrote {out_report}")
    return report
