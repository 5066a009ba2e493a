"""Batched evaluation of a saved actor (`run_experiment.py eval --num-envs N`, DESIGN.md §7.4).

N environments of one batch are reset once and stepped together with the deterministic actor and autoreset off for exactly
max_traj_len control steps: each environment's first episode is one sample.  After every step one launch
(BatchedHumanoidEnv.eval_accumulate, csrc/sim_core.h eval_accumulate_env) adds it to a per-env float64 accumulator record on the
device; the host reads the records once, at the end.  The control step (actor forward, step, accumulate) is captured as one
CUDA graph after an eager first step and replayed, as the rollout worker does.

The push-recovery sweep (`eval --num-envs N --push-speeds ...`, DESIGN.md §7.5) pushes every environment once, after control step
K = round(push_at / dt), between two replays of the same graph: env i gets the speed and heading-frame direction of grid cell
i mod (speeds x directions).  A fallen env is not pushed (a device-side `where` on its ended-by-done word), and the statistics come
from the same accumulator words: fell before the push (EV_DONE set and EV_LEN <= K), survived (EV_DONE clear at the horizon).

The command-tracking sweep (`eval --num-envs N --command forward:0,0.2 inplace:0.4 standing`, DESIGN.md §7.6) gives env i the held
command of cell i mod C (BatchedHumanoidEnv.set_command) after the reset, before the first step and outside the graph.  The graph
body then also launches BatchedHumanoidEnv.command_accumulate, whose per-env records give the signed mean velocities of each cell.

The footstep sweep (`eval --num-envs N --footsteps forward:0,0.05,0.1 lateral:left,right curved standing`, DESIGN.md §7.7, jvrc_step)
resets env i with the stepping-stone plan of cell i mod C (BatchedHumanoidEnv.reset_footsteps) in place of the one plain reset.  The
graph body is unchanged: the accumulator's footsteps-reached and sequence-length words already give each cell's progress.

The latency sweep (`eval --num-envs N --action-delays 0,0.005,0.01,0.02,0.025`, DESIGN.md §7.9) gives env i the action delay of
cell i mod C (BatchedHumanoidEnv.set_action_delay) after the reset, before the first step and outside the graph.  Autoreset is off,
so nothing redraws it; the graph body is unchanged but for its step, which is the delayed one.  Each cell's statistics are
summarize()'s over its envs.

The payload sweep (`eval --num-envs N --payloads 0,5,10,15,20 [--payload-at x,y,z]`, DESIGN.md §7.10) gives env i the payload mass
of cell i mod C, all at the one point --payload-at (BatchedHumanoidEnv.set_payload), after the reset, before the first step and
outside the graph.  Autoreset is off, so nothing redraws it; the graph body is unchanged but for its step, which is the payload
one.  Each cell's statistics are summarize()'s over its envs.

The motor-strength sweep (`eval --num-envs N --motor-strengths 0,0.5,0.8,1,1.2 [--motor-joints R_KNEE,L_KNEE]`, DESIGN.md §7.11)
gives env i the factor of cell i mod C on the named joints and 1 on the others (BatchedHumanoidEnv.set_motor_strength), after the
reset, before the first step and outside the graph.  Autoreset is off, so nothing redraws them; the graph body is unchanged but for
its step, which is the motor one.  Each cell's statistics are summarize()'s over its envs.

The sensor sweep (`eval --num-envs N --sensor-errors roll:-0.05,0.05 pitch:0.1 encoder:0.03 noise:1,2`, DESIGN.md §7.12) gives
env i the sensor errors of cell i mod C (BatchedHumanoidEnv.set_sensor_errors) before the reset, because the first observation
is a sensor reading too: a roll or pitch cell sets that IMU offset, an encoder cell every motor-position offset, a noise cell the
noise multiplier, and every other word of the cell is 0.  Autoreset is off, so nothing redraws them; the graph body is unchanged
but for the sensor pass after its step.  Cells are (kind, value) pairs, so each cell's statistics are summarize()'s over the envs
of its index.
"""
from __future__ import annotations

import json

import numpy as np
import torch

from ..envs.batched_env import FOOTSTEP_MODES

# the accumulator words of csrc/sim_core.h (EV_*), per env
LEN, RET, DONE, TERMS, TRACK, REACHED, SEQLEN, WORDS = 0, 1, 2, 3, 13, 25, 26, 27
MODES = ("STANDING", "INPLACE", "FORWARD")     # WalkingTask's modes, in the order of the kernel's mode word
TRACKED = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1")   # h1: its StandingTask, against zero references
# the command sweep's signed-velocity words of csrc/sim_core.h (CMD_*), per env
C_LEN, C_VF, C_VL, C_WZ, C_DONE, C_WORDS = 0, 1, 2, 3, 4, 5


def push_grid(n: int, speeds, directions: int):
    """Per env (speed m/s, direction in degrees) of the sweep: env i is cell c = i mod (S D), with speed speeds[c // D] and
    direction 360 (c mod D) / D in its heading frame (0 forward, 90 towards the robot's left)."""
    c = np.arange(n) % (len(speeds) * directions)
    return np.asarray(speeds, dtype=np.float64)[c // directions], 360.0 * (c % directions) / directions


def push_vectors(speed: np.ndarray, dir_deg: np.ndarray) -> np.ndarray:
    """[N, 2] heading-frame velocity changes (dx, dy) of the sweep."""
    th = np.deg2rad(dir_deg)
    return np.stack((speed * np.cos(th), speed * np.sin(th)), axis=1)


def command_grid(n: int, cells):
    """Per env (mode index, value) of the command sweep: env i is in cell i mod C of cells = [(mode name, value), ...]."""
    c = np.arange(n) % len(cells)
    return np.asarray([MODES.index(m) for m, _ in cells], dtype=np.int32)[c], np.asarray([v for _, v in cells], dtype=np.float64)[c]


def command_refs(mode: np.ndarray, value: np.ndarray) -> np.ndarray:
    """[N, 3] references (yaw_rate, vx, vy) of the sweep: FORWARD value -> (0, value, 0), INPLACE value -> (value, 0, 0), STANDING
    -> (0, 0, 0)."""
    ref = np.zeros((len(mode), 3))
    ref[mode == MODES.index("FORWARD"), 1] = value[mode == MODES.index("FORWARD")]
    ref[mode == MODES.index("INPLACE"), 0] = value[mode == MODES.index("INPLACE")]
    return ref


def footstep_grid(n: int, cells):
    """Per env (plan type index, value) of the footstep sweep: env i is in cell i mod C of cells = [(plan type name, value), ...]."""
    c = np.arange(n) % len(cells)
    return (np.asarray([FOOTSTEP_MODES.index(m) for m, _ in cells], dtype=np.int32)[c],
            np.asarray([v for _, v in cells], dtype=np.float64)[c])


def delay_grid(n: int, delays) -> np.ndarray:
    """Per env the action delay in seconds of the latency sweep: env i is in cell i mod C of delays."""
    return np.asarray(delays, dtype=np.float64)[np.arange(n) % len(delays)]


def payload_grid(n: int, masses) -> np.ndarray:
    """Per env the payload mass in kg of the payload sweep: env i is in cell i mod C of masses."""
    return np.asarray(masses, dtype=np.float64)[np.arange(n) % len(masses)]


def motor_grid(n: int, factors) -> np.ndarray:
    """Per env the strength factor of the motor-strength sweep: env i is in cell i mod C of factors."""
    return np.asarray(factors, dtype=np.float64)[np.arange(n) % len(factors)]


SENSOR_KINDS = ("roll", "pitch", "encoder", "noise")


def sensor_grid(n: int, cells, nu: int) -> tuple[np.ndarray, np.ndarray, np.ndarray]:
    """The sensor sweep's rows: per env its cell index (env i is in cell i mod C of cells = [(kind, value), ...]), noise
    multiplier [n] and offsets [n, 5 + nu] (roll, pitch, gyro x, y, z, the motor positions), 0 but for the cell's one kind."""
    m, b = np.zeros(len(cells)), np.zeros((len(cells), 5 + nu))
    for c, (kind, v) in enumerate(cells):
        if kind == "roll":
            b[c, 0] = v
        elif kind == "pitch":
            b[c, 1] = v
        elif kind == "encoder":
            b[c, 5:] = v
        elif kind == "noise":
            m[c] = v
        else:
            raise ValueError(f"unknown sensor error kind {kind!r}; expected one of {', '.join(SENSOR_KINDS)}")
    idx = np.arange(n) % len(cells)
    return idx, m[idx], b[idx]


@torch.no_grad()
def rollout(env, policy, steps: int, graph: bool = True, push=None, command=None, footsteps=None, delay=None, payload=None,
            motor=None, sensor=None):
    """Reset `env` once and run `steps` control steps of the deterministic `policy` with autoreset off; returns the
    [N, WORDS] float64 device accumulators.  graph=False runs every step eagerly (the same launches, in the same order).
    push = (K, d): after control step K (1 <= K < steps) every env whose episode has not ended gets the heading-frame velocity
    change d [N, 2] (BatchedHumanoidEnv.push); with push=None nothing but the control steps is launched.
    command = (mode [N], ref [N, 3]): held commands (BatchedHumanoidEnv.set_command) applied after the reset, and every step also
    adds to the [N, C_WORDS] signed-velocity records; then the return is (accumulators, signed-velocity records).
    footsteps = (mode [N], value [N]): the reset is BatchedHumanoidEnv.reset_footsteps with these plans instead of reset().
    delay = seconds [N]: action delays (BatchedHumanoidEnv.set_action_delay) set after the reset.
    payload = (mass [N], offset (x, y, z)): payloads (BatchedHumanoidEnv.set_payload) set after the reset.
    motor = strengths [N, act_dim]: motor strengths (BatchedHumanoidEnv.set_motor_strength) set after the reset.
    sensor = (noise [N], bias [N, 5 + act_dim]): sensor errors (BatchedHumanoidEnv.set_sensor_errors) set before the reset."""
    if env.eval_words() != WORDS:
        raise RuntimeError(f"the library's evaluation record has {env.eval_words()} words, this module knows {WORDS}")
    if command is not None and env.command_words() != C_WORDS:
        raise RuntimeError(f"the library's command record has {env.command_words()} words, this module knows {C_WORDS}")
    acc = torch.zeros(env.num_envs, WORDS, dtype=torch.float64, device=env.device)
    cacc = torch.zeros(env.num_envs, C_WORDS, dtype=torch.float64, device=env.device) if command is not None else None
    if sensor is not None:
        env.set_sensor_errors(*sensor)
    if footsteps is not None:
        env.reset_footsteps(*footsteps)
    else:
        env.reset()
    if command is not None:
        env.set_command(*command)
    if delay is not None:
        env.set_action_delay(delay)
    if payload is not None:
        env.set_payload(*payload)
    if motor is not None:
        env.set_motor_strength(motor)
    state = env.obs.float().clone()
    push_k, push_d = push if push is not None else (None, None)
    if push is not None:
        if not 1 <= push_k < steps:
            raise ValueError(f"the push must come after control step 1..{steps - 1}, got {push_k}")
        push_d = torch.as_tensor(push_d).to(device=env.device, dtype=env.dtype).reshape(env.num_envs, 2).contiguous()

    def after(t):     # after control step t (1-based)
        if t == push_k:
            env.push(torch.where(acc[:, DONE:DONE + 1] != 0, torch.zeros_like(push_d), push_d))   # the fallen stay where they lie

    def body():
        a = policy(state, deterministic=True)
        obs, _, _, _ = env.step(a if env.dtype == torch.float32 else a.double(), autoreset=False)
        env.eval_accumulate(acc)
        if cacc is not None:
            env.command_accumulate(cacc)
        state.copy_(obs.float())

    out = acc if command is None else (acc, cacc)
    if not graph or steps <= 1:
        for t in range(steps):
            body()
            after(t + 1)
        return out
    cur = torch.cuda.current_stream(env.device)
    s = torch.cuda.Stream(device=env.device)
    s.wait_stream(cur)
    with torch.cuda.stream(s):
        body()     # the first step, eagerly: it also warms up the actor's GEMMs before the capture
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=s):
            body()     # capturing does not execute: the replays run steps 2..steps
        after(1)
        env.bind()
        for t in range(2, steps + 1):
            g.replay()
            after(t)
    cur.wait_stream(s)
    return out


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


def push_summary(acc: np.ndarray, speed: np.ndarray, dir_deg: np.ndarray, speeds, directions: int, push_at: float,
                 push_step: int) -> dict:
    """The sweep's outcome per cell (speed x direction) and per speed: n, fell before the push, alive at the push, survived to the
    horizon, and survival = survived / alive at the push (None when no env was alive)."""
    fell = acc[:, DONE] != 0
    before = fell & (acc[:, LEN] <= push_step)
    surv = lambda s, a: float(s / a) if a else None
    cells = []
    for si, v in enumerate(speeds):
        for k in range(directions):
            m = (speed == float(v)) & (dir_deg == 360.0 * k / directions)
            n, b, ok = int(m.sum()), int((m & before).sum()), int((m & ~fell).sum())
            cells.append(dict(speed=float(v), direction_deg=360.0 * k / directions, n=n, fell_before_push=b, alive_at_push=n - b,
                              survived=ok, survival=surv(ok, n - b)))
    per_speed = []
    for v in speeds:
        cs = [c for c in cells if c["speed"] == float(v)]
        alive, ok = sum(c["alive_at_push"] for c in cs), sum(c["survived"] for c in cs)
        per_speed.append(dict(speed=float(v), alive_at_push=alive, survived=ok, survival=surv(ok, alive)))
    return dict(speeds=[float(v) for v in speeds], directions_deg=[360.0 * k / directions for k in range(directions)],
                push_at=float(push_at), push_step=int(push_step), cells=cells, per_speed=per_speed)


def format_push_table(p: dict) -> str:
    f = lambda v: "    -" if v is None else f"{v:5.3f}"
    lines = [f"  push recovery: one push after control step {p['push_step']} ({p['push_at']} s); survival = survived to the horizon / "
             "alive at the push",
             "    speed m/s \\ direction deg " + "".join(f"{d:>7.0f}" for d in p["directions_deg"]) + "    all"]
    nd = len(p["directions_deg"])
    for i, ps in enumerate(p["per_speed"]):
        row = p["cells"][i * nd:(i + 1) * nd]
        lines.append(f"    {ps['speed']:>27.3f} " + "".join(f"  {f(c['survival'])}" for c in row) + f"  {f(ps['survival'])}")
    return "\n".join(lines)


def command_summary(acc: np.ndarray, cacc: np.ndarray, mode: np.ndarray, value: np.ndarray, cells) -> dict:
    """The command sweep's outcome per cell: n, fall fraction, mean episode length; the achieved v_fwd, v_lat and w_z as the mean
    and standard deviation over the cell's envs of each env's per-step mean; and the §7.4 tracking errors of the held mode, the
    cell's error sums over its tracked steps."""
    v = cacc[:, [C_VF, C_VL, C_WZ]] / cacc[:, C_LEN:C_LEN + 1]
    out = []
    for name, val in cells:
        m_idx = MODES.index(name)
        m = (mode == m_idx) & (value == float(val))
        ref = command_refs(np.array([m_idx]), np.array([float(val)]))[0]
        t = acc[m, TRACK + 4 * m_idx:TRACK + 4 * m_idx + 4].sum(0)
        achieved = {k: dict(mean=float(v[m, j].mean()), std=float(v[m, j].std())) for j, k in enumerate(("v_fwd", "v_lat", "yaw_rate"))}
        out.append(dict(mode=name, value=float(val), ref=dict(yaw_rate=float(ref[0]), vx=float(ref[1]), vy=float(ref[2])), n=int(m.sum()),
                        fall_fraction=float((acc[m, DONE] != 0).mean()), mean_length=float(acc[m, LEN].mean()), achieved=achieved,
                        tracking=dict(steps=int(t[0]), vx_error=float(t[1] / t[0]), vy_error=float(t[2] / t[0]),
                                      yaw_rate_error=float(t[3] / t[0]))))
    return dict(cells=out)


def format_command_table(c: dict) -> str:
    f = lambda a: f"{a['mean']:>7.3f} +- {a['std']:.3f}"
    lines = ["  held commands: achieved = mean over the cell's envs of each env's per-step mean (+- std across envs)",
             "    command              n   fell  length        v_fwd m/s         v_lat m/s         w_z rad/s"
             "   |v_fwd-vx| |v_lat-vy| |w_z-yaw|"]
    for x in c["cells"]:
        a, t = x["achieved"], x["tracking"]
        name = x["mode"].lower() + ("" if x["mode"] == "STANDING" else f" {x['value']:g}")
        lines.append(f"    {name:<16s} {x['n']:>5d} {x['fall_fraction']:6.3f} {x['mean_length']:7.1f}  {f(a['v_fwd'])}  {f(a['v_lat'])}  "
                     f"{f(a['yaw_rate'])}  {t['vx_error']:10.4f} {t['vy_error']:10.4f} {t['yaw_rate_error']:9.4f}")
    return "\n".join(lines)


def footstep_label(name: str, value: float) -> str:
    """The cell as the command line writes it: forward:0.1, lateral:left, curved:17, curved (drawn), standing, backward."""
    if name == "LATERAL":
        return "lateral:" + ("left" if value > 0 else "right")
    if name == "FORWARD" or (name == "CURVED" and value >= 0):
        return f"{name.lower()}:{value:g}"
    return name.lower()


def footstep_summary(acc: np.ndarray, mode: np.ndarray, value: np.ndarray, cells) -> dict:
    """The footstep sweep's outcome per cell: n, fall fraction, mean episode length, mean footsteps reached and mean sequence
    length, completed fraction (reached >= sequence length - 1, as summarize counts it) and the mean return."""
    out = []
    for name, val in cells:
        m = (mode == FOOTSTEP_MODES.index(name)) & (value == float(val))
        reached, seq_len = acc[m, REACHED], acc[m, SEQLEN]
        out.append(dict(mode=name, value=float(val), label=footstep_label(name, float(val)), n=int(m.sum()),
                        fall_fraction=float((acc[m, DONE] != 0).mean()), mean_length=float(acc[m, LEN].mean()),
                        mean_reached=float(reached.mean()), mean_sequence_length=float(seq_len.mean()),
                        completed_fraction=float((reached >= seq_len - 1).mean()), return_mean=float(acc[m, RET].mean())))
    return dict(cells=out)


def format_footstep_table(f: dict) -> str:
    lines = ["  chosen footstep plans: reached = mean footsteps reached of the mean sequence length",
             "    plan                 n   fell  length     reached  completed    return"]
    for x in f["cells"]:
        lines.append(f"    {x['label']:<16s} {x['n']:>5d} {x['fall_fraction']:6.3f} {x['mean_length']:7.1f}  "
                     f"{x['mean_reached']:5.2f}/{x['mean_sequence_length']:<5.2f} {x['completed_fraction']:8.3f} {x['return_mean']:9.3f}")
    return "\n".join(lines)


def _cell_summary(acc: np.ndarray, per_env: np.ndarray, values, key: str, env_name: str, reward_names) -> list:
    """One sweep's outcome per cell: the cell's value under `key`, n, and summarize()'s fall fraction, episode length, return,
    per-mode tracking errors (walking tasks) and footsteps reached and completed (jvrc_step) over the envs whose per_env value
    is the cell's."""
    out = []
    for v in values:
        s = summarize(acc[per_env == float(v)], env_name, reward_names)
        cell = {key: float(v), "n": s["num_envs"], "fall_fraction": s["fall_fraction"], "mean_length": s["length"]["mean"],
                "return_mean": s["return"]["mean"]}
        cell.update({k: s[k] for k in ("tracking", "footsteps") if k in s})
        out.append(cell)
    return out


def _format_cells(d: dict, title: str, head: str, value) -> str:
    """The table of a sweep's cells: title, then per cell `value(cell)` followed by _cell_summary's statistics."""
    f = lambda v: "      -" if v is None else f"{v:7.4f}"
    lines = [f"  {title}: per cell the fall fraction, mean episode length and return"
             + ("; |v_fwd - vx_ref| per tracked mode" if "tracking" in d["cells"][0] else "")
             + ("; footsteps reached and sequences completed" if "footsteps" in d["cells"][0] else "")]
    head = f"    {head}      n   fell  length    return"
    if "tracking" in d["cells"][0]:
        head += "".join(f"  {m:>9s}" for m in d["cells"][0]["tracking"])
    if "footsteps" in d["cells"][0]:
        head += "     reached  completed"
    lines.append(head)
    for x in d["cells"]:
        row = f"    {value(x)} {x['n']:>6d} {x['fall_fraction']:6.3f} {x['mean_length']:7.1f} {x['return_mean']:9.3f}"
        if "tracking" in x:
            row += "".join(f"    {f(t['vx_error'])}" for t in x["tracking"].values())
        if "footsteps" in x:
            fs = x["footsteps"]
            row += f"  {fs['mean_reached']:5.2f}/{fs['mean_sequence_length']:<5.2f} {fs['completed_fraction']:8.3f}"
        lines.append(row)
    return "\n".join(lines)


def delay_summary(acc: np.ndarray, delay: np.ndarray, delays, env_name: str, reward_names) -> dict:
    """The latency sweep's outcome per cell: the delay in seconds, n, and summarize()'s fall fraction, episode length, return,
    per-mode tracking errors (walking tasks) and footsteps reached and completed (jvrc_step) over the cell's envs."""
    return dict(delays=[float(d) for d in delays], cells=_cell_summary(acc, delay, delays, "delay", env_name, reward_names))


def format_delay_table(d: dict) -> str:
    return _format_cells(d, "action delays", "delay ms", lambda x: f"{1000 * x['delay']:8.1f}")


def payload_summary(acc: np.ndarray, mass: np.ndarray, masses, at, env_name: str, reward_names) -> dict:
    """The payload sweep's outcome per cell: the payload mass in kg, n, and summarize()'s fall fraction, episode length, return,
    per-mode tracking errors (walking tasks) and footsteps reached and completed (jvrc_step) over the cell's envs; `at` is the
    payload's point, which every cell shares."""
    return dict(masses=[float(m) for m in masses], at=[float(v) for v in at],
                cells=_cell_summary(acc, mass, masses, "mass", env_name, reward_names))


def format_payload_table(d: dict) -> str:
    at = ", ".join(f"{v:g}" for v in d["at"])
    return _format_cells(d, f"payloads at ({at}) m", " mass kg", lambda x: f"{x['mass']:8.2f}")


def motor_summary(acc: np.ndarray, factor: np.ndarray, factors, joints, env_name: str, reward_names) -> dict:
    """The motor-strength sweep's outcome per cell: the strength factor, n, and summarize()'s fall fraction, episode length,
    return, per-mode tracking errors (walking tasks) and footsteps reached and completed (jvrc_step) over the cell's envs; `joints`
    are the joints that carry the factor, which every cell shares."""
    return dict(factors=[float(f) for f in factors], joints=list(joints),
                cells=_cell_summary(acc, factor, factors, "factor", env_name, reward_names))


def format_motor_table(d: dict) -> str:
    return _format_cells(d, f"motor strengths on {', '.join(d['joints'])}", "  factor", lambda x: f"{x['factor']:8.3f}")


def sensor_summary(acc: np.ndarray, cell: np.ndarray, cells, env_name: str, reward_names) -> dict:
    """The sensor sweep's outcome per cell: its kind and value, n, and summarize()'s fall fraction, episode length, return,
    per-mode tracking errors (walking tasks) and footsteps reached and completed (jvrc_step) over the envs of the cell's index."""
    out = _cell_summary(acc, cell, range(len(cells)), "cell", env_name, reward_names)
    for x, (kind, v) in zip(out, cells):
        x["cell"] = int(x["cell"])
        x.update(kind=kind, value=float(v))
    return dict(cells=out)


def format_sensor_table(d: dict) -> str:
    return _format_cells(d, "sensor errors", "   kind   value", lambda x: f"{x['kind']:>7s} {x['value']:7.3f}")


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


def evaluate_batched(policy, env, out_report=None, meta: dict | None = None, push: dict | None = None, commands=None,
                     footsteps=None, delays=None, payloads=None, motor=None, sensor=None) -> dict:
    """Roll `policy` out on every environment of `env` for env.max_traj_len control steps, print the table and, with
    out_report, write the JSON report (meta + summary + per-env arrays).  push = dict(speeds, directions, push_at): the
    push-recovery sweep, with its table and `summary.push`.  commands = [(mode name, value), ...]: the command-tracking sweep
    (env i holds the command of cell i mod len(commands)), with its table and `summary.commands`.  footsteps = [(plan type name,
    value), ...]: the footstep sweep (env i resets with the plan of cell i mod len(footsteps)), with its table and
    `summary.footsteps_sweep`.  delays = [seconds, ...]: the latency sweep (env i has the action delay of cell i mod len(delays)),
    with its table and `summary.delay`.  payloads = dict(masses=[kg, ...], at=(x, y, z)): the payload sweep (env i carries the
    mass of cell i mod len(masses) at `at`), with its table and `summary.payload`.  motor = dict(factors=[...], joints=[names],
    mask=[bool per joint]): the motor-strength sweep (env i's masked joints get the factor of cell i mod len(factors), the others 1),
    with its table and `summary.motor_strength`.  sensor = [(kind, value), ...]: the sensor sweep (env i observes with the
    errors of cell i mod len(sensor), sensor_grid), with its table and `summary.sensor`.  Returns the report."""
    if sum(x is not None for x in (push, commands, footsteps, delays, payloads, motor, sensor)) > 1:
        raise ValueError("the push, command, footstep, latency, payload, motor-strength and sensor sweeps are separate evaluations")
    sweep = held = plans = delay = load = None
    if push is not None:
        k = int(round(push["push_at"] / env.dt))
        speed, dir_deg = push_grid(env.num_envs, push["speeds"], push["directions"])
        sweep = (k, push_vectors(speed, dir_deg))
    if commands is not None:
        cmd_mode, cmd_value = command_grid(env.num_envs, commands)
        held = (cmd_mode, command_refs(cmd_mode, cmd_value))
    if footsteps is not None:
        fs_mode, fs_value = footstep_grid(env.num_envs, footsteps)
        plans = (fs_mode, fs_value)
    if delays is not None:
        delay = delay_grid(env.num_envs, delays)
    if payloads is not None:
        load = payload_grid(env.num_envs, payloads["masses"])
    strength = factor = None
    if motor is not None:
        factor = motor_grid(env.num_envs, motor["factors"])
        strength = np.where(np.asarray(motor["mask"], dtype=bool)[None, :], factor[:, None], 1.0)
    rows = cell = None
    if sensor is not None:
        cell, noise, bias = sensor_grid(env.num_envs, sensor, env.act_dim)
        rows = (noise, bias)
    out = rollout(env, policy, env.max_traj_len, push=sweep, command=held, footsteps=plans, delay=delay,
                  payload=None if load is None else (load, payloads["at"]), motor=strength, sensor=rows)
    acc, cacc = (out[0].cpu().numpy(), out[1].cpu().numpy()) if commands is not None else (out.cpu().numpy(), None)
    summary = summarize(acc, env.model_name, env.reward_names)
    pe = per_env(acc, env.model_name, env.reward_names)
    print(format_table(summary, env.max_traj_len))
    if push is not None:
        summary["push"] = push_summary(acc, speed, dir_deg, push["speeds"], push["directions"], push["push_at"], k)
        pe.update(push_speed=speed.tolist(), push_dir_deg=dir_deg.tolist())
        print(format_push_table(summary["push"]))
    if commands is not None:
        summary["commands"] = command_summary(acc, cacc, cmd_mode, cmd_value, commands)
        pe.update(command_mode=[MODES[m] for m in cmd_mode], command_value=cmd_value.tolist(),
                  command_steps=cacc[:, C_LEN].astype(int).tolist(), v_fwd_sum=cacc[:, C_VF].tolist(),
                  v_lat_sum=cacc[:, C_VL].tolist(), yaw_rate_sum=cacc[:, C_WZ].tolist())
        print(format_command_table(summary["commands"]))
    if footsteps is not None:
        summary["footsteps_sweep"] = footstep_summary(acc, fs_mode, fs_value, footsteps)
        pe.update(footstep_mode=[FOOTSTEP_MODES[m] for m in fs_mode], footstep_value=fs_value.tolist())
        print(format_footstep_table(summary["footsteps_sweep"]))
    if delays is not None:
        summary["delay"] = delay_summary(acc, delay, delays, env.model_name, env.reward_names)
        pe.update(action_delay=delay.tolist())
        print(format_delay_table(summary["delay"]))
    if payloads is not None:
        summary["payload"] = payload_summary(acc, load, payloads["masses"], payloads["at"], env.model_name, env.reward_names)
        pe.update(payload_mass=load.tolist())
        print(format_payload_table(summary["payload"]))
    if motor is not None:
        summary["motor_strength"] = motor_summary(acc, factor, motor["factors"], motor["joints"], env.model_name, env.reward_names)
        pe.update(motor_strength=factor.tolist())
        print(format_motor_table(summary["motor_strength"]))
    if sensor is not None:
        summary["sensor"] = sensor_summary(acc, cell, sensor, env.model_name, env.reward_names)
        pe.update(sensor_cell=cell.tolist())
        print(format_sensor_table(summary["sensor"]))
    report = dict(meta or {}, env=env.model_name, precision=env.precision, seed=env.seed, num_envs=env.num_envs,
                  max_traj_len=env.max_traj_len, summary=summary, per_env=pe)
    if out_report is not None:
        with open(out_report, "w") as f:
            json.dump(report, f, indent=1)
        print(f"Wrote {out_report}")
    return report
