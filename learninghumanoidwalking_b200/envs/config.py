"""Per-env YAML configuration (`partial(Env, path_to_yaml)`, run_experiment.py:115; envs/jvrc/configs/base.yaml,
envs/h1/configs/base.yaml; envs/common/config_builder.py): a user YAML is overlaid on the `cfg` block of the compiled model
before the constants are packed for the device.  Everything the reference reads from the YAML at ENV level is honoured — time
steps, PD gains, action smoothing, nominal pose, task timing / goal height, noise / perturbation / randomisation blocks.  Keys
that change the MJCF the reference would generate (`reduced_xml`, `ctrllimited`, `jointlimited`) cannot be applied to an
already compiled model: a value different from the compiled one is an error that names tools/compile_model.py."""
from __future__ import annotations

import copy
import math

import numpy as np

_STRUCTURAL = {"reduced_xml": True, "ctrllimited": False, "jointlimited": False}   # what model/h1.json was compiled with
_IGNORED = ("xml_export_path",)                                                    # where the reference caches generated XML


def load_yaml(path) -> dict:
    import yaml
    with open(path) as f:
        return yaml.safe_load(f) or {}


def apply_config(mj: dict, user: dict) -> dict:
    """A deep copy of the compiled model `mj` with `user` (a parsed YAML) applied; raises ValueError on what cannot be honoured."""
    mj = copy.deepcopy(mj)
    c = mj["cfg"]
    h1 = mj["name"] in ("h1", "h1_walk")     # the H1 robot: its MJCF keys, pose in radians, noise / push / randomisation blocks
    stand = mj["name"] == "h1"               # the standing task: no gait clock, no task block
    user = dict(user)
    for k in _IGNORED:
        user.pop(k, None)
    for k, compiled in _STRUCTURAL.items():
        if k in user and bool(user.pop(k)) != compiled and h1:
            raise ValueError(f"YAML key {k!r} changes the generated MJCF; recompile the model constants with tools/compile_model.py")
    if "sim_dt" in user or "control_dt" in user:
        sim_dt, control_dt = float(user.pop("sim_dt", c["sim_dt"])), float(user.pop("control_dt", c["control_dt"]))
        if round(control_dt % sim_dt, 6) != 0 and round(sim_dt - control_dt % sim_dt, 6) != 0:     # robots/robot_base.py:36-38
            raise ValueError("Control dt should be an integer multiple of Simulation dt.")
        c["sim_dt"], c["control_dt"], c["frame_skip"] = sim_dt, control_dt, int(round(control_dt / sim_dt))
        mj["opt"]["timestep"] = sim_dt
    if "obs_history_len" in user:
        if int(user.pop("obs_history_len")) != 1:
            raise ValueError("obs_history_len != 1: the device environments keep no observation history (every reference config uses 1)")
    if "action_smoothing" in user:
        c["action_smoothing"] = float(user.pop("action_smoothing"))
    nu = len(c["kp"])
    for k in ("kp", "kd"):
        if k in user:
            v = [float(x) for x in user.pop(k)]
            if len(v) != nu:
                raise ValueError(f"{k} needs {nu} entries")
            c[k] = v
    if "pdgains" in user:       # envs/h1/configs/base.yaml: {joint name: [kp, kd]}; only the actuated leg joints matter
        pd = user.pop("pdgains")
        names = [lk["joint"]["name"] for lk in mj["links"][1:]]
        for i, jn in enumerate(names):
            if jn in pd:
                c["kp"][i], c["kd"][i] = float(pd[jn][0]), float(pd[jn][1])
    if "half_sitting_pose" in user:
        pose = [float(x) for x in user.pop("half_sitting_pose")]
        if len(pose) != nu:
            raise ValueError(f"half_sitting_pose needs {nu} entries")
        if h1:          # radians, envs/h1/h1_base.py
            c["half_sitting_pose"] = pose
            c["nominal_qpos"] = c["nominal_qpos"][:7] + pose
        else:           # degrees, envs/jvrc/jvrc_base.py:55-60
            c["half_sitting_pose_deg"] = pose
            c["nominal_qpos"] = c["nominal_qpos"][:7] + [math.radians(x) for x in pose]
    if "task" in user:
        t = dict(user.pop("task"))
        if stand:
            raise ValueError("the H1 standing task has no YAML task block")
        for k in ("goal_height", "total_duration", "swing_duration", "stance_duration"):
            if k in t:
                c["task"][k] = float(t.pop(k))
        if t:
            raise ValueError(f"unknown task keys {sorted(t)}")
    if "init_noise" in user:
        c["init_noise_deg"] = float(user.pop("init_noise"))
    for blk in ("observation_noise", "perturbation", "dynamics_randomization"):
        if blk in user:
            if not h1:
                raise ValueError(f"{blk}: only the H1 environments implement it (as in the reference, envs/jvrc has none)")
            new = user.pop(blk)
            if blk == "observation_noise" and new.get("type", "uniform") != "uniform":
                raise ValueError("observation_noise.type: only 'uniform' is implemented on the device")
            if blk == "perturbation" and list(new.get("bodies", c[blk]["bodies"])) != list(c[blk]["bodies"]):
                raise ValueError("perturbation.bodies: the kernel applies wrenches to (pelvis, torso_link) only")
            merged = copy.deepcopy(c[blk])
            for k, v in new.items():
                if isinstance(v, dict):
                    merged[k] = {**merged.get(k, {}), **v}
                else:
                    merged[k] = v
            c[blk] = merged
    if user:
        raise ValueError(f"YAML keys this build does not know: {sorted(user)}")
    if not stand:
        period = int(math.floor(2 * c["task"]["total_duration"] * (1.0 / c["control_dt"])))      # tasks/walking_task.py:201
        if not 2 <= period <= 96:
            raise ValueError(f"gait period {period} control steps: the kernel's clock table holds at most 96 (csrc/sim_core.h MAXPERIOD)")
    assert len(c["nominal_qpos"]) == 7 + nu and np.isfinite(c["nominal_qpos"]).all()
    return mj
