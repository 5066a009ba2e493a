"""Load a compiled robot model (tools/compile_model.py output) and pack it for the C-ABI.

The flat float64 layout below is what lhw_sim_create() consumes (csrc/model_pack.h:fill_model).
"""
from __future__ import annotations

import json
import os

import numpy as np

from ..tasks.gait_clock import phase_clock_table

_HERE = os.path.dirname(os.path.abspath(__file__))


def load_model(name: str = "jvrc_walk") -> dict:
    with open(os.path.join(_HERE, name + ".json")) as f:
        return json.load(f)


def pack_model(mj: dict, tolerance: float | None = None, max_iter: int | None = None, kp=None, kd=None,
               self_collision: bool = True, observation_noise: bool = True, domain_randomization: bool = True,
               init_noise: bool = True, pd_gain_randomization: float = 0.0,
               iteration_count: float = float("inf")) -> np.ndarray:
    links = mj["links"]
    nl = len(links)
    assert (nl - 1) % 2 == 0, "expected a free root + two equal serial chains"
    nj = (nl - 1) // 2
    for c in range(2):
        for k in range(nj):
            i = 1 + c * nj + k
            assert links[i]["parent"] == (0 if k == 0 else i - 1), "links must be ordered root, chain0, chain1"
    assert {mj["rfoot_link"], mj["lfoot_link"]} == {nj, 2 * nj}
    # which chain ends in the right foot is compiled into the kernel (csrc/sim_core.h Cfg::RFOOT): chain 0 for JVRC-1, 1 for H1
    assert mj["rfoot_link"] == (2 * nj if mj["name"] in ("h1", "h1_walk") else nj)
    h1 = mj["name"] in ("h1", "h1_walk")  # the Unitree H1 robot: capsule feet, noise, randomisation, pushes
    stand = mj["name"] == "h1"          # Unitree H1 + StandingTask (csrc/sim_core.h Cfg<5, 0>)
    h1_walk = mj["name"] == "h1_walk"   # Unitree H1 + WalkingTask (csrc/sim_core.h Cfg<5, 3>)
    step = mj["name"] == "jvrc_step"    # JVRC-1 + SteppingTask (csrc/sim_core.h Cfg<6, 1>)
    terrain = mj.get("terrain")         # JVRC-1 + WalkingTask on terraces (extension; csrc/sim_core.h Cfg<6, 2>)
    b: list[float] = [nj + (100 if step else 200 if terrain else 300 if h1_walk else 0)]
    for lk in links:
        b += lk["pos"]
        b += list(np.asarray(lk["rot"], dtype=float).reshape(-1))
        b += lk["joint"].get("axis", [0.0, 0.0, 0.0])
        b.append(lk["mass"])
        b += lk["com"]
        b += lk["inertia"]
    nv = 6 + 2 * nj
    for d in range(nv):
        if d < 6:
            b += [0.0, 0.0, 0.0, 0.0, mj["dof_invweight0"][d]]
        else:
            j = links[d - 5]["joint"]
            lo, hi = j["range"] if j.get("limited", True) else (-1e30, 1e30)
            b += [j["armature"], j["damping"], lo, hi, mj["dof_invweight0"][d]]
    assert [g["link"] for g in mj["geoms"]] == [nj, 2 * nj], "one ground-contact geom set per foot, chain order"
    for g in mj["geoms"]:
        assert g["type"] == ("spheres" if h1 else "box")
        b += g.get("pos", [0.0, 0.0, 0.0])
        b += g.get("size", [0.0, 0.0, 0.0])
        b.append(mj["link_invweight0"][g["link"]][0])
    o = mj["opt"]
    b.append(o["timestep"])
    b += o["gravity"]
    b += o["solref"]
    b += o["solimp"]
    b += [o["friction"][0], o["impratio"], mj["meaninertia"],
          o["tolerance"] if tolerance is None else tolerance, o["iterations"] if max_iter is None else max_iter]
    c = mj["cfg"]
    b += list(c["kp"] if kp is None else kp)
    b += list(c["kd"] if kd is None else kd)
    b += c["nominal_qpos"]
    b += [c["action_smoothing"], c["frame_skip"]]
    b += mj.get("head_in_root", [0.0, 0.0, 0.0])
    if stand:
        b += [mj["total_mass"], 0.98, 0]       # no gait clock (tasks/standing_task.py)
    else:
        t = c["task"]
        period, table = phase_clock_table(t["swing_duration"], t["stance_duration"], 0.1, "grounded",
                                          1.0 / c["control_dt"], total_duration=t["total_duration"])
        # get_robot_mass() = mj_getTotalmass: in jvrc_step it also counts the 20 static boxes (SURVEY Appendix C-3)
        b += [mj.get("stepping", {}).get("task_mass", mj["total_mass"]), t["goal_height"], period]
        b += list(table.reshape(-1))
    # self-collision capsule proxies (termination flag; tools/fit_collision_proxies.py)
    sc = mj.get("self_collision") if self_collision else None
    caps = sc["capsules"] if sc else []
    b.append(len(caps))
    for cap in caps:
        b += [cap["link"]] + list(cap["p0"]) + list(cap["p1"]) + [cap["radius"]]
    pairs = sc["pairs"] if sc else []
    b.append(len(pairs))
    for a_, b_ in pairs:
        b += [a_, b_]
    # task / robot variant tail
    if h1:
        ns = c["observation_noise"] if observation_noise else {"enabled": False}
        lvl = ns["multiplier"] if ns["enabled"] else 0.0
        scales = [lvl * ns["scales"][k] for k in ("root_orient", "root_ang_vel", "motor_pos", "motor_vel", "motor_tau")] \
            if ns["enabled"] else [0.0] * 5
        pert, dyn = c["perturbation"], c["dynamics_randomization"]
        b += ([0.6, 1.4] if h1_walk else [0.9, 1.4]) + scales   # tasks/walking_task.py:192-193, tasks/standing_task.py:124-125
        b += [int(dyn["interval"] / c["control_dt"]) if dyn["enable"] and domain_randomization else 0,
              int(pert["interval"] / c["control_dt"]) if pert["enable"] and domain_randomization else 0,
              pert["force_magnitude"], pert["torque_magnitude"],
              c["init_noise_deg"] * np.pi / 180 if init_noise else 0.0]
    elif step:
        b += [0.6, 1e30] + [0.0] * 5 + [0, 0, 0.0, 0.0, 0.0]  # tasks/stepping_task.py:254-257 (relative height, no upper bound)
    else:
        b += [0.6, 1.4] + [0.0] * 5 + [0, 0, 0.0, 0.0, 0.0]   # tasks/walking_task.py:192-193
    for g in mj["geoms"]:
        pts = g.get("points", [])
        b += [len(pts), g.get("radius", 0.0)]
        for pt in pts:
            b += pt
    rp = mj.get("root_parts")
    if rp:
        sym = lambda A: [A[0][0], A[1][1], A[2][2], A[0][1], A[0][2], A[1][2]]
        b += [rp["pelvis"]["mass"]] + rp["pelvis"]["com"] + sym(rp["pelvis"]["Ic"])
        b += [rp["rest"]["mass"]] + rp["rest"]["mc"] + sym(rp["rest"]["Io"])
        b += rp["torso_com"]
    else:
        b += [0.0] * 23
    b.append(float(pd_gain_randomization))     # RobotBase(pdrand_k) (robots/robot_base.py:5,43-47); 0 = off
    if terrain:
        b += terrain["strip_half"] + [terrain["side_tol"], terrain["pitch"], terrain["bump"], terrain["z_lo"], terrain["z_hi"],
                                      terrain["xy"], terrain["interval"]] + terrain["contact_solref"] + [1 if terrain.get("side_faces", True) else 0]
    if step:
        st = mj["stepping"]
        for site in mj["foot_sites"]:
            b += site
        b += st["slab_half"]
        b += [st["target_radius"], st["side_tol"], st["delay_frames"], curriculum_height(iteration_count),
              1 if st.get("slab_contacts_are_floor") else 0, 1 if st.get("side_faces", True) else 0]
        b.append(len(st["plans"]))
        for plan in st["plans"]:
            b.append(len(plan))
            for row in plan:
                b += row
    # assumption switches (model JSON "assumptions", SURVEY.md Appendix A warnings): bit 0 = explicit Euler
    b.append(float(assumption_flags(mj)))
    return np.asarray(b, dtype=np.float64)


def assumption_flags(mj: dict) -> int:
    """The switchable modelling assumptions of model/*.json ("assumptions": SURVEY.md Appendix A, the details of mj_step that
    could not be checked against MuJoCo here) as the flags word at the end of the packed model."""
    a = mj.get("assumptions", {})
    return 0 if a.get("implicit_damping", True) else 1


def curriculum_height(iteration_count: float) -> float:
    """SteppingTask.reset (tasks/stepping_task.py:312): h = clip((iteration_count - 3000) / 8000, 0, 1) * 0.1.
    `env.robot.iteration_count` is inf unless the trainer sets it (robots/robot_base.py:35, rl/workers/rollout_worker.py:95)."""
    return float(np.clip((iteration_count - 3000) / 8000, 0, 1) * 0.1)
