#!/usr/bin/env python3
"""Model compiler: reference MJCF -> packed constant block for the on-device simulator.

Runs in the build container only (it reads /root/reference, which does not exist on
the GPU box); its OUTPUT (learninghumanoidwalking_b200/model/*.json) is committed.

What it restates (never copies) from the reference:
  * envs/jvrc/gen_xml.py:58-164   the MJCF surgery the reference performs with dm_control
    (drop every joint except `root` + LEG_JOINTS, fix the arm pose through body eulers,
    keep only leg collision geoms, add one collision box per foot, wrap the floor plane in
    a body, export with precision=5 i.e. '%.5g' on every numeric attribute).
  * models/jvrc_mj_description/xml/jvrc1.xml  (tree, inertials, joint axes/ranges/armature,
    defaults: joint damping 0.2 + limited, option timestep/solver/cone).
  * envs/jvrc/configs/base.yaml   (kp/kd, half-sitting pose, task durations).
  * MuJoCo compile-time constants the runtime needs (SURVEY.md Appendix A.3):
    body_invweight0 / dof_invweight0 / stat.meaninertia at qpos0 (mj_setConst).

dm_control and mujoco are not installed, so the surgery is re-done with xml.etree and the
jointless bodies are welded into their nearest jointed ancestor ("link"): dynamics are
identical (no DoF between them), 45 inertial bodies -> 13 links.
"""
from __future__ import annotations

import argparse
import json
import os
import xml.etree.ElementTree as ET

import numpy as np
import yaml

REF = os.environ.get("LHW_REFERENCE", "/root/reference")

JVRC_LEG_JOINTS = [
    "R_HIP_P", "R_HIP_R", "R_HIP_Y", "R_KNEE", "R_ANKLE_R", "R_ANKLE_P",
    "L_HIP_P", "L_HIP_R", "L_HIP_Y", "L_KNEE", "L_ANKLE_R", "L_ANKLE_P",
]
# gen_xml.py:92-101 — arm pose fixed through body eulers (radians, xyz)
JVRC_ARM_EULER = {
    "R_SHOULDER_P_S": [0, -0.052, 0],
    "R_SHOULDER_R_S": [-0.17, 0, 0],
    "R_ELBOW_P_S": [0, -0.524, 0],
    "L_SHOULDER_P_S": [0, -0.052, 0],
    "L_SHOULDER_R_S": [0.17, 0, 0],
    "L_ELBOW_P_S": [0, -0.524, 0],
}
# gen_xml.py:104-111 — bodies whose collision meshes are kept (self-collision only)
JVRC_COLLISION_BODIES = ["R_HIP_R_S", "R_HIP_Y_S", "R_KNEE_S", "L_HIP_R_S", "L_HIP_Y_S", "L_KNEE_S"]


# the modelling assumptions SURVEY.md Appendix A could not check against MuJoCo, as switchable / traceable entries of every
# compiled model (tests/test_assumption_switches.py measures what each one is worth)
ASSUMPTIONS = {
 "_doc": "Details of mujoco.mj_step / the MJCF export that SURVEY.md Appendix A could only take from MuJoCo's documentation (the library is not installable here). Each is a value in THIS file, so the day a MuJoCo recording exists (tools/record_reference.py) a mismatch can be traced by flipping one entry; tests/test_assumption_switches.py measures how far each one moves a trajectory.",
 "implicit_damping": True,
 "implicit_damping_doc": "mj_Euler solves (M + h diag(damping)) qacc' = M qacc before integrating (A.1). False = explicit Euler.",
 "export_rounding_digits": 5,
 "export_rounding_doc": "every number of links / geoms / opt above is already rounded with '%.5g' (dm_control export_with_assets(precision=5), envs/jvrc/gen_xml.py:161); carried by the numbers themselves.",
 "contact_diagapprox_doc": "R_n = (1 - imp) / imp * link_invweight0[foot][0] * (1 + mu^2) (A.3); carried by link_invweight0 / dof_invweight0 (mj_setConst at qpos0, frozen).",
 "pyramid_regulariser_doc": "every pyramid edge: R = 2 mu^2 R_n / impratio (A.3); carried by opt.impratio (1).",
 "planebox_corners_doc": "mjc_PlaneBox keeps the first (at most) 4 corners below the plane on the plane side of the box centre, in corner-index order (A.5); at most 4 corners can qualify unless the box stands exactly on an edge, so the order cannot matter (tested).",
 "solref_solimp_doc": "contacts and limits use the global defaults opt.solref (0.02, 1) / opt.solimp (0.9, 0.95, 0.001, 0.5, 2): nothing in the reference's XML overrides them (A.0)."
}


def r5(x: float) -> float:
    """dm_control export_with_assets(precision=5) writes every number as '%.5g'."""
    return float("%.5g" % float(x))


def vec(s, n=None, default=None):
    if s is None:
        return None if default is None else np.array(default, dtype=float)
    v = np.array([r5(t) for t in s.split()], dtype=float)
    if n is not None:
        assert v.shape == (n,), (s, n)
    return v


def quat2mat(q):
    q = np.asarray(q, dtype=float)
    q = q / np.linalg.norm(q)
    w, x, y, z = q
    return np.array([
        [1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
        [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
        [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)],
    ])


def euler_xyz2mat(e):
    """MuJoCo eulerseq 'xyz' (intrinsic): R = Rx(e0) Ry(e1) Rz(e2)."""
    cx, sx = np.cos(e[0]), np.sin(e[0])
    cy, sy = np.cos(e[1]), np.sin(e[1])
    cz, sz = np.cos(e[2]), np.sin(e[2])
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]])
    Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    return Rx @ Ry @ Rz


def skew(v):
    return np.array([[0, -v[2], v[1]], [v[2], 0, -v[0]], [-v[1], v[0], 0]])


class Link:
    def __init__(self, name, parent, pos, rot):
        self.name = name
        self.parent = parent  # link index or -1
        self.pos = pos        # origin in parent-link frame
        self.rot = rot        # orientation in parent-link frame (3x3)
        self.joint = None     # dict(type, axis, armature, damping, range, name)
        self.mass = 0.0
        self.mc = np.zeros(3)         # sum m*c (link frame)
        self.Io = np.zeros((3, 3))    # inertia about link origin (link frame)
        self.members = {}     # xml body name -> (pos, rot) in link frame
        self.geoms = []

    def add_inertial(self, m, c, Ic):
        """Add a rigid piece: mass m, com c, inertia about its com Ic — all in link frame."""
        self.mass += m
        self.mc += m * c
        self.Io += Ic + m * (np.dot(c, c) * np.eye(3) - np.outer(c, c))

    def finalize(self):
        c = self.mc / self.mass
        Ic = self.Io - self.mass * (np.dot(c, c) * np.eye(3) - np.outer(c, c))
        return c, 0.5 * (Ic + Ic.T)


def compile_jvrc(boxes: bool = False):
    xml_dir = os.path.join(REF, "models/jvrc_mj_description/xml")
    root = ET.parse(os.path.join(xml_dir, "jvrc1.xml")).getroot()
    cfg = yaml.safe_load(open(os.path.join(REF, "envs/jvrc/configs/base.yaml")))

    opt = root.find("option").attrib
    timestep = r5(opt["timestep"])
    assert opt["solver"] == "Newton" and opt["cone"] == "pyramidal"
    jdef = root.find("default").find("joint").attrib
    joint_damping_default = r5(jdef["damping"])
    assert jdef["limited"] == "true"

    keep = set(JVRC_LEG_JOINTS)
    links: list[Link] = []

    def walk(body, link_idx, pos_in_link, rot_in_link):
        """body: xml element; (pos,rot) of this xml body's frame expressed in link link_idx."""
        name = body.attrib["name"]
        jel = body.find("joint")
        fj = body.find("freejoint")
        jointed = fj is not None or (jel is not None and jel.attrib["name"] in keep)
        if jointed:
            lk = Link(name, link_idx, pos_in_link, rot_in_link)
            if fj is not None:
                # <freejoint> takes no defaults: damping 0, armature 0 (MuJoCo XML reference)
                lk.joint = dict(type="free", name=fj.attrib["name"])
            else:
                lk.joint = dict(
                    type="hinge", name=jel.attrib["name"],
                    axis=vec(jel.attrib["axis"], 3),
                    armature=r5(jel.attrib.get("armature", 0)),
                    damping=r5(jel.attrib.get("damping", joint_damping_default)),
                    range=vec(jel.attrib["range"], 2),
                )
                assert np.allclose(vec(jel.attrib.get("pos", "0 0 0"), 3), 0)
            links.append(lk)
            link_idx = len(links) - 1
            pos_in_link, rot_in_link = np.zeros(3), np.eye(3)
        lk = links[link_idx]
        lk.members[name] = (pos_in_link.copy(), rot_in_link.copy())
        ine = body.find("inertial")
        m = r5(ine.attrib["mass"])
        ipos = vec(ine.attrib.get("pos", "0 0 0"), 3)
        iquat = vec(ine.attrib.get("quat", "1 0 0 0"), 4)
        diag = vec(ine.attrib["diaginertia"], 3)
        Ri = rot_in_link @ quat2mat(iquat)
        lk.add_inertial(m, pos_in_link + rot_in_link @ ipos, Ri @ np.diag(diag) @ Ri.T)
        for child in body.findall("body"):
            cpos = vec(child.attrib.get("pos", "0 0 0"), 3)
            crot = np.eye(3)
            if "quat" in child.attrib:
                crot = quat2mat(vec(child.attrib["quat"], 4))
            if child.attrib["name"] in JVRC_ARM_EULER:
                crot = euler_xyz2mat([r5(e) for e in JVRC_ARM_EULER[child.attrib["name"]]])
            walk(child, link_idx, pos_in_link + rot_in_link @ cpos, rot_in_link @ crot)

    pelvis = root.find("worldbody").find("body")
    assert pelvis.attrib["name"] == "PELVIS_S"
    qpos0_root = vec(pelvis.attrib["pos"], 3)
    walk(pelvis, -1, np.zeros(3), np.eye(3))

    # dof order = joint order in the XML depth-first traversal == LEG_JOINTS order (gen_xml.py:42-55)
    names = [lk.joint["name"] for lk in links[1:]]
    assert names == JVRC_LEG_JOINTS, names

    model = dict(name="jvrc_step" if boxes else "jvrc_walk")
    model["opt"] = dict(
        timestep=timestep, gravity=[0.0, 0.0, -9.81],
        solver="Newton", iterations=int(opt["iterations"]), tolerance=float(opt["tolerance"]),
        cone="pyramidal", impratio=1.0,
        # MuJoCo defaults, nothing in the reference overrides them (SURVEY Appendix A.0)
        solref=[0.02, 1.0], solimp=[0.9, 0.95, 0.001, 0.5, 2.0], friction=[1.0, 0.005, 0.0001],
    )
    out_links = []
    for i, lk in enumerate(links):
        c, Ic = lk.finalize()
        d = dict(name=lk.name, parent=lk.parent, pos=lk.pos.tolist(), rot=lk.rot.tolist(),
                 mass=lk.mass, com=c.tolist(),
                 inertia=[Ic[0, 0], Ic[1, 1], Ic[2, 2], Ic[0, 1], Ic[0, 2], Ic[1, 2]],
                 members=sorted(lk.members))
        j = lk.joint
        if j["type"] == "free":
            d["joint"] = dict(type="free", name=j["name"])
        else:
            d["joint"] = dict(type="hinge", name=j["name"], axis=j["axis"].tolist(), armature=j["armature"],
                              damping=j["damping"], range=j["range"].tolist())
        out_links.append(d)
    model["links"] = out_links
    model["qpos0"] = qpos0_root.tolist() + [1.0, 0.0, 0.0, 0.0] + [0.0] * 12

    # feet: gen_xml.py:125-130 (collision box per foot, class collision => condim 3)
    foot_size = [r5(0.1), r5(0.05), r5(0.01)]
    foot_pos = [r5(0.029), 0.0, r5(-0.09778)]
    li = {lk.name: i for i, lk in enumerate(links)}
    model["geoms"] = [
        dict(name="R_ANKLE_P_S-foot", type="box", link=li["R_ANKLE_P_S"], pos=foot_pos, size=foot_size),
        dict(name="L_ANKLE_P_S-foot", type="box", link=li["L_ANKLE_P_S"], pos=foot_pos, size=foot_size),
    ]
    model["rfoot_link"] = li["R_ANKLE_P_S"]
    model["lfoot_link"] = li["L_ANKLE_P_S"]
    # head body NECK_P_S is welded into the root link; its origin in the root frame:
    model["head_in_root"] = links[0].members["NECK_P_S"][0].tolist()
    model["total_mass"] = float(sum(lk.mass for lk in links))

    # env config (envs/jvrc/configs/base.yaml, envs/jvrc/jvrc_base.py:38-67)
    model["cfg"] = dict(
        sim_dt=cfg["sim_dt"], control_dt=cfg["control_dt"], frame_skip=int(round(cfg["control_dt"] / cfg["sim_dt"])),
        action_smoothing=cfg["action_smoothing"], obs_history_len=cfg["obs_history_len"],
        kp=[float(x) for x in cfg["kp"]], kd=[float(x) for x in cfg["kd"]],
        half_sitting_pose_deg=[float(x) for x in cfg["half_sitting_pose"]],
        nominal_qpos=[0.0, 0.0, 0.81, 1.0, 0.0, 0.0, 0.0] + np.deg2rad(cfg["half_sitting_pose"]).tolist(),
        task=dict(cfg["task"]),
    )
    if boxes:
        # envs/jvrc/jvrc_step.py + tasks/stepping_task.py: force-sensor sites (gen_xml.py:143-144), 20 stepping-stone slabs
        # (gen_xml.py:147-153; re-sized to 0.15 x 1 x box_h at every task reset, stepping_task.py:322-329), footstep plans
        site = [r5(0.03), 0.0, r5(-0.1)]
        model["foot_sites"] = [site, site]          # rf_force, lf_force in the foot link frame
        plans, seq = [], []
        for line in open(os.path.join(REF, "utils/footstep_plans.txt")):
            line = line.strip()
            if line == "---":                       # stepping_task.py:57-64 (a trailing block without '---' is dropped)
                if seq:
                    plans.append(seq)
                seq = []
            else:
                seq.append([float(v) for v in line.split(",")])
        t = cfg["task"]
        model["stepping"] = dict(
            nboxes=20, slab_half=[0.15, 1.0, r5(0.1)], target_radius=0.20,
            delay_frames=int(np.floor(t["swing_duration"] / cfg["control_dt"])),
            # not in the reference: penetration depth up to which a slab's top face always supports a point (beyond it the
            # point must be at least as far from the slab's side faces), see oracle/sim_oracle.c:slab_supports
            side_tol=0.02,
            # SURVEY Appendix C-3: SteppingTask normalises the foot forces with RobotInterface.get_robot_mass() = mj_getTotalmass,
            # which sums EVERY body: the 20 static boxes are compiled from `size="1 1 0.1"` (gen_xml.py:151) at the default
            # density 1000 kg/m^3 = 800 kg each, and later geom_size edits do not touch body_mass
            task_mass=float(sum(lk.mass for lk in links)) + 20 * (2 * 1.0) * (2 * 1.0) * (2 * r5(0.1)) * 1000.0,
            # SURVEY Appendix C-2: get_*_floor_contacts skips contacts whose geom1 is a robot geom; a foot box precedes a stone box
            # in MuJoCo's (type, id) pair ordering, so stone contacts are invisible to the task (GRF, contact_point_z).
            # True = count them as floor (the physically meant behaviour), False = the reference's behaviour
            slab_contacts_are_floor=False,
            side_faces=True,         # slab side faces (stair risers) stop foot-box corners; False = round-1 behaviour (they pass through)
            mode_probs=[0.15, 0.05, 0.2, 0.3, 0.3],  # CURVED, STANDING, BACKWARD, LATERAL, FORWARD
            plans=plans)
    add_setconst(model)
    return model


# ----------------------------------------------------------------------------------------------
# mj_setConst restatement: mass matrix at qpos0 -> dof_invweight0, body_invweight0, meaninertia
# (numpy, generic tree; also used by tests as a third independent mass-matrix implementation)
# ----------------------------------------------------------------------------------------------

def kinematics(model, qpos):
    links = model["links"]
    n = len(links)
    xpos = np.zeros((n, 3))
    xmat = np.zeros((n, 3, 3))
    adr = 7
    for i, lk in enumerate(links):
        if lk["joint"]["type"] == "free":
            xpos[i] = qpos[0:3]
            xmat[i] = quat2mat(qpos[3:7])
        else:
            p = lk["parent"]
            ax = np.array(lk["joint"]["axis"])
            q = qpos[adr]
            adr += 1
            K = skew(ax / np.linalg.norm(ax))
            Rj = np.eye(3) + np.sin(q) * K + (1 - np.cos(q)) * K @ K
            xpos[i] = xpos[p] + xmat[p] @ np.array(lk["pos"])
            xmat[i] = xmat[p] @ np.array(lk["rot"]) @ Rj
    return xpos, xmat


def dof_jacobians(model, qpos, point, link):
    """3xnv translational jacobian of world `point` rigidly attached to `link`, and 3xnv rotational."""
    links = model["links"]
    xpos, xmat = kinematics(model, qpos)
    nv = 6 + len(links) - 1
    jp = np.zeros((3, nv))
    jr = np.zeros((3, nv))
    b = link
    while b >= 0:
        lk = links[b]
        if lk["joint"]["type"] == "free":
            jp[:, 0:3] = np.eye(3)
            for k in range(3):
                a = xmat[b][:, k]
                jr[:, 3 + k] = a
                jp[:, 3 + k] = np.cross(a, point - xpos[b])
        else:
            d = 6 + (b - 1)
            a = xmat[b] @ np.array(lk["joint"]["axis"])
            jr[:, d] = a
            jp[:, d] = np.cross(a, point - xpos[b])
        b = lk["parent"]
    return jp, jr


def mass_matrix(model, qpos):
    links = model["links"]
    xpos, xmat = kinematics(model, qpos)
    nv = 6 + len(links) - 1
    M = np.zeros((nv, nv))
    for i, lk in enumerate(links):
        c = xpos[i] + xmat[i] @ np.array(lk["com"])
        a = lk["inertia"]
        Ib = np.array([[a[0], a[3], a[4]], [a[3], a[1], a[5]], [a[4], a[5], a[2]]])
        Iw = xmat[i] @ Ib @ xmat[i].T
        jp, jr = dof_jacobians(model, qpos, c, i)
        M += lk["mass"] * jp.T @ jp + jr.T @ Iw @ jr
    for i, lk in enumerate(links):
        if lk["joint"]["type"] == "hinge":
            M[6 + i - 1, 6 + i - 1] += lk["joint"]["armature"]
    return M


def add_setconst(model):
    qpos0 = np.array(model["qpos0"])
    M = mass_matrix(model, qpos0)
    Minv = np.linalg.inv(M)
    nv = M.shape[0]
    dofw = np.diag(Minv).copy()
    # free joint: translational and rotational dofs each share their mean (engine_setconst.c set0)
    dofw[0:3] = dofw[0:3].mean()
    dofw[3:6] = dofw[3:6].mean()
    xpos, xmat = kinematics(model, qpos0)
    bw = []
    for i, lk in enumerate(model["links"]):
        c = xpos[i] + xmat[i] @ np.array(lk["com"])
        jp, jr = dof_jacobians(model, qpos0, c, i)
        J = np.vstack([jp, jr])
        A = J @ Minv @ J.T
        bw.append([float(np.trace(A[:3, :3]) / 3), float(np.trace(A[3:, 3:]) / 3)])
    model["dof_invweight0"] = dofw.tolist()
    model["link_invweight0"] = bw
    model["meaninertia"] = float(np.trace(M) / nv)
    # MuJoCo's body_invweight0 is per *xml body*; the only bodies that ever carry contact rows here
    # are the feet (leaf links, no welded children => identical to the link value) and the world (0).
    # For welded members that differ from their link com the value would differ; record the caveat.
    model["notes"] = [
        "numeric attributes rounded with '%.5g' (dm_control export precision=5) — unverified against a live export",
        "link_invweight0 evaluated at the LINK com; equals MuJoCo body_invweight0 only for links without welded children",
    ]



# ==============================================================================================
# Unitree H1 (envs/h1/gen_xml.py:64-126, envs/h1/h1_env.py:17-33, envs/h1/h1_base.py:38-70,
# models/mujoco_menagerie/unitree_h1/h1.xml)
# ==============================================================================================
H1_LEG_JOINTS = ["left_hip_yaw", "left_hip_roll", "left_hip_pitch", "left_knee", "left_ankle",
                 "right_hip_yaw", "right_hip_roll", "right_hip_pitch", "right_knee", "right_ankle"]


def r5v(v):
    """%.5g export rounding (mjcf.export_with_assets(precision=5)) of a vector."""
    return [r5(x) for x in np.asarray(v, dtype=float)]


def compile_h1():
    """H1Env: torso + arm joints removed (unused_joints), jointlimited=False, ctrllimited=False, minimal XML.
    Post-compile the reference overrides body masses (pelvis 8.89, torso_link 21.289, h1_base.py:40-41) WITHOUT
    re-running mj_setConst: inertia tensors and *_invweight0 keep their compile-time values (SURVEY Appendix C-7)."""
    xml_dir = os.path.join(REF, "models/mujoco_menagerie/unitree_h1")
    root = ET.parse(os.path.join(xml_dir, "h1.xml")).getroot()
    cfg = yaml.safe_load(open(os.path.join(REF, "envs/h1/configs/base.yaml")))
    dflt = root.find("default").find("default")          # class h1
    assert dflt.attrib["class"] == "h1"
    jd = dflt.find("joint").attrib
    j_damping, j_armature = r5(jd["damping"]), r5(jd["armature"])
    foot_cls = {}
    for d in dflt.iter("default"):
        if d.attrib.get("class", "").startswith("foot") and d.find("geom") is not None and "fromto" in d.find("geom").attrib:
            foot_cls[d.attrib["class"]] = vec(d.find("geom").attrib["fromto"], 6)
    foot_radius = r5(0.014)
    keep = set(H1_LEG_JOINTS)
    mass_override = {"pelvis": 8.89, "torso_link": 21.289}
    links: list[Link] = []
    parts = {}      # xml body name -> dict(link, mass0, mass, com (link frame), Ic (link frame))
    foot_pts = {}
    leg_caps = []   # exact capsule / sphere collision primitives of the leg links (self-collision termination flag)
    root_caps = []  # ... and the torso's "hip" capsule, the one upper-body primitive the legs reach before termination

    def walk(body, link_idx, pos_in_link, rot_in_link):
        name = body.attrib["name"]
        jel, fj = body.find("joint"), body.find("freejoint")
        jointed = fj is not None or (jel is not None and jel.attrib["name"] in keep)
        if jointed:
            lk = Link(name, link_idx, pos_in_link, rot_in_link)
            if fj is not None:
                lk.joint = dict(type="free", name="root")
            else:
                lk.joint = dict(type="hinge", name=jel.attrib["name"], axis=vec(jel.attrib["axis"], 3),
                                armature=r5(jel.attrib.get("armature", j_armature)), damping=r5(jel.attrib.get("damping", j_damping)),
                                range=vec(jel.attrib["range"], 2), limited=False)   # jointlimited: false (configs/base.yaml)
            links.append(lk)
            link_idx = len(links) - 1
            pos_in_link, rot_in_link = np.zeros(3), np.eye(3)
        lk = links[link_idx]
        lk.members[name] = (pos_in_link.copy(), rot_in_link.copy())
        ine = body.find("inertial")
        m0 = r5(ine.attrib["mass"])
        ipos = vec(ine.attrib.get("pos", "0 0 0"), 3)
        Ri = rot_in_link @ quat2mat(vec(ine.attrib.get("quat", "1 0 0 0"), 4))
        Ic = Ri @ np.diag(vec(ine.attrib["diaginertia"], 3)) @ Ri.T
        parts[name] = dict(link=link_idx, mass0=m0, mass=mass_override.get(name, m0), com=pos_in_link + rot_in_link @ ipos, Ic=Ic)
        for g in body.findall("geom"):
            c = g.attrib.get("class", "")
            if c in foot_cls:
                ft = foot_cls[c]
                foot_pts.setdefault(link_idx, []).extend([(pos_in_link + rot_in_link @ ft[0:3]).tolist(),
                                                          (pos_in_link + rot_in_link @ ft[3:6]).tolist()])
                leg_caps.append(dict(link=link_idx, p0=r5v(pos_in_link + rot_in_link @ ft[0:3]),
                                     p1=r5v(pos_in_link + rot_in_link @ ft[3:6]), radius=foot_radius, name=name + ":" + c))
            elif c == "collision" and link_idx > 0 and g.attrib.get("type") == "capsule":
                ft = vec(g.attrib["fromto"], 6)
                leg_caps.append(dict(link=link_idx, p0=r5v(pos_in_link + rot_in_link @ ft[0:3]),
                                     p1=r5v(pos_in_link + rot_in_link @ ft[3:6]), radius=r5(g.attrib["size"]), name=name + ":capsule"))
            elif c == "collision" and link_idx == 0 and g.attrib.get("name") == "hip":     # h1.xml:154, on the welded torso
                ft = vec(g.attrib["fromto"], 6)
                root_caps.append(dict(link=0, p0=r5v(pos_in_link + rot_in_link @ ft[0:3]),
                                      p1=r5v(pos_in_link + rot_in_link @ ft[3:6]), radius=r5(g.attrib["size"]), name="torso_link:hip"))
            elif c == "collision" and link_idx > 0 and g.attrib.get("type") == "sphere":
                ctr = r5v(pos_in_link + rot_in_link @ vec(g.attrib["pos"], 3))
                leg_caps.append(dict(link=link_idx, p0=ctr, p1=ctr, radius=r5(g.attrib["size"]), name=name + ":sphere"))
        for child in body.findall("body"):
            cpos = vec(child.attrib.get("pos", "0 0 0"), 3)
            crot = quat2mat(vec(child.attrib["quat"], 4)) if "quat" in child.attrib else np.eye(3)
            walk(child, link_idx, pos_in_link + rot_in_link @ cpos, rot_in_link @ crot)

    pelvis = root.find("worldbody").find("body")
    assert pelvis.attrib["name"] == "pelvis"
    qpos0_root = vec(pelvis.attrib["pos"], 3)
    walk(pelvis, -1, np.zeros(3), np.eye(3))
    assert [lk.joint["name"] for lk in links[1:]] == H1_LEG_JOINTS

    def assemble(use_override):
        for lk in links:
            lk.mass, lk.mc, lk.Io = 0.0, np.zeros(3), np.zeros((3, 3))
        for nm, pt in parts.items():
            links[pt["link"]].add_inertial(pt["mass"] if use_override else pt["mass0"], pt["com"], pt["Ic"])
        out = []
        for lk in links:
            c, Ic = lk.finalize()
            d = dict(name=lk.name, parent=lk.parent, pos=lk.pos.tolist(), rot=lk.rot.tolist(), mass=lk.mass, com=c.tolist(),
                     inertia=[Ic[0, 0], Ic[1, 1], Ic[2, 2], Ic[0, 1], Ic[0, 2], Ic[1, 2]], members=sorted(lk.members))
            j = lk.joint
            d["joint"] = dict(type="free", name="root") if j["type"] == "free" else dict(
                type="hinge", name=j["name"], axis=j["axis"].tolist(), armature=j["armature"], damping=j["damping"],
                range=j["range"].tolist(), limited=False)
            out.append(d)
        return out

    model = dict(name="h1")
    model["opt"] = dict(timestep=float(cfg["sim_dt"]), gravity=[0.0, 0.0, -9.81], solver="Newton", iterations=100, tolerance=1e-8,
                        cone="pyramidal", impratio=1.0, solref=[0.02, 1.0], solimp=[0.9, 0.95, 0.001, 0.5, 2.0],
                        friction=[1.0, 0.005, 0.0001])
    model["qpos0"] = qpos0_root.tolist() + [1.0, 0.0, 0.0, 0.0] + [0.0] * 10
    model["cfg"] = dict(sim_dt=cfg["sim_dt"], control_dt=cfg["control_dt"], frame_skip=int(round(cfg["control_dt"] / cfg["sim_dt"])),
                        action_smoothing=cfg["action_smoothing"], obs_history_len=cfg["obs_history_len"], init_noise_deg=cfg["init_noise"])
    # mj_setConst quantities with the COMPILE-TIME masses (the override happens afterwards and does not refresh them)
    model["links"] = assemble(False)
    add_setconst(model)
    frozen = {k: model[k] for k in ("dof_invweight0", "link_invweight0", "meaninertia")}
    # runtime model: overridden masses
    model["links"] = assemble(True)
    model.update(frozen)
    gains = cfg["pdgains"]
    model["cfg"].update(kp=[float(gains[j][0]) for j in H1_LEG_JOINTS], kd=[float(gains[j][1]) for j in H1_LEG_JOINTS],
                        half_sitting_pose=[float(x) for x in cfg["half_sitting_pose"]],
                        nominal_qpos=[0.0, 0.0, 0.98, 1.0, 0.0, 0.0, 0.0] + [float(x) for x in cfg["half_sitting_pose"]],
                        observation_noise=cfg["observation_noise"], perturbation=cfg["perturbation"],
                        dynamics_randomization=cfg["dynamics_randomization"])
    li = {lk.name: i for i, lk in enumerate(links)}
    model["lfoot_link"], model["rfoot_link"] = li["left_ankle_link"], li["right_ankle_link"]
    model["geoms"] = [dict(name=links[l].name + "-feet", type="spheres", link=l, radius=foot_radius, points=foot_pts[l])
                      for l in (li["left_ankle_link"], li["right_ankle_link"])]
    model["total_mass"] = float(sum(lk.mass for lk in links))
    # self-collision (StandingTask.done -> check_self_collisions, robot_interface.py:472-484): MuJoCo collides every pair of
    # collision geoms on different, non-adjacent (weld-aware) bodies.  Modelled exactly: all capsule / sphere primitives of one
    # leg against those of the other leg (thigh x2, shin, knee sphere, 3 foot capsules = 7 per leg, 49 pairs), and the torso's
    # "hip" capsule (welded to the pelvis, h1.xml:154) against the thigh / shin / knee primitives of both legs (8 pairs): the
    # contact that ends episodes under large actions (tools/eval_h1_self_collision.py: every self-contact an oracle rollout
    # at sigma = 1.0 reaches before the 0.9 m height termination involves it).  Not modelled: the hip cylinders, the torso box,
    # head and the welded arms (no pose of that study reaches them without also closing a modelled pair).
    nj = len(H1_LEG_JOINTS) // 2
    left = [i for i, c_ in enumerate(leg_caps) if c_["link"] <= nj]
    right = [i for i, c_ in enumerate(leg_caps) if c_["link"] > nj]
    assert len(left) == len(right) == 7 and len(root_caps) == 1, (len(left), len(right), len(root_caps))
    caps = leg_caps + root_caps
    hip = len(leg_caps)
    upper_leg = [i for i, c_ in enumerate(leg_caps) if ":foot" not in c_["name"]]
    model["self_collision"] = dict(capsules=caps, pairs=[[a, b] for a in left for b in right] + [[a, hip] for a in upper_leg],
                                   source="exact primitives from unitree_h1/h1.xml (capsule and sphere geoms of the leg bodies, "
                                          "the torso's hip capsule)")
    # the root link is pelvis + torso + arms welded; randomize_dynamics (domain_randomization.py:46-56) only touches the
    # pelvis BODY (mass x U(.95,1.05), ipos + U(+-.01)) and the leg bodies, so keep the pelvis separable from the rest
    pel = parts["pelvis"]
    rest_m = sum(p_["mass"] for n_, p_ in parts.items() if p_["link"] == 0 and n_ != "pelvis")
    rest_mc = sum(p_["mass"] * p_["com"] for n_, p_ in parts.items() if p_["link"] == 0 and n_ != "pelvis")
    rest_Io = sum(p_["Ic"] + p_["mass"] * (np.dot(p_["com"], p_["com"]) * np.eye(3) - np.outer(p_["com"], p_["com"]))
                  for n_, p_ in parts.items() if p_["link"] == 0 and n_ != "pelvis")
    model["root_parts"] = dict(pelvis=dict(mass=pel["mass"], com=pel["com"].tolist(), Ic=pel["Ic"].tolist()),
                               rest=dict(mass=float(rest_m), mc=np.asarray(rest_mc).tolist(), Io=np.asarray(rest_Io).tolist()),
                               torso_com=(parts["torso_link"]["com"]).tolist())
    model["notes"] = ["dof_invweight0 / link_invweight0 / meaninertia evaluated with the XML masses (pelvis 5.39, torso 17.789); "
                      "dynamics use the overridden ones (8.89, 21.289) with unchanged inertia tensors (h1_base.py:40-41)",
                      "ground contacts: the 3 foot capsules per foot (6 end spheres, radius 0.014); other collision primitives "
                      "(legs, torso, arms) only touch the floor after the 0.9 m termination height and are not modelled",
                      "self-collision flag: leg-vs-leg capsule / sphere primitives and the torso's hip capsule vs thighs / shins (exact); "
                      "hip cylinders, torso box, head and the welded arms are not modelled (tests/golden/h1_self_collision_eval.json)"]
    return model


# h1_walk: the H1 robot of h1.json with a WalkingTask.  The reference's envs/h1/h1_walk.py is not read here, so these values are
# this build's choices (DESIGN.md §4.6): jvrc_walk's gait durations, the standing task's goal height (tasks/standing_task.py), and
# the torso's centre of mass (on the torso welded to the pelvis, in the root-link frame) as the upper-body reward's head point
H1_WALK_TASK = dict(goal_height=0.98, total_duration=1.1, swing_duration=0.75, stance_duration=0.35)


def derive_h1_walk(h1: dict) -> dict:
    """model/h1_walk.json from model/h1.json: the same robot plus a walking `task` block and `head_in_root`."""
    hw = json.loads(json.dumps(h1))
    hw["name"] = "h1_walk"
    hw["head_in_root"] = list(h1["root_parts"]["torso_com"])
    hw["cfg"]["task"] = dict(H1_WALK_TASK)
    return hw


def write_h1_walk(out: str) -> str:
    h1 = json.load(open(os.path.join(out, "h1.json")))
    path = os.path.join(out, "h1_walk.json")
    with open(path, "w") as f:
        json.dump(derive_h1_walk(h1), f, indent=1)
    return path


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(os.path.dirname(__file__), "..",
                                                  "learninghumanoidwalking_b200", "model"))
    ap.add_argument("--h1-walk-only", action="store_true",
                    help="only derive h1_walk.json from the h1.json already in --out (needs no reference checkout)")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.h1_walk_only:
        print("wrote", write_h1_walk(args.out))
        return
    m = compile_jvrc()
    path = os.path.join(args.out, "jvrc_walk.json")
    if os.path.exists(path):   # tools/fit_collision_proxies.py adds this block afterwards; keep it across recompiles
        old = json.load(open(path))
        if "self_collision" in old:
            m["self_collision"] = old["self_collision"]
    m["assumptions"] = ASSUMPTIONS
    with open(path, "w") as f:
        json.dump(m, f, indent=1)
    print("wrote", path, "mass", m["total_mass"], "links", len(m["links"]), "meaninertia", m["meaninertia"])
    for lk in m["links"]:
        print(f"  {lk['name']:14s} parent {lk['parent']:2d} mass {lk['mass']:.4f} com {np.round(lk['com'], 4)}")
    print("foot invweight0", m["link_invweight0"][m["rfoot_link"]], "dof_invweight0", np.round(m["dof_invweight0"], 4))
    st = compile_jvrc(boxes=True)
    if "self_collision" in m:
        st["self_collision"] = m["self_collision"]
    st["assumptions"] = ASSUMPTIONS
    json.dump(st, open(os.path.join(args.out, "jvrc_step.json"), "w"), indent=1)
    print("wrote jvrc_step.json plans", len(st["stepping"]["plans"]), "delay_frames", st["stepping"]["delay_frames"])
    # uneven / compliant terrain EXTENSION (BASELINE configs[4]; SURVEY F7: the reference has only the unused
    # WalkingTask(manip_hfield) hook and no height-field asset).  jvrc_walk on 20 terraces re-posed with the hook's ranges
    # (tasks/walking_task.py:172-179: x, y ~ U(-0.5, 0.5), z ~ U(-0.035, -0.015), w.p. 1/200 per control step outside
    # STANDING); terrace tops bump ~ U(0, 0.05) above that offset; softer foot-ground contacts (solref timeconst 0.04 s)
    tm = dict(m)
    tm["name"] = "jvrc_walk_terrain"
    tm["terrain"] = dict(strip_half=[0.15, 1.0, 0.1], side_tol=0.02, pitch=0.3, bump=0.05, z_lo=-0.035, z_hi=-0.015, xy=0.5,
                         interval=200, contact_solref=[0.04, 1.0], side_faces=True)
    json.dump(tm, open(os.path.join(args.out, "jvrc_walk_terrain.json"), "w"), indent=1)
    h = compile_h1()
    h["assumptions"] = ASSUMPTIONS
    json.dump(h, open(os.path.join(args.out, "h1.json"), "w"), indent=1)
    print("wrote h1.json mass", h["total_mass"], "links", len(h["links"]), "meaninertia", h["meaninertia"])
    for lk in h["links"]:
        print(f"  {lk['name']:22s} parent {lk['parent']:2d} mass {lk['mass']:.4f} com {np.round(lk['com'], 4)}")
    print("  foot points", np.round(h["geoms"][0]["points"], 4).tolist())
    print("wrote", write_h1_walk(args.out))


if __name__ == "__main__":
    main()
