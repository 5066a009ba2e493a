"""h1_walk: the Unitree H1 robot (Cfg<5, 0>) with the WalkingTask (Cfg<6, 0>), as the step kernel's variant Cfg<5, 3>.

CPU tier: the committed model constants are what tools/compile_model.py derives from h1.json; the mirror lists fit the
kernel's observation layout; the kernel source (CPU lane emulation, tests/emu) agrees with oracle/ over closed-loop runs with
mode switches, randomisation, pushes and resets; the YAML overlay; the fp32 kernel source one control step at a time."""
import json
import os

import numpy as np
import pytest

from h1_walk_oracle import TORQUES, H1WalkOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MODEL_DIR = os.path.join(ROOT, "learninghumanoidwalking_b200", "model")
NQ, NV, NU = 17, 16, 10
# state record (csrc/sim_core.h Persist + PersistRand): act_len, act_vel, then the per-env parameters and the pushes
ACT_LEN, ACT_VEL = NQ + 2 * NV, NQ + 2 * NV + NU
P_MASS, P_FLOSS, XFRC = slice(103, 114), slice(163, 173), slice(176, 188)


def _attrs():
    """The env attributes BatchedHumanoidEnv sets for h1_walk (pure numpy; no device needed)."""
    from learninghumanoidwalking_b200.envs.batched_env import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.model import load_model
    env = BatchedHumanoidEnv.__new__(BatchedHumanoidEnv)
    env._iteration_count = float("inf")
    env._setup_reference_attributes("h1_walk", load_model("h1_walk")["cfg"])
    return env


def test_model_constants_are_derived_from_h1_json():
    from tools.compile_model import H1_WALK_TASK, derive_h1_walk
    h1 = json.load(open(os.path.join(MODEL_DIR, "h1.json")))
    with open(os.path.join(MODEL_DIR, "h1_walk.json")) as f:
        committed = f.read()
    assert json.dumps(derive_h1_walk(h1), indent=1) == committed
    hw = json.loads(committed)
    assert hw["head_in_root"] == h1["root_parts"]["torso_com"] and hw["head_in_root"][2] > 0.1   # on the torso, above the pelvis
    assert hw["cfg"]["task"] == H1_WALK_TASK and (hw["lfoot_link"], hw["rfoot_link"]) == (h1["lfoot_link"], h1["rfoot_link"])
    from learninghumanoidwalking_b200.model import pack_model
    flat = pack_model(hw)
    assert flat[0] == 305


def test_mirror_lists_are_involutions_of_the_right_length():
    env = _attrs()
    r = env.robot
    assert len(r.mirrored_obs) == 43 == len(env.obs_mean) == len(env.obs_std) and len(r.mirrored_acts) == NU
    assert list(r.clock_inds) == [35, 36] and list(env.reward_names)[6] == "upper_body_reward"
    for lst in (r.mirrored_obs, r.mirrored_acts):
        idx = np.abs(np.asarray(lst)).astype(int)
        sign = np.sign(lst)
        assert sorted(idx) == list(range(len(lst)))
        for i in range(len(lst)):
            assert idx[idx[i]] == i and sign[idx[i]] == sign[i]
    # h1's 35 robot-state entries, then jvrc_walk's 8 walking-task words
    gold = json.load(open(os.path.join(ROOT, "tests", "golden", "env_attributes.json")))
    assert np.array_equal(env.obs_mean, np.concatenate((gold["h1"]["obs_mean"], gold["jvrc_walk"]["obs_mean"][-8:])))
    assert np.array_equal(env.obs_std, np.concatenate((gold["h1"]["obs_std"], gold["jvrc_walk"]["obs_std"][-8:])))


def _mirror_record(sr, mirrored_acts):
    """The mirror image (in the sagittal plane) of a state record: root y, the quaternion's x and z, the angular velocity's x
    and z, and every joint quantity by the action mirror list (legs swapped, hip yaw / roll negated)."""
    idx = np.abs(np.asarray(mirrored_acts)).astype(int)
    sgn = np.sign(mirrored_acts)
    m = sr.copy()
    joints = lambda v: v[idx] * sgn
    m[1] = -sr[1]
    m[4], m[6] = -sr[4], -sr[6]
    m[7:NQ] = joints(sr[7:NQ])
    m[NQ + 1] = -sr[NQ + 1]
    m[NQ + 3], m[NQ + 5] = -sr[NQ + 3], -sr[NQ + 5]
    m[NQ + 6:NQ + NV] = joints(sr[NQ + 6:NQ + NV])
    for off in (ACT_LEN, ACT_VEL):
        m[off:off + NU] = joints(sr[off:off + NU])
    return m


def test_mirrored_state_gives_the_mirrored_observation_in_the_kernel_source():
    """The mirror lists against the kernel's own observation: a control step without physics (frame_skip 0) observes the
    record as it is, so the observation of a mirrored record must be the mirror of the observation, exactly, apart from the
    clock words (SymmetricEnv shifts the phase by half a period; here both records keep theirs)."""
    from emu_variants import Emu
    from learninghumanoidwalking_b200.model import load_model, pack_model
    env = _attrs()
    mo, ma = env.robot.mirrored_obs, env.robot.mirrored_acts
    P = np.zeros((43, 43))
    P[np.arange(43), np.abs(np.asarray(mo)).astype(int)] = np.sign(mo)
    mj = load_model("h1_walk")
    run = Emu(pack_model(mj, observation_noise=False), 64, 8, seed=4)
    run.reset()
    rng = np.random.RandomState(1)
    for _ in range(15):
        run.step(rng.normal(size=(8, NU)) * 0.3)
    frozen = json.loads(json.dumps(mj))
    frozen["cfg"]["frame_skip"] = 0
    flat = pack_model(frozen, observation_noise=False)
    checked = 0
    for i in range(8):
        if not np.isfinite(run.sr[i]).all():
            continue
        outs = []
        for rec in (run.sr[i], _mirror_record(run.sr[i], ma)):
            e = Emu(flat, 64, 1, seed=4, first_id=i)     # a fresh emulation: the step sees only this record
            e.sr[0], e.si[0] = rec, run.si[i]
            outs.append(e.step(np.zeros((1, NU)), autoreset=0)[0][0])
        o, om = outs
        keep = np.ones(43, bool)
        keep[env.robot.clock_inds] = False
        assert np.array_equal((o @ P)[keep], om[keep]), np.abs(o @ P - om)[keep].max()
        assert np.abs(o[5:15]).max() > 0.01 and np.abs(o[15:25]).max() > 0.01        # joints moved: the test sees them
        checked += 1
    assert checked >= 6


def test_kernel_source_matches_oracle_h1_walk_fp64():
    from emu_variants import Emu
    from learninghumanoidwalking_b200.model import load_model, pack_model
    o = H1WalkOracle(tolerance=1e-14)
    N, seed = 16, 11
    e = Emu(pack_model(load_model("h1_walk"), tolerance=1e-14), 64, N, seed=seed, first_id=5)
    assert e.nobs == 43 and e.nu == NU
    envs = o.make_envs(N, seed=seed, first_id=5)
    assert np.abs(o.batch_reset(envs, N) - e.reset()).max() < 1e-10
    rng = np.random.RandomState(2)
    n_end = n_fall = switches = 0
    pushed, worst = False, 0.0
    mode = e.si[:, 1].copy()
    for t in range(300):
        a = rng.normal(size=(N, NU)) * 0.3
        oo, to, tt, rr, dd, ee = o.batch_step(envs, N, a, max_traj_len=60)
        eo, et, etm, er, ed, een, eplen, eprew = e.step(a, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        oq = np.stack([o.field(envs, i, "qpos")[:NQ] for i in range(N)])
        ov = np.stack([o.field(envs, i, "qvel")[:NV] for i in range(N)])
        worst = max(worst, np.abs(oo - eo).max(), np.abs(tt - etm).max(), np.abs(rr - er).max(), np.abs(oq - e.qpos).max(),
                    np.abs(ov - e.qvel).max())
        m = ee.astype(bool)
        if m.any():   # the oracle's terminal observation has no torque words (the env has been reset since)
            assert np.nanmax(np.abs(to[m] - et[m])) < 1e-7 and np.isnan(to[m][:, TORQUES]).all()
        n_end += int(m.sum()); n_fall += int(dd.sum())
        switches += int(((e.si[:, 1] != mode) & ~m).sum())
        mode = e.si[:, 1].copy()
        x = np.stack([o.field(envs, i, "xfrc") for i in range(N)])
        pushed |= bool(np.any(x))
        assert np.array_equal(x, e.sr[:, XFRC])            # the same pushes and the same coin flips
        assert (np.stack([o.field(envs, i, "mode") for i in range(N)])[:, 0] == e.si[:, 1]).all()
        assert (np.stack([o.field(envs, i, "phase") for i in range(N)])[:, 0] == e.si[:, 0]).all()
    assert worst < 1e-7, worst
    assert n_fall > 0 and n_end > n_fall and switches > 0 and pushed, (n_fall, n_end, switches, pushed)
    for i in range(N):   # the per-env randomised parameters
        assert np.array_equal(o.field(envs, i, "P_frictionloss")[6:16], e.sr[i, P_FLOSS])
        assert np.abs(o.field(envs, i, "P_mass")[:11] - e.sr[i, P_MASS]).max() < 1e-13


def test_yaml_overlay_for_h1_walk():
    from learninghumanoidwalking_b200.envs.config import apply_config
    from learninghumanoidwalking_b200.model import load_model, pack_model
    mj = load_model("h1_walk")
    out = apply_config(mj, {"task": {"goal_height": 0.95, "swing_duration": 0.7, "stance_duration": 0.3, "total_duration": 1.0},
                            "half_sitting_pose": [0.0, 0.0, -0.3, 0.6, -0.3] * 2,
                            "pdgains": {mj["links"][1]["joint"]["name"]: [123.0, 4.5]},
                            "observation_noise": {"multiplier": 0.5}, "perturbation": {"force_magnitude": 20},
                            "dynamics_randomization": {"interval": 1.0}, "init_noise": 2})
    c = out["cfg"]
    assert c["task"] == dict(goal_height=0.95, total_duration=1.0, swing_duration=0.7, stance_duration=0.3)
    assert c["half_sitting_pose"] == [0.0, 0.0, -0.3, 0.6, -0.3] * 2 and c["nominal_qpos"][7:] == c["half_sitting_pose"]  # radians
    assert (c["kp"][0], c["kd"][0]) == (123.0, 4.5)
    assert c["observation_noise"]["multiplier"] == 0.5 and c["perturbation"]["force_magnitude"] == 20
    assert c["dynamics_randomization"]["interval"] == 1.0 and c["init_noise_deg"] == 2
    assert pack_model(out)[0] == 305
    for bad in ({"reduced_xml": False}, {"jointlimited": True}, {"task": {"foo": 1}}, {"observation_noise": {"type": "gaussian"}}):
        with pytest.raises(ValueError):
            apply_config(mj, bad)


def test_fp32_one_step_error_against_fp64_h1_walk():
    """tools/fp32_local_error.py on h1_walk at the bounds of the other variants (tests/test_fp32_local_error.py)."""
    from tools import fp32_local_error as L
    res = L.run(L.EmulationBackend("h1_walk", 8, seed=3, first_id=7), "h1_walk", 120, regime="noisy")
    n = res["env_steps"]
    assert res["falls"] > 0 and res["ended"] > 0 and res["param_events"] > 0
    assert not res["mismatch"], res["mismatch"][:5]
    assert not res["fail"], res["fail"][:5]
    assert len(res["exempt"]) <= 0.01 * n, len(res["exempt"])
    for q, bound in (("qpos", 1e-6), ("qvel", 1e-5), ("obs", 1e-5), ("reward", 1e-5), ("rew_terms", 1e-5)):
        assert np.median(res["errors"][q]) < bound, (q, np.median(res["errors"][q]))


REF = os.environ.get("LHW_REFERENCE", "/root/reference")


@pytest.mark.skipif(not os.path.exists(os.path.join(REF, "envs", "h1", "h1_walk.py")), reason="no reference checkout")
def test_build_defined_attributes_agree_with_a_reference_checkout():
    """Where a reference checkout has envs/h1/h1_walk.py, its own normalisation and mirror methods (lifted by AST, as
    tools/gen_golden_env_attrs.py does) must give what this build defines."""
    import types
    import yaml
    from tools.gen_golden_env_attrs import lift
    half = yaml.safe_load(open(os.path.join(REF, "envs", "h1", "configs", "base.yaml")))["half_sitting_pose"]
    holder = types.SimpleNamespace(half_sitting_pose=half, history_len=1, robot=types.SimpleNamespace(),
                                   _get_num_external_obs=lambda: 8)
    lift("envs/h1/h1_walk.py", "H1WalkEnv", "_setup_obs_normalization")(holder)
    env = _attrs()
    assert np.allclose(holder.obs_mean, env.obs_mean) and np.allclose(holder.obs_std, env.obs_std)
    try:
        lift("envs/h1/h1_walk.py", "H1WalkEnv", "_setup_mirror_indices")(holder)
    except StopIteration:
        return
    assert [float(x) for x in holder.robot.mirrored_obs] == [float(x) for x in env.robot.mirrored_obs]
    assert [float(x) for x in holder.robot.mirrored_acts] == [float(x) for x in env.robot.mirrored_acts]
