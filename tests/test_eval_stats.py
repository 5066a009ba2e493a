"""Evaluation statistics (`eval --num-envs`, DESIGN.md §7.4), CPU tier.

The product's accumulator body (csrc/sim_core.h eval_accumulate_env, the per-env body of lhw_sim_eval_accumulate) runs on the
host (tests/emu/eval_emu.cpp) over roll-outs of the kernel source's host emulation of every variant, at fp64 and fp32, with
autoreset off as the batched evaluation steps.  The roll-outs mix falls and truncations, and the walking tasks switch modes and
h1 is pushed.  The accumulators must equal a float64 numpy recomputation from the per-step records, which takes the record
layout from the dimensions alone (not from the header).  Also: the report's summary, and the command line's refusals."""
import ctypes
import os

import numpy as np
import pytest

import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
NREW, NSLAB = 10, 20
LEN, RET, DONE, TERMS, TRACK, REACHED, SEQLEN, WORDS = 0, 1, 2, 3, 13, 25, 26, 27
STANDING, INPLACE, FORWARD = 0, 1, 2
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
H1_XFRC = slice(176, 188)      # the pushes in h1's record (tests/test_h1_walk.py)


def _lib():
    lib = emu_variants._build("eval_emu.cpp", "eval_emu.cpp", os.path.join(HERE, "emu", "_build", "libeval_emu.so"), [])
    L = ctypes.CDLL(lib)
    L.eval_emu_accumulate.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 4
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def recompute(env_name, nj, records, n):
    """float64 numpy recomputation of the accumulators from per-step (sr, si, reward, rew_terms, done) of an autoreset-off run."""
    nv, nu = 6 + 2 * nj, 2 * nj
    nq = nv + 1
    mode_ref = nq + 2 * nv + 5 * nu      # qpos qvel qacc_warm, then act_len act_vel prev_pred prev_action prev_torque
    tk = mode_ref + 4 + 4 * NSLAB        # mode_ref[3] ep_rew, the footstep sequence [20][4], then the task counters
    acc = np.zeros((n, WORDS))
    for sr, si, rew, terms, done in records:
        sr = sr.astype(np.float64)
        for i in range(n):
            a = acc[i]
            if a[DONE] != 0:
                continue
            a[LEN] += 1
            a[RET] += float(rew[i])
            a[TERMS:TERMS + NREW] += terms[i].astype(np.float64)
            if env_name == "jvrc_step":
                a[REACHED], a[SEQLEN] = sr[i, tk + 1], sr[i, tk]
            else:
                mode = STANDING if env_name == "h1" else int(si[i, 1])
                yaw_ref, vx, vy = sr[i, mode_ref:mode_ref + 3]
                if mode == STANDING:
                    yaw_ref = vx = vy = 0.0
                elif mode == INPLACE:
                    vx = vy = 0.0
                else:
                    yaw_ref = 0.0
                qw, x, y, z = sr[i, 3:7]
                s = 2 / (qw * qw + x * x + y * y + z * z)
                X, Y, Z = x * s, y * s, z * s
                wX, wY, wZ, xX, xY, xZ, yY, yZ, zZ = qw * X, qw * Y, qw * Z, x * X, x * Y, x * Z, y * Y, y * Z, z * Z
                v0, v1, v2 = sr[i, nq:nq + 3]
                vf = (1 - (yY + zZ)) * v0 + (xY + wZ) * v1 + (xZ - wY) * v2
                vl = (xY - wZ) * v0 + (1 - (xX + zZ)) * v1 + (yZ + wX) * v2
                t = a[TRACK + 4 * mode:TRACK + 4 * mode + 4]
                t += (1.0, abs(vf - vx), abs(vl - vy), abs(sr[i, nq + 5] - yaw_ref))
            if done[i]:
                a[DONE] = 1
    return acc


def _rollout(env_name, precision, n=16, seed=3):
    """An autoreset-off roll-out of the host emulation with random actions (large ones on half of the envs, so that they fall),
    accumulated step by step through the product's body; returns (acc, per-step records, facts about the run).  h1 is pushed
    every 0.1 s on average here (its default is every 5 s), and its standing task ends at 0.9 m, which the untrained actions
    below reach after 11 steps, so its roll-out is shorter."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    mj = load_model(env_name)
    if env_name in ("h1", "h1_walk"):
        mj["cfg"]["perturbation"] = dict(mj["cfg"]["perturbation"], enable=True, interval=0.1)
    steps = 10 if env_name == "h1" else 40
    flat = pack_model(mj, tolerance=None if precision == 64 else 1e-6)
    var = int(flat[0])
    e = emu_variants.Emu(flat, precision, n, seed=seed)
    L = _lib()
    assert L.eval_emu_words() == WORDS
    e.reset()
    acc = np.zeros((n, WORDS))
    rng = np.random.RandomState(seed)
    scale = np.where(np.arange(n) % 2 == 0, 1.5, 0.02)[:, None]
    records, modes, pushed = [], set(), False
    for _ in range(steps):
        _, _, terms, rew, done, _, _, _ = e.step(rng.normal(size=(n, e.nu)) * scale, max_traj_len=steps, autoreset=0)
        assert L.eval_emu_accumulate(var, precision, _p(e.sr), _p(e.si), n, _p(rew), _p(terms),
                                     _p(done), _p(acc)) == 0
        records.append((e.sr.copy(), e.si.copy(), rew.copy(), terms.copy(), done.copy()))
        modes |= {tuple(m) for m in enumerate(e.si[:, 1])}
        if env_name in ("h1", "h1_walk"):
            pushed |= bool(np.abs(e.sr[:, H1_XFRC]).max() > 0)
    switched = len(modes) > n
    return acc, records, dict(pushed=pushed, switched=switched)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("env_name", VARIANTS)
def test_accumulators_equal_numpy_recomputation(env_name, precision):
    nj = 5 if env_name.startswith("h1") else 6
    acc, records, facts = _rollout(env_name, precision)
    n = acc.shape[0]
    want = recompute(env_name, nj, records, n)
    assert np.array_equal(acc, want), np.abs(acc - want).max()
    # the roll-out has what the statistics are about: falls and truncated episodes, and where the task has them, mode switches,
    # pushes and footsteps
    fell = acc[:, DONE] != 0
    assert fell.any() and (~fell).any(), acc[:, LEN]
    assert (acc[~fell, LEN] == len(records)).all() and (acc[fell, LEN] <= len(records)).all()
    assert np.array_equal(acc[:, TERMS:TERMS + NREW].sum(1) != 0, np.ones(n, bool))
    if env_name in ("jvrc_walk", "jvrc_walk_terrain", "h1_walk"):
        assert facts["switched"]
        assert np.array_equal(acc[:, [TRACK, TRACK + 4, TRACK + 8]].sum(1), acc[:, LEN])
    if env_name == "h1":
        assert np.array_equal(acc[:, TRACK], acc[:, LEN]) and not acc[:, TRACK + 4:TRACK + 12].any()
    if env_name in ("h1", "h1_walk"):
        assert facts["pushed"]
    if env_name == "jvrc_step":
        assert (acc[:, SEQLEN] >= 1).all() and (acc[:, REACHED] <= acc[:, SEQLEN] - 1).all()
        assert not acc[:, TRACK:TRACK + 12].any()
    else:
        assert not acc[:, REACHED:].any()


def test_summary_of_known_records():
    from learninghumanoidwalking_b200.rl import evaluation as ev
    acc = np.zeros((4, WORDS))
    acc[:, LEN] = [400, 100, 400, 20]
    acc[:, RET] = [40.0, 10.0, 38.0, 2.0]
    acc[:, DONE] = [0, 1, 0, 1]
    acc[:, TERMS] = acc[:, LEN] * 0.5
    acc[:, TRACK] = [400, 50, 0, 20]
    acc[:, TRACK + 1] = [40, 5, 0, 2]
    acc[:, TRACK + 8] = [0, 50, 400, 0]
    acc[:, TRACK + 11] = [0, 10, 30, 0]
    names = [f"t{k}" for k in range(NREW)]
    s = ev.summarize(acc, "jvrc_walk", names)
    assert s["num_envs"] == 4 and s["fall_fraction"] == 0.5
    assert s["length"] == dict(mean=230.0, min=20.0, p5=np.percentile([400, 100, 400, 20], 5), median=250.0)
    assert s["return"]["mean"] == 22.5 and s["return"]["std"] == pytest.approx(np.std([40, 10, 38, 2]))
    assert s["reward_terms"]["t0"] == 0.5 and s["reward_terms"]["t1"] == 0.0
    assert s["tracking"]["STANDING"] == dict(steps=470, vx_error=47 / 470, vy_error=0.0, yaw_rate_error=0.0)
    assert s["tracking"]["INPLACE"]["steps"] == 0 and s["tracking"]["INPLACE"]["vx_error"] is None
    assert s["tracking"]["FORWARD"]["yaw_rate_error"] == 40 / 450
    assert "footsteps" not in s
    step = np.zeros((2, WORDS))
    step[:, LEN] = 10
    step[:, REACHED] = [3, 19]
    step[:, SEQLEN] = [20, 20]
    fs = ev.summarize(step, "jvrc_step", names)["footsteps"]
    assert fs == dict(mean_reached=11.0, mean_sequence_length=20.0, completed_fraction=0.5)
    assert "tracking" not in ev.summarize(step, "jvrc_step", names)
    assert list(ev.summarize(acc, "h1", names)["tracking"]) == ["STANDING"]
    assert "FORWARD" in ev.format_table(s, 400) and "sequences completed" in ev.format_table(ev.summarize(step, "jvrc_step", names), 10)
    pe = ev.per_env(acc, "jvrc_walk", names)
    assert pe["length"] == [400, 100, 400, 20] and pe["fell"] == [False, True, False, True]
    assert pe["tracking"]["FORWARD"]["yaw_rate_error_sum"] == [0, 10, 30, 0]


@pytest.mark.parametrize("extra, message", [(["--num-envs", "0"], "at least one environment"),
                                            (["--num-envs", "4", "--out-dir", "x"], "cannot be combined"),
                                            (["--report", "r.json"], "add --num-envs"),
                                            (["--precision", "32"], "add --num-envs")])
def test_command_line_refuses_before_building_anything(tmp_path, extra, message):
    """The refusals come before the actor is even looked for (the run directory here does not exist)."""
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(tmp_path / "missing"), *extra])


def test_op_and_c_abi_are_registered():
    """torch.ops.lhw.sim_eval_accumulate exists and checks its handle before anything else; the C-ABI's word count is the
    accumulator width this module and rl/evaluation.py assume."""
    import torch
    import __graft_entry__
    __graft_entry__.build()
    from learninghumanoidwalking_b200 import _lib
    from learninghumanoidwalking_b200.rl import evaluation
    assert _lib.lib().lhw_sim_eval_words() == WORDS == evaluation.WORDS
    r = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="null sim handle"):
        _lib.ops().sim_eval_accumulate(0, r, r.int(), r[:, 0], r, r[:, 0].int(), r.double())
