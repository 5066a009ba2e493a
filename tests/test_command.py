"""Held walking commands (`env.set_command`, `eval --command`, DESIGN.md §7.6), CPU tier.

The product's command body and signed-velocity accumulator (csrc/sim_core.h set_command_env / command_accumulate_env, the per-env
bodies of lhw_sim_set_command and lhw_sim_command_accumulate) run on the host (tests/emu/command_emu.cpp) over records of the
kernel source's host emulation of the three walking variants, at fp64 and fp32.  The command body must write exactly what a numpy
recomputation from the record layout says, the accumulator must equal a float64 numpy recomputation, and closed-loop roll-outs of
the emulation with held commands must stay with the oracle given the same commands.  Also: the sweep's cells and summary, and the
command line's grammar and refusals."""
import ctypes
import os
import pickle
from argparse import Namespace

import numpy as np
import pytest

import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
WALKING = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk")
STANDING, INPLACE, FORWARD = 0, 1, 2
HELD = 1 << 30
C_WORDS, EV_LEN, EV_WORDS = 5, 0, 27


def _lib():
    lib = emu_variants._build("command_emu.cpp", "command_emu.cpp", os.path.join(HERE, "emu", "_build", "libcommand_emu.so"), [])
    L = ctypes.CDLL(lib)
    L.command_emu_set.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 4
    L.command_emu_accumulate.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _layout(nu):
    """Record positions from the dimensions alone: mode_ref follows qpos qvel qacc_warm and five NU-blocks; the obs task words are
    the last six (after the robot state and the two clock words)."""
    nv = 6 + nu
    nq = nv + 1
    return nq, nq + 2 * nv + 5 * nu


def set_command(L, var, prec, e, mode, ref, obs):
    given = np.zeros(e.n, np.int32)
    rc = L.command_emu_set(var, prec, _p(e.sr), _p(e.si), e.n, _p(np.ascontiguousarray(mode, np.int32)),
                           _p(np.ascontiguousarray(ref, e.dt)), _p(obs), _p(given))
    return rc, given.astype(bool)


def _records(name, prec, n=48, seed=5):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    flat = pack_model(load_model(name), tolerance=None if prec == 64 else 1e-6)
    e = emu_variants.Emu(flat, prec, n, seed=seed)
    e.reset()
    rng = np.random.RandomState(seed)
    obs = None
    for _ in range(20):
        obs = e.step(rng.normal(size=(n, e.nu)) * 0.5, max_traj_len=400)[0]
    return int(flat[0]), e, obs


def _command(n, seed):
    rng = np.random.RandomState(seed)
    mode = rng.randint(-1, 3, size=n).astype(np.int32)
    ref = rng.uniform(-1, 1, size=(n, 3))
    return mode, ref


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", WALKING)
def test_command_body_equals_numpy(name, precision):
    L = _lib()
    var, e, obs = _records(name, precision)
    nq, mode_ref = _layout(e.nu)
    mode, ref = _command(e.n, 1)
    ref = ref.astype(e.dt)
    sr0, si0, obs0 = e.sr.copy(), e.si.copy(), obs.copy()
    rc, given = set_command(L, var, precision, e, mode, ref, obs)
    assert rc == 0 and np.array_equal(given, mode >= 0) and 0 < given.sum() < e.n
    # untouched rows, and every other word of the touched ones, are bit-equal
    assert np.array_equal(e.sr[~given], sr0[~given]) and np.array_equal(e.si[~given], si0[~given])
    assert np.array_equal(obs[~given], obs0[~given])
    other = np.ones(e.nr, bool)
    other[mode_ref:mode_ref + 3] = False
    assert np.array_equal(e.sr[:, other], sr0[:, other])
    assert np.array_equal(e.sr[given, mode_ref:mode_ref + 3], ref[given])
    si_other = np.ones(e.si.shape[1], bool)
    si_other[1] = False
    assert np.array_equal(e.si[:, si_other], si0[:, si_other])
    assert np.array_equal(e.si[given, 1], mode[given] | HELD)
    task = np.zeros((e.n, 6), e.dt)
    task[:, 0], task[:, 1], task[:, 2] = mode == FORWARD, mode == INPLACE, mode == STANDING
    task[:, 3:] = ref
    assert np.array_equal(obs[given, -6:], task[given])
    assert np.array_equal(obs[:, :-6], obs0[:, :-6])
    # what env_obs writes for the held record: the next step's task words of every env that did not end
    nxt = e.step(np.zeros((e.n, e.nu)), max_traj_len=400)
    alive = given & (nxt[5] == 0)
    assert alive.sum() > 0
    assert np.array_equal(nxt[0][alive, -6:], task[alive])
    assert np.array_equal(e.si[alive, 1], mode[alive] | HELD)


@pytest.mark.parametrize("name", ["h1", "jvrc_step"])
def test_command_body_refuses_other_tasks(name):
    L = _lib()
    from learninghumanoidwalking_b200.model import load_model, pack_model
    flat = pack_model(load_model(name))
    e = emu_variants.Emu(flat, 64, 4)
    e.reset()
    si0 = e.si.copy()
    rc, _ = set_command(L, int(flat[0]), 64, e, np.full(4, FORWARD), np.zeros((4, 3)), np.zeros((4, e.nobs)))
    assert rc == -2 and np.array_equal(e.si, si0)


def _oracle(name):
    from oracle.oracle import Oracle
    if name == "h1_walk":
        from h1_walk_oracle import H1WalkOracle
        return H1WalkOracle(tolerance=1e-14)
    return Oracle(name, tolerance=1e-14)


@pytest.mark.parametrize("name", WALKING)
def test_held_rollout_matches_oracle(name):
    """16 envs x 300 closed-loop autoreset steps: env i % 4 == 3 is never commanded, the others hold FORWARD, INPLACE or STANDING
    (i % 3) and get their command again after each reset, in the emulation through the host command body.  The oracle has no
    hold: it gets the same mode and mode_ref through its fields, and after every step in which its random switch fired for a
    commanded env (its terminal observation's task words differ from the command) the command is written back.  The oracle's
    switch runs after the physics of its step, so only that step's reward terms and task words of that env are its own; they are
    left out of the comparison, and the emulation's must be the command's.  A held mode never changes within an episode, every
    reset clears the hold, the uncommanded envs still switch, and obs, reward terms, qpos and qvel agree within the bound of the
    pushed roll-outs."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    L = _lib()
    N, seed, first_id = 16, 13, 2
    flat = pack_model(load_model(name), tolerance=1e-14)
    var = int(flat[0])
    o = _oracle(name)
    e = emu_variants.Emu(flat, 64, N, seed=seed, first_id=first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    eo = e.reset()
    assert np.abs(o.batch_reset(envs, N) - eo).max() < 1e-10
    nq, nv = e.nq, e.nv
    mr = _layout(e.nu)[1]
    cmd_mode = np.where(np.arange(N) % 4 == 3, -1, np.arange(N) % 3).astype(np.int32)
    cmd_ref = np.array([[0, 0, 0], [0.3, 0, 0], [0, 0.25, 0]])[np.maximum(cmd_mode, 0)]
    cmd_ref[cmd_mode < 0] = 0
    held = cmd_mode >= 0
    task = np.zeros((N, 6))
    task[:, 0], task[:, 1], task[:, 2] = cmd_mode == FORWARD, cmd_mode == INPLACE, cmd_mode == STANDING
    task[:, 3:] = cmd_ref

    def command(which):
        m = np.where(which, cmd_mode, -1).astype(np.int32)
        rc, given = set_command(L, var, 64, e, m, cmd_ref, np.zeros((N, e.nobs)))
        assert rc == 0

    def oracle_command(which):
        for i in np.flatnonzero(which & held):
            o.set_field(envs, i, "mode", cmd_mode[i])
            o.set_field(envs, i, "mode_ref", cmd_ref[i])

    command(np.ones(N, bool))
    oracle_command(np.ones(N, bool))
    rng = np.random.RandomState(4)
    worst, n_end, n_fired, free_modes = 0.0, 0, 0, [set() for _ in range(N)]
    for t in range(300):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = o.batch_step(envs, N, a, max_traj_len=60)
        eo_, et, etm, er, ed, een, _, _ = e.step(a, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        ended = een != 0
        # the emulation's step kept the command: its observation carries it (the terminal one where the step ended the env)
        assert np.array_equal(np.where(ended[:, None], et, eo_)[held, -6:], task[held]), t
        fired = held & (np.abs(to[:, -6:] - task).max(1) > 0)
        n_fired += int(fired.sum())
        assert (e.si[held & ~ended, 1] == (cmd_mode | HELD)[held & ~ended]).all(), t
        assert (e.si[ended, 1] & HELD == 0).all(), t
        assert np.array_equal(e.sr[held & ~ended, mr:mr + 3], cmd_ref[held & ~ended])
        for i in np.flatnonzero(~held & ~ended):
            free_modes[i].add(int(e.si[i, 1]))
        same = ~fired
        task_words = np.ones(oo.shape[1], bool)
        task_words[-6:] = False
        oq = np.stack([o.field(envs, i, "qpos")[:nq] for i in range(N)])
        ov = np.stack([o.field(envs, i, "qvel")[:nv] for i in range(N)])
        worst = max(worst, np.abs(oo[same] - eo_[same]).max(initial=0), np.abs(oo[:, task_words] - eo_[:, task_words]).max(),
                    np.abs((oo - eo_)[ended]).max(initial=0), np.abs(tt[same] - etm[same]).max(initial=0),
                    np.abs(rr[same] - er[same]).max(initial=0), np.abs(oq - e.qpos).max(), np.abs(ov - e.qvel).max())
        n_end += int(ended.sum())
        command(ended)
        oracle_command(ended | fired)
    assert worst < 1e-7, worst
    assert n_end > 0 and n_fired > 0 and any(len(m) > 1 for m in free_modes), (n_end, n_fired, free_modes)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", WALKING)
def test_accumulator_equals_numpy(name, precision):
    """An autoreset-off roll-out with held commands (large actions on half of the envs, so that they fall): the signed-velocity
    records equal a float64 numpy recomputation bit for bit, and their step counts equal the evaluation accumulator's EV_LEN."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    eval_lib = ctypes.CDLL(emu_variants._build("eval_emu.cpp", "eval_emu.cpp", os.path.join(HERE, "emu", "_build", "libeval_emu.so"), []))
    eval_lib.eval_emu_accumulate.argtypes = [ctypes.c_int, ctypes.c_int] + [ctypes.c_void_p] * 2 + [ctypes.c_int] + [ctypes.c_void_p] * 4
    L = _lib()
    assert L.command_emu_words() == C_WORDS
    n, steps = 16, 40
    flat = pack_model(load_model(name), tolerance=None if precision == 64 else 1e-6)
    var = int(flat[0])
    e = emu_variants.Emu(flat, precision, n, seed=9)
    obs = e.reset()
    nq = e.nq
    mode = (np.arange(n) % 3).astype(np.int32)
    ref = np.array([[0, 0, 0], [-0.4, 0, 0], [0, 0.3, 0]])[mode]
    assert set_command(L, var, precision, e, mode, ref, obs)[0] == 0
    acc, ev = np.zeros((n, C_WORDS)), np.zeros((n, EV_WORDS))
    want = np.zeros((n, C_WORDS))
    rng = np.random.RandomState(9)
    scale = np.where(np.arange(n) % 2 == 0, 1.5, 0.02)[:, None]
    for _ in range(steps):
        _, _, terms, rew, done, _, _, _ = e.step(rng.normal(size=(n, e.nu)) * scale, max_traj_len=steps, autoreset=0)
        assert L.command_emu_accumulate(var, precision, _p(e.sr), n, _p(done), _p(acc)) == 0
        assert eval_lib.eval_emu_accumulate(var, precision, _p(e.sr), _p(e.si), n, _p(rew), _p(terms), _p(done), _p(ev)) == 0
        sr = e.sr.astype(np.float64)
        for i in range(n):
            if want[i, 4] != 0:
                continue
            qw, x, y, z = sr[i, 3:7]
            s = 2 / (qw * qw + x * x + y * y + z * z)
            X, Y, Z = x * s, y * s, z * s
            wX, wY, wZ, xX, xY, xZ, yY, yZ, zZ = qw * X, qw * Y, qw * Z, x * X, x * Y, x * Z, y * Y, y * Z, z * Z
            v0, v1, v2 = sr[i, nq:nq + 3]
            want[i, :4] += (1.0, (1 - (yY + zZ)) * v0 + (xY + wZ) * v1 + (xZ - wY) * v2,
                            (xY - wZ) * v0 + (1 - (xX + zZ)) * v1 + (yZ + wX) * v2, sr[i, nq + 5])
            if done[i]:
                want[i, 4] = 1
    assert np.array_equal(acc, want), np.abs(acc - want).max()
    assert np.array_equal(acc[:, 0], ev[:, EV_LEN])
    fell = acc[:, 4] != 0
    assert fell.any() and (~fell).any() and (acc[~fell, 0] == steps).all()
    # the held mode is the only one tracked
    for m in range(3):
        assert np.array_equal(ev[:, 13 + 4 * m], np.where(mode == m, ev[:, EV_LEN], 0))


def test_sweep_cells_and_summary():
    from learninghumanoidwalking_b200.rl import evaluation as ev
    cells = [("FORWARD", 0.0), ("FORWARD", 0.2), ("INPLACE", -0.4), ("STANDING", 0.0)]
    mode, value = ev.command_grid(10, cells)
    assert mode.tolist() == [2, 2, 1, 0] * 2 + [2, 2] and value.tolist() == [0, 0.2, -0.4, 0] * 2 + [0, 0.2]
    ref = ev.command_refs(mode, value)
    assert ref[1].tolist() == [0, 0.2, 0] and ref[2].tolist() == [-0.4, 0, 0] and ref[3].tolist() == [0, 0, 0]
    acc, cacc = np.zeros((10, ev.WORDS)), np.zeros((10, ev.C_WORDS))
    acc[:, ev.LEN] = cacc[:, ev.C_LEN] = [400, 400, 100, 400, 400, 200, 400, 400, 400, 400]
    acc[:, ev.DONE] = cacc[:, ev.C_DONE] = [0, 0, 1, 0, 0, 1, 0, 0, 0, 0]
    cacc[:, ev.C_VF] = cacc[:, ev.C_LEN] * np.array([0.0, 0.25, 0, 0, 0.1, 0.15, 0, 0, 0.05, 0.2])
    cacc[:, ev.C_WZ] = cacc[:, ev.C_LEN] * np.array([0, 0, -0.3, 0, 0, 0, -0.5, 0, 0, 0])
    for i in range(10):
        m = int(mode[i])
        acc[i, ev.TRACK + 4 * m] = acc[i, ev.LEN]
        acc[i, ev.TRACK + 4 * m + 1] = 0.01 * acc[i, ev.LEN] * (i + 1)
    c = ev.command_summary(acc, cacc, mode, value, cells)["cells"]
    assert [x["n"] for x in c] == [3, 3, 2, 2]
    f = c[1]    # FORWARD 0.2: envs 1, 5, 9 -> per-env means 0.25, 0.15, 0.2
    assert f["mode"] == "FORWARD" and f["ref"] == dict(yaw_rate=0.0, vx=0.2, vy=0.0)
    assert f["fall_fraction"] == pytest.approx(1 / 3) and f["mean_length"] == pytest.approx(1000 / 3)
    assert f["achieved"]["v_fwd"]["mean"] == pytest.approx(0.2) and f["achieved"]["v_fwd"]["std"] == pytest.approx(np.std([0.25, 0.15, 0.2]))
    assert f["tracking"]["steps"] == 1000 and f["tracking"]["vx_error"] == pytest.approx(0.01 * (400 * 2 + 200 * 6 + 400 * 10) / 1000)
    assert c[2]["achieved"]["yaw_rate"]["mean"] == pytest.approx(-0.4) and c[2]["fall_fraction"] == 0.5
    table = ev.format_command_table(dict(cells=c))
    assert "forward 0.2" in table and "inplace -0.4" in table and "standing " in table


def _eval_args(**kw):
    base = dict(command=None, num_envs=None, push_speeds=None)
    base.update(kw)
    return Namespace(**base)


def test_command_grammar():
    import run_experiment as rx
    cells = rx.command_cells(_eval_args(command=["forward:0,0.2,0.4", "inplace:-0.4,0.4", "standing"], num_envs=256))
    assert cells == [("FORWARD", 0.0), ("FORWARD", 0.2), ("FORWARD", 0.4), ("INPLACE", -0.4), ("INPLACE", 0.4), ("STANDING", 0.0)]
    assert rx.command_cells(_eval_args(command=["forward:0.9"])) == [("FORWARD", 0.9)]    # outside the training range: allowed
    assert rx.command_cells(_eval_args()) is None
    # repeatable and nargs="+" alike
    import argparse
    p = argparse.ArgumentParser()
    for flag, kw in rx.EVAL_FLAGS:
        p.add_argument(flag, **kw)
    assert p.parse_args(["--command", "forward:0.1", "standing", "--command", "inplace:0.2"]).command == \
        ["forward:0.1", "standing", "inplace:0.2"]


@pytest.mark.parametrize("extra, message", [(["--command", "sideways:1"], "unknown mode"),
                                            (["--command", "standing:0"], "standing takes no values"),
                                            (["--command", "forward:"], "comma-separated numbers"),
                                            (["--command", "forward:0.1,x"], "comma-separated numbers"),
                                            (["--command", "forward:nan"], "must be finite"),
                                            (["--command", "inplace:inf"], "must be finite"),
                                            (["--command", "forward:0.1,0.2"], "add --num-envs"),
                                            (["--command", "forward:0.1", "standing"], "add --num-envs"),
                                            (["--num-envs", "2", "--command", "forward:0,0.2", "standing"], "3 cells"),
                                            (["--num-envs", "64", "--command", "standing", "--push-speeds", "1"], "separate sweeps")])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Every refusal comes before an actor is looked for (the run directory here has none)."""
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(tmp_path / "no_run"), *extra])


@pytest.mark.parametrize("env_name", ["h1", "jvrc_step"])
@pytest.mark.parametrize("extra", [[], ["--num-envs", "8"]])
def test_eval_refuses_runs_without_a_walking_command(tmp_path, env_name, extra):
    """The run's env comes from its experiment.pkl, which is read before the actor is loaded (the directory has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env=env_name, max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=f"{env_name} has no walking command"):
        rx.main(["eval", "--path", str(run), "--command", "standing", *extra])


def test_ops_and_c_abi_are_registered():
    """torch.ops.lhw.sim_set_command and .sim_command_accumulate exist and check their handle before anything else."""
    import torch
    import __graft_entry__
    __graft_entry__.build()
    from learninghumanoidwalking_b200 import _lib as lhw
    assert lhw.lib().lhw_version() == 3 and lhw.lib().lhw_sim_command_words() == C_WORDS
    r = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="null sim handle"):
        lhw.ops().sim_set_command(0, r, r.int(), r[:, 0].int().contiguous(), r, r)
    with pytest.raises(RuntimeError, match="null sim handle"):
        lhw.ops().sim_command_accumulate(0, r, r[:, 0].int().contiguous(), r.double())
