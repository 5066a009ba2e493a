"""Root-velocity pushes (`train --push-vel`, `eval --push-speeds`, DESIGN.md §7.5), CPU tier.

The product's push body (csrc/sim_core.h push_env, the per-env body of lhw_sim_push) runs on the host (tests/emu/push_emu.cpp)
over records of the kernel source's host emulation of every variant, at fp64 and fp32.  Its pushed set and velocity changes must
equal a float64 numpy recomputation that draws with the oracle's Philox and takes the record layout from the dimensions alone.
Pushed closed-loop roll-outs of the emulation must stay with the oracle, which gets the same kicks through its qvel field.  Also:
the sweep's grid and statistics, and the command line's refusals."""
import ctypes
import os
import pickle
from argparse import Namespace

import numpy as np
import pytest

import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
PUSH_STREAM = 70


def _lib():
    lib = emu_variants._build("push_emu.cpp", "push_emu.cpp", os.path.join(HERE, "emu", "_build", "libpush_emu.so"), [])
    L = ctypes.CDLL(lib)
    L.push_emu.argtypes = ([ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_uint32,
                            ctypes.c_void_p, ctypes.c_double, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p])
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(ctypes.c_void_p)


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def push(L, var, prec, e, seed, first_id, ended=None, vel=0.0, interval=1, d=None):
    """One launch of the host push body over the emulation's records; returns the pushed flags."""
    pushed = np.zeros(e.n, np.int32)
    assert L.push_emu(var, prec, _p(e.sr), _p(e.si), e.n, seed, first_id, _p(ended), vel, interval, _p(d), _p(pushed)) == 0
    return pushed


def heading_dv(sr, nq, d):
    """float64 numpy: Rz(psi) d per env, psi = yaw of the (normalised) root quaternion sr[:, 3:7]."""
    q = sr[:, 3:7].astype(np.float64)
    q = q / np.linalg.norm(q, axis=1, keepdims=True)
    w, x, y, z = q.T
    psi = np.arctan2(2 * (w * z + x * y), 1 - 2 * (y * y + z * z))
    c, s = np.cos(psi), np.sin(psi)
    return np.stack((c * d[:, 0] - s * d[:, 1], s * d[:, 0] + c * d[:, 1]), axis=1)


def random_draws(philox, seed, first_id, si, ended, vel, interval):
    """float64 numpy: which envs the random mode pushes and their heading-frame (dx, dy)."""
    n = si.shape[0]
    pushed, d = np.zeros(n, bool), np.zeros((n, 2))
    for i in range(n):
        u = philox(seed, first_id + i, int(si[i, 4]) & 0xFFFFFFFF, PUSH_STREAM)
        if ended[i] or (u[0] * interval) >> 32 != 0:
            continue
        pushed[i] = True
        d[i] = vel * (2 * ((u[1] >> 8) / 16777216.0) - 1), vel * (2 * ((u[2] >> 8) / 16777216.0) - 1)
    return pushed, d


def check_push(before, after, nq, pushed, d, rel):
    """`after` equals `before` everywhere but qvel[0:2] of the pushed envs, which is old + Rz(psi) d."""
    other = np.ones(before.shape[1], bool)
    other[nq:nq + 2] = False
    assert np.array_equal(after[:, other], before[:, other])
    assert np.array_equal(after[~pushed], before[~pushed])
    want = before[pushed, nq:nq + 2].astype(np.float64) + heading_dv(before[pushed], nq, d[pushed])
    err = np.abs(after[pushed, nq:nq + 2] - want) / np.maximum(1.0, np.abs(want))
    assert err.max(initial=0) <= rel, err.max()


def _records(name, prec, n=64, seed=7, first_id=3):
    """An emulation batch after a closed-loop autoreset roll-out with large actions: varied headings, some envs just ended."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    e = emu_variants.Emu(pack_model(load_model(name), tolerance=None if prec == 64 else 1e-6), prec, n, seed=seed, first_id=first_id)
    e.reset()
    rng = np.random.RandomState(seed)
    ended = np.zeros(n, np.int32)
    for _ in range(25):
        ended = e.step(rng.normal(size=(n, e.nu)) * 0.8, max_traj_len=400)[5].astype(np.int32)
    return e, ended


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_push_body_equals_numpy(name, precision, philox):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    L = _lib()
    var = int(pack_model(load_model(name))[0])
    seed, first_id = 7, 3
    e, ended = _records(name, precision, seed=seed, first_id=first_id)
    nq = e.nq
    rel = 1e-12 if precision == 64 else 1e-6
    ended[::5] = 1                                          # and some more, so that skipping them is seen
    # random mode: a push every 3 control steps on average, up to 1.5 m/s per axis
    before = e.sr.copy()
    got = push(L, var, precision, e, seed, first_id, ended=ended, vel=1.5, interval=3).astype(bool)
    want, d = random_draws(philox, seed, first_id, e.si, ended, 1.5, 3)
    assert np.array_equal(got, want)
    assert 0 < want.sum() < e.n and not (want & (ended != 0)).any()
    check_push(before, e.sr, nq, want, d, rel)
    assert np.array_equal(e.sr[ended != 0], before[ended != 0])
    # interval 1: every env that did not just end
    before = e.sr.copy()
    got = push(L, var, precision, e, seed, first_id, ended=ended, vel=0.25, interval=1).astype(bool)
    assert np.array_equal(got, ended == 0)
    check_push(before, e.sr, nq, got, random_draws(philox, seed, first_id, e.si, ended, 0.25, 1)[1], rel)
    # explicit mode: a random d, with some rows exactly zero (skipped) and some with one zero component (pushed)
    rng = np.random.RandomState(1)
    d = (rng.normal(size=(e.n, 2)) * 2).astype(e.dt)
    d[::4] = 0
    d[1::8, 0] = 0
    before = e.sr.copy()
    got = push(L, var, precision, e, seed, first_id, d=d).astype(bool)
    assert np.array_equal(got, np.abs(d).sum(1) != 0)
    check_push(before, e.sr, nq, got, d.astype(np.float64), rel)
    assert np.array_equal(e.sr[::4], before[::4])
    # the heading frame: a forward push of a robot facing +y moves it along +y
    e.sr[0, 3:7] = np.array([np.cos(np.pi / 4), 0, 0, np.sin(np.pi / 4)], dtype=e.dt)
    v0 = e.sr[0, nq:nq + 2].astype(np.float64).copy()
    one = np.zeros((e.n, 2), e.dt)
    one[0] = 1, 0
    push(L, var, precision, e, seed, first_id, d=one)
    assert np.abs(e.sr[0, nq:nq + 2] - v0 - [0, 1]).max() < (1e-15 if precision == 64 else 1e-6)


def _oracle(name):
    from oracle.oracle import Oracle
    if name == "h1_walk":
        from h1_walk_oracle import H1WalkOracle
        return H1WalkOracle(tolerance=1e-14)
    return Oracle(name, tolerance=1e-14)


@pytest.mark.parametrize("name", VARIANTS)
def test_pushed_rollout_matches_oracle(name):
    """16 envs x 300 closed-loop steps with a random push about every 20 steps (1 m/s per axis at most): after each step the host
    push body kicks the emulation's records, and the oracle's qvel[0:2] gets the same values.  Falls, truncations and resets
    included; obs, reward terms, qpos and qvel agree within the bound of the h1_walk kernel-source test."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    L = _lib()
    N, seed, first_id = 16, 11, 5
    flat = pack_model(load_model(name), tolerance=1e-14)
    var = int(flat[0])
    o = _oracle(name)
    e = emu_variants.Emu(flat, 64, N, seed=seed, first_id=first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    assert np.abs(o.batch_reset(envs, N) - e.reset()).max() < 1e-10
    nq, nv = e.nq, e.nv
    rng = np.random.RandomState(2)
    worst, n_push, n_end = 0.0, 0, 0
    for t in range(300):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = o.batch_step(envs, N, a, max_traj_len=60)
        eo, et, etm, er, ed, een, _, _ = e.step(a, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        pushed = push(L, var, 64, e, seed, first_id, ended=een.astype(np.int32), vel=1.0, interval=20).astype(bool)
        for i in np.flatnonzero(pushed):
            qv = o.field(envs, i, "qvel")
            qv[0:2] = e.sr[i, nq:nq + 2]
            o.set_field(envs, i, "qvel", qv)
        n_push += int(pushed.sum())
        n_end += int(een.sum())
        oq = np.stack([o.field(envs, i, "qpos")[:nq] for i in range(N)])
        ov = np.stack([o.field(envs, i, "qvel")[:nv] for i in range(N)])
        worst = max(worst, np.abs(oo - eo).max(), np.abs(tt - etm).max(), np.abs(rr - er).max(), np.abs(oq - e.qpos).max(),
                    np.abs(ov - e.qvel).max())
    assert worst < 1e-7, worst
    assert n_push > 150 and n_end > 0, (n_push, n_end)


def test_sweep_grid_and_statistics():
    from learninghumanoidwalking_b200.rl import evaluation as ev
    speed, deg = ev.push_grid(10, [0.0, 1.5], 4)
    assert speed.tolist() == [0, 0, 0, 0, 1.5, 1.5, 1.5, 1.5, 0, 0] and deg.tolist() == [0, 90, 180, 270] * 2 + [0, 90]
    d = ev.push_vectors(speed, deg)
    assert np.allclose(d[4], [1.5, 0]) and np.allclose(d[5], [0, 1.5]) and np.allclose(d[6], [-1.5, 0]) and not d[:4].any()
    acc = np.zeros((10, ev.WORDS))
    acc[:, ev.LEN] = [400, 30, 400, 400, 400, 100, 50, 400, 20, 400]
    acc[:, ev.DONE] = [0, 1, 0, 0, 0, 1, 1, 0, 1, 0]
    p = ev.push_summary(acc, speed, deg, [0.0, 1.5], 4, 2.0, 50)
    c = p["cells"]
    assert [x["n"] for x in c] == [2, 2, 1, 1, 1, 1, 1, 1]
    assert c[0] == dict(speed=0.0, direction_deg=0.0, n=2, fell_before_push=1, alive_at_push=1, survived=1, survival=1.0)
    assert c[1]["fell_before_push"] == 1 and c[1]["survival"] == 1.0             # env 1 fell at step 30, env 9 stood
    assert c[5]["alive_at_push"] == 1 and c[5]["survived"] == 0 and c[5]["survival"] == 0.0   # fell at 100, after the push
    assert c[6]["fell_before_push"] == 1 and c[6]["survival"] is None            # fell at step 50 = K: before the push
    assert p["per_speed"][1] == dict(speed=1.5, alive_at_push=3, survived=2, survival=2 / 3)
    assert p["directions_deg"] == [0, 90, 180, 270] and p["push_step"] == 50
    table = ev.format_push_table(p)
    assert "0.667" in table and "1.000" in table and "-" in table


def test_env_refuses_bad_push_arguments():
    from learninghumanoidwalking_b200.envs.batched_env import push_interval_steps
    assert push_interval_steps(1.0, 15.0, 0.025) == 600 and push_interval_steps(0.0, 0.025, 0.025) == 1
    for vel, interval in ((-0.1, 15.0), (float("nan"), 15.0), (float("inf"), 15.0), (1.0, 0.01), (1.0, float("nan")), (1.0, 0.0)):
        with pytest.raises(ValueError):
            push_interval_steps(vel, interval, 0.025)


@pytest.mark.parametrize("extra, message", [(["--push-vel", "-1"], "finite speed"), (["--push-vel", "nan"], "finite speed"),
                                            (["--push-vel", "1", "--push-interval", "0.01"], "at least one control step")])
def test_train_refuses_before_building_anything(tmp_path, extra, message, monkeypatch):
    import run_experiment as rx
    monkeypatch.setattr(rx, "make_env_fn", lambda *a, **k: pytest.fail("an environment was built"))
    with pytest.raises(SystemExit, match=message):
        rx.main(["train", "--env", "jvrc_walk", "--logdir", str(tmp_path / "logs"), *extra])
    assert not (tmp_path / "logs").exists()


@pytest.mark.parametrize("extra, message", [(["--push-speeds", "0,1"], "add --num-envs"),
                                            (["--push-at", "1"], "add --num-envs"),
                                            (["--num-envs", "4", "--push-directions", "2"], "add --push-speeds"),
                                            (["--num-envs", "15", "--push-speeds", "0,1"], "16 cells"),
                                            (["--num-envs", "64", "--push-speeds", "0,-1"], "finite and >= 0"),
                                            (["--num-envs", "64", "--push-speeds", "0,inf"], "finite and >= 0"),
                                            (["--num-envs", "64", "--push-speeds", "0,x"], "comma-separated"),
                                            (["--num-envs", "64", "--push-speeds", "1", "--push-directions", "0"], "at least one direction"),
                                            (["--num-envs", "64", "--push-speeds", "1", "--push-at", "nan"], "finite"),
                                            (["--num-envs", "64", "--push-speeds", "1", "--push-at", "0"], "after control step 0"),
                                            (["--num-envs", "64", "--push-speeds", "1", "--push-at", "10"], "after control step 400")])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """The grid refusals come before the actor is looked for; the push step's, which need the run's control step and horizon,
    after its experiment.pkl is read and before the actor is loaded (the run directory here has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(run), *extra])


def test_op_and_c_abi_are_registered():
    """torch.ops.lhw.sim_push exists and checks its handle before anything else."""
    import torch
    import __graft_entry__
    __graft_entry__.build()
    from learninghumanoidwalking_b200 import _lib as lhw
    assert lhw.lib().lhw_version() == 3
    r = torch.zeros(4, 3)
    with pytest.raises(RuntimeError, match="null sim handle"):
        lhw.ops().sim_push(0, r, r.int(), 0, 0, None, 0.0, 1, r[:, :2].contiguous())
