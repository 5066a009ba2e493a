"""Sensor errors for every environment (`train --sensor-noise M --sensor-bias O,G,E`, `eval --sensor-errors ...`, DESIGN.md §7.12),
CPU tier.

The sensor pass (csrc/sim_core.h sensor_env, the body of lhw_sim_sense's kernel) runs on the host (tests/emu/sensor_emu.cpp) for
every variant's (NROBOT, NU, obs_dim) at fp64 and fp32 and is held bit for bit to a numpy restatement with the oracle's Philox: in
both phases, with and without autoreset, with masks, ended flags, random and explicit rows and the draw.  Task words are never
written, an all-zero row leaves every bit of an observation, without autoreset term_obs stays equal to obs, and closed-loop
roll-outs of the host step plus the pass keep the records, rewards and dones of roll-outs without it.  Also: the noise scales
against model/h1.json, and every refusal of the env helpers and the command line."""
import ctypes
import json
import os
import pickle
import re
from argparse import Namespace

import numpy as np
import pytest

import emu
import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
# (NROBOT, NU, obs_dim) of each variant: the robot-state words lead the observation (csrc/sim_core.h Dims::NROBOT)
DIMS = {"jvrc_walk": (29, 12, 37), "jvrc_walk_terrain": (29, 12, 37), "jvrc_step": (29, 12, 39), "h1": (35, 10, 35),
        "h1_walk": (35, 10, 43)}
BIAS_STREAM, OBS_STREAM, TERM_STREAM = 80, 96, 112
SCALES = (0.05, 0.05, 0.02, 0.05, 5.0)     # orient, gyro, motor_pos, motor_vel, motor_tau
BOUNDS = (0.2, 0.5, 0.2)                   # roll / pitch, gyro, encoder


def _lib_path():
    return emu_variants._build("sensor_emu.cpp", "sim_emu_variants.cpp", os.path.join(HERE, "emu", "_build", "libsensor_emu.so"), [])


def _lib():
    return ctypes.CDLL(_lib_path())


class SensorEmu(emu_variants.Emu):
    """emu_variants.Emu on the library of sensor_emu.cpp (sim_emu_variants.cpp's entry points plus sensor_emu_sense)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = _lib_path()
        self.raw = ctypes.CDLL(lib)
        self.lib = emu_variants._Lib(lib, "emu_", "emuv_")
        self.lib.emu_create.restype = ctypes.c_void_p
        flat = np.ascontiguousarray(flat, dtype=np.float64)
        self.h = ctypes.c_void_p(self.lib.emu_create(flat.ctypes.data_as(ctypes.c_void_p), len(flat), precision))
        assert self.h.value, "emu_create failed"
        self.prec, self.n, self.seed, self.first_id = precision, n, seed, first_id
        self.dt = np.float64 if precision == 64 else np.float32
        self.nr = self.lib.emu_state_words(self.h)
        self.nobs = self.lib.emu_obs_dim(self.h)
        self.nu = 2 * (int(flat[0]) % 100)
        self.nq, self.nv = 7 + self.nu, 6 + self.nu
        self.sr = np.zeros((n, self.nr), dtype=self.dt)
        self.si = np.zeros((n, emu.NSTATE_I), dtype=np.int32)


def sense(precision, si, seed, first_id, sel, after_step, autoreset, draw, nrobot, nu, sensor, obs, term_obs):
    """One host pass over every env (sensor_emu_sense); sensor, obs and term_obs are written in place."""
    dt = np.float64 if precision == 64 else np.float32
    for a in (sensor, obs) + (() if term_obs is None else (term_obs,)):
        assert a.dtype == dt and a.flags.c_contiguous
    p = lambda a: None if a is None else a.ctypes.data_as(ctypes.c_void_p)
    s = None if sel is None else np.ascontiguousarray(sel, np.int32)
    d = None if draw is None else np.ascontiguousarray(draw, np.float64)
    _lib().sensor_emu_sense(precision, p(np.ascontiguousarray(si, np.int32)), len(obs), ctypes.c_uint32(seed), ctypes.c_uint32(first_id),
                            p(s), int(after_step), int(autoreset), p(d), nrobot, nu, obs.shape[1], p(sensor), p(obs), p(term_obs))


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def _u01(x):
    return float(int(x) >> 8) * (1.0 / 16777216.0)


def _scale(i, nu):
    return SCALES[0 if i < 2 else 1 if i < 5 else 2 if i < 5 + nu else 3 if i < 5 + 2 * nu else 4]


def sense_numpy(philox, seed, first_id, si, sel, after_step, autoreset, draw, nrobot, nu, sensor, obs, term_obs):
    """numpy restatement of sensor_env over every env: returns new (sensor, obs, term_obs).  Float64 arithmetic, one rounding to
    the arrays' dtype per written word."""
    sensor, obs = sensor.copy(), obs.copy()
    term_obs = None if term_obs is None else term_obs.copy()
    dt = obs.dtype.type

    def apply(i_env, x, stream):
        row, ctr = sensor[i_env], int(si[i_env, 4]) & 0xFFFFFFFF
        m = float(row[0])
        for i in range(nrobot):
            b = float(row[1 + i]) if i < 5 + nu else 0.0
            a = m * _scale(i, nu)
            if b == 0 and a == 0:
                continue
            u = philox(seed, first_id + i_env, ctr, stream + i // 4)
            x[i] = dt(float(x[i]) + b + a * (2 * _u01(u[i % 4]) - 1))

    for e in range(len(obs)):
        s = 1 if sel is None else int(sel[e])
        if not after_step and not s:
            continue
        new_episode = not after_step or (autoreset and s)
        if after_step and new_episode:
            apply(e, term_obs[e], TERM_STREAM)
        if new_episode and draw is not None:
            ctr = int(si[e, 4]) & 0xFFFFFFFF
            for k in range(5 + nu):
                u = philox(seed, first_id + e, ctr, BIAS_STREAM + k // 4)
                sensor[e, 1 + k] = dt(draw[0 if k < 2 else 1 if k < 5 else 2] * (2 * _u01(u[k % 4]) - 1))
        apply(e, obs[e], OBS_STREAM)
        if after_step and not autoreset:
            term_obs[e, :nrobot] = obs[e, :nrobot]
    return sensor, obs, term_obs


def random_rows(rng, n, nu, dt):
    """Explicit rows of every kind: per-env multipliers in [0, 4] and offsets within their bounds, all-zero rows, noise-only rows,
    offset-only rows and rows with single zero offsets."""
    rows = np.zeros((n, 6 + nu))
    rows[:, 0] = rng.uniform(0, 4, size=n)
    bound = np.repeat(BOUNDS, [2, 3, nu])
    rows[:, 1:] = rng.uniform(-1, 1, size=(n, 5 + nu)) * bound
    rows[::5] = 0                         # error-free
    rows[1::5, 1:] = 0                    # noise only
    rows[2::5, 0] = 0                     # offsets only
    rows[3::5, 1 + rng.randint(0, 5 + nu, size=4)] = 0
    return rows.astype(dt)


def random_obs(rng, n, obs_dim, dt):
    obs = rng.normal(size=(n, obs_dim)).astype(dt)
    obs[::3, 3] = -0.0
    obs[1::4, 6] = -0.0
    return obs


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_pass_equals_numpy(name, precision, philox):
    """The host pass against the numpy restatement bit for bit (rows, obs and term_obs): after a reset (every env, a mask) and
    after a step with autoreset (random ended flags) and without, each with and without the draw, with explicit rows of every
    kind and per-env multipliers, at counters that differ per env."""
    nrobot, nu, obs_dim = DIMS[name]
    N, seed, first_id = 24, 13, 5
    dt = np.float64 if precision == 64 else np.float32
    rng = np.random.RandomState(1)
    si = np.zeros((N, emu.NSTATE_I), np.int32)
    si[:, 4] = rng.randint(0, 1 << 30, size=N)
    for after_step, autoreset in ((False, False), (True, True), (True, False)):
        for sel in (None, (rng.uniform(size=N) < 0.4).astype(np.int32) * rng.randint(1, 7, size=N)):
            if after_step and sel is None:
                continue
            for draw in (None, (0.2, 0.5, 0.2), (0.05, 0.0, 0.03)):
                sensor, obs = random_rows(rng, N, nu, dt), random_obs(rng, N, obs_dim, dt)
                term = None
                if after_step:
                    term = obs.copy() if not autoreset else random_obs(rng, N, obs_dim, dt)
                want = sense_numpy(philox, seed, first_id, si, sel, after_step, autoreset, draw, nrobot, nu, sensor, obs, term)
                sense(precision, si, seed, first_id, sel, after_step, autoreset, draw, nrobot, nu, sensor, obs, term)
                case = (after_step, autoreset, sel is None, draw)
                assert sensor.tobytes() == want[0].tobytes(), case
                assert obs.tobytes() == want[1].tobytes(), case
                if term is not None:
                    assert term.tobytes() == want[2].tobytes(), case


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_task_words_and_error_free_rows_are_untouched(name, precision):
    """The task words after NROBOT are never written, whatever the rows; an all-zero row leaves its env's obs and term_obs
    bit-identical, planted -0.0 words included; and without autoreset term_obs equals the treated obs bit for bit."""
    nrobot, nu, obs_dim = DIMS[name]
    N = 30
    dt = np.float64 if precision == 64 else np.float32
    rng = np.random.RandomState(2)
    si = np.zeros((N, emu.NSTATE_I), np.int32)
    si[:, 4] = np.arange(N) * 7
    rows = random_rows(rng, N, nu, dt)
    zero = ~rows.any(axis=1)
    assert zero.sum() >= 5 and (~zero).sum() >= 20
    for after_step, autoreset in ((False, False), (True, True), (True, False)):
        obs = random_obs(rng, N, obs_dim, dt)
        term = (obs.copy() if not autoreset else random_obs(rng, N, obs_dim, dt)) if after_step else None
        o0, t0 = obs.copy(), None if term is None else term.copy()
        ended = np.ones(N, np.int32) if after_step else None
        sense(precision, si, 3, 0, ended, after_step, autoreset, None, nrobot, nu, rows, obs, term)
        assert obs[:, nrobot:].tobytes() == o0[:, nrobot:].tobytes()
        assert obs[zero].tobytes() == o0[zero].tobytes()
        assert (obs[~zero, :nrobot] != o0[~zero, :nrobot]).any(axis=1).all()
        if term is not None:
            assert term[:, nrobot:].tobytes() == t0[:, nrobot:].tobytes() and term[zero].tobytes() == t0[zero].tobytes()
            if not autoreset:
                assert term.tobytes() == obs.tobytes()


@pytest.mark.parametrize("precision", [64, 32])
def test_draw_writes_only_offsets_within_bounds(precision, philox):
    """The draw of a reset: selected envs get offsets in their bounds (velocity and torque words have none), the multiplier is
    never written, unselected envs keep their rows and observations; the draw equals numpy."""
    nrobot, nu, obs_dim = DIMS["h1_walk"]
    N, seed = 200, 9
    dt = np.float64 if precision == 64 else np.float32
    rng = np.random.RandomState(4)
    si = np.zeros((N, emu.NSTATE_I), np.int32)
    si[:, 4] = rng.randint(0, 1000, size=N)
    rows = np.zeros((N, 6 + nu), dt)
    rows[:, 0] = rng.uniform(0, 4, size=N)
    rows[:, 1:] = 7          # no valid offset: every selected word must be redrawn
    mask = (rng.uniform(size=N) < 0.5).astype(np.int32)
    obs = random_obs(rng, N, obs_dim, dt)
    before_rows, before_obs = rows.copy(), obs.copy()
    want = sense_numpy(philox, seed, 0, si, mask, False, False, (0.1, 0.3, 0.05), nrobot, nu, rows, obs, None)
    sense(precision, si, seed, 0, mask, False, False, (0.1, 0.3, 0.05), nrobot, nu, rows, obs, None)
    assert rows.tobytes() == want[0].tobytes() and obs.tobytes() == want[1].tobytes()
    on = mask != 0
    assert rows[:, 0].tobytes() == before_rows[:, 0].tobytes()
    assert rows[~on].tobytes() == before_rows[~on].tobytes() and obs[~on].tobytes() == before_obs[~on].tobytes()
    b = rows[on, 1:].astype(np.float64)
    assert (np.abs(b[:, :2]) <= 0.1).all() and (np.abs(b[:, 2:5]) <= 0.3).all() and (np.abs(b[:, 5:]) <= 0.05).all()
    assert np.abs(b[:, 5:]).max() > 0.04 and np.abs(b[:, 2:5]).max() > 0.25


def _flat(name, prec):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model(name), tolerance=None if prec == 64 else 1e-6)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_closed_loop_records_are_those_without_the_pass(name, precision):
    """24 envs x 60 autoreset steps of max_traj_len 20 under one fixed action sequence: the host step followed by the pass in
    random mode (a multiplier of 2 and offsets redrawn at every auto-reset) against the host step alone.  Records, rewards, reward
    terms, done, ended and the episode words are bit-identical; the observations are not."""
    nrobot, nu, obs_dim = DIMS[name]
    flat = _flat(name, precision)
    N, seed, first_id = 24, 5, 3
    e, p = SensorEmu(flat, precision, N, seed, first_id), emu_variants.Emu(flat, precision, N, seed, first_id)
    assert (e.nobs, e.nu) == (obs_dim, nu)
    rows = np.zeros((N, 6 + nu), e.dt)
    rows[:, 0] = 2
    draw = (0.2, 0.5, 0.2)
    obs = e.reset()
    assert obs.tobytes() == p.reset().tobytes()
    sense(precision, e.si, seed, first_id, None, False, False, draw, nrobot, nu, rows, obs, None)
    rng = np.random.RandomState(0)
    n_end, differ = 0, 0
    for t in range(60):
        a = rng.normal(size=(N, nu)) * np.where(np.arange(N) % 4 == 3, 1.0, 0.15)[:, None]
        got, want = e.step(a, max_traj_len=20), p.step(a, max_traj_len=20)
        sense(precision, e.si, seed, first_id, got[5], True, True, draw, nrobot, nu, rows, got[0], got[1])
        for g, w in zip(got[2:], want[2:]):
            assert g.tobytes() == w.tobytes(), t
        assert e.sr.tobytes() == p.sr.tobytes() and np.array_equal(e.si, p.si), t
        assert got[0][:, nrobot:].tobytes() == want[0][:, nrobot:].tobytes(), t
        differ += int((got[0][:, :nrobot] != want[0][:, :nrobot]).any(axis=1).sum())
        n_end += int(got[5].sum())
    assert n_end > 0 and differ == 60 * N


def test_noise_scales_are_the_h1_scales():
    """The one table of noise scales in sim_core.h equals the reference's H1 observation_noise.scales (model/h1.json)."""
    src = open(os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", "sim_core.h")).read()
    got = {k: float(v) for k, v in re.findall(r"SENSOR_SCALE_(\w+) = ([0-9.]+)", src)}
    scales = json.load(open(os.path.join(ROOT, "learninghumanoidwalking_b200", "model", "h1.json")))["cfg"]["observation_noise"]["scales"]
    assert got == dict(ORIENT=scales["root_orient"], GYRO=scales["root_ang_vel"], POS=scales["motor_pos"], VEL=scales["motor_vel"],
                       TAU=scales["motor_tau"])
    assert SCALES == (got["ORIENT"], got["GYRO"], got["POS"], got["VEL"], got["TAU"])


def test_sensor_streams_are_new():
    """The sensor streams 80-84, 96-104 and 112-120 are not among the fixed stream numbers of any other philox( call of csrc/."""
    used = set()
    for f in os.listdir(os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc")):
        src = open(os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", f)).read()
        for arg in re.findall(r"philox\([^;]*?,[^;]*?,[^;]*?,\s*([^,;]+?),\s*\w+\)", src):
            used.update(int(x) for x in re.findall(r"\b(\d+)\b", arg))
    assert {0, 3, 40, 50, 60} <= used
    assert not used & (set(range(80, 85)) | set(range(96, 105)) | set(range(112, 121)))


def test_sensor_checks_and_refusals():
    from learninghumanoidwalking_b200.envs.batched_env import check_sensor_bias, check_sensor_noise, check_sensor_range
    assert check_sensor_noise([0, 1, 4]).tolist() == [0, 1, 4]
    for v in (float("nan"), float("inf"), -0.1, 4.01, [1, 5]):
        with pytest.raises(ValueError, match="noise multiplier must lie in"):
            check_sensor_noise(v)
    ok = np.concatenate([[0.2, -0.2], [0.5, -0.5, 0.1], np.full(12, -0.2)])
    assert check_sensor_bias(ok, 12).tolist() == ok.tolist()
    for k, v, group in ((0, 0.21, "roll / pitch"), (1, float("nan"), "roll / pitch"), (3, -0.51, "gyro"), (9, 0.3, "encoder"),
                        (16, float("inf"), "encoder")):
        bad = ok.copy()
        bad[k] = v
        with pytest.raises(ValueError, match=f"a {group} offset must lie in"):
            check_sensor_bias(bad, 12)
    with pytest.raises(ValueError, match="17 words"):
        check_sensor_bias(np.zeros(15), 12)
    assert check_sensor_range(1, (0.05, 0.1, 0.02)) == (1.0, (0.05, 0.1, 0.02))
    for noise, bias, msg in ((float("nan"), (0, 0, 0), "noise multiplier"), (5, (0, 0, 0), "noise multiplier"),
                             (1, (0, 0), "three numbers"), (1, (-0.1, 0, 0), "roll / pitch offset range"),
                             (1, (0, 0.6, 0), "gyro offset range"), (1, (0, 0, float("nan")), "encoder offset range"),
                             (1, (0, 0, 0.25), "encoder offset range")):
        with pytest.raises(ValueError, match=msg):
            check_sensor_range(noise, bias)


@pytest.mark.parametrize("extra, message", [
    (["--sensor-noise", "nan"], "noise multiplier must lie in"),
    (["--sensor-noise", "-1"], "noise multiplier must lie in"),
    (["--sensor-noise", "4.5"], "noise multiplier must lie in"),
    (["--sensor-bias", "0.05,x,0"], "three comma-separated numbers"),
    (["--sensor-bias", "0.05,0.1"], "three numbers"),
    (["--sensor-bias", "0.3,0,0"], "roll / pitch offset range"),
    (["--sensor-bias", "0,0.6,0"], "gyro offset range"),
    (["--sensor-bias", "0,0,-0.01"], "encoder offset range"),
    (["--sensor-bias", "0,0,inf"], "encoder offset range"),
])
def test_train_refuses_before_anything_exists(tmp_path, extra, message):
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["train", "--env", "jvrc_walk", *extra, "--logdir", str(tmp_path / "logs"), "--n-itr", "1"])
    assert not (tmp_path / "logs").exists()


@pytest.mark.parametrize("extra, message", [
    (["--num-envs", "64", "--sensor-errors", "yaw:0.1"], "unknown kind"),
    (["--num-envs", "64", "--sensor-errors", "roll"], "comma-separated numbers"),
    (["--num-envs", "64", "--sensor-errors", "roll:0.1,x"], "comma-separated numbers"),
    (["--num-envs", "64", "--sensor-errors", "roll:0.3"], "must lie in"),
    (["--num-envs", "64", "--sensor-errors", "pitch:-0.25"], "must lie in"),
    (["--num-envs", "64", "--sensor-errors", "encoder:nan"], "must lie in"),
    (["--num-envs", "64", "--sensor-errors", "noise:-1"], "must lie in"),
    (["--num-envs", "64", "--sensor-errors", "noise:5"], "must lie in"),
    (["--sensor-errors", "roll:0.1", "noise:1"], "need the batched evaluation"),
    (["--sensor-errors", "roll:0.1,0.2"], "need the batched evaluation"),
    (["--num-envs", "2", "--sensor-errors", "roll:0,0.1", "noise:1"], "every cell needs"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--push-speeds", "0,1"], "separate sweeps"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--command", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--footsteps", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--action-delays", "0,0.01"], "separate sweeps"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--payloads", "0,5"], "separate sweeps"),
    (["--num-envs", "64", "--sensor-errors", "noise:1", "--motor-strengths", "0,1"], "separate sweeps"),
])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Grammar, kinds, ranges, cell counts and combinations are refused before the actor is looked for (the run directory here
    has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(run), *extra])


def test_eval_cells_follow_the_grammar():
    import run_experiment as rx
    args = Namespace(sensor_errors=["roll:-0.05,0.05", "pitch:-0.1,0,0.1", "encoder:0.03", "noise:1,2"], num_envs=64,
                     push_speeds=None, command=None, footsteps=None, action_delays=None, payloads=None, motor_strengths=None)
    assert rx.sensor_cells(args) == [("roll", -0.05), ("roll", 0.05), ("pitch", -0.1), ("pitch", 0.0), ("pitch", 0.1),
                                     ("encoder", 0.03), ("noise", 1.0), ("noise", 2.0)]


def test_env_gets_the_run_values_and_old_runs_are_off(monkeypatch):
    """make_env_fn hands --sensor-noise and --sensor-bias (as check_sensor_flags leaves it) to the env, which `resume` rebuilds
    from experiment.pkl; a pickle written before the flags existed means no sensor errors."""
    import run_experiment as rx
    got = []

    class FakeEnv:
        def __init__(self, n, **kw):
            got.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(rx, "import_env", lambda name: FakeEnv)
    base = dict(env="jvrc_walk", num_procs=8, seed=1, precision=32, max_traj_len=400, yaml=None, no_mirror=True)
    args = Namespace(**base, sensor_noise=1.0, sensor_bias="0.05,0.1,0.02")
    rx.check_sensor_flags(args)
    assert args.sensor_bias == (0.05, 0.1, 0.02)
    rx.make_env_fn(pickle.loads(pickle.dumps(args)), 0, 1, 0)()
    rx.make_env_fn(pickle.loads(pickle.dumps(Namespace(**base))), 0, 1, 0)()
    assert [(g["sensor_noise"], g["sensor_bias"]) for g in got] == [(1.0, (0.05, 0.1, 0.02))] * 2 + [(0.0, (0.0, 0.0, 0.0))] * 2


def test_system_info_prints_sensor_errors_only_when_on(capsys):
    import run_experiment as rx
    base = dict(env="jvrc_walk", logdir="x", num_procs=8, lr=1e-4, max_traj_len=400, n_itr=1, seed=0)
    rx.print_system_info(Namespace(**base), training=True)
    rx.print_system_info(Namespace(**base, sensor_noise=0.0, sensor_bias=(0.0, 0.0, 0.0)), training=True)
    assert "Sensor errors" not in capsys.readouterr().out
    rx.print_system_info(Namespace(**base, sensor_noise=1.0, sensor_bias=(0.05, 0.1, 0.02)), training=True)
    assert "Sensor errors: noise x1; offsets up to 0.05 rad roll / pitch, 0.1 rad/s gyro, 0.02 rad encoders" in capsys.readouterr().out


def test_sweep_grid_and_cell_statistics():
    """Env i gets cell i mod C; a cell's row is 0 but for its one kind; each cell's statistics are summarize()'s over the envs of
    its index, so cells of equal value stay apart."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    cells = [("roll", 0.05), ("pitch", 0.05), ("encoder", 0.03), ("noise", 2.0)]
    idx, m, b = ev.sensor_grid(9, cells, 12)
    assert idx.tolist() == [0, 1, 2, 3, 0, 1, 2, 3, 0] and m.tolist() == [0, 0, 0, 2, 0, 0, 0, 2, 0]
    assert b.shape == (9, 17) and b[0].tolist() == [0.05] + [0] * 16 and b[1].tolist() == [0, 0.05] + [0] * 15
    assert b[2].tolist() == [0] * 5 + [0.03] * 12 and not b[3].any()
    with pytest.raises(ValueError, match="unknown sensor error kind"):
        ev.sensor_grid(4, [("yaw", 0.1)], 12)
    rng = np.random.RandomState(0)
    acc = np.zeros((9, ev.WORDS))
    acc[:, ev.LEN] = rng.randint(1, 400, size=9)
    acc[:, ev.RET] = rng.normal(size=9)
    acc[:, ev.DONE] = [1, 0, 1, 1, 0, 0, 0, 1, 0]
    acc[:, ev.TRACK:ev.TRACK + 12] = rng.uniform(1, 2, size=(9, 12))
    s = ev.sensor_summary(acc, idx, cells, "jvrc_walk", ["r"] * 10)
    c0, c1 = s["cells"][0], s["cells"][1]
    assert (c0["cell"], c0["kind"], c0["value"], c0["n"]) == (0, "roll", 0.05, 3) and c0["fall_fraction"] == pytest.approx(1 / 3)
    assert (c1["kind"], c1["value"], c1["n"]) == ("pitch", 0.05, 2) and c1["mean_length"] == pytest.approx(acc[[1, 5], ev.LEN].mean())
    assert set(c0["tracking"]) == set(ev.MODES)
    table = ev.format_sensor_table(s)
    assert "sensor errors" in table and "encoder" in table and "noise" in table


def test_op_and_c_abi_are_declared():
    src = open(os.path.join(ROOT, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_sense"' in src
    hdr = open(os.path.join(ROOT, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_sense(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_sense" in _lib.SIGNATURES
    from learninghumanoidwalking_b200.rl.ppo import _PER_ENV
    assert _PER_ENV["sensor"] == ("sensor errors", "--sensor-noise / --sensor-bias")
