"""Action delays for every environment (`train --action-delay S`, `eval --action-delays ...`, DESIGN.md §7.9), CPU tier.

The delayed step (csrc/sim_core.h env_step with DELAY = true, the body of lhw_sim_step_delay's kernels) and the random draw
(delay_draw_env, the body of lhw_sim_draw_delay's kernel) run on the host (tests/emu/delay_emu.cpp) for all five variants at fp64
and fp32.  At delay 0 the delayed step must be the plain step bit for bit; the first step of an episode must be the plain step
for any delay; with delays, closed-loop roll-outs must stay with the oracle given the same per-env delays; the draw must equal a
numpy restatement; on jvrc_step the stair curriculum must compose with the delay.  Also: every refusal of the env helpers and the
command line."""
import ctypes
import os
import pickle
import subprocess
from argparse import Namespace

import numpy as np
import pytest

import emu
import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
DELAY_STREAM, FRAME_SKIP = 71, 25


class DelayEmu(emu_variants.Emu):
    """emu_variants.Emu on the library of delay_emu.cpp (sim_emu_variants.cpp's entry points plus delay_emu_step / _draw)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = emu_variants._build("delay_emu.cpp", "sim_emu_variants.cpp", os.path.join(HERE, "emu", "_build", "libdelay_emu.so"), [])
        raw = ctypes.CDLL(lib)
        self.raw = raw
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

    def step_delay(self, actions, delay, max_traj_len=400, autoreset=1, level=None, n_levels=0):
        """One delayed step of every env; level: the stair curriculum's levels as well (jvrc_step)."""
        n = self.n
        a = np.ascontiguousarray(actions, dtype=self.dt).reshape(n, self.nu)
        d = np.ascontiguousarray(delay, dtype=np.int32)
        assert d.shape == (n,)
        sr, si = self.sr, self.si
        obs, tobs = np.zeros((n, self.nobs), self.dt), np.zeros((n, self.nobs), self.dt)
        rew, terms, eprew = np.zeros(n, self.dt), np.zeros((n, emu.NREW), self.dt), np.zeros(n, self.dt)
        done, ended, eplen = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        if level is not None:
            assert level.dtype == np.int32 and level.flags.c_contiguous
        rc = self.raw.delay_emu_step(self.h, self.prec, self._p(sr), self._p(si), n, ctypes.c_uint32(self.seed),
                                     ctypes.c_uint32(self.first_id), self._p(a), max_traj_len, autoreset, self._p(obs), self._p(tobs),
                                     self._p(rew), self._p(terms), self._p(done), self._p(ended), self._p(eplen), self._p(eprew),
                                     self._p(d), None if level is None else self._p(level), n_levels)
        assert rc == 0
        return obs, tobs, terms, rew, done, ended, eplen, eprew

    def draw(self, mask, max_delay, delay):
        m = None if mask is None else self._p(np.ascontiguousarray(mask, np.int32))
        self.raw.delay_emu_draw(self._p(self.si), self.n, ctypes.c_uint32(self.seed), ctypes.c_uint32(self.first_id), m, max_delay,
                                self._p(delay))


def _flat(name, prec, tolerance=None):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model(name), tolerance=tolerance if tolerance is not None else (None if prec == 64 else 1e-6))


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def draws(philox, seed, first_id, si, sel, max_delay, before):
    """numpy restatement of delay_draw_env: a selected env gets randint(u[0], D + 1) of u = philox(seed, env id, rng_ctr, 71)."""
    out = before.copy()
    for i in range(len(out)):
        if sel is None or sel[i]:
            u = philox(seed, first_id + i, int(si[i, 4]) & 0xFFFFFFFF, DELAY_STREAM)
            out[i] = (int(u[0]) * (max_delay + 1)) >> 32
    return out


def _actions(rng, n, nu, t):
    scale = np.where(np.arange(n) % 4 == 3, 1.0, 0.15)[:, None]     # every fourth env falls now and then
    return rng.normal(size=(n, nu)) * scale


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_zero_delay_is_the_plain_step(name, precision):
    """24 envs x 80 closed-loop autoreset steps with falls and truncations: the delayed step at delay 0 gives the plain step's
    records, observations, terminal observations, rewards, reward terms, done / ended and episode words bit for bit."""
    flat = _flat(name, precision)
    N, seed, first_id = 24, 3, 7
    d, p = DelayEmu(flat, precision, N, seed, first_id), emu_variants.Emu(flat, precision, N, seed, first_id)
    assert d.reset().tobytes() == p.reset().tobytes()
    rng = np.random.RandomState(0)
    zero = np.zeros(N, np.int32)
    n_end = 0
    for t in range(80):
        a = _actions(rng, N, d.nu, t)
        got, want = d.step_delay(a, zero, max_traj_len=30), p.step(a, max_traj_len=30)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert d.sr.tobytes() == p.sr.tobytes() and np.array_equal(d.si, p.si), t
        n_end += int(got[5].sum())
    assert n_end > 0


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_first_step_of_an_episode_is_never_delayed(name, precision):
    """After a fresh reset every env's first step equals the plain one bit for bit, whatever its delay (0 .. 25, and -3 and 40,
    which are clamped); the second step of a delayed env differs from the plain one."""
    flat = _flat(name, precision)
    N, seed, first_id = 30, 8, 2
    d, p = DelayEmu(flat, precision, N, seed, first_id), emu_variants.Emu(flat, precision, N, seed, first_id)
    d.reset(), p.reset()
    delay = np.array([-3, 40] + list(range(N - 2)), np.int32)
    rng = np.random.RandomState(1)
    a = rng.normal(size=(N, d.nu)) * 0.3
    got, want = d.step_delay(a, delay), p.step(a)
    for g, w in zip(got, want):
        assert g.tobytes() == w.tobytes()
    assert d.sr.tobytes() == p.sr.tobytes()
    a = rng.normal(size=(N, d.nu)) * 0.3
    d.step_delay(a, delay), p.step(a)
    same = [d.sr[i].tobytes() == p.sr[i].tobytes() for i in range(N)]
    assert same[0] and [i for i in range(N) if same[i]] == [0] + [i for i in range(2, N) if delay[i] == 0]


def _oracle(name):
    from oracle.oracle import Oracle
    if name == "h1_walk":
        from h1_walk_oracle import H1WalkOracle
        return H1WalkOracle(tolerance=1e-14)
    return Oracle(name, tolerance=1e-14)


def _delay_oracle_lib():
    """tests/emu/delay_oracle.c: the unchanged oracle source plus its control step with an action delay."""
    root = os.path.dirname(HERE)
    srcs = [os.path.join(HERE, "emu", "delay_oracle.c"), os.path.join(root, "oracle", "sim_oracle.c"),
            os.path.join(root, "oracle", "sim_oracle.h")]
    lib = os.path.join(HERE, "emu", "_build", "libdelay_oracle.so")
    if not os.path.exists(lib) or any(os.path.getmtime(s) > os.path.getmtime(lib) for s in srcs):
        os.makedirs(os.path.dirname(lib), exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-std=gnu11", "-fvisibility=hidden", "-o", lib, srcs[0], "-lm"])
    return ctypes.CDLL(lib)


def delayed_oracle_step(lib, o, envs, n, actions, delay, max_traj_len):
    """o.batch_step(envs, n, actions, max_traj_len) with per-env delays [n] in substeps (the oracle's own step at delay 0); the
    h1_walk oracle's observation words are completed as its batch_step completes them."""
    from oracle.oracle import NREW
    p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    actions = np.ascontiguousarray(actions, dtype=np.float64)
    d = np.ascontiguousarray(delay, dtype=np.int32)
    nobs = getattr(o, "nobs")
    obs, tobs, terms = np.zeros((n, nobs)), np.zeros((n, nobs)), np.zeros((n, NREW))
    rew, done, ended = np.zeros(n), np.zeros(n, dtype=np.int32), np.zeros(n, dtype=np.int32)
    lib.delay_oracle_step(o._model, envs, n, p(actions), p(d), max_traj_len, p(obs), p(tobs), p(terms), p(rew), p(done), p(ended))
    if hasattr(o, "observe"):
        obs, tobs = o.observe(envs, obs), o.observe(envs, tobs, back=ended)
    return obs, tobs, terms, rew, done, ended


@pytest.mark.parametrize("name", VARIANTS)
def test_delay_oracle_at_zero_is_the_oracle(name):
    """The test oracle's delayed step at delay 0 against the oracle's own orc_batch_step_autoreset: 8 envs x 120 closed-loop
    autoreset steps with falls and truncations, outputs and env records bit for bit (prev_action over the model's nu joints: the
    oracle copies its whole ORC_NU target array, whose tail it never writes)."""
    from oracle.oracle import _ENV_FIELDS
    N, seed = 8, 4
    o, lib = _oracle(name), _delay_oracle_lib()
    a_envs, b_envs = o.make_envs(N, seed=seed), o.make_envs(N, seed=seed)
    o.batch_reset(a_envs, N), o.batch_reset(b_envs, N)
    rng = np.random.RandomState(6)
    n_end = 0
    for t in range(120):
        act = _actions(rng, N, o.nu, t)
        want = o.batch_step(a_envs, N, act, max_traj_len=40)
        got = delayed_oracle_step(lib, o, b_envs, N, act, np.zeros(N, np.int32), 40)
        for g, w in zip(got, want):
            assert np.array_equal(g, w, equal_nan=True), t
        for i in range(N):
            for f in _ENV_FIELDS:
                x, y = o.field(a_envs, i, f), o.field(b_envs, i, f)
                if f == "prev_action":
                    x, y = x[:o.nu], y[:o.nu]
                assert x.tobytes() == y.tobytes(), (t, i, f)
        n_end += int(want[5].sum())
    assert n_end > 0


@pytest.mark.parametrize("name", VARIANTS)
def test_delayed_rollout_matches_oracle(name):
    """16 envs x 300 closed-loop autoreset steps at fp64 with per-env delays 0 .. 25 substeps (frame_skip included), redrawn from
    U{0..25} by the draw body after every auto-reset and given to the test oracle's delayed step (tests/emu/delay_oracle.c): observations, reward terms,
    rewards, qpos and qvel agree within 1e-7 (the pushed roll-outs' bound); falls, truncations and resets included."""
    N, seed, first_id = 16, 11, 5
    flat = _flat(name, 64, tolerance=1e-14)
    o, lib = _oracle(name), _delay_oracle_lib()
    e = DelayEmu(flat, 64, N, seed, first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    assert np.abs(o.batch_reset(envs, N) - e.reset()).max() < 1e-10
    delay = np.array([0, FRAME_SKIP] + [(7 * i) % (FRAME_SKIP + 1) for i in range(2, N)], np.int32)
    rng = np.random.RandomState(2)
    worst, n_end, seen = 0.0, 0, set(delay.tolist())
    for t in range(300):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = delayed_oracle_step(lib, o, envs, N, a, delay, 60)
        eo, et, etm, er, ed, een, _, _ = e.step_delay(a, delay, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        e.draw(een, FRAME_SKIP, delay)
        seen |= set(delay[een != 0].tolist())
        n_end += int(een.sum())
        oq = np.stack([o.field(envs, i, "qpos")[:e.nq] for i in range(N)])
        ov = np.stack([o.field(envs, i, "qvel")[:e.nv] for i in range(N)])
        worst = max(worst, np.abs(oo - eo).max(), np.abs(tt - etm).max(), np.abs(rr - er).max(), np.abs(oq - e.qpos).max(),
                    np.abs(ov - e.qvel).max())
    assert worst < 1e-7, worst
    assert n_end > 0 and len(seen) > 10, (n_end, seen)


@pytest.mark.parametrize("name", VARIANTS)
def test_draw_equals_numpy(name, philox):
    """The draw body against the numpy restatement bit for bit: every env (no mask), masked envs, and the envs a step ended,
    for D = 0, 1, 7 and 25; unselected envs keep their word."""
    flat = _flat(name, 64)
    N, seed, first_id = 40, 21, 9
    e = DelayEmu(flat, 64, N, seed, first_id)
    e.reset()
    rng = np.random.RandomState(3)
    for t in range(6):
        e.step_delay(rng.normal(size=(N, e.nu)) * 0.2, np.zeros(N, np.int32))
    e.si[:, 4] += np.arange(N, dtype=np.int32) * 3            # counters differ per env
    for D in (0, 1, 7, FRAME_SKIP):
        for sel in (None, (np.arange(N) % 3 == 0).astype(np.int32), (rng.uniform(size=N) < 0.3).astype(np.int32) * 5):
            before = rng.randint(-5, 30, size=N).astype(np.int32)
            got = before.copy()
            e.draw(sel, D, got)
            want = draws(philox, seed, first_id, e.si, sel, D, before)
            assert np.array_equal(got, want), (D, sel)
            picked = got if sel is None else got[sel != 0]
            assert picked.min() >= 0 and picked.max() <= D
    big = np.zeros(4000, np.int32)
    e4 = DelayEmu(flat, 64, 4000, seed, 0)
    e4.si[:, 4] = 1
    e4.draw(None, FRAME_SKIP, big)
    assert set(big.tolist()) == set(range(FRAME_SKIP + 1))     # every value of U{0..25} occurs


@pytest.mark.parametrize("precision", [64, 32])
def test_stairs_compose_with_delays(precision):
    """jvrc_step with the stair curriculum and delays together: with every delay 0 the curriculum + delay step equals the
    curriculum step alone bit for bit (levels included); with delays 0 .. 25, each env's step equals the delay-only step of a copy
    of its record in a sim whose step height is its level's height (the level the curriculum step left), so its resets are the
    delay-only resets at that height."""
    from test_stair_curriculum import StairEmu, _force_far, height
    flat = _flat("jvrc_step", precision)
    K, N, seed, first_id, max_len = 5, 24, 9, 40, 25
    both, stairs = DelayEmu(flat, precision, N, seed, first_id), StairEmu(flat, precision, N, seed, first_id)
    plain = DelayEmu(flat, precision, 1, seed, first_id)
    lv_b = np.array([(i % (K + 2)) - 1 for i in range(N)], np.int32)
    lv_s = lv_b.copy()
    stairs.reset_stairs(lv_s, K, fresh=True)
    both.sr[:], both.si[:] = stairs.sr, stairs.si
    rng = np.random.RandomState(5)
    zero = np.zeros(N, np.int32)
    for t in range(60):
        for i in range(0, N, 2):
            _force_far(both.sr, both.si, i, max_len)
            _force_far(stairs.sr, stairs.si, i, max_len)
        a = _actions(rng, N, 12, t)
        got = both.step_delay(a, zero, max_traj_len=max_len, level=lv_b, n_levels=K)
        want = stairs.step_stairs(a, lv_s, K, max_traj_len=max_len)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert both.sr.tobytes() == stairs.sr.tobytes() and np.array_equal(lv_b, lv_s), t
    delay = np.array([(5 * i) % (FRAME_SKIP + 1) for i in range(N)], np.int32)
    n_end, moved = 0, 0
    for t in range(120):
        for i in range(0, N, 2):
            _force_far(both.sr, both.si, i, max_len)
        a = _actions(rng, N, 12, t)
        sr0, si0, lv0 = both.sr.copy(), both.si.copy(), lv_b.copy()
        obs, tobs, _, rew, done, ended, eplen, eprew = both.step_delay(a, delay, max_traj_len=max_len, level=lv_b, n_levels=K)
        moved += int((lv_b != lv0).sum())
        n_end += int(ended.sum())
        for i in range(N):
            plain.sr[0], plain.si[0] = sr0[i], si0[i]
            plain.lib.emu_set_step_height(plain.h, precision, ctypes.c_double(height(lv_b[i], K)))
            plain.first_id = first_id + i
            po, pt, _, pr, pd, pe, pl, pw = plain.step_delay(a[i:i + 1], delay[i:i + 1], max_traj_len=max_len)
            assert plain.sr[0].tobytes() == both.sr[i].tobytes() and np.array_equal(plain.si[0], both.si[i]), (t, i)
            assert po.tobytes() == obs[i:i + 1].tobytes() and pr[0] == rew[i] and pd[0] == done[i] and pe[0] == ended[i]
            if ended[i]:
                assert pt.tobytes() == tobs[i:i + 1].tobytes() and pl[0] == eplen[i] and pw[0] == eprew[i]
    assert n_end > 0 and moved > 0, (n_end, moved)


def test_delay_substeps_and_refusals():
    from learninghumanoidwalking_b200.envs.batched_env import action_delay_substeps
    assert action_delay_substeps(0.0, 0.001, 0.025).tolist() == [0]
    assert action_delay_substeps([0, 0.005, 0.01, 0.02, 0.025], 0.001, 0.025).tolist() == [0, 5, 10, 20, 25]
    assert action_delay_substeps(0.003, 0.0005, 0.02).tolist() == [6]
    for bad, msg in ((float("nan"), "must lie in"), (float("inf"), "must lie in"), (-0.001, "must lie in"), (0.026, "must lie in"),
                     (0.0015, "whole number"), ([0.01, 0.0001], "whole number")):
        with pytest.raises(ValueError, match=msg):
            action_delay_substeps(bad, 0.001, 0.025)


@pytest.mark.parametrize("value, message", [("nan", "must lie in"), ("inf", "must lie in"), ("-0.005", "must lie in"),
                                            ("0.03", "must lie in"), ("0.0125", "whole number")])
def test_train_refuses_before_anything_exists(tmp_path, value, message):
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["train", "--env", "jvrc_walk", "--action-delay", value, "--logdir", str(tmp_path / "logs"), "--n-itr", "1"])
    assert not (tmp_path / "logs").exists()


def test_train_checks_against_the_yaml_model(tmp_path):
    """A YAML with 0.5 ms physics substeps accepts a 10.5 ms delay that the shipped model (1 ms substeps) refuses."""
    import run_experiment as rx
    y = tmp_path / "cfg.yaml"
    y.write_text("sim_dt: 0.0005\ncontrol_dt: 0.025\n")
    rx.check_action_delay(Namespace(env="jvrc_walk", yaml=str(y), action_delay=0.0105))
    with pytest.raises(SystemExit, match="whole number of physics substeps of 0.001 s"):
        rx.check_action_delay(Namespace(env="jvrc_walk", yaml=None, action_delay=0.0105))


@pytest.mark.parametrize("extra, message", [
    (["--action-delays", "0,x"], "comma-separated"),
    (["--action-delays", "0,-0.005"], "finite and >= 0"),
    (["--action-delays", "0,inf"], "finite and >= 0"),
    (["--action-delays", "0,0.01"], "need the batched evaluation"),
    (["--num-envs", "2", "--action-delays", "0,0.01,0.02"], "every cell needs"),
    (["--num-envs", "64", "--action-delays", "0,0.01", "--push-speeds", "0,1"], "separate sweeps"),
    (["--num-envs", "64", "--action-delays", "0,0.01", "--command", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--action-delays", "0,0.01", "--footsteps", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--action-delays", "0,0.0105"], "whole number"),
    (["--num-envs", "64", "--action-delays", "0,0.03"], "must lie in"),
    (["--action-delays", "0.0305"], "must lie in"),
])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Grammar and combinations are refused before the actor is looked for; the values against the run's model after its
    experiment.pkl is read and before the actor is loaded (the run directory here has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(run), *extra])


def test_env_gets_the_run_value_and_old_runs_are_off(monkeypatch):
    """make_env_fn hands --action-delay to the env, which `resume` rebuilds from experiment.pkl; a pickle written before the flag
    existed means no delay."""
    import run_experiment as rx
    got = []

    class FakeEnv:
        def __init__(self, n, **kw):
            got.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(rx, "import_env", lambda name: FakeEnv)
    base = dict(env="jvrc_walk", num_procs=8, seed=1, precision=32, max_traj_len=400, yaml=None, no_mirror=True)
    rx.make_env_fn(Namespace(**base, action_delay=0.02), 0, 1, 0)()
    rx.make_env_fn(pickle.loads(pickle.dumps(Namespace(**base))), 0, 1, 0)()
    assert [g["action_delay"] for g in got] == [0.02, 0.02, 0.0, 0.0]


def test_sweep_grid_and_cell_statistics():
    """Env i gets cell i mod C; each cell's statistics are summarize()'s over its envs."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    d = ev.delay_grid(7, [0, 0.01, 0.025])
    assert d.tolist() == [0, 0.01, 0.025, 0, 0.01, 0.025, 0]
    rng = np.random.RandomState(0)
    acc = np.zeros((7, ev.WORDS))
    acc[:, ev.LEN] = rng.randint(1, 400, size=7)
    acc[:, ev.RET] = rng.normal(size=7)
    acc[:, ev.DONE] = [1, 0, 1, 1, 0, 0, 0]
    acc[:, ev.TRACK:ev.TRACK + 12] = rng.uniform(1, 2, size=(7, 12))
    s = ev.delay_summary(acc, d, [0, 0.01, 0.025], "jvrc_walk", ["r"] * 10)
    c0 = s["cells"][0]
    assert c0["n"] == 3 and c0["fall_fraction"] == pytest.approx(2 / 3)
    assert c0["mean_length"] == pytest.approx(acc[[0, 3, 6], ev.LEN].mean())
    assert c0["return_mean"] == pytest.approx(acc[[0, 3, 6], ev.RET].mean())
    assert set(c0["tracking"]) == set(ev.MODES)
    assert "delay ms" in ev.format_delay_table(s)


def test_op_and_c_abi_are_declared():
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_step_delay"' in src and 'm.impl("sim_draw_delay"' in src
    hdr = open(os.path.join(root, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_step_delay(" in hdr and "int lhw_sim_draw_delay(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_step_delay" in _lib.SIGNATURES and "lhw_sim_draw_delay" in _lib.SIGNATURES
