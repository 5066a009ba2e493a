"""Motor strength for every environment (`train --motor-strength R`, `eval --motor-strengths ...`, DESIGN.md §7.11), CPU tier.

The motor step (csrc/sim_core.h env_step with MOTOR = true, the body of lhw_sim_step_motor's kernels) and the random draw
(motor_draw_env, the body of lhw_sim_draw_motor's kernel) run on the host (tests/emu/motor_emu.cpp) for all five variants at fp64
and fp32.  Strength 1 on every joint must be the plain step bit for bit; with strengths, closed-loop roll-outs must stay with the
unchanged oracle given a model whose kp, kd are multiplied by each env's factors (in numpy); a limp joint must deliver no torque;
the draw must equal a numpy restatement; strength must compose with delays, payloads and the stair curriculum.  Also: every
refusal of the env helpers and the command line."""
import ctypes
import os
import pickle
from argparse import Namespace

import numpy as np
import pytest

import emu
import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = ("jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step")
MOTOR_STREAM = 73


class MotorEmu(emu_variants.Emu):
    """emu_variants.Emu on the library of motor_emu.cpp (sim_emu_variants.cpp's entry points plus motor_emu_step / _draw)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = emu_variants._build("motor_emu.cpp", "sim_emu_variants.cpp", os.path.join(HERE, "emu", "_build", "libmotor_emu.so"), [])
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

    @property
    def prev_torque(self):
        """The record's prev_torque: the act_force of the last substep of the env's last control step (0 after a reset)."""
        k = self.nq + 2 * self.nv + 4 * self.nu
        return self.sr[:, k:k + self.nu]

    def step_motor(self, actions, strength, payload=None, delay=None, max_traj_len=400, autoreset=1, level=None, n_levels=0):
        """One motor step of every env; payload, delay: payloads and action delays as well; level: the stair curriculum's levels
        as well (jvrc_step)."""
        n = self.n
        a = np.ascontiguousarray(actions, dtype=self.dt).reshape(n, self.nu)
        assert strength.dtype == self.dt and strength.shape == (n, self.nu) and strength.flags.c_contiguous
        if payload is not None:
            assert payload.dtype == self.dt and payload.shape == (n, 4) and payload.flags.c_contiguous
        d = None if delay is None else np.ascontiguousarray(delay, dtype=np.int32)
        obs, tobs = np.zeros((n, self.nobs), self.dt), np.zeros((n, self.nobs), self.dt)
        rew, terms, eprew = np.zeros(n, self.dt), np.zeros((n, emu.NREW), self.dt), np.zeros(n, self.dt)
        done, ended, eplen = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        if level is not None:
            assert level.dtype == np.int32 and level.flags.c_contiguous
        rc = self.raw.motor_emu_step(self.h, self.prec, self._p(self.sr), self._p(self.si), n, ctypes.c_uint32(self.seed),
                                     ctypes.c_uint32(self.first_id), self._p(a), max_traj_len, autoreset, self._p(obs),
                                     self._p(tobs), self._p(rew), self._p(terms), self._p(done), self._p(ended), self._p(eplen),
                                     self._p(eprew), self._p(strength), None if payload is None else self._p(payload),
                                     None if d is None else self._p(d), None if level is None else self._p(level), n_levels)
        assert rc == 0
        return obs, tobs, terms, rew, done, ended, eplen, eprew

    def draw(self, mask, max_dev, strength):
        assert strength.dtype == self.dt and strength.shape == (self.n, self.nu)
        m = None if mask is None else self._p(np.ascontiguousarray(mask, np.int32))
        self.raw.motor_emu_draw(self.prec, self._p(self.si), self.n, ctypes.c_uint32(self.seed), ctypes.c_uint32(self.first_id), m,
                                ctypes.c_double(max_dev), self.nu, self._p(strength))


def _flat(name, prec, tolerance=None, pdrand=0.0):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model(name), tolerance=tolerance if tolerance is not None else (None if prec == 64 else 1e-6),
                      pd_gain_randomization=pdrand)


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def draws(philox, seed, first_id, si, sel, max_dev, nu, before):
    """numpy restatement of motor_draw_env: a selected env's joint l gets 1 + R (2 u01(u[l % 4]) - 1) of
    u = philox(seed, env id, rng_ctr, 73 + l / 4), in float64 rounded once to the strength's dtype."""
    out = before.copy()
    u01 = lambda x: float(int(x) >> 8) * (1.0 / 16777216.0)
    for i in range(len(out)):
        if sel is None or sel[i]:
            for b in range((nu + 3) // 4):
                u = philox(seed, first_id + i, int(si[i, 4]) & 0xFFFFFFFF, MOTOR_STREAM + b)
                for k in range(min(4, nu - 4 * b)):
                    out[i, 4 * b + k] = 1 + max_dev * (2 * u01(u[k]) - 1)
    return out


def _actions(rng, n, nu):
    scale = np.where(np.arange(n) % 4 == 3, 1.0, 0.15)[:, None]     # every fourth env falls now and then
    return rng.normal(size=(n, nu)) * scale


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_unit_strength_is_the_plain_step(name, precision):
    """24 envs x 80 closed-loop autoreset steps with falls and truncations: the motor step with every factor 1 (and no payload or
    delay) gives the plain step's records, observations, terminal observations, rewards, reward terms, done / ended and episode
    words bit for bit."""
    flat = _flat(name, precision)
    N, seed, first_id = 24, 3, 7
    e, p = MotorEmu(flat, precision, N, seed, first_id), emu_variants.Emu(flat, precision, N, seed, first_id)
    assert e.reset().tobytes() == p.reset().tobytes()
    rng = np.random.RandomState(0)
    ones = np.ones((N, e.nu), e.dt)
    n_end = 0
    for t in range(80):
        a = _actions(rng, N, e.nu)
        got, want = e.step_motor(a, ones, max_traj_len=30), p.step(a, max_traj_len=30)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert e.sr.tobytes() == p.sr.tobytes() and np.array_equal(e.si, p.si), t
        n_end += int(got[5].sum())
    assert n_end > 0


class ScaledOracle:
    """The unchanged oracle with one model per env, whose cfg kp and kd are the compiled gains times that env's factors (numpy);
    each env steps (with the oracle's own auto-reset) on its own model, rebuilt whenever its factors change."""

    def __init__(self, name, n, seed, first_id, pdrand=0.0):
        from oracle import oracle as O
        self.O, self.name, self.n, self.pdrand = O, name, n, pdrand
        if name == "h1_walk":
            from h1_walk_oracle import H1WalkOracle
            self.o = H1WalkOracle(tolerance=1e-14)
        else:
            self.o = O.Oracle(name, tolerance=1e-14, pdrand_k=pdrand)
        self.envs = self.o.make_envs(n, seed=seed, first_id=first_id)
        self.models, self.factors = [None] * n, [None] * n

    def _model(self, s):
        import copy
        mj = copy.deepcopy(self.o.mj)
        mj["cfg"]["kp"] = list(np.asarray(mj["cfg"]["kp"], np.float64) * s)
        mj["cfg"]["kd"] = list(np.asarray(mj["cfg"]["kd"], np.float64) * s)
        if self.name == "h1_walk":
            from h1_walk_oracle import pack_oracle_model
            flat = pack_oracle_model(mj, self.o.clocks, 1e-14)
        else:
            flat = self.O.pack_model(mj, self.o.clocks, 1e-14, pdrand_k=self.pdrand)
        buf = ctypes.create_string_buffer(self.o.lib.orc_sizeof_model())
        assert self.o.lib.orc_model_from_flat(buf, flat.ctypes.data_as(ctypes.c_void_p), len(flat)) == 0
        return buf

    def set(self, strength):
        for i in range(self.n):
            s = np.asarray(strength[i], np.float64)
            if self.factors[i] is None or s.tobytes() != self.factors[i].tobytes():
                self.factors[i], self.models[i] = s.copy(), self._model(s)

    def step(self, actions, max_traj_len, delay=None, delay_lib=None):
        """One autoreset step of every env on its own model (with delay [n] substeps through tests/emu/delay_oracle.c)."""
        from oracle.oracle import NREW
        o, n = self.o, self.n
        p = lambda a: a.ctypes.data_as(ctypes.c_void_p)
        obs, tobs, terms = np.zeros((n, o.nobs)), np.zeros((n, o.nobs)), np.zeros((n, NREW))
        rew, done, ended = np.zeros(n), np.zeros(n, np.int32), np.zeros(n, np.int32)
        for i in range(n):
            a = np.ascontiguousarray(actions[i], np.float64)
            args = (p(a),)
            if delay is not None:
                args += (p(np.array([delay[i]], np.int32)),)
            args += (max_traj_len, p(obs[i]), p(tobs[i]), p(terms[i]), p(rew[i:i + 1]), p(done[i:i + 1]), p(ended[i:i + 1]))
            env = ctypes.byref(self.envs, i * o.env_size)
            if delay is None:
                o.lib.orc_batch_step_autoreset(self.models[i], env, 1, *args, 0)
            else:
                delay_lib.delay_oracle_step(self.models[i], env, 1, *args)
        if hasattr(o, "observe"):
            obs, tobs = o.observe(self.envs, obs), o.observe(self.envs, tobs, back=ended)
        return obs, tobs, terms, rew, done, ended

    def qpos_qvel(self, nq, nv):
        o = self.o
        return (np.stack([o.field(self.envs, i, "qpos")[:nq] for i in range(self.n)]),
                np.stack([o.field(self.envs, i, "qvel")[:nv] for i in range(self.n)]))


def _rollout_against_oracle(name, steps, pdrand=0.0, delay=None):
    N, seed, first_id = 16, 11, 5
    flat = _flat(name, 64, tolerance=1e-14, pdrand=pdrand)
    so = ScaledOracle(name, N, seed, first_id, pdrand)
    e = MotorEmu(flat, 64, N, seed, first_id)
    assert np.abs(so.o.batch_reset(so.envs, N) - e.reset()).max() < 1e-10
    s = np.ones((N, e.nu))
    e.draw(None, 1.0, s)
    s[::5] = 1.0                     # a few envs at the plain gains
    s[1, :2] = 0.0                   # and limp joints
    so.set(s)
    delay_lib = None
    if delay is not None:
        from test_action_delay import _delay_oracle_lib
        delay_lib = _delay_oracle_lib()
    rng = np.random.RandomState(2)
    worst, n_end = 0.0, 0
    for t in range(steps):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = so.step(a, 60, delay, delay_lib)
        eo, et, etm, er, ed, een, _, _ = e.step_motor(a, s, delay=delay, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        e.draw(een, 1.0, s)
        so.set(s)
        n_end += int(een.sum())
        oq, ov = so.qpos_qvel(e.nq, e.nv)
        worst = max(worst, np.abs(oo - eo).max(), np.abs(tt - etm).max(), np.abs(rr - er).max(), np.abs(oq - e.qpos).max(),
                    np.abs(ov - e.qvel).max())
    assert worst < 1e-7, worst
    assert n_end > 0, n_end


@pytest.mark.parametrize("name", VARIANTS)
def test_motor_rollout_matches_oracle(name):
    """16 envs x 200 closed-loop autoreset steps at fp64 with random strengths at R = 1 (factors in [0, 2]), redrawn by the draw
    body after every auto-reset; the unchanged oracle steps each env on a model whose kp, kd are scaled by its factors:
    observations, reward terms, rewards, qpos and qvel agree within 1e-7; falls, truncations and resets included."""
    _rollout_against_oracle(name, 200)


def test_motor_rollout_with_pd_gain_randomization():
    """As above on jvrc_walk with pd_gain_randomization = 0.2: the strength scales the gains the pdrand_k draw gave."""
    _rollout_against_oracle("jvrc_walk", 150, pdrand=0.2)


@pytest.mark.parametrize("name", ["jvrc_walk", "h1_walk"])
def test_strength_and_delay_match_the_delay_oracle(name):
    """Factors in [0, 2] together with action delays of 0..25 substeps: the motor step against tests/emu/delay_oracle.c given
    each env's scaled gains, within 1e-7."""
    _rollout_against_oracle(name, 150, delay=np.array([(7 * i) % 26 for i in range(16)], np.int32))


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_limp_joint_delivers_no_torque(name, precision):
    """A joint with factor 0 has act_force exactly 0 at every step (the record's prev_torque, which the step copies from the last
    substep's act_force), while the other joints still deliver torque."""
    flat = _flat(name, precision)
    N = 8
    e = MotorEmu(flat, precision, N, 2, 0)
    e.reset()
    s = np.ones((N, e.nu), e.dt)
    limp = np.arange(e.nu) % 3 == 0
    s[:, limp] = 0
    rng = np.random.RandomState(1)
    for t in range(40):
        e.step_motor(_actions(rng, N, e.nu), s, max_traj_len=25)
        assert (e.prev_torque[:, limp] == 0).all(), t
    assert (np.abs(e.prev_torque[:, ~limp]) > 0).any()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", ["jvrc_walk", "h1"])
def test_draw_equals_numpy(name, precision, philox):
    """The draw body against the numpy restatement bit for bit: every env (no mask), masked envs and the envs a step ended, for
    several ranges; unselected envs keep their words."""
    flat = _flat(name, precision)
    N, seed, first_id = 40, 21, 9
    e = MotorEmu(flat, precision, N, seed, first_id)
    e.reset()
    e.si[:, 4] += np.arange(N, dtype=np.int32) * 3            # counters differ per env
    rng = np.random.RandomState(3)
    for R in (0.0, 0.3, 1.0):
        for sel in (None, (np.arange(N) % 3 == 0).astype(np.int32), (rng.uniform(size=N) < 0.3).astype(np.int32) * 5):
            before = rng.normal(size=(N, e.nu)).astype(e.dt)
            got = before.copy()
            e.draw(sel, R, got)
            want = draws(philox, seed, first_id, e.si, sel, R, e.nu, before.astype(np.float64)).astype(e.dt)
            assert got.tobytes() == want.tobytes(), (R, sel)
            picked = got if sel is None else got[sel != 0]
            assert (picked >= 1 - R).all() and (picked <= 1 + R).all()


@pytest.mark.parametrize("precision", [64, 32])
def test_unit_strength_composes_with_delays_payloads_and_stairs(precision):
    """jvrc_step with the stair curriculum, action delays and payloads: with every factor 1 the motor step equals the payload +
    delay + curriculum step bit for bit (levels included), through auto-resets; and on jvrc_walk, factor 1 with delays only equals
    the delay step."""
    from test_action_delay import DelayEmu
    from test_payload import PayloadEmu
    from test_stair_curriculum import _force_far
    flat = _flat("jvrc_step", precision)
    K, N, seed, first_id, max_len = 5, 24, 9, 40, 25
    both, ref = MotorEmu(flat, precision, N, seed, first_id), PayloadEmu(flat, precision, N, seed, first_id)
    ref.reset(), both.reset()
    lv_b = np.array([(i % (K + 2)) - 1 for i in range(N)], np.int32)
    lv_r = lv_b.copy()
    delay = np.array([(5 * i) % 26 for i in range(N)], np.int32)
    rng = np.random.RandomState(5)
    pay = np.zeros((N, 4), both.dt)
    ref.draw(None, 20.0, 0.2, pay)
    ones = np.ones((N, 12), both.dt)
    n_end = 0
    for t in range(80):
        for i in range(0, N, 2):
            _force_far(both.sr, both.si, i, max_len)
            _force_far(ref.sr, ref.si, i, max_len)
        a = _actions(rng, N, 12)
        got = both.step_motor(a, ones, pay, delay, max_traj_len=max_len, level=lv_b, n_levels=K)
        want = ref.step_payload(a, pay, delay, max_traj_len=max_len, level=lv_r, n_levels=K)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert both.sr.tobytes() == ref.sr.tobytes() and np.array_equal(lv_b, lv_r), t
        n_end += int(got[5].sum())
    assert n_end > 0
    flat = _flat("jvrc_walk", precision)
    both, ref = MotorEmu(flat, precision, N, seed, first_id), DelayEmu(flat, precision, N, seed, first_id)
    ref.reset(), both.reset()
    for t in range(40):
        a = _actions(rng, N, 12)
        got, want = both.step_motor(a, ones, delay=delay, max_traj_len=max_len), ref.step_delay(a, delay, max_traj_len=max_len)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t


def test_motor_checks_and_refusals():
    from learninghumanoidwalking_b200.envs.batched_env import check_motor_strength, check_motor_strength_range
    assert check_motor_strength([0, 1, 2]).tolist() == [0, 1, 2]
    for v in (float("nan"), float("inf"), -0.1, 2.01, [1, 1, 3]):
        with pytest.raises(ValueError, match="must lie in"):
            check_motor_strength(v)
    for r in (0, 0.3, 1):
        check_motor_strength_range(r)
    for r in (float("nan"), float("inf"), -0.1, 1.01):
        with pytest.raises(ValueError, match="range must lie in"):
            check_motor_strength_range(r)


@pytest.mark.parametrize("value", ["nan", "inf", "-0.1", "1.5"])
def test_train_refuses_before_anything_exists(tmp_path, value):
    import run_experiment as rx
    with pytest.raises(SystemExit, match="range must lie in"):
        rx.main(["train", "--env", "jvrc_walk", "--motor-strength", value, "--logdir", str(tmp_path / "logs"), "--n-itr", "1"])
    assert not (tmp_path / "logs").exists()


@pytest.mark.parametrize("extra, message", [
    (["--motor-strengths", "0,x"], "comma-separated"),
    (["--motor-strengths", "0,-0.5"], "must lie in"),
    (["--motor-strengths", "0,2.5"], "must lie in"),
    (["--motor-strengths", "0,nan"], "must lie in"),
    (["--motor-strengths", "0,1"], "need the batched evaluation"),
    (["--num-envs", "2", "--motor-strengths", "0,0.5,1"], "every cell needs"),
    (["--num-envs", "64", "--motor-joints", "R_KNEE"], "add --motor-strengths"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--motor-joints", "R_KNEE,,L_KNEE"], "comma-separated joint names"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--motor-joints", "R_KNEE,ELBOW"], "ELBOW is not a joint"),
    (["--motor-strengths", "0.5", "--motor-joints", "KNEE"], "KNEE is not a joint"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--push-speeds", "0,1"], "separate sweeps"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--command", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--footsteps", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--action-delays", "0,0.01"], "separate sweeps"),
    (["--num-envs", "64", "--motor-strengths", "0,1", "--payloads", "0,5"], "separate sweeps"),
])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Grammar, range and combinations are refused before the actor is looked for; the joint names against the run's model after
    its experiment.pkl is read and before the actor is loaded (the run directory here has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(run), *extra])


def test_joint_mask_follows_the_run_model():
    import run_experiment as rx
    from learninghumanoidwalking_b200.model import load_model
    names = [lk["joint"]["name"] for lk in load_model("jvrc_walk")["links"][1:]]
    motor = dict(factors=[0.5], joints=["R_KNEE", "L_KNEE"])
    mask = rx.motor_joint_mask(motor, Namespace(env="jvrc_walk"), None)
    assert mask == [n in ("R_KNEE", "L_KNEE") for n in names] and sum(mask) == 2
    motor = dict(factors=[0.5], joints=None)
    assert rx.motor_joint_mask(motor, Namespace(env="h1"), None) == [True] * 10 and len(motor["joints"]) == 10


def test_env_gets_the_run_values_and_old_runs_are_off(monkeypatch):
    """make_env_fn hands --motor-strength to the env, which `resume` rebuilds from experiment.pkl; a pickle written before the
    flag existed means no strengths."""
    import run_experiment as rx
    got = []

    class FakeEnv:
        def __init__(self, n, **kw):
            got.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(rx, "import_env", lambda name: FakeEnv)
    base = dict(env="jvrc_walk", num_procs=8, seed=1, precision=32, max_traj_len=400, yaml=None, no_mirror=True)
    rx.make_env_fn(Namespace(**base, motor_strength=0.3), 0, 1, 0)()
    rx.make_env_fn(pickle.loads(pickle.dumps(Namespace(**base))), 0, 1, 0)()
    assert [g["motor_strength"] for g in got] == [0.3] * 2 + [0.0] * 2


def test_system_info_prints_strengths_only_when_on(capsys):
    import run_experiment as rx
    base = dict(env="jvrc_walk", logdir="x", num_procs=8, lr=1e-4, max_traj_len=400, n_itr=1, seed=0)
    rx.print_system_info(Namespace(**base), training=True)
    assert "Motor strength" not in capsys.readouterr().out
    rx.print_system_info(Namespace(**base, motor_strength=0.3), training=True)
    assert "Motor strengths: U(0.7, 1.3)" in capsys.readouterr().out


def test_sweep_grid_and_cell_statistics():
    """Env i gets cell i mod C; each cell's statistics are summarize()'s over its envs."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    f = ev.motor_grid(7, [0, 0.5, 1])
    assert f.tolist() == [0, 0.5, 1, 0, 0.5, 1, 0]
    rng = np.random.RandomState(0)
    acc = np.zeros((7, ev.WORDS))
    acc[:, ev.LEN] = rng.randint(1, 400, size=7)
    acc[:, ev.RET] = rng.normal(size=7)
    acc[:, ev.DONE] = [1, 0, 1, 1, 0, 0, 0]
    acc[:, ev.TRACK:ev.TRACK + 12] = rng.uniform(1, 2, size=(7, 12))
    s = ev.motor_summary(acc, f, [0, 0.5, 1], ["R_KNEE", "L_KNEE"], "jvrc_walk", ["r"] * 10)
    c0 = s["cells"][0]
    assert c0["factor"] == 0 and c0["n"] == 3 and c0["fall_fraction"] == pytest.approx(2 / 3)
    assert c0["mean_length"] == pytest.approx(acc[[0, 3, 6], ev.LEN].mean())
    assert set(c0["tracking"]) == set(ev.MODES) and s["joints"] == ["R_KNEE", "L_KNEE"]
    assert "factor" in ev.format_motor_table(s) and "R_KNEE" in ev.format_motor_table(s)


def test_op_and_c_abi_are_declared():
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_step_motor"' in src and 'm.impl("sim_draw_motor"' in src
    hdr = open(os.path.join(root, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_step_motor(" in hdr and "int lhw_sim_draw_motor(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_step_motor" in _lib.SIGNATURES and "lhw_sim_draw_motor" in _lib.SIGNATURES
    from learninghumanoidwalking_b200.rl.ppo import _PER_ENV
    assert _PER_ENV["motor_strength"] == ("motor strengths", "--motor-strength")
