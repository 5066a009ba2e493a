"""Carried payloads for every environment (`train --payload-mass M`, `eval --payloads ...`, DESIGN.md §7.10), CPU tier.

The payload step (csrc/sim_core.h env_step with PAYLOAD = true, the body of lhw_sim_step_payload's kernels) and the random draw
(payload_draw_env, the body of lhw_sim_draw_payload's kernel) run on the host (tests/emu/payload_emu.cpp) for all five variants at
fp64 and fp32.  A payload of mass 0 must be the plain step bit for bit; with payloads, closed-loop roll-outs must stay with the
unchanged oracle whose root link is given the composite of link and payload (computed here in numpy); the draw must equal a numpy restatement; on jvrc_step the stair curriculum and the action
delays must compose with the payload.  Also: every refusal of the env helpers and the command line."""
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
PAYLOAD_STREAM = 72


class PayloadEmu(emu_variants.Emu):
    """emu_variants.Emu on the library of payload_emu.cpp (sim_emu_variants.cpp's entry points plus payload_emu_step / _draw)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = emu_variants._build("payload_emu.cpp", "sim_emu_variants.cpp", os.path.join(HERE, "emu", "_build", "libpayload_emu.so"),
                                  [])
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

    def step_payload(self, actions, payload, delay=None, max_traj_len=400, autoreset=1, level=None, n_levels=0):
        """One payload step of every env; delay: action delays as well; level: the stair curriculum's levels as well (jvrc_step)."""
        n = self.n
        a = np.ascontiguousarray(actions, dtype=self.dt).reshape(n, self.nu)
        assert payload.dtype == self.dt and payload.shape == (n, 4) and payload.flags.c_contiguous
        d = None if delay is None else np.ascontiguousarray(delay, dtype=np.int32)
        obs, tobs = np.zeros((n, self.nobs), self.dt), np.zeros((n, self.nobs), self.dt)
        rew, terms, eprew = np.zeros(n, self.dt), np.zeros((n, emu.NREW), self.dt), np.zeros(n, self.dt)
        done, ended, eplen = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        if level is not None:
            assert level.dtype == np.int32 and level.flags.c_contiguous
        rc = self.raw.payload_emu_step(self.h, self.prec, self._p(self.sr), self._p(self.si), n, ctypes.c_uint32(self.seed),
                                       ctypes.c_uint32(self.first_id), self._p(a), max_traj_len, autoreset, self._p(obs),
                                       self._p(tobs), self._p(rew), self._p(terms), self._p(done), self._p(ended), self._p(eplen),
                                       self._p(eprew), self._p(payload), None if d is None else self._p(d),
                                       None if level is None else self._p(level), n_levels)
        assert rc == 0
        return obs, tobs, terms, rew, done, ended, eplen, eprew

    def draw(self, mask, max_mass, max_offset, payload):
        assert payload.dtype == self.dt and payload.shape == (self.n, 4)
        m = None if mask is None else self._p(np.ascontiguousarray(mask, np.int32))
        self.raw.payload_emu_draw(self.prec, self._p(self.si), self.n, ctypes.c_uint32(self.seed), ctypes.c_uint32(self.first_id), m,
                                  ctypes.c_double(max_mass), ctypes.c_double(max_offset), self._p(payload))


def _flat(name, prec, tolerance=None):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model(name), tolerance=tolerance if tolerance is not None else (None if prec == 64 else 1e-6))


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def draws(philox, seed, first_id, si, sel, max_mass, max_offset, before):
    """numpy restatement of payload_draw_env: a selected env gets (M u01(u[0]), R (2 u01(u[1..3]) - 1)) of
    u = philox(seed, env id, rng_ctr, 72), in float64 rounded once to the payload's dtype."""
    out = before.copy()
    u01 = lambda x: float(int(x) >> 8) * (1.0 / 16777216.0)
    for i in range(len(out)):
        if sel is None or sel[i]:
            u = philox(seed, first_id + i, int(si[i, 4]) & 0xFFFFFFFF, PAYLOAD_STREAM)
            out[i] = [max_mass * u01(u[0])] + [max_offset * (2 * u01(u[1 + k]) - 1) for k in range(3)]
    return out


def _actions(rng, n, nu):
    scale = np.where(np.arange(n) % 4 == 3, 1.0, 0.15)[:, None]     # every fourth env falls now and then
    return rng.normal(size=(n, nu)) * scale


def composite(ms, c, I, m, p):
    """numpy float64: the root link (mass ms, centre of mass c, 3x3 inertia I about c) with a point mass m at p, all in the link
    frame: (M', c', I' about c')."""
    M = ms + m
    cc = (ms * c + m * p) / M
    d1, d2 = c - cc, p - cc
    E = np.eye(3)
    Ic = I + ms * (d1 @ d1 * E - np.outer(d1, d1)) + m * (d2 @ d2 * E - np.outer(d2, d2))
    return M, cc, Ic


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_zero_mass_is_the_plain_step(name, precision):
    """24 envs x 80 closed-loop autoreset steps with falls and truncations: the payload step with mass 0 and non-zero offsets
    gives the plain step's records, observations, terminal observations, rewards, reward terms, done / ended and episode words
    bit for bit."""
    flat = _flat(name, precision)
    N, seed, first_id = 24, 3, 7
    e, p = PayloadEmu(flat, precision, N, seed, first_id), emu_variants.Emu(flat, precision, N, seed, first_id)
    assert e.reset().tobytes() == p.reset().tobytes()
    rng = np.random.RandomState(0)
    pay = np.zeros((N, 4), e.dt)
    pay[:, 1:] = rng.uniform(-0.25, 0.25, size=(N, 3))
    n_end = 0
    for t in range(80):
        a = _actions(rng, N, e.nu)
        got, want = e.step_payload(a, pay, max_traj_len=30), p.step(a, max_traj_len=30)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert e.sr.tobytes() == p.sr.tobytes() and np.array_equal(e.si, p.si), t
        n_end += int(got[5].sum())
    assert n_end > 0


def _oracle(name, model_dict=None):
    from oracle.oracle import Oracle
    if name == "h1_walk":
        from h1_walk_oracle import H1WalkOracle
        return H1WalkOracle(tolerance=1e-14)
    return Oracle(name, tolerance=1e-14, model_dict=model_dict)


class OraclePayload:
    """Writes env i's composite root link into the oracle's P_mass[0], P_com[0] and P_inertia[0], composed on the plain values
    the oracle last set there itself (its reset, and H1's re-randomisation)."""

    def __init__(self, o, envs, n):
        self.o, self.envs, self.n = o, envs, n
        self.base = [None] * n
        self.written = [None] * n
        self.com0 = np.asarray(o.mj["links"][0]["com"], dtype=np.float64)

    def _read(self, i):
        f = lambda k: self.o.field(self.envs, i, k)
        return f("P_mass")[0], f("P_com")[:3].copy(), f("P_inertia")[:9].reshape(3, 3).copy()

    def apply(self, payload):
        for i in range(self.n):
            cur = self._read(i)
            if self.written[i] is None or any(a.tobytes() != b.tobytes() for a, b in zip(map(np.asarray, cur),
                                                                                         map(np.asarray, self.written[i]))):
                self.base[i] = cur
            ms, c, I = self.base[i]
            m = float(payload[i, 0])
            if m != 0:
                ms, c, I = composite(ms, c, I, m, self.com0 + payload[i, 1:].astype(np.float64))
            self._write(i, ms, c, I)
            self.written[i] = self._read(i)

    def _write(self, i, ms, c, I):
        self.o.set_field(self.envs, i, "P_mass", np.concatenate([[ms], self.o.field(self.envs, i, "P_mass")[1:]]))
        pc = self.o.field(self.envs, i, "P_com")
        pc[:3] = c
        self.o.set_field(self.envs, i, "P_com", pc)
        pI = self.o.field(self.envs, i, "P_inertia")
        pI[:9] = I.reshape(-1)
        self.o.set_field(self.envs, i, "P_inertia", pI)

    def batch_step(self, actions, max_traj_len):
        """o.batch_step with autoreset, except that every reset runs on the plain root link: the H1 oracles' resets re-randomise
        it themselves; for the JVRC-1 variants, orc_step_autoreset is restated per env with the plain link written back before
        orc_reset."""
        from oracle.oracle import NREW
        o, n = self.o, self.n
        if "h1" in o.mj["name"]:
            return o.batch_step(self.envs, n, actions, max_traj_len)
        out = [np.zeros((n, o.nobs)), np.zeros((n, o.nobs)), np.zeros((n, NREW)), np.zeros(n),
               np.zeros(n, np.int32), np.zeros(n, np.int32)]
        for i in range(n):
            obs, r, d, terms = o.step(self.envs, i, actions[i])
            f = lambda k: o.field(self.envs, i, k)
            o.set_field(self.envs, i, "traj_len", f("traj_len") + 1)
            o.set_field(self.envs, i, "ep_len", f("ep_len") + 1)
            o.set_field(self.envs, i, "ep_rew", f("ep_rew") + r)
            end = d or f("traj_len")[0] >= max_traj_len
            out[1][i], out[2][i], out[3][i], out[4][i], out[5][i] = obs, terms, r, d, end
            if end:
                o.set_field(self.envs, i, "status", 0)
                self._write(i, *self.base[i])
                obs = o.reset(self.envs, i)
            out[0][i] = obs
        return tuple(out)


@pytest.mark.parametrize("name", VARIANTS)
def test_payload_rollout_matches_oracle(name):
    """16 envs x 300 closed-loop autoreset steps at fp64 with random payloads up to 20 kg at offsets up to 0.25 m (a third of the
    envs at mass 0), redrawn by the draw body after every auto-reset; the unchanged oracle is given each env's composite root link
    after each of its resets (and, on H1, after each re-randomisation), and its resets run on the plain link: observations, reward terms, rewards, qpos and qvel agree
    within 1e-7; falls, truncations and resets included."""
    N, seed, first_id = 16, 11, 5
    flat = _flat(name, 64, tolerance=1e-14)
    o = _oracle(name)
    e = PayloadEmu(flat, 64, N, seed, first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    assert np.abs(o.batch_reset(envs, N) - e.reset()).max() < 1e-10
    pay = np.zeros((N, 4))
    e.draw(None, 20.0, 0.25, pay)
    pay[::3, 0] = 0
    op = OraclePayload(o, envs, N)
    op.apply(pay)
    rng = np.random.RandomState(2)
    worst, n_end = 0.0, 0
    for t in range(300):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = op.batch_step(a, 60)
        eo, et, etm, er, ed, een, _, _ = e.step_payload(a, pay, max_traj_len=60)
        assert (dd == ed).all() and (ee == een).all(), t
        e.draw(een, 20.0, 0.25, pay)
        op.apply(pay)
        n_end += int(een.sum())
        oq = np.stack([o.field(envs, i, "qpos")[:e.nq] for i in range(N)])
        ov = np.stack([o.field(envs, i, "qvel")[:e.nv] for i in range(N)])
        worst = max(worst, np.abs(oo - eo).max(), np.abs(tt - etm).max(), np.abs(rr - er).max(), np.abs(oq - e.qpos).max(),
                    np.abs(ov - e.qvel).max())
    assert worst < 1e-7, worst
    assert n_end > 0, n_end


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", ["jvrc_walk", "h1"])
def test_draw_equals_numpy(name, precision, philox):
    """The draw body against the numpy restatement bit for bit: every env (no mask), masked envs and the envs a step ended, for
    several ranges; unselected envs keep their words."""
    flat = _flat(name, precision)
    N, seed, first_id = 40, 21, 9
    e = PayloadEmu(flat, precision, N, seed, first_id)
    e.reset()
    e.si[:, 4] += np.arange(N, dtype=np.int32) * 3            # counters differ per env
    rng = np.random.RandomState(3)
    for M, R in ((0.0, 0.0), (5.0, 0.0), (20.0, 0.25), (31.2, 0.1)):
        for sel in (None, (np.arange(N) % 3 == 0).astype(np.int32), (rng.uniform(size=N) < 0.3).astype(np.int32) * 5):
            before = rng.normal(size=(N, 4)).astype(e.dt)
            got = before.copy()
            e.draw(sel, M, R, got)
            want = draws(philox, seed, first_id, e.si, sel, M, R, before.astype(np.float64)).astype(e.dt)
            assert got.tobytes() == want.tobytes(), (M, R, sel)
            picked = got if sel is None else got[sel != 0]
            assert (picked[:, 0] >= 0).all() and (picked[:, 0] <= M).all() and (np.abs(picked[:, 1:]) <= R).all()


@pytest.mark.parametrize("precision", [64, 32])
def test_stairs_and_delays_compose_with_payloads(precision):
    """jvrc_step with the stair curriculum and action delays: with every payload mass 0 the payload step equals the curriculum +
    delay step bit for bit (levels included); with payloads, each env's step equals the payload + delay step of a copy of its record
    in a sim whose step height is its level's height (the level the curriculum step left)."""
    from test_action_delay import DelayEmu
    from test_stair_curriculum import _force_far, height
    flat = _flat("jvrc_step", precision)
    K, N, seed, first_id, max_len = 5, 24, 9, 40, 25
    both, ref = PayloadEmu(flat, precision, N, seed, first_id), DelayEmu(flat, precision, N, seed, first_id)
    plain = PayloadEmu(flat, precision, 1, seed, first_id)
    ref.reset(), both.reset()
    lv_b = np.array([(i % (K + 2)) - 1 for i in range(N)], np.int32)
    lv_r = lv_b.copy()
    delay = np.array([(5 * i) % 26 for i in range(N)], np.int32)
    rng = np.random.RandomState(5)
    pay = np.zeros((N, 4), both.dt)
    pay[:, 1:] = 0.1
    for t in range(60):
        for i in range(0, N, 2):
            _force_far(both.sr, both.si, i, max_len)
            _force_far(ref.sr, ref.si, i, max_len)
        a = _actions(rng, N, 12)
        got = both.step_payload(a, pay, delay, max_traj_len=max_len, level=lv_b, n_levels=K)
        want = ref.step_delay(a, delay, max_traj_len=max_len, level=lv_r, n_levels=K)
        for g, w in zip(got, want):
            assert g.tobytes() == w.tobytes(), t
        assert both.sr.tobytes() == ref.sr.tobytes() and np.array_equal(lv_b, lv_r), t
    both.draw(None, 20.0, 0.2, pay)
    n_end, moved = 0, 0
    for t in range(120):
        for i in range(0, N, 2):
            _force_far(both.sr, both.si, i, max_len)
        a = _actions(rng, N, 12)
        sr0, si0, lv0 = both.sr.copy(), both.si.copy(), lv_b.copy()
        obs, tobs, _, rew, done, ended, eplen, eprew = both.step_payload(a, pay, delay, max_traj_len=max_len, level=lv_b, n_levels=K)
        moved += int((lv_b != lv0).sum())
        n_end += int(ended.sum())
        for i in range(N):
            plain.sr[0], plain.si[0] = sr0[i], si0[i]
            plain.lib.emu_set_step_height(plain.h, precision, ctypes.c_double(height(lv_b[i], K)))
            plain.first_id = first_id + i
            po, pt, _, pr, pd, pe, pl, pw = plain.step_payload(a[i:i + 1], pay[i:i + 1].copy(), delay[i:i + 1], max_traj_len=max_len)
            assert plain.sr[0].tobytes() == both.sr[i].tobytes() and np.array_equal(plain.si[0], both.si[i]), (t, i)
            assert po.tobytes() == obs[i:i + 1].tobytes() and pr[0] == rew[i] and pd[0] == done[i] and pe[0] == ended[i]
            if ended[i]:
                assert pt.tobytes() == tobs[i:i + 1].tobytes() and pl[0] == eplen[i] and pw[0] == eprew[i]
        both.draw(ended, 20.0, 0.2, pay)
    assert n_end > 0 and moved > 0, (n_end, moved)


def test_payload_checks_and_refusals():
    from learninghumanoidwalking_b200.envs.batched_env import check_payload, check_payload_range
    m, r = check_payload([0, 5, 31.2], [0.25, -0.25, 0], 62.4)
    assert m.tolist() == [0, 5, 31.2] and r.tolist() == [0.25, -0.25, 0]
    for mass, off, msg in ((float("nan"), 0, "mass must lie"), (float("inf"), 0, "mass must lie"), (-1, 0, "mass must lie"),
                           (31.3, 0, "mass must lie"), (1, float("nan"), "offset must lie"), (1, 0.26, "offset must lie"),
                           (1, [0, 0, -0.3], "offset must lie"), (1, float("inf"), "offset must lie")):
        with pytest.raises(ValueError, match=msg):
            check_payload(mass, off, 62.4)
    check_payload_range(10, 0.1, 62.4)
    with pytest.raises(ValueError, match="needs a payload mass"):
        check_payload_range(0, 0.1, 62.4)
    with pytest.raises(ValueError, match=">= 0 m"):
        check_payload_range(10, -0.1, 62.4)


@pytest.mark.parametrize("extra, message", [
    (["--payload-mass", "nan"], "mass must lie"), (["--payload-mass", "inf"], "mass must lie"),
    (["--payload-mass", "-1"], "mass must lie"), (["--payload-mass", "31.3"], "mass must lie"),
    (["--payload-mass", "10", "--payload-offset", "0.3"], "offset must lie"),
    (["--payload-mass", "10", "--payload-offset", "nan"], "offset must lie"),
    (["--payload-mass", "10", "--payload-offset", "-0.1"], ">= 0 m"),
    (["--payload-offset", "0.1"], "needs a payload mass"),
])
def test_train_refuses_before_anything_exists(tmp_path, extra, message):
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["train", "--env", "jvrc_walk", *extra, "--logdir", str(tmp_path / "logs"), "--n-itr", "1"])
    assert not (tmp_path / "logs").exists()


def test_train_checks_against_the_robot_of_the_run(tmp_path):
    """Half the robot's mass after the YAML: 31.2 kg for JVRC-1, 29.2 kg for H1; a YAML that changes other keys keeps the bound."""
    import run_experiment as rx
    y = tmp_path / "cfg.yaml"
    y.write_text("sim_dt: 0.0005\ncontrol_dt: 0.025\n")
    rx.check_payload_mass(Namespace(env="jvrc_walk", yaml=str(y), payload_mass=31.2, payload_offset=0.0))
    rx.check_payload_mass(Namespace(env="h1", yaml=None, payload_mass=29.2, payload_offset=0.25))
    with pytest.raises(SystemExit, match="29.2"):
        rx.check_payload_mass(Namespace(env="h1", yaml=None, payload_mass=29.3, payload_offset=0.0))
    with pytest.raises(SystemExit, match="31.2"):
        rx.check_payload_mass(Namespace(env="jvrc_step", yaml=str(y), payload_mass=31.3, payload_offset=0.0))


@pytest.mark.parametrize("extra, message", [
    (["--payloads", "0,x"], "comma-separated"),
    (["--payloads", "0,-5"], "finite and >= 0"),
    (["--payloads", "0,inf"], "finite and >= 0"),
    (["--payloads", "0,10"], "need the batched evaluation"),
    (["--num-envs", "2", "--payloads", "0,5,10"], "every cell needs"),
    (["--num-envs", "64", "--payloads", "0,5", "--payload-at", "0,0"], "one point"),
    (["--num-envs", "64", "--payloads", "0,5", "--payload-at", "0,0,0.3"], "within 0.25"),
    (["--num-envs", "64", "--payloads", "0,5", "--payload-at", "0,nan,0"], "within 0.25"),
    (["--num-envs", "64", "--payload-at", "0,0,0.1"], "add --payloads"),
    (["--num-envs", "64", "--payloads", "0,5", "--push-speeds", "0,1"], "separate sweeps"),
    (["--num-envs", "64", "--payloads", "0,5", "--command", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--payloads", "0,5", "--footsteps", "standing"], "separate sweeps"),
    (["--num-envs", "64", "--payloads", "0,5", "--action-delays", "0,0.01"], "separate sweeps"),
    (["--num-envs", "64", "--payloads", "0,31.3"], "mass must lie"),
    (["--payloads", "40"], "mass must lie"),
])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Grammar, offset and combinations are refused before the actor is looked for; the masses against the run's model after its
    experiment.pkl is read and before the actor is loaded (the run directory here has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(run), *extra])


def test_env_gets_the_run_values_and_old_runs_are_off(monkeypatch):
    """make_env_fn hands --payload-mass / --payload-offset to the env, which `resume` rebuilds from experiment.pkl; a pickle
    written before the flags existed means no payload."""
    import run_experiment as rx
    got = []

    class FakeEnv:
        def __init__(self, n, **kw):
            got.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(rx, "import_env", lambda name: FakeEnv)
    base = dict(env="jvrc_walk", num_procs=8, seed=1, precision=32, max_traj_len=400, yaml=None, no_mirror=True)
    rx.make_env_fn(Namespace(**base, payload_mass=20.0, payload_offset=0.1), 0, 1, 0)()
    rx.make_env_fn(pickle.loads(pickle.dumps(Namespace(**base))), 0, 1, 0)()
    assert [(g["payload_mass"], g["payload_offset"]) for g in got] == [(20.0, 0.1)] * 2 + [(0.0, 0.0)] * 2


def test_system_info_prints_payloads_only_when_on(capsys):
    import run_experiment as rx
    base = dict(env="jvrc_walk", logdir="x", num_procs=8, lr=1e-4, max_traj_len=400, n_itr=1, seed=0)
    rx.print_system_info(Namespace(**base), training=True)
    assert "Payload" not in capsys.readouterr().out
    rx.print_system_info(Namespace(**base, payload_mass=20.0, payload_offset=0.1), training=True)
    assert "Payloads: up to 20 kg" in capsys.readouterr().out


def test_sweep_grid_and_cell_statistics():
    """Env i gets cell i mod C; each cell's statistics are summarize()'s over its envs."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    m = ev.payload_grid(7, [0, 10, 20])
    assert m.tolist() == [0, 10, 20, 0, 10, 20, 0]
    rng = np.random.RandomState(0)
    acc = np.zeros((7, ev.WORDS))
    acc[:, ev.LEN] = rng.randint(1, 400, size=7)
    acc[:, ev.RET] = rng.normal(size=7)
    acc[:, ev.DONE] = [1, 0, 1, 1, 0, 0, 0]
    acc[:, ev.TRACK:ev.TRACK + 12] = rng.uniform(1, 2, size=(7, 12))
    s = ev.payload_summary(acc, m, [0, 10, 20], (0, 0, 0.1), "jvrc_walk", ["r"] * 10)
    c0 = s["cells"][0]
    assert c0["mass"] == 0 and c0["n"] == 3 and c0["fall_fraction"] == pytest.approx(2 / 3)
    assert c0["mean_length"] == pytest.approx(acc[[0, 3, 6], ev.LEN].mean())
    assert c0["return_mean"] == pytest.approx(acc[[0, 3, 6], ev.RET].mean())
    assert set(c0["tracking"]) == set(ev.MODES) and s["at"] == [0, 0, 0.1]
    assert "mass kg" in ev.format_payload_table(s)


def test_op_and_c_abi_are_declared():
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_step_payload"' in src and 'm.impl("sim_draw_payload"' in src
    hdr = open(os.path.join(root, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_step_payload(" in hdr and "int lhw_sim_draw_payload(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_step_payload" in _lib.SIGNATURES and "lhw_sim_draw_payload" in _lib.SIGNATURES
