"""The stair curriculum of jvrc_step (`train --stair-curriculum H`, DESIGN.md §7.8), CPU tier.

The curriculum's step and reset (csrc/sim_core.h env_step / env_reset with STAIRS = true, the bodies of lhw_sim_step_stairs's and
lhw_sim_reset_stairs's kernels) run on the host (tests/emu/stairs_emu.cpp) next to the kernel source's host emulation of jvrc_step,
at fp64 and fp32.  A reset of an env at level L must be, bit for bit, the plain reset of the same record in a sim whose step height
is 0.01 L; over closed-loop roll-outs the levels must follow a numpy restatement of the rule, and the roll-outs must stay with the
unchanged oracle given each env's level height before its resets.  Also: the refusals of the env constructor and the command line."""
import ctypes
import os
import pickle
from argparse import Namespace

import numpy as np
import pytest

import emu
import emu_variants

HERE = os.path.dirname(os.path.abspath(__file__))
CURVED, STANDING, BACKWARD, LATERAL, FORWARD = range(5)
NSLAB = 20
# jvrc_step's record: qpos qvel qacc_warm, five NU-blocks, 3 + 1 words, then the plan: seq [20][4] and tk [5] (sim_core.h Dims)
SEQ = 19 + 18 + 18 + 5 * 12 + 3 + 1
TK = SEQ + 4 * NSLAB
I_MODE, I_TRAJ_LEN = 1, 2


class StairEmu(emu.Emu):
    """emu.Emu on the library of stairs_emu.cpp (sim_emu.cpp's entry points plus stairs_emu_reset / stairs_emu_step)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = emu_variants._build("stairs_emu.cpp", "sim_emu.cpp", os.path.join(HERE, "emu", "_build", "libstairs_emu.so"), [])
        self.lib = ctypes.CDLL(lib)
        self.lib.emu_create.restype = ctypes.c_void_p
        flat = np.ascontiguousarray(flat, dtype=np.float64)
        self.h = ctypes.c_void_p(self.lib.emu_create(flat.ctypes.data_as(ctypes.c_void_p), len(flat), precision))
        assert self.h.value, "emu_create failed"
        self.prec, self.n, self.seed, self.first_id = precision, n, seed, first_id
        self.dt = np.float64 if precision == 64 else np.float32
        self.nr = self.lib.emu_state_words(self.h)
        self.nobs = self.lib.emu_obs_dim(self.h)
        self.nu = 12
        self.nq, self.nv = 7 + self.nu, 6 + self.nu
        self.sr = np.zeros((n, self.nr), dtype=self.dt)
        self.si = np.zeros((n, emu.NSTATE_I), dtype=np.int32)

    def reset_stairs(self, level, n_levels, fresh=False, mask=None):
        obs = np.zeros((self.n, self.nobs), dtype=self.dt)
        m = None if mask is None else self._p(np.ascontiguousarray(mask, np.int32))
        rc = self.lib.stairs_emu_reset(self.h, self.prec, self._p(self.sr), self._p(self.si), self.n, ctypes.c_uint32(self.seed),
                                       ctypes.c_uint32(self.first_id), m, self._p(level), n_levels, self._p(obs), int(fresh))
        assert rc == 0
        return obs

    def step_stairs(self, actions, level, n_levels, max_traj_len=400, autoreset=1):
        assert level.dtype == np.int32 and level.flags.c_contiguous
        a = np.ascontiguousarray(actions, dtype=self.dt).reshape(self.n, self.nu)
        n = self.n
        obs, tobs = np.zeros((n, self.nobs), self.dt), np.zeros((n, self.nobs), self.dt)
        rew, terms, eprew = np.zeros(n, self.dt), np.zeros((n, emu.NREW), self.dt), np.zeros(n, self.dt)
        done, ended, eplen = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        rc = self.lib.stairs_emu_step(self.h, self.prec, self._p(self.sr), self._p(self.si), n, ctypes.c_uint32(self.seed),
                                      ctypes.c_uint32(self.first_id), self._p(a), max_traj_len, autoreset, self._p(obs), self._p(tobs),
                                      self._p(rew), self._p(terms), self._p(done), self._p(ended), self._p(eplen), self._p(eprew),
                                      self._p(level), n_levels)
        assert rc == 0
        return obs, tobs, terms, rew, done, ended, eplen, eprew

    def set_step_height(self, h):
        self.lib.emu_set_step_height(self.h, self.prec, ctypes.c_double(h))

    def plain_step_one(self, i, sr, si, action, max_traj_len, autoreset):
        """The plain step of one env from the record (sr, si), which it updates in place: (obs, term_obs, reward, done, ended,
        ep_len, ep_rew)."""
        obs, tobs = np.zeros((1, self.nobs), self.dt), np.zeros((1, self.nobs), self.dt)
        rew, terms, eprew = np.zeros(1, self.dt), np.zeros((1, emu.NREW), self.dt), np.zeros(1, self.dt)
        done, ended, eplen = np.zeros(1, np.int32), np.zeros(1, np.int32), np.zeros(1, np.int32)
        a = np.ascontiguousarray(action, dtype=self.dt)
        self.lib.emu_step(self.h, self.prec, self._p(sr), self._p(si), 1, ctypes.c_uint32(self.seed), ctypes.c_uint32(self.first_id + i),
                          self._p(a), max_traj_len, autoreset, self._p(obs), self._p(tobs), self._p(rew), self._p(terms), self._p(done),
                          self._p(ended), self._p(eplen), self._p(eprew))
        return obs[0], tobs[0], rew[0], done[0], ended[0], eplen[0], eprew[0]


def _flat(prec, iteration_count=float("inf")):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model("jvrc_step"), tolerance=None if prec == 64 else 1e-6, iteration_count=iteration_count)


def rule(level, n_levels, mode, fell, reached, seq_len):
    """numpy restatement of the level rule (DESIGN.md §7.8) for an env whose episode just ended: the level word afterwards."""
    if mode != FORWARD:
        return level                      # other plan types leave the word alone
    lv = min(max(level, 0), n_levels - 1)
    if not fell and 2 * reached >= seq_len:
        return min(lv + 1, n_levels - 1)
    if fell and 2 * reached < seq_len:
        return max(lv - 1, 0)
    return lv


def height(level, n_levels):
    return 0.01 * min(max(int(level), 0), n_levels - 1)


def _force_far(sr, si, i, max_traj_len):
    """Make env i's FORWARD episode have reached half its footsteps just before it is truncated, so that the roll-outs see
    levels go up (random actions never get that far): t1 = ceil(n / 2), t2 = t1 + 1, as step_update_targets leaves them."""
    if si[i, I_MODE] != FORWARD or si[i, I_TRAJ_LEN] + 1 < max_traj_len:
        return None
    n = int(sr[i, TK])
    k = (n + 1) // 2
    if sr[i, TK + 1] >= k:
        return None
    sr[i, TK + 1], sr[i, TK + 2] = k, min(k + 1, n - 1)
    return k, min(k + 1, n - 1)


@pytest.mark.parametrize("precision", [64, 32])
def test_reset_equals_plain_reset_at_the_level_height(precision):
    """Every env of a batch, fresh and then twice more mid-episode (every third one masked out the last time), resets at its level
    (every level of a 21-level curriculum, and -1 and 21, clamped) exactly as the plain reset does in a sim whose step height is
    0.01 L: record and observation bit for bit.  FORWARD plans of both signs occur; the level words are only read."""
    flat = _flat(precision)
    K, N, seed, first_id = 21, 69, 5, 3
    cur, plain = StairEmu(flat, precision, N, seed, first_id), StairEmu(flat, precision, N, seed, first_id)
    level = np.array([(i % (K + 2)) - 1 for i in range(N)], np.int32)
    signs = set()
    for rnd in range(3):
        mask = None if rnd < 2 else (np.arange(N) % 3 != 0).astype(np.int32)
        before = level.copy()
        co = cur.reset_stairs(level, K, fresh=rnd == 0, mask=mask)
        assert np.array_equal(level, before)
        po = np.zeros_like(co)
        for i in range(N):
            if mask is not None and not mask[i]:
                continue
            plain.set_step_height(height(level[i], K))
            po[i] = plain.reset_one(i)
        assert np.array_equal(cur.si, plain.si), rnd
        assert cur.sr.tobytes() == plain.sr.tobytes(), rnd
        assert co.tobytes() == po.tobytes(), rnd
        for i in range(N):
            if cur.si[i, I_MODE] == FORWARD and height(level[i], K) > 0:
                signs.add(np.sign(cur.sr[i, SEQ:SEQ + 4 * NSLAB].reshape(NSLAB, 4)[NSLAB - 1, 2]))
        a = np.random.RandomState(rnd).normal(size=(N, 12)) * 0.2
        for _ in range(4):
            cur.step_stairs(a, level, K, autoreset=0)
            plain.step(a, autoreset=0)
        assert np.array_equal(level, before)            # autoreset off never moves a level
        assert cur.sr.tobytes() == plain.sr.tobytes()
    assert signs == {-1.0, 1.0}, signs


@pytest.mark.parametrize("precision", [64, 32])
def test_autoreset_equals_plain_and_levels_follow_the_rule(precision):
    """Closed-loop autoreset roll-outs of 24 envs on a 5-level curriculum, with falls (large actions), truncations (max_traj_len
    25) and every plan type, levels starting at -1 .. 5.  Before every step each env's record is copied; the plain step of that copy
    in a sim whose step height is 0.01 x (the level the curriculum step left) gives the curriculum step's record, observations,
    reward and episode words bit for bit.  The plain step of the copy with autoreset off gives the ending episode's plan type,
    footsteps reached and sequence length, and the levels follow the numpy rule.  Some FORWARD episodes are given half their
    footsteps just before truncation, so that levels go up; every branch of the rule, both clamps included, is taken."""
    flat = _flat(precision)
    K, N, seed, first_id, T, max_len = 5, 24, 9, 40, 160, 25
    cur, plain = StairEmu(flat, precision, N, seed, first_id), StairEmu(flat, precision, N, seed, first_id)
    level = np.array([(i % (K + 2)) - 1 for i in range(N)], np.int32)
    cur.reset_stairs(level, K, fresh=True)
    rng = np.random.RandomState(1)
    scale = np.where(np.arange(N) % 4 == 3, 1.0, 0.1)[:, None]
    seen = set()
    modes = set()
    for t in range(T):
        for i in range(N):
            if i % 2 == 0:
                _force_far(cur.sr, cur.si, i, max_len)
        a = rng.normal(size=(N, 12)) * scale
        sr0, si0, lv0 = cur.sr.copy(), cur.si.copy(), level.copy()
        out = cur.step_stairs(a, level, K, max_traj_len=max_len)
        obs, tobs, _, rew, done, ended, eplen, eprew = out
        for i in range(N):
            r0, i0 = sr0[i].copy(), si0[i].copy()
            _, _, _, d0, e0, _, _ = plain.plain_step_one(i, r0, i0, a[i], max_len, 0)   # the ending step, without the reset
            assert d0 == done[i] and e0 == ended[i]
            if ended[i]:
                mode, reached, n = int(i0[I_MODE]), float(r0[TK + 1]), float(r0[TK])
                modes.add(mode)
                want = rule(int(lv0[i]), K, mode, bool(done[i]), reached, n)
                assert level[i] == want, (t, i, lv0[i], mode, done[i], reached, n, level[i])
                if mode == FORWARD:
                    lv = min(max(int(lv0[i]), 0), K - 1)
                    seen.add(("up" if want > lv else "down" if want < lv else "stay", lv == 0, lv == K - 1, bool(done[i]),
                              2 * reached >= n))
            else:
                assert level[i] == lv0[i]
            r1, i1 = sr0[i].copy(), si0[i].copy()
            plain.set_step_height(height(level[i], K))
            po, pt, pr, pd, pe, pl, pw = plain.plain_step_one(i, r1, i1, a[i], max_len, 1)
            assert r1.tobytes() == cur.sr[i].tobytes() and np.array_equal(i1, cur.si[i]), (t, i)
            assert po.tobytes() == obs[i].tobytes() and pr == rew[i] and pd == done[i] and pe == ended[i]
            if ended[i]:
                assert pt.tobytes() == tobs[i].tobytes() and pl == eplen[i] and pw == eprew[i]
    kinds = {k[0] for k in seen}
    assert kinds == {"up", "down", "stay"}, seen
    assert ("stay", True, False, True, False) in seen, seen      # a fall short of half at level 0 stays at 0
    assert ("stay", False, True, False, True) in seen, seen      # half the footsteps without a fall at the top level stays there
    assert ("stay", False, False, False, False) in seen, seen    # neither: a truncation short of half
    assert {CURVED, STANDING, BACKWARD, LATERAL, FORWARD} <= modes, modes


def test_rollout_matches_oracle_given_the_level_heights():
    """16 envs x 300 closed-loop autoreset steps at fp64 on a 16-level curriculum (0 .. 0.15 m), with falls and truncations: the
    unchanged oracle, whose step height is set per env to that env's level height before each of its steps (so before each of its
    resets), stays within 1e-7 of the emulation, and the FORWARD plans of both sides carry the same stair heights."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    from oracle.oracle import Oracle
    K, N, seed, first_id, max_len = 16, 16, 13, 2, 60
    flat = pack_model(load_model("jvrc_step"), tolerance=1e-14)
    o = Oracle("jvrc_step", tolerance=1e-14)
    e = StairEmu(flat, 64, N, seed, first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    level = np.array([3 * i % K for i in range(N)], np.int32)
    set_h = lambda h: o.lib.orc_set_step_height(o._model, ctypes.c_double(h))
    eo = e.reset_stairs(level, K, fresh=True)
    oo = np.zeros_like(eo)
    for i in range(N):
        set_h(height(level[i], K))
        oo[i] = o.batch_reset(o.env_ptr(envs, i), 1)[0]
    assert np.abs(oo - eo).max() < 1e-10
    rng = np.random.RandomState(4)
    scale = np.where(np.arange(N) % 4 == 3, 0.6, 0.15)[:, None]
    worst, n_end, n_fell, moved = 0.0, 0, 0, 0
    for t in range(300):
        for i in range(0, N, 2):
            f = _force_far(e.sr, e.si, i, max_len)
            if f is not None:
                o.set_field(envs, i, "t1", f[0])
                o.set_field(envs, i, "t2", f[1])
        a = rng.normal(size=(N, 12)) * scale
        lv0 = level.copy()
        eo_, et, etm, er, ed, een, _, _ = e.step_stairs(a, level, K, max_traj_len=max_len)
        moved += int((level != lv0).sum())
        for i in range(N):
            set_h(height(level[i], K))
            oo_, to, tt, rr, dd, ee = o.batch_step(o.env_ptr(envs, i), 1, a[i:i + 1], max_traj_len=max_len)
            assert dd[0] == ed[i] and ee[0] == een[i], (t, i)
            oq = o.field(envs, i, "qpos")[:e.nq]
            worst = max(worst, np.abs(oo_[0] - eo_[i]).max(), np.abs(tt[0] - etm[i]).max(), abs(rr[0] - er[i]),
                        np.abs(oq - e.qpos[i]).max())
            if een[i]:
                worst = max(worst, np.abs(to[0] - et[i]).max())
                assert np.abs(o.field(envs, i, "seq") - e.sr[i, SEQ:SEQ + 4 * NSLAB]).max() < 1e-9
        n_end += int(een.sum())
        n_fell += int(ed.sum())
    assert worst < 1e-7, worst
    assert n_end > 0 and n_fell > 0 and moved > 0, (n_end, n_fell, moved)


def test_stair_levels_and_env_refusals():
    from learninghumanoidwalking_b200.envs.batched_env import BatchedHumanoidEnv, stair_levels
    assert stair_levels("jvrc_step", 0.0) == 0 and stair_levels("jvrc_walk", 0.0) == 0
    assert stair_levels("jvrc_step", 0.01) == 2 and stair_levels("jvrc_step", 0.15) == 16 and stair_levels("jvrc_step", 0.2) == 21
    assert stair_levels("jvrc_step", 0.07) == 8 and stair_levels("jvrc_step", 0.29 - 0.19) == 11
    for model in ("jvrc_walk", "h1", "jvrc_walk_terrain", "h1_walk"):
        with pytest.raises(ValueError, match=f"{model} has no stair curriculum"):
            BatchedHumanoidEnv(8, model=model, stair_curriculum=0.1)      # refused before any device is looked for
    for bad, msg in ((float("nan"), "stair height in"), (float("inf"), "stair height in"), (-0.05, "stair height in"),
                     (0.21, "stair height in"), (0.155, "multiple of 0.01"), (0.001, "multiple of 0.01")):
        with pytest.raises(ValueError, match=msg):
            BatchedHumanoidEnv(8, model="jvrc_step", stair_curriculum=bad)


@pytest.mark.parametrize("env_name, value, message", [
    ("jvrc_walk", "0.1", "jvrc_walk has no stair curriculum"),
    ("h1", "0.1", "h1 has no stair curriculum"),
    ("jvrc_walk_terrain", "0.05", "jvrc_walk_terrain has no stair curriculum"),
    ("h1_walk", "0.2", "h1_walk has no stair curriculum"),
    ("jvrc_step", "nan", "stair height in"),
    ("jvrc_step", "inf", "stair height in"),
    ("jvrc_step", "-0.1", "stair height in"),
    ("jvrc_step", "0.25", "stair height in"),
    ("jvrc_step", "0.125", "multiple of 0.01"),
])
def test_train_refuses_before_anything_exists(tmp_path, env_name, value, message):
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["train", "--env", env_name, "--stair-curriculum", value, "--logdir", str(tmp_path / "logs"), "--n-itr", "1"])
    assert not (tmp_path / "logs").exists()


def test_env_gets_the_run_value_and_old_runs_are_off(monkeypatch):
    """make_env_fn hands --stair-curriculum to the env, which `resume` rebuilds from experiment.pkl; a pickle written before the
    flag existed means off."""
    import run_experiment as rx
    got = []

    class FakeEnv:
        def __init__(self, n, **kw):
            got.append(kw)

        def close(self):
            pass

    monkeypatch.setattr(rx, "import_env", lambda name: FakeEnv)
    base = dict(env="jvrc_step", num_procs=8, seed=1, precision=32, max_traj_len=400, yaml=None, no_mirror=True)
    rx.make_env_fn(Namespace(**base, stair_curriculum=0.15), 0, 1, 0)()
    old = pickle.loads(pickle.dumps(Namespace(**base)))
    rx.make_env_fn(old, 0, 1, 0)()
    assert [g["stair_curriculum"] for g in got] == [0.15, 0.15, 0.0, 0.0]


def test_op_and_c_abi_are_declared():
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_step_stairs"' in src and 'm.impl("sim_reset_stairs"' in src
    hdr = open(os.path.join(root, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_step_stairs(" in hdr and "int lhw_sim_reset_stairs(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_step_stairs" in _lib.SIGNATURES and "lhw_sim_reset_stairs" in _lib.SIGNATURES
