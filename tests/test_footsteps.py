"""Chosen stepping-stone plans (`env.reset_footsteps`, `eval --footsteps`, DESIGN.md §7.7), CPU tier.

The reset with a chosen plan (csrc/sim_core.h env_reset<..., PLAN = true>, the body of lhw_sim_reset_footsteps's kernel) runs on
the host (tests/emu/footsteps_emu.cpp) next to the kernel source's host emulation of jvrc_step, at fp64 and fp32.  Given the plan a
plain reset draws, it must write the plain reset's record and observation bit for bit; given any plan, the sequence must be a numpy
restatement of generate_step_sequence + transform_sequence from the settled pose; closed-loop roll-outs of chosen plans must stay
with the oracle given the same plan.  Also: the sweep's cells and summary, and the command line's grammar and refusals."""
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


class FootEmu(emu.Emu):
    """emu.Emu on the library of footsteps_emu.cpp (sim_emu.cpp's entry points plus footsteps_emu_reset)."""

    def __init__(self, flat, precision=64, n=1, seed=0, first_id=0):
        lib = emu_variants._build("footsteps_emu.cpp", "sim_emu.cpp", os.path.join(HERE, "emu", "_build", "libfootsteps_emu.so"), [])
        self.lib = ctypes.CDLL(lib)
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

    def reset_footsteps(self, mode, value, fresh=False):
        obs = np.zeros((self.n, self.nobs), dtype=self.dt)
        rc = self.lib.footsteps_emu_reset(self.h, self.prec, self._p(self.sr), self._p(self.si), self.n, ctypes.c_uint32(self.seed),
                                          ctypes.c_uint32(self.first_id), self._p(np.ascontiguousarray(mode, np.int32)),
                                          self._p(np.ascontiguousarray(value, self.dt)), self._p(obs), int(fresh))
        assert rc == 0
        return obs


def _model(iteration_count=float("inf")):
    from learninghumanoidwalking_b200.model import load_model
    return load_model("jvrc_step"), iteration_count


def _flat(prec, iteration_count):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    return pack_model(load_model("jvrc_step"), tolerance=None if prec == 64 else 1e-6, iteration_count=iteration_count)


def _oracle(iteration_count=float("inf")):
    from oracle.oracle import Oracle
    return Oracle("jvrc_step", tolerance=1e-14, iteration_count=iteration_count)


def _u01(u, dt):
    return dt(u >> 8) * dt(1.0 / 16777216.0)


def _randint(u, n):
    return int((int(u) * n) >> 32)


def drawn_plan(o, seed, env_id, ctr, height, dt):
    """The plan a plain reset draws at event counter ctr (sim_core.h step_task_reset): (mode, value)."""
    u, v = o.philox(seed, env_id, ctr, 3), o.philox(seed, env_id, ctr, 4)
    cm = _u01(u[0], dt)
    mode = (CURVED if cm < dt(0.15) else STANDING if cm < dt(0.15 + 0.05) else BACKWARD if cm < dt(0.15 + 0.05 + 0.2)
            else LATERAL if cm < dt(0.15 + 0.05 + 0.2 + 0.3) else FORWARD)
    nplan = len(_model()[0]["stepping"]["plans"])
    value = {CURVED: float(_randint(u[2], nplan)), STANDING: 0.0, BACKWARD: 0.0,
             LATERAL: -1.0 if _randint(u[2], 2) == 0 else 1.0, FORWARD: -height if _randint(v[0], 2) == 0 else height}[mode]
    return mode, value


@pytest.mark.parametrize("height", [0.0, 0.1])
@pytest.mark.parametrize("precision", [64, 32])
def test_given_the_drawn_plan_equals_plain_reset(precision, height):
    """Every env of a batch, fresh and then again mid-episode, gets the plan its plain reset draws (type, +- curriculum height,
    plan index, lateral side, recomputed with the oracle's Philox): record and observation are the plain reset's, bit for bit.
    This pins every draw that is not part of the plan (phase, first-step offset, randint(2, 4), init noise, rng_ctr)."""
    ic = 3000 + 8000 * height / 0.1
    flat = _flat(precision, ic)
    N, seed, first_id = 64, 7, 3
    o = _oracle()
    plain, chosen = FootEmu(flat, precision, N, seed, first_id), FootEmu(flat, precision, N, seed, first_id)
    dt = plain.dt
    modes = set()
    for rnd in range(2):
        ctr = plain.si[:, 4] + 1      # the reset's event counter
        plan = [drawn_plan(o, seed, first_id + i, int(ctr[i]), height, dt) for i in range(N)]
        mode = np.array([p[0] for p in plan], np.int32)
        value = np.array([p[1] for p in plan])
        modes |= set(mode.tolist())
        if rnd == 0:
            po = plain.reset()
        else:     # mid-episode, every third env is left out: its row is untouched, as a plain reset's masked-out row is
            mode[::3] = -1
            po = np.zeros_like(plain.sr[:, :plain.nobs])
            for i in np.flatnonzero(mode >= 0):
                po[i] = plain.reset_one(i)
        co = chosen.reset_footsteps(mode, value, fresh=rnd == 0)
        assert np.array_equal(plain.si, chosen.si), rnd
        assert plain.sr.tobytes() == chosen.sr.tobytes(), rnd
        assert po.tobytes() == co.tobytes(), rnd
        assert np.array_equal(plain.si[mode >= 0, 1], mode[mode >= 0])
        a = np.random.RandomState(rnd).normal(size=(N, plain.nu)) * 0.3
        for _ in range(5):
            plain.step(a, autoreset=0)
            chosen.step(a, autoreset=0)
    assert modes == set(range(5)), modes


def _period():
    from learninghumanoidwalking_b200.model.loader import phase_clock_table
    mj = _model()[0]
    t = mj["cfg"]["task"]
    return phase_clock_table(t["swing_duration"], t["stance_duration"], 0.1, "grounded", 1.0 / mj["cfg"]["control_dt"],
                             total_duration=t["total_duration"])[0]


def numpy_plan(mode, value, phase, u2, u3, plans, period):
    """tasks/stepping_task.py generate_step_sequence: the plan relative to the feet, rows (x, y, z, theta)."""
    if mode == CURVED:
        k = int(value) if value >= 0 else _randint(u2, len(plans))
        return [(x, y, 0.0, th) for x, y, th in plans[k]]
    if mode == LATERAL:
        y, rows = 0.0, []
        for i in range(1, NSLAB):
            y = y + 0.4 if i % 2 else y - (2.0 / 3.0) * 0.4
            rows.append((0.0, value * y, 0.0, 0.0))
        return rows
    step_size = -0.1 if mode == BACKWARD else 0.3
    num_steps = 1 if mode == STANDING else NSLAB
    height = value if mode == FORWARD else 0.0
    first = 0.095 + (0.105 - 0.095) * _u01(u2, np.float64)
    if phase == period // 2 and period % 2 == 0:
        rows, y = [(0.0, -first, 0.0, 0.0)], -0.15
    else:
        rows, y = [(0.0, first, 0.0, 0.0)], 0.15
    x = z = 0.0
    c = 2 + _randint(u3, 2)
    for i in range(1, num_steps - 1):
        x += step_size
        y *= -1
        if i > c:
            z += height
        rows.append((x, y, z, 0.0))
    rows.append((x + step_size, -y, z, 0.0))
    return rows


def numpy_transform(rows, root_xmat, foot_xpos):
    """transform_sequence: about the mid-point of the two foot bodies, yawed with the root; unused boxes at (0, 0, -1, 0)."""
    R = np.asarray(root_xmat).reshape(3, 3)
    yaw = np.arctan2(R[1, 0], R[0, 0])
    f = np.asarray(foot_xpos).reshape(2, 3)
    mid = (f[0, :2] + f[1, :2]) / 2
    seq = np.zeros((NSLAB, 4))
    seq[:, 2] = -1
    for i, (x, y, z, th) in enumerate(rows):
        seq[i] = (mid[0] + x * np.cos(yaw) - y * np.sin(yaw), mid[1] + x * np.sin(yaw) + y * np.cos(yaw), z, yaw + th)
    return seq


@pytest.mark.parametrize("precision", [64, 32])
def test_plans_equal_numpy(precision):
    """For every plan type and a set of stair heights, plan indices and sides, the record's seq and tk of a fresh env are the
    numpy restatement built from the oracle's settled pose; the mode word is the type, the unused boxes sit below the floor; rows
    with mode -1 are not touched (not even zeroed)."""
    flat = _flat(precision, float("inf"))
    mj = _model()[0]
    plans, period = mj["stepping"]["plans"], _period()
    cells = ([(FORWARD, h) for h in (-0.2, -0.1, 0.0, 0.05, 0.1, 0.15, 0.2)] + [(LATERAL, 1.0), (LATERAL, -1.0)]
             + [(CURVED, k) for k in (-1.0, 0.0, 17.0, len(plans) - 1.0)] + [(STANDING, 0.0), (BACKWARD, 0.0), (-1, 0.0)])
    N, seed, first_id = 2 * len(cells), 11, 5
    mode = np.array([cells[i % len(cells)][0] for i in range(N)], np.int32)
    value = np.array([cells[i % len(cells)][1] for i in range(N)])
    e = FootEmu(flat, precision, N, seed, first_id)
    obs = e.reset_footsteps(mode, value, fresh=True)
    o = _oracle()
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    o.batch_reset(envs, N)
    tol = 1e-9 if precision == 64 else 2e-4
    for i in range(N):
        if mode[i] < 0:
            assert not e.sr[i].any() and not e.si[i].any() and not obs[i].any()
            continue
        ctr = int(e.si[i, 4])
        u = o.philox(seed, first_id + i, ctr, 3)
        rows = numpy_plan(int(mode[i]), float(e.dt(value[i])), int(e.si[i, 0]), u[2], u[3], plans, period)
        assert int(o.field(envs, i, "rng_ctr")[0]) == ctr     # the oracle's settled pose is that of the same reset
        want = numpy_transform(rows, o.field(envs, i, "root_xmat"), o.field(envs, i, "foot_xpos"))
        seq = e.sr[i, SEQ:SEQ + 4 * NSLAB].reshape(NSLAB, 4).astype(np.float64)
        assert e.si[i, 1] == mode[i]
        assert e.sr[i, TK] == len(rows) and e.sr[i, TK + 1] == 0 and e.sr[i, TK + 2] == 1, (i, e.sr[i, TK:TK + 5])
        assert np.abs(seq - want).max() < tol, (i, mode[i], value[i], np.abs(seq - want).max())


def test_chosen_plan_rollout_matches_oracle():
    """16 envs x 300 closed-loop autoreset steps at fp64, plans of every type with stair heights up to 0.15 m: the emulation resets
    with the chosen plans; the oracle, whose reset is unchanged, resets plainly and then gets the same plan words (mode, seq,
    sequence length, targets).  The roll-outs agree within the bound of the held-command roll-outs, falls included, and after each
    env's autoreset its plan is drawn again on both sides."""
    from learninghumanoidwalking_b200.model import load_model, pack_model
    N, seed, first_id = 16, 13, 2
    flat = pack_model(load_model("jvrc_step"), tolerance=1e-14)
    o = _oracle()
    e = FootEmu(flat, 64, N, seed, first_id)
    envs = o.make_envs(N, seed=seed, first_id=first_id)
    cells = [(FORWARD, 0.15), (FORWARD, -0.1), (FORWARD, 0.05), (LATERAL, 1.0), (LATERAL, -1.0), (CURVED, 3.0), (CURVED, -1.0),
             (STANDING, 0.0), (BACKWARD, 0.0)]
    mode = np.array([cells[i % len(cells)][0] for i in range(N)], np.int32)
    value = np.array([cells[i % len(cells)][1] for i in range(N)])
    eo = e.reset_footsteps(mode, value, fresh=True)
    oo = o.batch_reset(envs, N)
    for i in range(N):
        o.set_field(envs, i, "mode", e.si[i, 1])
        o.set_field(envs, i, "seq", e.sr[i, SEQ:SEQ + 4 * NSLAB])
        o.set_field(envs, i, "seq_len", int(e.sr[i, TK]))
        o.set_field(envs, i, "t1", int(e.sr[i, TK + 1]))
        o.set_field(envs, i, "t2", int(e.sr[i, TK + 2]))
    assert np.abs(oo - eo).max() < 1e-10      # the reset's observation does not see the plan (its goal words are zero)
    rng = np.random.RandomState(4)
    worst, n_end, n_fell = 0.0, 0, 0
    for t in range(300):
        a = rng.normal(size=(N, e.nu)) * 0.25
        oo, to, tt, rr, dd, ee = o.batch_step(envs, N, a, max_traj_len=120)
        eo_, et, etm, er, ed, een, _, _ = e.step(a, max_traj_len=120)
        assert (dd == ed).all() and (ee == een).all(), t
        oq = np.stack([o.field(envs, i, "qpos")[:e.nq] for i in range(N)])
        ended = een != 0      # the terminal observation is written where the step ended the env
        worst = max(worst, np.abs(oo - eo_).max(), np.abs(to - et)[ended].max(initial=0), np.abs(tt - etm).max(), np.abs(rr - er).max(),
                    np.abs(oq - e.qpos).max())
        n_end += int(een.sum())
        n_fell += int(ed.sum())
    assert worst < 1e-7, worst
    assert n_end > 0 and n_fell > 0, (n_end, n_fell)


def _eval_args(**kw):
    base = dict(num_envs=None, footsteps=None, command=None, push_speeds=None)
    base.update(kw)
    return Namespace(**base)


def test_footstep_grammar_cells_and_summary():
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import evaluation as ev
    cells = rx.footstep_cells(_eval_args(num_envs=64, footsteps=["forward:0,0.05,-0.1", "lateral:left,right", "backward", "curved",
                                                                  "curved:3,17", "standing"]))
    assert cells == [("FORWARD", 0.0), ("FORWARD", 0.05), ("FORWARD", -0.1), ("LATERAL", 1.0), ("LATERAL", -1.0), ("BACKWARD", 0.0),
                     ("CURVED", -1.0), ("CURVED", 3.0), ("CURVED", 17.0), ("STANDING", 0.0)]
    assert rx.footstep_cells(_eval_args()) is None
    mode, value = ev.footstep_grid(23, cells)
    assert list(mode[:10]) == [4, 4, 4, 3, 3, 2, 0, 0, 0, 1] and list(mode[10:13]) == [4, 4, 4] and value[22] == -0.1
    acc = np.zeros((23, ev.WORDS))
    acc[:, ev.LEN] = np.arange(23) + 10
    acc[:, ev.RET] = 2.0
    acc[:, ev.SEQLEN] = 18
    acc[:, ev.REACHED] = np.where(np.arange(23) % 2 == 0, 17, 3)
    acc[::5, ev.DONE] = 1
    s = ev.footstep_summary(acc, mode, value, cells)["cells"]
    assert [c["label"] for c in s] == ["forward:0", "forward:0.05", "forward:-0.1", "lateral:left", "lateral:right", "backward",
                                       "curved", "curved:3", "curved:17", "standing"]
    for c, (name, val) in zip(s, cells):
        m = (mode == ev.FOOTSTEP_MODES.index(name)) & (value == val)
        assert c["n"] == m.sum() and c["mean_length"] == acc[m, ev.LEN].mean()
        assert c["fall_fraction"] == (acc[m, ev.DONE] != 0).mean()
        assert c["completed_fraction"] == (acc[m, ev.REACHED] >= 17).mean() and c["mean_sequence_length"] == 18
        assert c["return_mean"] == 2.0
    assert "lateral:left" in ev.format_footstep_table(dict(cells=s))


@pytest.mark.parametrize("extra, message", [
    (["--footsteps", "sideways"], "unknown plan type"),
    (["--footsteps", "standing:0"], "takes no values"),
    (["--footsteps", "backward:1"], "takes no values"),
    (["--footsteps", "forward:x"], "stair heights"),
    (["--footsteps", "forward:nan"], "finite"),
    (["--footsteps", "forward:0.25"], "must lie in"),
    (["--footsteps", "lateral:up"], "lateral:left"),
    (["--footsteps", "curved:1.5"], "plan index"),
    (["--footsteps", "curved:109"], "plan index"),
    (["--footsteps", "forward:0.1", "--command", "standing"], "separate sweeps"),
    (["--footsteps", "forward:0.1", "--push-speeds", "0.5", "--num-envs", "8"], "separate sweeps"),
    (["--footsteps", "forward:0,0.1"], "need the batched evaluation"),
    (["--footsteps", "forward:0,0.1", "lateral:left,right", "--num-envs", "3"], "every cell needs"),
])
def test_eval_refuses_before_loading_anything(tmp_path, extra, message):
    """Every refusal comes before an actor is looked for (the run directory here has none)."""
    import run_experiment as rx
    with pytest.raises(SystemExit, match=message):
        rx.main(["eval", "--path", str(tmp_path / "no_run"), *extra])


@pytest.mark.parametrize("env_name", ["jvrc_walk", "h1", "jvrc_walk_terrain", "h1_walk"])
@pytest.mark.parametrize("extra", [[], ["--num-envs", "8"]])
def test_eval_refuses_runs_without_footstep_plans(tmp_path, env_name, extra):
    """The run's env comes from its experiment.pkl, which is read before the actor is loaded (the directory has no actor)."""
    import run_experiment as rx
    run = tmp_path / "run"
    run.mkdir()
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env=env_name, max_traj_len=400, yaml=None), f)
    with pytest.raises(SystemExit, match=f"{env_name} has no footstep plan"):
        rx.main(["eval", "--path", str(run), "--footsteps", "forward:0.1", *extra])


def test_op_and_c_abi_are_declared():
    root = os.path.dirname(HERE)
    src = open(os.path.join(root, "learninghumanoidwalking_b200", "csrc", "torch_ops.cpp")).read()
    assert 'm.impl("sim_reset_footsteps"' in src
    hdr = open(os.path.join(root, "include", "lhw_b200.h")).read()
    assert "int lhw_sim_reset_footsteps(" in hdr and "int lhw_sim_footstep_limits(" in hdr
    from learninghumanoidwalking_b200 import _lib
    assert "lhw_sim_reset_footsteps" in _lib.SIGNATURES and "lhw_sim_footstep_limits" in _lib.SIGNATURES
