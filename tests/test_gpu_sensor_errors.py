"""Sensor errors on the device (DESIGN.md §7.12): the sensor kernel against the host body bit for bit for every variant at both
precisions and in both phases; the op's refusals before any launch; sensors off launching exactly what the env launched before;
with sensors on, records equal to the sensor-free records under fixed actions, and eager, graph-replayed, step_slice-halved and
sharded roll-outs agreeing bit for bit; a `train --snapshot` run resuming with its rows; the sweep's all-zero cell against a
nominal evaluation; and `train --sensor-noise --sensor-bias` then `eval --sensor-errors --report` end to end."""
import json
import pickle

import numpy as np
import pytest
import torch

from test_sensor_errors import DIMS, VARIANTS, random_obs, random_rows, sense, sense_numpy
from test_gpu_command import _actions, _graph_stepper

pytestmark = pytest.mark.gpu


def _env(name, precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, **kw)


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_kernel_equals_host_body(name, precision, philox):
    """torch.ops.lhw.sim_sense on 3000 envs (not a multiple of a block) against the host body, bit for bit: after a reset (every
    env, a mask) and after a step with and without autoreset (random ended flags), with and without the draw, at counters that
    differ per env; a sliced launch with its own first env id as well.  The first small case is also held to numpy."""
    from learninghumanoidwalking_b200 import _lib
    nrobot, nu, obs_dim = DIMS[name]
    n, seed = 3000, 11
    env = _env(name, precision, n, seed=seed)
    assert (env.obs_dim, env.act_dim) == (obs_dim, nu)
    dt = np.float64 if precision == 64 else np.float32
    rng = np.random.RandomState(5)
    env.state_i[:, 4] = torch.from_numpy(rng.randint(0, 1 << 30, size=n).astype(np.int32)).to(env.device)
    si = env.state_i.cpu().numpy()
    dev = lambda a: None if a is None else torch.from_numpy(np.ascontiguousarray(a)).to(env.device)
    checked_numpy = False
    for after_step, autoreset in ((False, False), (True, True), (True, False)):
        for sel in (None, ((rng.uniform(size=n) < 0.4) * rng.randint(1, 5, size=n)).astype(np.int32)):
            if after_step and sel is None:
                continue
            for draw in (None, (0.2, 0.5, 0.2)):
                rows, obs = random_rows(rng, n, nu, dt), random_obs(rng, n, obs_dim, dt)
                term = (obs.copy() if not autoreset else random_obs(rng, n, obs_dim, dt)) if after_step else None
                d_rows, d_obs, d_term = dev(rows), dev(obs), dev(term)
                _lib.ops().sim_sense(env._h.value, env.state_i, seed, 0, dev(sel), after_step, autoreset,
                                     None if draw is None else list(draw), d_rows, d_obs, d_term)
                if not checked_numpy:
                    want = sense_numpy(philox, seed, 0, si[:40], None if sel is None else sel[:40], after_step, autoreset, draw,
                                       nrobot, nu, rows[:40], obs[:40], None if term is None else term[:40])
                sense(precision, si, seed, 0, sel, after_step, autoreset, draw, nrobot, nu, rows, obs, term)
                case = (after_step, autoreset, sel is None, draw)
                assert d_rows.cpu().numpy().tobytes() == rows.tobytes(), case
                assert d_obs.cpu().numpy().tobytes() == obs.tobytes(), case
                if term is not None:
                    assert d_term.cpu().numpy().tobytes() == term.tobytes(), case
                if not checked_numpy:
                    assert rows[:40].tobytes() == want[0].tobytes() and obs[:40].tobytes() == want[1].tobytes()
                    checked_numpy = True
    rows, obs = random_rows(rng, n, nu, dt), random_obs(rng, n, obs_dim, dt)
    d_rows, d_obs = dev(rows), dev(obs)
    _lib.ops().sim_sense(env._h.value, env.state_i[1000:], seed, 1000, None, False, False, [0.1, 0.2, 0.1], d_rows[1000:],
                         d_obs[1000:], None)
    r2, o2 = rows[1000:].copy(), obs[1000:].copy()
    sense(precision, si[1000:], seed, 1000, None, False, False, (0.1, 0.2, 0.1), nrobot, nu, r2, o2, None)
    assert d_rows.cpu().numpy()[1000:].tobytes() == r2.tobytes() and d_obs.cpu().numpy()[1000:].tobytes() == o2.tobytes()
    assert d_rows.cpu().numpy()[:1000].tobytes() == rows[:1000].tobytes() and d_obs.cpu().numpy()[:1000].tobytes() == obs[:1000].tobytes()
    env.close()


def test_op_and_env_refuse_bad_arguments():
    from learninghumanoidwalking_b200 import _lib
    env = _env("jvrc_walk", 64, 8, seed=1)
    env.reset()
    dev = env.device
    good = torch.zeros(8, 18, dtype=torch.float64, device=dev)
    m = torch.ones(8, dtype=torch.int32, device=dev)

    def sense(sensor=good, sel=None, after_step=False, draw=None, obs=env.obs, term=None):
        _lib.ops().sim_sense(env._h.value, env.state_i, 1, 0, sel, after_step, True, draw, sensor, obs, term)

    c0 = _lib.lib().lhw_launch_count()
    for bad, msg in [(good.cpu(), "CUDA tensor"), (good.float(), "dtype"), (good[:4], "shape"), (good[:, :17].contiguous(), "shape"),
                     (torch.zeros(8, 36, dtype=torch.float64, device=dev)[:, ::2], "contiguous")]:
        with pytest.raises(RuntimeError, match=msg):
            sense(bad)
    for bad, msg in [(env.obs.cpu(), "CUDA tensor"), (env.obs.float(), "dtype"), (env.obs[:4], "shape")]:
        with pytest.raises(RuntimeError, match=msg):
            sense(obs=bad)
        with pytest.raises(RuntimeError, match=msg):
            sense(after_step=True, sel=m, term=bad)
    for bad, msg in [(m.cpu(), "CUDA tensor"), (m.long(), "dtype"), (m[:4], "shape")]:
        with pytest.raises(RuntimeError, match=msg):
            sense(sel=bad)
    with pytest.raises(RuntimeError, match="term_obs"):
        sense(after_step=True, sel=m)
    with pytest.raises(RuntimeError, match="draw must be"):
        sense(draw=[0.1, 0.1])
    for draw, msg in [([0.3, 0, 0], "roll / pitch"), ([0, 0.6, 0], "gyro"), ([0, 0, -0.1], "encoder"),
                      ([float("nan"), 0, 0], "roll / pitch"), ([0, 0, float("inf")], "encoder")]:
        with pytest.raises(RuntimeError, match=msg):
            sense(draw=draw)
    assert _lib.lib().lhw_launch_count() == c0           # every refusal came before a launch
    for noise, bias, msg in ((float("nan"), (0, 0, 0), "noise multiplier"), (5.0, (0, 0, 0), "noise multiplier"),
                             (1.0, (0.3, 0, 0), "offset range"), (1.0, (0, 0), "three numbers")):
        with pytest.raises(ValueError, match=msg):
            _env("jvrc_walk", 64, 8, sensor_noise=noise, sensor_bias=bias)
    for noise, bias, msg in ((5.0, None, "noise multiplier"), ([1.0] * 7, None, "noise must be"),
                             (1.0, np.zeros(16), "bias must be"), (1.0, np.zeros((7, 17)), "bias must be"),
                             (1.0, np.full(17, 0.25), "offset must lie in"), (1.0, [float("nan")] + [0] * 16, "offset must lie in")):
        with pytest.raises(ValueError, match=msg):
            env.set_sensor_errors(noise, bias)
    assert env.sensor is None
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_sensors_off_is_the_plain_env(precision):
    """sensor_noise=0 and no bias is the env as it was: no sensor tensor, one launch per step and per reset, and 300 autoreset
    steps bit for bit equal to an env built without the arguments.  With random sensor errors a step is two launches (the step,
    then the pass) and so is a reset; explicit rows make the same one extra launch."""
    from learninghumanoidwalking_b200 import _lib
    L = _lib.lib()
    a, b = _env("jvrc_walk", precision, 512, seed=2), _env("jvrc_walk", precision, 512, seed=2, sensor_noise=0.0,
                                                           sensor_bias=(0.0, 0.0, 0.0))
    assert b.sensor is None
    ga, gb = (torch.Generator(device=a.device).manual_seed(4) for _ in range(2))
    c0 = L.lhw_launch_count()
    a.reset()
    b.reset()
    assert L.lhw_launch_count() - c0 == 2
    for t in range(300):
        c0 = L.lhw_launch_count()
        b.step(_actions(b, gb))
        assert L.lhw_launch_count() - c0 == 1
        a.step(_actions(a, ga))
        for x in ("state_r", "state_i", "obs", "term_obs", "reward", "done", "ended"):
            assert torch.equal(getattr(a, x), getattr(b, x)), (x, t)
    r = _env("jvrc_walk", precision, 64, seed=2, sensor_noise=1.0, sensor_bias=(0.05, 0.1, 0.02))
    c0 = L.lhw_launch_count()
    r.reset()
    r.step(_actions(r, ga))
    assert L.lhw_launch_count() - c0 == 4
    x = _env("jvrc_walk", precision, 64, seed=2)
    x.set_sensor_errors(0.0)
    c0 = L.lhw_launch_count()
    x.reset()
    x.step(_actions(x, ga))
    assert L.lhw_launch_count() - c0 == 4
    for e in (a, b, r, x):
        e.close()


@pytest.mark.parametrize("name, extra", [("jvrc_walk", {}), ("h1", dict(payload_mass=10.0, action_delay=0.01, motor_strength=0.3)),
                                         ("jvrc_step", dict(action_delay=0.02, stair_curriculum=0.05)),
                                         ("h1_walk", dict(push_vel=0.5, push_interval=0.5))])
@pytest.mark.parametrize("precision", [64, 32])
def test_records_are_the_sensor_free_records(name, extra, precision):
    """300 autoreset steps of max_traj_len 30 under one fixed action sequence (with the other randomisations of the row on): the
    env with random sensor errors (multiplier 2, offsets redrawn at every auto-reset) against the same env without them.  Records,
    rewards, reward terms, dones, ended flags and episode words are bit-identical; the robot-state words of obs differ, the task
    words do not."""
    n, kw = 256, dict(seed=3, max_traj_len=30, **extra)
    a, b = _env(name, precision, n, **kw), _env(name, precision, n, sensor_noise=2.0, sensor_bias=(0.1, 0.2, 0.05), **kw)
    a.reset()
    b.reset()
    nrobot = DIMS[name][0]
    g = torch.Generator(device=a.device).manual_seed(8)
    n_end = 0
    for t in range(300):
        act = _actions(a, g)
        a.step(act)
        b.step(act)
        for x in ("state_r", "state_i", "reward", "rew_terms", "done", "ended", "ep_len", "ep_rew"):
            assert torch.equal(getattr(a, x), getattr(b, x)), (x, t)
        assert torch.equal(a.obs[:, nrobot:], b.obs[:, nrobot:]), t
        assert (a.obs[:, :nrobot] != b.obs[:, :nrobot]).any(dim=1).all(), t
        n_end += int(a.ended.sum())
    assert n_end > 0
    a.close()
    b.close()


@pytest.mark.parametrize("name, extra", [("jvrc_walk", {}), ("h1", dict(payload_mass=10.0, action_delay=0.01, motor_strength=0.3)),
                                         ("jvrc_step", dict(action_delay=0.02, stair_curriculum=0.05))])
@pytest.mark.parametrize("precision", [64, 32])
def test_eager_graph_halves_and_shards_agree(name, extra, precision):
    """Random sensor errors (with other randomisations on): four copies of a batch under the same actions for 300 autoreset
    steps of max_traj_len 30, stepped eagerly, through a replayed CUDA graph, as two step_slice halves, and as two env shards
    (first_env_id 0 and n/2).  Records, observations, terminal observations and sensor rows are bit-identical after every step,
    and the rows are redrawn."""
    n = 512
    kw = dict(seed=6, max_traj_len=30, sensor_noise=1.5, sensor_bias=(0.1, 0.3, 0.1), **extra)
    envs = {k: _env(name, precision, n, **kw) for k in ("eager", "graph", "halves")}
    shards = [_env(name, precision, n // 2, first_env_id=k * n // 2, **kw) for k in range(2)]
    for e in list(envs.values()) + shards:
        e.reset()
    start = envs["eager"].sensor.clone()
    assert start[:, 1:].abs().max() > 0 and (start[:, 0] == 1.5).all()
    gens = {k: torch.Generator(device=e.device).manual_seed(7) for k, e in envs.items()}
    gs = torch.Generator(device=shards[0].device).manual_seed(7)
    graph_step = _graph_stepper(envs["graph"], gens["graph"])
    cat = lambda x: torch.cat([getattr(s, x) for s in shards])
    for t in range(300):
        envs["eager"].step(_actions(envs["eager"], gens["eager"]))
        graph_step()
        a = _actions(envs["halves"], gens["halves"])
        envs["halves"].step_slice(0, n // 2, a[:n // 2].contiguous())
        envs["halves"].step_slice(n // 2, n, a[n // 2:].contiguous())
        a = (torch.randn(n, shards[0].act_dim, generator=gs, device=shards[0].device) * 0.5).to(shards[0].dtype)
        shards[0].step(a[:n // 2].contiguous())
        shards[1].step(a[n // 2:].contiguous())
        e = envs["eager"]
        for k in ("graph", "halves"):
            o = envs[k]
            for x in ("state_r", "state_i", "obs", "term_obs", "sensor", "reward"):
                assert torch.equal(getattr(o, x), getattr(e, x)), (k, x, t)
        for x in ("state_r", "obs", "term_obs", "sensor"):
            assert torch.equal(cat(x), getattr(e, x)), (x, t)
    assert not torch.equal(envs["eager"].sensor, start)
    for x in list(envs.values()) + shards:
        x.close()


def test_explicit_rows_hold_and_apply_from_the_next_reset():
    """set_sensor_errors does not rewrite the current obs; the rows apply from the next reset's observation on, hold through
    steps and masked resets, and term_obs equals obs without autoreset."""
    n = 64
    a, b = _env("h1_walk", 64, n, seed=2), _env("h1_walk", 64, n, seed=2)
    a.reset()
    b.reset()
    rows = np.zeros((n, 16))
    rows[:, 0] = 1.0
    rows[:, 6:] = 0.1
    before = b.obs.clone()
    b.set_sensor_errors(rows[:, 0], rows[:, 1:])
    assert torch.equal(b.obs, before)
    a.reset()
    b.reset()
    assert torch.equal(b.sensor.cpu(), torch.from_numpy(rows))
    d = (b.obs - a.obs)[:, 5:15]
    assert (d.abs() <= 0.1 + 0.02 + 1e-12).all() and (d > 0.07).all()
    act = torch.zeros(n, b.act_dim, dtype=b.dtype, device=b.device)
    for _ in range(5):
        a.step(act, autoreset=False)
        b.step(act, autoreset=False)
        assert torch.equal(b.term_obs, b.obs) and torch.equal(a.state_r, b.state_r)
    mask = torch.arange(n, device=b.device) % 2 == 0
    a.reset(mask)
    b.reset(mask)
    assert torch.equal(b.sensor.cpu(), torch.from_numpy(rows)) and (b.obs[:, 5:15] - a.obs[:, 5:15] > 0.07).all()
    a.close()
    b.close()


TRAIN = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
         "--eval-freq", "2", "--snapshot", "--sensor-noise", "1", "--sensor-bias", "0.05,0.05,0.02"]


def test_resume_carries_the_rows(tmp_path):
    """`train --snapshot --sensor-noise 1 --sensor-bias 0.05,0.05,0.02` for 4 iterations against 3 iterations then
    `resume --n-itr 4`: the same final snapshot, sensor rows included, and the same checkpoints.  A sensor run whose snapshot has
    no rows is refused."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl.snapshot import SnapshotError
    from test_gpu_resume import _compare_runs
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + TRAIN)
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    rx.main(["resume", "--path", str(run_b), "--n-itr", "4"])
    _compare_runs(run_a, run_b, 1)
    sa, sb = (torch.load(d / "snapshot" / "itr_3" / "rank_0.pt", weights_only=True) for d in (run_a, run_b))
    assert torch.equal(sa["sensor"], sb["sensor"]) and sa["sensor"].shape == (64, 18)
    plain = TRAIN[:-4]
    rx.main(["train", "--logdir", str(tmp_path / "c"), "--n-itr", "2"] + plain)
    (run_c,) = list((tmp_path / "c").iterdir())
    assert "sensor" not in torch.load(run_c / "snapshot" / "itr_1" / "rank_0.pt", weights_only=True)
    with open(run_c / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    args.sensor_noise = 1.0
    with open(run_c / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    with pytest.raises(SnapshotError, match="no sensor errors"):
        rx.main(["resume", "--path", str(run_c), "--n-itr", "3"])


def test_train_then_eval_sweep(tmp_path, capsys):
    """`train --sensor-noise 1 --sensor-bias 0.05,0.05,0.02` then `eval --num-envs 240 --sensor-errors roll:0,0.1 pitch:-0.1
    encoder:0.05 noise:2 --report`: the start-up line, the table and the report's `summary.sensor` and per-env column.  Then the
    sweep's all-zero cell against a nominal batched evaluation of the same env ids: the accumulator rows are bit-identical."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import evaluation as ev
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    rx.main(["train", "--env", "jvrc_walk", "--sensor-noise", "1", "--sensor-bias", "0.05,0.05,0.02", "--logdir", str(tmp_path / "logs"),
             "--num-procs", "64", "--n-itr", "2", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
             "--eval-freq", "2"])
    assert "Sensor errors: noise x1; offsets up to 0.05 rad roll / pitch" in capsys.readouterr().out
    report = tmp_path / "r.json"
    spec = ["roll:0,0.1", "pitch:-0.1", "encoder:0.05", "noise:2"]
    cells = [("roll", 0.0), ("roll", 0.1), ("pitch", -0.1), ("encoder", 0.05), ("noise", 2.0)]
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "240", "--sensor-errors", *spec, "--report", str(report)])
    assert "sensor errors" in capsys.readouterr().out
    r = json.loads(report.read_text())
    s = r["summary"]["sensor"]
    assert [(c["kind"], c["value"]) for c in s["cells"]] == cells and [c["cell"] for c in s["cells"]] == list(range(5))
    assert sum(c["n"] for c in s["cells"]) == 240 and all({"fall_fraction", "mean_length", "return_mean", "tracking"} <= set(c)
                                                         for c in s["cells"])
    assert r["per_env"]["sensor_cell"] == (np.arange(240) % 5).tolist()
    install_reference_aliases()
    (run,) = list((tmp_path / "logs").iterdir())
    policy = torch.load(run / "actor.pt", weights_only=False).cuda().eval()
    n, accs = 240, []
    for sweep in (True, False):
        env = _env("jvrc_walk", 64, n, max_traj_len=40)
        rows = ev.sensor_grid(n, cells, env.act_dim)[1:] if sweep else None
        accs.append(ev.rollout(env, policy, 40, sensor=rows).cpu().numpy())
        env.close()
    cell0 = np.arange(n) % len(cells) == 0
    assert accs[0][cell0].tobytes() == accs[1][cell0].tobytes()
    assert accs[0][~cell0].tobytes() != accs[1][~cell0].tobytes()
