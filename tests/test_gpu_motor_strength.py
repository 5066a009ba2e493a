"""Motor strengths on the device (DESIGN.md §7.11): the MOTOR step kernels, single-warp and lock-step, at strength 1 against the
plain kernels bit for bit and with strengths against the host body; the draw kernel against numpy; the ops' refusals; strengths
off launching exactly the plain kernels; eager, graph-replayed, step_slice-halved and sharded roll-outs agreeing bit for bit with
random strengths, alone and with delays, payloads and the stair curriculum; a `train --snapshot` run resuming with its strengths;
the sweep's 1.0 cell against a nominal evaluation; limp robots falling; and `train --motor-strength` then
`eval --motor-strengths --report` end to end."""
import json
import pickle

import numpy as np
import pytest
import torch

from test_motor_strength import VARIANTS, MotorEmu, _flat, draws
from test_gpu_command import _actions, _graph_stepper

pytestmark = pytest.mark.gpu


def _env(name, precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, **kw)


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


@pytest.mark.parametrize("wpb", ["1", None])
@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_unit_strength_kernels_are_the_plain_kernels(name, precision, wpb, monkeypatch):
    """One-warp (LHW_WARPS_PER_BLOCK=1) and lock-step blocks: 300 envs (not a multiple of a block) given strength 1 through
    set_motor_strength, 60 autoreset steps of max_traj_len 20 against an env without strengths: records and every output bit for
    bit."""
    if wpb is not None:
        monkeypatch.setenv("LHW_WARPS_PER_BLOCK", wpb)
    n = 300
    a, b = _env(name, precision, n, seed=4, max_traj_len=20), _env(name, precision, n, seed=4, max_traj_len=20)
    b.set_motor_strength(np.ones(n))
    a.reset()
    b.reset()
    g = torch.Generator(device=a.device).manual_seed(2)
    for t in range(60):
        act = _actions(a, g)
        a.step(act)
        b.step(act)
        for x in ("state_r", "state_i", "obs", "term_obs", "reward", "rew_terms", "done", "ended", "ep_len", "ep_rew"):
            assert torch.equal(getattr(a, x), getattr(b, x)), (x, t)
    a.close()
    b.close()


@pytest.mark.parametrize("wpb", ["1", None])
@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_device_equals_host_body(name, precision, wpb, philox, monkeypatch):
    """300 envs with random strengths at R = 1 (factors in [0, 2]), 40 autoreset steps of max_traj_len 20: before every step the
    device records and strengths are copied to the host body, and both take the step; then the host draw body redraws for the
    ended envs.  Strengths, done / ended and the integer words (but the solver's count) agree exactly; at fp64 the record and
    observation to 1e-8 (the device fuses multiply-adds), at fp32 only the exact words, as for payloads.  The first draws also
    equal the numpy restatement."""
    if wpb is not None:
        monkeypatch.setenv("LHW_WARPS_PER_BLOCK", wpb)
    n, seed = 300, 3
    env = _env(name, precision, n, seed=seed, max_traj_len=20, motor_strength=1.0)
    host = MotorEmu(_flat(name, precision), precision, n, seed, 0)
    env.reset()
    si = env.state_i.cpu().numpy()
    want = draws(philox, seed, 0, si, None, 1.0, env.act_dim, np.zeros((n, env.act_dim))).astype(host.dt)
    assert env.motor_strength.cpu().numpy().tobytes() == want.tobytes()
    g = torch.Generator(device=env.device).manual_seed(1)
    close = lambda x, y: precision == 32 or np.abs(x - y).max() < 1e-8
    n_end = 0
    for t in range(40):
        host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
        s = env.motor_strength.cpu().numpy().copy()
        a = _actions(env, g)
        hobs, _, _, _, hdone, hended, _, _ = host.step_motor(a.cpu().numpy(), s, max_traj_len=20)
        host.draw(hended, 1.0, s)
        env.step(a)
        assert np.array_equal(env.done.cpu().numpy(), hdone) and np.array_equal(env.ended.cpu().numpy(), hended), t
        assert env.motor_strength.cpu().numpy().tobytes() == s.tobytes(), t
        assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7]), t
        assert close(env.state_r.cpu().numpy(), host.sr) and close(env.obs.cpu().numpy(), hobs), t
        n_end += int(hended.sum())
    assert n_end > 0
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", ["jvrc_walk", "h1"])
def test_draw_kernel_equals_numpy(name, precision, philox):
    """The draw kernel on 5000 envs with counters 0 .. 4999: no mask, a mask, and a sliced launch with its own first env id;
    unselected envs keep their words."""
    from learninghumanoidwalking_b200 import _lib
    n, seed = 5000, 17
    env = _env(name, precision, n, seed=seed)
    nu = env.act_dim
    dt = np.float64 if precision == 64 else np.float32
    env.state_i[:, 4] = torch.arange(n, dtype=torch.int32, device=env.device)
    si = env.state_i.cpu().numpy()
    rng = np.random.RandomState(0)
    for R in (0.0, 0.3, 1.0):
        for mask in (None, (rng.uniform(size=n) < 0.4).astype(np.int32)):
            before = rng.normal(size=(n, nu)).astype(dt)
            p = torch.from_numpy(before).to(env.device)
            m = None if mask is None else torch.from_numpy(mask).to(env.device)
            _lib.ops().sim_draw_motor(env._h.value, env.state_i, seed, 0, m, R, p)
            want = draws(philox, seed, 0, si, mask, R, nu, before.astype(np.float64)).astype(dt)
            assert p.cpu().numpy().tobytes() == want.tobytes(), (R, mask is None)
    p = torch.zeros(n, nu, dtype=env.dtype, device=env.device)
    _lib.ops().sim_draw_motor(env._h.value, env.state_i[1000:], seed, 1000, None, 0.5, p[1000:])
    want = draws(philox, seed, 0, si, None, 0.5, nu, np.zeros((n, nu))).astype(dt)
    assert p.cpu().numpy()[1000:].tobytes() == want[1000:].tobytes() and not p[:1000].any()
    env.close()


def test_ops_and_env_refuse_bad_arguments():
    from learninghumanoidwalking_b200 import _lib
    env = _env("jvrc_walk", 64, 8, seed=1)
    env.reset()
    dev = env.device
    a = torch.zeros(8, env.act_dim, dtype=env.dtype, device=dev)
    good = torch.ones(8, 12, dtype=torch.float64, device=dev)
    pay = torch.zeros(8, 4, dtype=torch.float64, device=dev)
    d = torch.zeros(8, dtype=torch.int32, device=dev)

    def step(strength, payload=None, delay=None, level=None, k=0, e=env, act=a):
        _lib.ops().sim_step_motor(e._h.value, e.state_r, e.state_i, 1, 0, act, 400, True, e.obs, e.term_obs, e.reward, e.rew_terms,
                                  e.done, e.ended, e.ep_len, e.ep_rew, strength, payload, delay, level, k)

    c0 = _lib.lib().lhw_launch_count()
    for bad, msg in [(good.cpu(), "CUDA tensor"), (good.float(), "dtype"), (good[:4], "shape"), (good[:, :10].contiguous(), "shape"),
                     (torch.ones(8, 24, dtype=torch.float64, device=dev)[:, ::2], "contiguous")]:
        with pytest.raises(RuntimeError, match=msg):
            step(bad)
        with pytest.raises(RuntimeError, match=msg):
            _lib.ops().sim_draw_motor(env._h.value, env.state_i, 1, 0, None, 0.3, bad)
    for bad, msg in [(pay.cpu(), "CUDA tensor"), (pay.float(), "dtype"), (pay[:, :3].contiguous(), "shape")]:
        with pytest.raises(RuntimeError, match=msg):
            step(good, bad)
    for bad, msg in [(d.cpu(), "CUDA tensor"), (d.long(), "dtype"), (d[:4], "shape")]:
        with pytest.raises(RuntimeError, match=msg):
            step(good, None, bad)
    with pytest.raises(RuntimeError, match="mask"):
        _lib.ops().sim_draw_motor(env._h.value, env.state_i, 1, 0, d[:4], 0.3, good)
    for R in (-0.1, 1.5, float("nan"), float("inf")):
        with pytest.raises(RuntimeError, match="deviation"):
            _lib.ops().sim_draw_motor(env._h.value, env.state_i, 1, 0, None, R, good)
    with pytest.raises(RuntimeError, match="lhw_sim_step_motor: jvrc_walk has no stair curriculum"):
        step(good, None, None, d, 11)
    assert _lib.lib().lhw_launch_count() == c0           # every refusal came before a launch
    stairs = _env("jvrc_step", 64, 8, seed=1, stair_curriculum=0.1)
    stairs.reset()
    with pytest.raises(RuntimeError, match="n_levels"):
        step(good, None, None, stairs.stair_level, 22, e=stairs, act=torch.zeros(8, 12, dtype=torch.float64, device=dev))
    for R in (float("nan"), -0.1, 1.01):
        with pytest.raises(ValueError, match="range must lie in"):
            _env("jvrc_walk", 64, 8, motor_strength=R)
    for s, msg in (([2.5] * 8, "must lie in"), ([float("nan")] * 8, "must lie in"), ([-1.0] * 8, "must lie in"),
                   ([1.0] * 7, "strength must be"), (np.ones((8, 10)), "strength must be")):
        with pytest.raises(ValueError, match=msg):
            env.set_motor_strength(s)
    assert env.motor_strength is None
    stairs.close()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_strengths_off_is_the_plain_env(precision):
    """motor_strength=0 is the env as it was: no strength tensor, one launch per step and per reset, and 300 autoreset steps bit
    for bit equal to an env built without the argument.  With random strengths a step is two launches (the step, then the draw)
    and so is a reset."""
    from learninghumanoidwalking_b200 import _lib
    L = _lib.lib()
    a, b = _env("jvrc_walk", precision, 512, seed=2), _env("jvrc_walk", precision, 512, seed=2, motor_strength=0.0)
    assert b.motor_strength is None
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
        assert torch.equal(a.state_r, b.state_r) and torch.equal(a.state_i, b.state_i) and torch.equal(a.obs, b.obs), t
    r = _env("jvrc_walk", precision, 64, seed=2, motor_strength=0.3)
    c0 = L.lhw_launch_count()
    r.reset()
    r.step(_actions(r, ga))
    assert L.lhw_launch_count() - c0 == 4
    for x in (a, b, r):
        x.close()


@pytest.mark.parametrize("name, extra", [("jvrc_walk", {}), ("h1", dict(payload_mass=10.0, action_delay=0.01)),
                                         ("jvrc_step", dict(action_delay=0.02, payload_mass=10.0, stair_curriculum=0.05))])
@pytest.mark.parametrize("precision", [64, 32])
def test_eager_graph_halves_and_shards_agree(name, extra, precision):
    """Random strengths at R = 0.5 (with random delays and payloads, and on jvrc_step the stair curriculum as well): four copies
    of a batch under the same actions for 300 autoreset steps of max_traj_len 30, stepped eagerly, through a replayed CUDA graph,
    as two step_slice halves, and as two env shards (first_env_id 0 and n/2).  Records, outputs and strengths are bit-identical
    after every step; the strengths are redrawn."""
    n = 512
    kw = dict(seed=6, max_traj_len=30, motor_strength=0.5, **extra)
    envs = {k: _env(name, precision, n, **kw) for k in ("eager", "graph", "halves")}
    shards = [_env(name, precision, n // 2, first_env_id=k * n // 2, **kw) for k in range(2)]
    for e in list(envs.values()) + shards:
        e.reset()
    start = envs["eager"].motor_strength.clone()
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
            assert torch.equal(o.state_r, e.state_r) and torch.equal(o.state_i, e.state_i) and torch.equal(o.obs, e.obs), (k, t)
            assert torch.equal(o.motor_strength, e.motor_strength) and torch.equal(o.reward, e.reward), (k, t)
        assert torch.equal(cat("state_r"), e.state_r) and torch.equal(cat("motor_strength"), e.motor_strength), t
    assert not torch.equal(envs["eager"].motor_strength, start)
    for x in list(envs.values()) + shards:
        x.close()


@pytest.mark.parametrize("name", ["jvrc_walk", "h1_walk"])
def test_limp_robots_fall(name):
    """End to end on the device: with factor 0 on every joint (set after the reset, autoreset off) every env falls before the
    episode's 200 control steps end."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    n, steps = 256, 200
    env = _env(name, 64, n, seed=5, max_traj_len=steps)
    env.reset()
    env.set_motor_strength(np.zeros(n))
    acc = torch.zeros(n, ev.WORDS, dtype=torch.float64, device=env.device)
    for t in range(steps):
        env.step(torch.zeros(n, env.act_dim, dtype=env.dtype, device=env.device), autoreset=False)
        env.eval_accumulate(acc)
    limp = acc.cpu().numpy()
    env.close()
    assert (limp[:, ev.DONE] == 1).all() and (limp[:, ev.LEN] < steps).all()


TRAIN = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
         "--eval-freq", "2", "--snapshot", "--motor-strength", "0.3"]


def test_resume_carries_the_strengths(tmp_path):
    """`train --snapshot --motor-strength 0.3` for 4 iterations against 3 iterations then `resume --n-itr 4`: the same final
    snapshot, records and strengths included, and the same checkpoints.  A strength run whose snapshot has no strengths is
    refused."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl.snapshot import SnapshotError
    from test_gpu_resume import _compare_runs
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + TRAIN)
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    rx.main(["resume", "--path", str(run_b), "--n-itr", "4"])
    _compare_runs(run_a, run_b, 1)
    sa, sb = (torch.load(d / "snapshot" / "itr_3" / "rank_0.pt", weights_only=True) for d in (run_a, run_b))
    assert torch.equal(sa["motor_strength"], sb["motor_strength"]) and sa["motor_strength"].shape == (64, 12)
    plain = TRAIN[:-2]
    rx.main(["train", "--logdir", str(tmp_path / "c"), "--n-itr", "2"] + plain)
    (run_c,) = list((tmp_path / "c").iterdir())
    assert "motor_strength" not in torch.load(run_c / "snapshot" / "itr_1" / "rank_0.pt", weights_only=True)
    with open(run_c / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    args.motor_strength = 0.3
    with open(run_c / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    with pytest.raises(SnapshotError, match="no motor strengths"):
        rx.main(["resume", "--path", str(run_c), "--n-itr", "3"])


def test_train_then_eval_sweep(tmp_path, capsys):
    """`train --motor-strength 0.3` then `eval --num-envs 250 --motor-strengths 0,0.5,0.8,1,1.2 --motor-joints R_KNEE,L_KNEE
    --report`: the start-up line, the table and the report's `summary.motor_strength` and per-env column.  Then the sweep's 1.0
    cell against a nominal batched evaluation of the same env ids: the accumulator rows are bit-identical."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import evaluation as ev
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    rx.main(["train", "--env", "jvrc_walk", "--motor-strength", "0.3", "--logdir", str(tmp_path / "logs"), "--num-procs", "64",
             "--n-itr", "2", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    assert "Motor strengths: U(0.7, 1.3)" in capsys.readouterr().out
    report = tmp_path / "r.json"
    factors = [0.0, 0.5, 0.8, 1.0, 1.2]
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "250", "--motor-strengths", ",".join(map(str, factors)),
             "--motor-joints", "R_KNEE,L_KNEE", "--report", str(report)])
    assert "factor" in capsys.readouterr().out
    r = json.loads(report.read_text())
    s = r["summary"]["motor_strength"]
    assert s["factors"] == factors and [c["factor"] for c in s["cells"]] == factors and s["joints"] == ["R_KNEE", "L_KNEE"]
    assert sum(c["n"] for c in s["cells"]) == 250 and all({"fall_fraction", "mean_length", "return_mean", "tracking"} <= set(c)
                                                         for c in s["cells"])
    assert r["per_env"]["motor_strength"] == ev.motor_grid(250, factors).tolist()
    install_reference_aliases()
    (run,) = list((tmp_path / "logs").iterdir())
    policy = torch.load(run / "actor.pt", weights_only=False).cuda().eval()
    n = 250
    accs = []
    names = None
    for sweep in (True, False):
        env = _env("jvrc_walk", 64, n, max_traj_len=40)
        names = env.interface.get_motor_names()
        knee = np.array([x in ("R_KNEE", "L_KNEE") for x in names])
        strength = np.where(knee[None, :], ev.motor_grid(n, factors)[:, None], 1.0) if sweep else None
        accs.append(ev.rollout(env, policy, 40, motor=strength).cpu().numpy())
        env.close()
    assert sum(x in ("R_KNEE", "L_KNEE") for x in names) == 2
    cell1 = np.arange(n) % len(factors) == 3
    assert accs[0][cell1].tobytes() == accs[1][cell1].tobytes()
    assert accs[0][~cell1].tobytes() != accs[1][~cell1].tobytes()
