"""Action delays on the device (DESIGN.md §7.9): the DELAY step kernels, single-warp and lock-step, at delay 0 against the plain
kernels bit for bit and with delays against the host body; the draw kernel against numpy; the ops' refusals; delays off launching
exactly the plain kernels; eager, graph-replayed, step_slice-halved and sharded roll-outs agreeing bit for bit with random delays;
a `train --snapshot` run resuming with its delays; the latency sweep's 0-delay cell against an undelayed evaluation; and
`train --action-delay` then `eval --action-delays --report` end to end."""
import json
import pickle

import numpy as np
import pytest
import torch

from test_action_delay import VARIANTS, DelayEmu, _flat, draws
from test_gpu_command import _actions, _graph_stepper

pytestmark = pytest.mark.gpu


def _env(name, precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, **kw)


@pytest.mark.parametrize("wpb", ["1", None])
@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_zero_delay_kernels_are_the_plain_kernels(name, precision, wpb, monkeypatch):
    """One-warp (LHW_WARPS_PER_BLOCK=1) and lock-step blocks: 300 envs (not a multiple of a block) given delay 0 through
    set_action_delay, 60 autoreset steps of max_traj_len 20 against an env without delays: records and every output bit for
    bit."""
    if wpb is not None:
        monkeypatch.setenv("LHW_WARPS_PER_BLOCK", wpb)
    n = 300
    a, b = _env(name, precision, n, seed=4, max_traj_len=20), _env(name, precision, n, seed=4, max_traj_len=20)
    b.set_action_delay(np.zeros(n))
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


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_device_equals_host_body(name, precision, philox):
    """256 envs with random delays up to 25 substeps (action_delay = 0.025 s), 40 autoreset steps of max_traj_len 20: before every
    step the device records and delays are copied to the host body, and both take the step; then the host draw body redraws for
    the ended envs.  Delays, done / ended and the integer words (but the solver's count) agree exactly; at fp64 the record and
    observation to 1e-8 (the device fuses multiply-adds), at fp32 only the exact words, as for the stair curriculum.  The draws
    also equal the numpy restatement."""
    n, seed = 256, 3
    env = _env(name, precision, n, seed=seed, max_traj_len=20, action_delay=0.025)
    host = DelayEmu(_flat(name, precision), precision, n, seed, 0)
    env.reset()
    si = env.state_i.cpu().numpy()
    assert np.array_equal(env.action_delay.cpu().numpy(), draws(philox, seed, 0, si, None, 25, np.zeros(n, np.int32)))
    g = torch.Generator(device=env.device).manual_seed(1)
    close = lambda x, y: precision == 32 or np.abs(x - y).max() < 1e-8
    n_end = 0
    for t in range(40):
        host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
        delay = env.action_delay.cpu().numpy().copy()
        a = _actions(env, g)
        hobs, _, _, _, hdone, hended, _, _ = host.step_delay(a.cpu().numpy(), delay, max_traj_len=20)
        host.draw(hended, 25, delay)
        env.step(a)
        assert np.array_equal(env.done.cpu().numpy(), hdone) and np.array_equal(env.ended.cpu().numpy(), hended), t
        assert np.array_equal(env.action_delay.cpu().numpy(), delay), t
        assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7]), t
        assert close(env.state_r.cpu().numpy(), host.sr) and close(env.obs.cpu().numpy(), hobs), t
        n_end += int(hended.sum())
    assert n_end > 0
    env.close()


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def test_draw_kernel_equals_numpy(philox):
    """The draw kernel on 5000 envs with counters 0 .. 4999: no mask, a mask, and a sliced launch with its own first env id, for
    D = 0, 1, 13 and 25; unselected envs keep their word."""
    from learninghumanoidwalking_b200 import _lib
    n, seed = 5000, 17
    env = _env("jvrc_walk", 32, n, seed=seed)
    env.state_i[:, 4] = torch.arange(n, dtype=torch.int32, device=env.device)
    si = env.state_i.cpu().numpy()
    rng = np.random.RandomState(0)
    for D in (0, 1, 13, 25):
        for mask in (None, (rng.uniform(size=n) < 0.4).astype(np.int32)):
            before = rng.randint(-3, 30, size=n).astype(np.int32)
            d = torch.from_numpy(before).to(env.device)
            m = None if mask is None else torch.from_numpy(mask).to(env.device)
            _lib.ops().sim_draw_delay(env._h.value, env.state_i, seed, 0, m, D, d)
            assert np.array_equal(d.cpu().numpy(), draws(philox, seed, 0, si, mask, D, before)), (D, mask is None)
    d = torch.zeros(n, dtype=torch.int32, device=env.device)
    _lib.ops().sim_draw_delay(env._h.value, env.state_i[1000:], seed, 1000, None, 25, d[1000:])
    want = draws(philox, seed, 0, si, None, 25, np.zeros(n, np.int32))
    assert np.array_equal(d.cpu().numpy()[1000:], want[1000:]) and not d[:1000].any()
    env.close()


def test_ops_and_env_refuse_bad_arguments():
    from learninghumanoidwalking_b200 import _lib
    env = _env("jvrc_walk", 64, 8, seed=1)
    env.reset()
    dev = env.device
    a = torch.zeros(8, env.act_dim, dtype=env.dtype, device=dev)
    good = torch.zeros(8, dtype=torch.int32, device=dev)

    def step(delay, level=None, k=0, e=env, act=a):
        _lib.ops().sim_step_delay(e._h.value, e.state_r, e.state_i, 1, 0, act, 400, True, e.obs, e.term_obs, e.reward, e.rew_terms,
                                  e.done, e.ended, e.ep_len, e.ep_rew, delay, level, k)

    for delay, msg in [(good.cpu(), "CUDA tensor"), (good.long(), "dtype"), (good[:4], "shape"),
                       (torch.zeros(16, dtype=torch.int32, device=dev)[::2], "contiguous")]:
        with pytest.raises(RuntimeError, match=msg):
            step(delay)
        with pytest.raises(RuntimeError, match=msg):
            _lib.ops().sim_draw_delay(env._h.value, env.state_i, 1, 0, None, 5, delay)
    with pytest.raises(RuntimeError, match="mask"):
        _lib.ops().sim_draw_delay(env._h.value, env.state_i, 1, 0, good[:4], 5, good)
    for D, msg in ((-1, "non-negative"), (26, "must lie in 0..25")):
        with pytest.raises(RuntimeError, match=msg):
            _lib.ops().sim_draw_delay(env._h.value, env.state_i, 1, 0, None, D, good)
    with pytest.raises(RuntimeError, match="lhw_sim_step_delay: jvrc_walk has no stair curriculum"):
        step(good, good, 11)
    stairs = _env("jvrc_step", 64, 8, seed=1, stair_curriculum=0.1)
    stairs.reset()
    with pytest.raises(RuntimeError, match="n_levels"):
        step(good, stairs.stair_level, 22, e=stairs, act=torch.zeros(8, 12, dtype=torch.float64, device=dev))
    for bad, msg in ((float("nan"), "must lie in"), (-0.001, "must lie in"), (0.026, "must lie in"), (0.0025, "whole number")):
        with pytest.raises(ValueError, match=msg):
            _env("jvrc_walk", 64, 8, action_delay=bad)
        with pytest.raises(ValueError, match=msg):
            env.set_action_delay([bad] * 8)
    with pytest.raises(ValueError, match="8 numbers"):
        env.set_action_delay([0.0] * 7)
    assert env.action_delay is None
    stairs.close()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_delays_off_is_the_plain_env(precision):
    """action_delay=0 is the env as it was: no delay tensor, one launch per step and per reset, and 300 autoreset steps bit for
    bit equal to an env built without the argument.  With random delays a step is two launches (the step, then the draw) and so
    is a reset."""
    from learninghumanoidwalking_b200 import _lib
    L = _lib.lib()
    a, b = _env("jvrc_walk", precision, 512, seed=2), _env("jvrc_walk", precision, 512, seed=2, action_delay=0.0)
    assert b.action_delay is None and b.action_delay_max == 0
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
    r = _env("jvrc_walk", precision, 64, seed=2, action_delay=0.01)
    c0 = L.lhw_launch_count()
    r.reset()
    r.step(_actions(r, ga))
    assert L.lhw_launch_count() - c0 == 4
    for x in (a, b, r):
        x.close()


@pytest.mark.parametrize("name", ["jvrc_walk", "jvrc_step"])
@pytest.mark.parametrize("precision", [64, 32])
def test_eager_graph_halves_and_shards_agree(name, precision):
    """Random delays up to 20 ms (jvrc_step: with the stair curriculum as well): four copies of a batch under the same actions for
    300 autoreset steps of max_traj_len 30, stepped eagerly, through a replayed CUDA graph, as two step_slice halves, and as two
    env shards (first_env_id 0 and n/2).  Records, outputs and delays are bit-identical after every step; the delays are redrawn."""
    n = 512
    kw = dict(seed=6, max_traj_len=30, action_delay=0.02, **(dict(stair_curriculum=0.05) if name == "jvrc_step" else {}))
    envs = {k: _env(name, precision, n, **kw) for k in ("eager", "graph", "halves")}
    shards = [_env(name, precision, n // 2, first_env_id=k * n // 2, **kw) for k in range(2)]
    for e in list(envs.values()) + shards:
        e.reset()
    start = envs["eager"].action_delay.clone()
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
            assert torch.equal(o.action_delay, e.action_delay) and torch.equal(o.reward, e.reward), (k, t)
        assert torch.equal(cat("state_r"), e.state_r) and torch.equal(cat("action_delay"), e.action_delay), t
    assert not torch.equal(envs["eager"].action_delay, start)
    for x in list(envs.values()) + shards:
        x.close()


TRAIN = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
         "--eval-freq", "2", "--snapshot", "--action-delay", "0.02"]


def test_resume_carries_the_delays(tmp_path):
    """`train --snapshot --action-delay 0.02` for 4 iterations against 3 iterations then `resume --n-itr 4`: the same final
    snapshot, records and delays included, and the same checkpoints.  A delay run whose snapshot has no delays is refused."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl.snapshot import SnapshotError
    from test_gpu_resume import _compare_runs
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + TRAIN)
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    rx.main(["resume", "--path", str(run_b), "--n-itr", "4"])
    _compare_runs(run_a, run_b, 1)
    sa, sb = (torch.load(d / "snapshot" / "itr_3" / "rank_0.pt", weights_only=True) for d in (run_a, run_b))
    assert torch.equal(sa["action_delay"], sb["action_delay"]) and sa["action_delay"].dtype == torch.int32
    plain = [x if x != "0.02" else "0" for x in TRAIN]
    rx.main(["train", "--logdir", str(tmp_path / "c"), "--n-itr", "2"] + plain)
    (run_c,) = list((tmp_path / "c").iterdir())
    assert "action_delay" not in torch.load(run_c / "snapshot" / "itr_1" / "rank_0.pt", weights_only=True)
    with open(run_c / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    args.action_delay = 0.02
    with open(run_c / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    with pytest.raises(SnapshotError, match="no action delays"):
        rx.main(["resume", "--path", str(run_c), "--n-itr", "3"])


def test_train_then_eval_sweep(tmp_path, capsys):
    """`train --action-delay 0.02` then `eval --num-envs 256 --action-delays 0,0.005,0.01,0.02,0.025 --report`: the start-up line,
    the table and the report's `summary.delay` and per-env column.  Then the sweep's 0-delay cell against an undelayed batched
    evaluation of the same env ids: the accumulator rows are bit-identical."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import evaluation as ev
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    rx.main(["train", "--env", "jvrc_walk", "--action-delay", "0.02", "--logdir", str(tmp_path / "logs"), "--num-procs", "64",
             "--n-itr", "2", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    assert "Action delays: up to 20 ms, drawn at every reset" in capsys.readouterr().out
    report = tmp_path / "r.json"
    delays = [0, 0.005, 0.01, 0.02, 0.025]
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "256", "--action-delays", ",".join(map(str, delays)),
             "--report", str(report)])
    assert "delay ms" in capsys.readouterr().out
    r = json.loads(report.read_text())
    s = r["summary"]["delay"]
    assert s["delays"] == delays and [c["delay"] for c in s["cells"]] == delays
    assert sum(c["n"] for c in s["cells"]) == 256 and all({"fall_fraction", "mean_length", "return_mean", "tracking"} <= set(c)
                                                         for c in s["cells"])
    assert r["per_env"]["action_delay"] == ev.delay_grid(256, delays).tolist()
    install_reference_aliases()
    (run,) = list((tmp_path / "logs").iterdir())
    policy = torch.load(run / "actor.pt", weights_only=False).cuda().eval()
    n = 256
    accs = []
    for delay in (ev.delay_grid(n, delays), None):
        env = _env("jvrc_walk", 64, n, max_traj_len=40)
        accs.append(ev.rollout(env, policy, 40, delay=delay).cpu().numpy())
        env.close()
    cell0 = np.arange(n) % len(delays) == 0
    assert accs[0][cell0].tobytes() == accs[1][cell0].tobytes()
    assert accs[0][~cell0].tobytes() != accs[1][~cell0].tobytes()
