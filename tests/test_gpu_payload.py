"""Carried payloads on the device (DESIGN.md §7.10): the PAYLOAD step kernels, single-warp and lock-step, at mass 0 against the
plain kernels bit for bit and with payloads against the host body; the draw kernel against numpy; the ops' refusals; payloads off
launching exactly the plain kernels; eager, graph-replayed, step_slice-halved and sharded roll-outs agreeing bit for bit with random
payloads, with and without delays; a `train --snapshot` run resuming with its payloads; the sweep's 0-kg cell against an
evaluation without payloads; and `train --payload-mass` then `eval --payloads --report` end to end."""
import json
import pickle

import numpy as np
import pytest
import torch

from test_payload import VARIANTS, PayloadEmu, _flat, draws
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
def test_zero_mass_kernels_are_the_plain_kernels(name, precision, wpb, monkeypatch):
    """One-warp (LHW_WARPS_PER_BLOCK=1) and lock-step blocks: 300 envs (not a multiple of a block) given mass 0 at an offset
    through set_payload, 60 autoreset steps of max_traj_len 20 against an env without payloads: records and every output bit for
    bit."""
    if wpb is not None:
        monkeypatch.setenv("LHW_WARPS_PER_BLOCK", wpb)
    n = 300
    a, b = _env(name, precision, n, seed=4, max_traj_len=20), _env(name, precision, n, seed=4, max_traj_len=20)
    b.set_payload(np.zeros(n), (0.1, -0.2, 0.25))
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
    """300 envs with random payloads up to 20 kg at offsets up to 0.2 m, 40 autoreset steps of max_traj_len 20: before every step
    the device records and payloads are copied to the host body, and both take the step; then the host draw body redraws for the
    ended envs.  Payloads, done / ended and the integer words (but the solver's count) agree exactly; at fp64 the record and
    observation to 1e-8 (the device fuses multiply-adds), at fp32 only the exact words, as for the action delays.  The first
    draws also equal the numpy restatement."""
    if wpb is not None:
        monkeypatch.setenv("LHW_WARPS_PER_BLOCK", wpb)
    n, seed = 300, 3
    env = _env(name, precision, n, seed=seed, max_traj_len=20, payload_mass=20.0, payload_offset=0.2)
    host = PayloadEmu(_flat(name, precision), precision, n, seed, 0)
    env.reset()
    si = env.state_i.cpu().numpy()
    want = draws(philox, seed, 0, si, None, 20.0, 0.2, np.zeros((n, 4))).astype(host.dt)
    assert env.payload.cpu().numpy().tobytes() == want.tobytes()
    g = torch.Generator(device=env.device).manual_seed(1)
    close = lambda x, y: precision == 32 or np.abs(x - y).max() < 1e-8
    n_end = 0
    for t in range(40):
        host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
        pay = env.payload.cpu().numpy().copy()
        a = _actions(env, g)
        hobs, _, _, _, hdone, hended, _, _ = host.step_payload(a.cpu().numpy(), pay, max_traj_len=20)
        host.draw(hended, 20.0, 0.2, pay)
        env.step(a)
        assert np.array_equal(env.done.cpu().numpy(), hdone) and np.array_equal(env.ended.cpu().numpy(), hended), t
        assert env.payload.cpu().numpy().tobytes() == pay.tobytes(), t
        assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7]), t
        assert close(env.state_r.cpu().numpy(), host.sr) and close(env.obs.cpu().numpy(), hobs), t
        n_end += int(hended.sum())
    assert n_end > 0
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_draw_kernel_equals_numpy(precision, philox):
    """The draw kernel on 5000 envs with counters 0 .. 4999: no mask, a mask, and a sliced launch with its own first env id;
    unselected envs keep their words."""
    from learninghumanoidwalking_b200 import _lib
    n, seed = 5000, 17
    env = _env("jvrc_walk", precision, n, seed=seed)
    dt = np.float64 if precision == 64 else np.float32
    env.state_i[:, 4] = torch.arange(n, dtype=torch.int32, device=env.device)
    si = env.state_i.cpu().numpy()
    rng = np.random.RandomState(0)
    for M, R in ((0.0, 0.0), (10.0, 0.25), (31.2, 0.05)):
        for mask in (None, (rng.uniform(size=n) < 0.4).astype(np.int32)):
            before = rng.normal(size=(n, 4)).astype(dt)
            p = torch.from_numpy(before).to(env.device)
            m = None if mask is None else torch.from_numpy(mask).to(env.device)
            _lib.ops().sim_draw_payload(env._h.value, env.state_i, seed, 0, m, M, R, p)
            want = draws(philox, seed, 0, si, mask, M, R, before.astype(np.float64)).astype(dt)
            assert p.cpu().numpy().tobytes() == want.tobytes(), (M, R, mask is None)
    p = torch.zeros(n, 4, dtype=env.dtype, device=env.device)
    _lib.ops().sim_draw_payload(env._h.value, env.state_i[1000:], seed, 1000, None, 20.0, 0.1, p[1000:])
    want = draws(philox, seed, 0, si, None, 20.0, 0.1, np.zeros((n, 4))).astype(dt)
    assert p.cpu().numpy()[1000:].tobytes() == want[1000:].tobytes() and not p[:1000].any()
    env.close()


def test_ops_and_env_refuse_bad_arguments():
    from learninghumanoidwalking_b200 import _lib
    env = _env("jvrc_walk", 64, 8, seed=1)
    env.reset()
    dev = env.device
    a = torch.zeros(8, env.act_dim, dtype=env.dtype, device=dev)
    good = torch.zeros(8, 4, dtype=torch.float64, device=dev)
    d = torch.zeros(8, dtype=torch.int32, device=dev)

    def step(payload, delay=None, level=None, k=0, e=env, act=a):
        _lib.ops().sim_step_payload(e._h.value, e.state_r, e.state_i, 1, 0, act, 400, True, e.obs, e.term_obs, e.reward, e.rew_terms,
                                    e.done, e.ended, e.ep_len, e.ep_rew, payload, delay, level, k)

    for bad, msg in [(good.cpu(), "CUDA tensor"), (good.float(), "dtype"), (good[:4], "shape"), (good[:, :3].contiguous(), "shape"),
                     (torch.zeros(8, 8, dtype=torch.float64, device=dev)[:, ::2], "contiguous")]:
        with pytest.raises(RuntimeError, match=msg):
            step(bad)
        with pytest.raises(RuntimeError, match=msg):
            _lib.ops().sim_draw_payload(env._h.value, env.state_i, 1, 0, None, 5.0, 0.0, bad)
    for bad, msg in [(d.cpu(), "CUDA tensor"), (d.long(), "dtype"), (d[:4], "shape")]:
        with pytest.raises(RuntimeError, match=msg):
            step(good, bad)
    with pytest.raises(RuntimeError, match="mask"):
        _lib.ops().sim_draw_payload(env._h.value, env.state_i, 1, 0, d[:4], 5.0, 0.0, good)
    for M, R, msg in ((-1.0, 0.0, "mass"), (float("nan"), 0.0, "mass"), (float("inf"), 0.0, "mass"), (5.0, 0.3, "offset"),
                      (5.0, -0.1, "offset"), (5.0, float("nan"), "offset")):
        with pytest.raises(RuntimeError, match=msg):
            _lib.ops().sim_draw_payload(env._h.value, env.state_i, 1, 0, None, M, R, good)
    with pytest.raises(RuntimeError, match="lhw_sim_step_payload: jvrc_walk has no stair curriculum"):
        step(good, None, d, 11)
    stairs = _env("jvrc_step", 64, 8, seed=1, stair_curriculum=0.1)
    stairs.reset()
    with pytest.raises(RuntimeError, match="n_levels"):
        step(good, None, stairs.stair_level, 22, e=stairs, act=torch.zeros(8, 12, dtype=torch.float64, device=dev))
    for kw, msg in ((dict(payload_mass=float("nan")), "mass must lie"), (dict(payload_mass=-1.0), "mass must lie"),
                    (dict(payload_mass=31.3), "mass must lie"), (dict(payload_mass=5.0, payload_offset=0.3), "offset must lie"),
                    (dict(payload_offset=0.1), "needs a payload mass")):
        with pytest.raises(ValueError, match=msg):
            _env("jvrc_walk", 64, 8, **kw)
    with pytest.raises(ValueError, match="mass must lie"):
        _env("h1", 64, 8, payload_mass=29.3)
    for mass, off, msg in (([31.3] * 8, None, "mass must lie"), ([float("nan")] * 8, None, "mass must lie"),
                           ([1.0] * 8, (0, 0, 0.3), "offset must lie"), ([1.0] * 7, None, "8 numbers"),
                           ([1.0] * 8, (0, 0), "offset must be")):
        with pytest.raises(ValueError, match=msg):
            env.set_payload(mass, off)
    assert env.payload is None
    stairs.close()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_payloads_off_is_the_plain_env(precision):
    """payload_mass=0 is the env as it was: no payload tensor, one launch per step and per reset, and 300 autoreset steps bit for
    bit equal to an env built without the argument.  With random payloads a step is two launches (the step, then the draw) and so
    is a reset."""
    from learninghumanoidwalking_b200 import _lib
    L = _lib.lib()
    a, b = _env("jvrc_walk", precision, 512, seed=2), _env("jvrc_walk", precision, 512, seed=2, payload_mass=0.0)
    assert b.payload is None
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
    r = _env("jvrc_walk", precision, 64, seed=2, payload_mass=10.0)
    c0 = L.lhw_launch_count()
    r.reset()
    r.step(_actions(r, ga))
    assert L.lhw_launch_count() - c0 == 4
    for x in (a, b, r):
        x.close()


@pytest.mark.parametrize("name, extra", [("jvrc_walk", {}), ("jvrc_walk", dict(action_delay=0.02)), ("h1", {}),
                                         ("jvrc_step", dict(action_delay=0.02, stair_curriculum=0.05))])
@pytest.mark.parametrize("precision", [64, 32])
def test_eager_graph_halves_and_shards_agree(name, extra, precision):
    """Random payloads up to 20 kg within 0.1 m (with random delays, and on jvrc_step the stair curriculum as well): four copies
    of a batch under the same actions for 300 autoreset steps of max_traj_len 30, stepped eagerly, through a replayed CUDA graph,
    as two step_slice halves, and as two env shards (first_env_id 0 and n/2).  Records, outputs and payloads are bit-identical after
    every step; the payloads are redrawn."""
    n = 512
    kw = dict(seed=6, max_traj_len=30, payload_mass=20.0, payload_offset=0.1, **extra)
    envs = {k: _env(name, precision, n, **kw) for k in ("eager", "graph", "halves")}
    shards = [_env(name, precision, n // 2, first_env_id=k * n // 2, **kw) for k in range(2)]
    for e in list(envs.values()) + shards:
        e.reset()
    start = envs["eager"].payload.clone()
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
            assert torch.equal(o.payload, e.payload) and torch.equal(o.reward, e.reward), (k, t)
        assert torch.equal(cat("state_r"), e.state_r) and torch.equal(cat("payload"), e.payload), t
    assert not torch.equal(envs["eager"].payload, start)
    for x in list(envs.values()) + shards:
        x.close()


TRAIN = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
         "--eval-freq", "2", "--snapshot", "--payload-mass", "10", "--payload-offset", "0.05"]


def test_resume_carries_the_payloads(tmp_path):
    """`train --snapshot --payload-mass 10` for 4 iterations against 3 iterations then `resume --n-itr 4`: the same final
    snapshot, records and payloads included, and the same checkpoints.  A payload run whose snapshot has no payloads is refused."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl.snapshot import SnapshotError
    from test_gpu_resume import _compare_runs
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + TRAIN)
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    rx.main(["resume", "--path", str(run_b), "--n-itr", "4"])
    _compare_runs(run_a, run_b, 1)
    sa, sb = (torch.load(d / "snapshot" / "itr_3" / "rank_0.pt", weights_only=True) for d in (run_a, run_b))
    assert torch.equal(sa["payload"], sb["payload"]) and sa["payload"].shape == (64, 4)
    plain = TRAIN[:-4]
    rx.main(["train", "--logdir", str(tmp_path / "c"), "--n-itr", "2"] + plain)
    (run_c,) = list((tmp_path / "c").iterdir())
    assert "payload" not in torch.load(run_c / "snapshot" / "itr_1" / "rank_0.pt", weights_only=True)
    with open(run_c / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    args.payload_mass = 10.0
    with open(run_c / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    with pytest.raises(SnapshotError, match="no payloads"):
        rx.main(["resume", "--path", str(run_c), "--n-itr", "3"])


def test_train_then_eval_sweep(tmp_path, capsys):
    """`train --payload-mass 10` then `eval --num-envs 256 --payloads 0,5,10,15,20 --payload-at 0,0,0.1 --report`: the start-up
    line, the table and the report's `summary.payload` and per-env column.  Then the sweep's 0-kg cell against a batched evaluation
    without payloads of the same env ids: the accumulator rows are bit-identical."""
    import run_experiment as rx
    from learninghumanoidwalking_b200.rl import evaluation as ev
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    rx.main(["train", "--env", "jvrc_walk", "--payload-mass", "10", "--logdir", str(tmp_path / "logs"), "--num-procs", "64",
             "--n-itr", "2", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    assert "Payloads: up to 10 kg" in capsys.readouterr().out
    report = tmp_path / "r.json"
    masses = [0.0, 5.0, 10.0, 15.0, 20.0]
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "256", "--payloads", ",".join(map(str, masses)),
             "--payload-at", "0,0,0.1", "--report", str(report)])
    assert "mass kg" in capsys.readouterr().out
    r = json.loads(report.read_text())
    s = r["summary"]["payload"]
    assert s["masses"] == masses and [c["mass"] for c in s["cells"]] == masses and s["at"] == [0, 0, 0.1]
    assert sum(c["n"] for c in s["cells"]) == 256 and all({"fall_fraction", "mean_length", "return_mean", "tracking"} <= set(c)
                                                         for c in s["cells"])
    assert r["per_env"]["payload_mass"] == ev.payload_grid(256, masses).tolist()
    install_reference_aliases()
    (run,) = list((tmp_path / "logs").iterdir())
    policy = torch.load(run / "actor.pt", weights_only=False).cuda().eval()
    n = 256
    accs = []
    for load in ((ev.payload_grid(n, masses), (0, 0, 0.1)), None):
        env = _env("jvrc_walk", 64, n, max_traj_len=40)
        accs.append(ev.rollout(env, policy, 40, payload=load).cpu().numpy())
        env.close()
    cell0 = np.arange(n) % len(masses) == 0
    assert accs[0][cell0].tobytes() == accs[1][cell0].tobytes()
    assert accs[0][~cell0].tobytes() != accs[1][~cell0].tobytes()
