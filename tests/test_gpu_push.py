"""Root-velocity pushes on the device (DESIGN.md §7.5): lhw_sim_push in explicit and random mode against a host recomputation
from the device records, pushes off against an env built without them, graph replay / the two rollout halves / sharding with
pushes on, bit-identical resume of a pushed run, and the push-recovery sweep of `eval --num-envs`."""
import json
import pickle
import shutil
from argparse import Namespace

import numpy as np
import pytest
import torch

from test_gpu_eval_stats import TRAINED
from test_gpu_resume import LOGGED, _args, _close, _compare_runs, _same, _state_dicts_equal
from test_push import check_push, random_draws

pytestmark = pytest.mark.gpu
VARIANTS = ["jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step"]


@pytest.fixture(scope="module")
def philox():
    from oracle.oracle import Oracle
    return Oracle().philox


def _env(name, precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, **kw)


def _walk(env, steps, seed=1, scale=0.8):
    g = torch.Generator(device=env.device).manual_seed(seed)
    for _ in range(steps):
        env.step(torch.randn(env.num_envs, env.act_dim, generator=g, device=env.device).to(env.dtype) * scale)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_explicit_push_adds_the_rotated_velocity_and_nothing_else(name, precision):
    env = _env(name, precision, 512, seed=4, first_env_id=9)
    env.reset()
    _walk(env, 20)
    rng = np.random.RandomState(2)
    d = rng.normal(size=(env.num_envs, 2)) * 2
    d[::3] = 0
    before = env.state_r.cpu().numpy()
    si_before = env.state_i.clone()
    env.push(torch.as_tensor(d, dtype=env.dtype, device=env.device))
    after = env.state_r.cpu().numpy()
    pushed = np.abs(d).sum(1) != 0
    d_env = d.astype(np.float64 if precision == 64 else np.float32).astype(np.float64)
    check_push(before, after, env.nq, pushed, d_env, 1e-12 if precision == 64 else 1e-6)
    assert np.array_equal(after[::3].view(np.uint8), before[::3].view(np.uint8))     # zero rows: bitwise untouched
    assert torch.equal(env.state_i, si_before)
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_random_push_equals_host_recomputation(name, precision, philox):
    seed, first = 6, 33
    env = _env(name, precision, 512, seed=seed, first_env_id=first, push_vel=1.5, push_interval=1.0)
    env.push_interval_steps = 3            # a push every 3 control steps on average
    env.reset()
    vel, seen_pushed, seen_ended = env.push_vel, 0, 0
    for t in range(12):
        env.push_vel = 0.0                 # step without the push, look at the records, then push as step() does
        _walk(env, 1, seed=t)
        env.push_vel = vel
        before, si, ended = env.state_r.cpu().numpy(), env.state_i.cpu().numpy(), env.ended.cpu().numpy()
        env._push_random(0, env.num_envs)
        after = env.state_r.cpu().numpy()
        want, d = random_draws(philox, seed, first, si, ended, vel, 3)
        changed = (after != before).any(1)
        assert not (changed & ~want).any()
        check_push(before, after, env.nq, want, d, 1e-12 if precision == 64 else 1e-6)
        seen_pushed += int(want.sum())
        seen_ended += int(ended.sum())
    assert seen_pushed > 12 * 512 / 3 * 0.8 and seen_ended > 0
    env.close()


def _worker(env, obs_dim, act_dim):
    from learninghumanoidwalking_b200.rl import DeviceRolloutWorker, FF_V, Gaussian_FF_Actor
    torch.manual_seed(5)
    pol, cri = Gaussian_FF_Actor(obs_dim, act_dim, init_std=0.223).cuda(), FF_V(obs_dim).cuda()
    pol.obs_mean = cri.obs_mean = torch.tensor(env.obs_mean, dtype=torch.float32, device="cuda")
    pol.obs_std = cri.obs_std = torch.tensor(env.obs_std, dtype=torch.float32, device="cuda")
    return DeviceRolloutWorker(env, pol, cri, seed=9)


def _samples(env, iters=2, T=30):
    w = _worker(env, env.obs_dim, env.act_dim)
    out = []
    for _ in range(iters):
        b = w.sample(0.99, 0.95, T, 60)
        out.append([t.clone() for t in (b.states, b.actions, b.rewards, b.returns, b.dones)])
    out.append([env.state_r.clone(), env.state_i.clone()])
    return out


def _equal(x, y):
    return all(torch.equal(p, q) for a, b in zip(x, y) for p, q in zip(a, b))


@pytest.mark.parametrize("name, precision", [("jvrc_walk", 32), ("h1", 64)])
def test_pushes_off_is_the_env_without_pushes(name, precision):
    from learninghumanoidwalking_b200 import _lib
    runs = []
    for kw in ({}, dict(push_vel=0.0, push_interval=0.5)):
        env = _env(name, precision, 1024, seed=3, **kw)
        n0 = _lib.lib().lhw_launch_count()
        runs.append((_samples(env), _lib.lib().lhw_launch_count() - n0))
        env.close()
    assert _equal(runs[0][0], runs[1][0])
    assert runs[0][1] == runs[1][1]            # and not one launch more


@pytest.mark.parametrize("name, precision", [("jvrc_walk", 32), ("h1_walk", 64)])
def test_pushed_rollout_replay_halves_and_shards(name, precision, monkeypatch):
    """With pushes on: the worker's replayed per-half graphs equal its eager loop over the same halves, bit for bit.  An env's
    trajectory under given actions does not depend on how it is launched: the two halves stepped with step_slice, and the upper
    half alone as a shard with first_env_id 512, equal the full-batch step.  (The worker's single-stream rollout differs from the
    halves by the MLP's batch-size-dependent rounding even without pushes, tests/test_gpu_ppo.py, so the env-level check is the
    bitwise one.)"""
    kw = dict(push_vel=1.0, push_interval=0.25)
    ref = _samples(_env(name, precision, 1024, seed=3, **kw))
    monkeypatch.setenv("LHW_ROLLOUT_GRAPH", "0")
    assert _equal(ref, _samples(_env(name, precision, 1024, seed=3, **kw)))
    monkeypatch.delenv("LHW_ROLLOUT_GRAPH")
    assert not _equal(ref, _samples(_env(name, precision, 1024, seed=3)))      # pushes happened, and they changed the roll-out
    full, halves = _env(name, precision, 1024, seed=3, **kw), _env(name, precision, 1024, seed=3, **kw)
    tail = _env(name, precision, 512, seed=3, first_env_id=512, **kw)
    for e in (full, halves, tail):
        e.reset()
    g = torch.Generator(device=full.device).manual_seed(4)
    for _ in range(60):
        a = torch.randn(1024, full.act_dim, generator=g, device=full.device).to(full.dtype) * 0.5
        full.step(a)
        halves.step_slice(0, 512, a[:512].contiguous())
        halves.step_slice(512, 1024, a[512:].contiguous())
        tail.step(a[512:].contiguous())
    assert torch.equal(full.state_r, halves.state_r) and torch.equal(full.state_i, halves.state_i)
    assert torch.equal(full.state_r[512:], tail.state_r) and torch.equal(full.state_i[512:], tail.state_i)
    for e in (full, halves, tail):
        e.close()


def _push_env_fn(model, precision):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(64, model=model, precision=precision, seed=7, push_vel=1.0, push_interval=0.25)
    probe = base()
    r = probe.robot
    probe.close()
    if not hasattr(r, "mirrored_obs"):
        return base
    return lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)


@pytest.mark.parametrize("model, precision", [("jvrc_walk", 32), ("h1", 64)])
def test_pushed_run_resumes_bit_identically(tmp_path, monkeypatch, model, precision):
    """tests/test_gpu_resume.py's check with random pushes on: the push decisions come from the records' Philox counters, so the
    snapshot needs nothing new."""
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    env_fn = _push_env_fn(model, precision)
    a = PPO(env_fn, _args(tmp_path / "a"), seed=11)
    log_a = a.train(None, 4, verbose=False)
    fin_a = [t.clone() for t in (a._flat_param, a._flat_m, a._flat_v, a.env.state_r, a.env.state_i)]
    _close(a)
    b = PPO(env_fn, _args(tmp_path / "b", snapshot=True), seed=11)
    log_b = b.train(None, 2, verbose=False)
    _close(b)
    del b
    b = PPO(env_fn, _args(tmp_path / "b", snapshot=True), seed=11)
    assert b.restore(tmp_path / "b") == 1
    log_b += b.train(None, 4, verbose=False, start_itr=2)
    for name, x, y in zip(("params", "exp_avg", "exp_avg_sq", "state_r", "state_i"), fin_a,
                          (b._flat_param, b._flat_m, b._flat_v, b.env.state_r, b.env.state_i)):
        assert torch.equal(x, y), name
    for ea, eb in zip(log_a[2:], log_b[2:]):
        for k in LOGGED:
            if k in ea or k in eb:
                assert _same(ea[k], eb[k]), (ea["itr"], k, ea[k], eb[k])
    for name in ("actor_3.pt", "critic_3.pt"):
        assert _state_dicts_equal(tmp_path / "a" / name, tmp_path / "b" / name), name
    _close(b)


def test_command_line_train_push_resume(tmp_path, capsys):
    """`train --push-vel 1 --push-interval 0.5 --snapshot` records the two values, and `resume` rebuilds the pushed env from them."""
    import run_experiment as rx
    train = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
             "--eval-freq", "2", "--snapshot", "--push-vel", "1", "--push-interval", "0.5"]
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + train)
    assert "Random pushes: up to 1.0 m/s about every 0.5 s" in capsys.readouterr().out
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + train)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    with open(run_b / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    assert (args.push_vel, args.push_interval) == (1.0, 0.5)
    rx.main(["resume", "--path", str(run_b), "--n-itr", "4"])
    _compare_runs(run_a, run_b, 1)


def _policy():
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    return torch.load(TRAINED, weights_only=False).cuda().eval()


def test_sweep_on_the_trained_actor(tmp_path, capsys):
    """0 m/s envs are bit-equal to an un-pushed evaluation; the trained actor survives all of them (DESIGN §7.4 saw no falls) and
    a 3 m/s shove in any direction topples some; the graph replay equals the eager loop; the CLI report's schema."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    policy = _policy()
    n, speeds, D = 1024, [0.0, 3.0], 8
    speed, deg = ev.push_grid(n, speeds, D)
    k = 80                                                     # 2.0 s at jvrc_walk's 0.025 s control step

    def run(**kw):        # a fresh env each time: a second reset of the same env starts other episodes (its event counter moved on)
        env = _env("jvrc_walk", 64, n, seed=0)
        acc = ev.rollout(env, policy, env.max_traj_len, **kw).cpu().numpy()
        env.close()
        return acc
    plain = run()
    pushed = run(push=(k, ev.push_vectors(speed, deg)))
    eager = run(graph=False, push=(k, ev.push_vectors(speed, deg)))
    assert np.array_equal(pushed, eager)
    zero = speed == 0
    assert np.array_equal(pushed[zero], plain[zero])
    p = ev.push_summary(pushed, speed, deg, speeds, D, 2.0, k)
    assert p["per_speed"][0]["survival"] == 1.0 and p["per_speed"][0]["alive_at_push"] == n // 2
    assert all(c["survival"] < 1.0 for c in p["cells"][D:]), [c["survival"] for c in p["cells"][D:]]
    print(ev.format_push_table(p))
    # the command line: an actor with its experiment.pkl
    run = tmp_path / "run"
    run.mkdir()
    shutil.copy(TRAINED, run / "actor.pt")
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    import run_experiment as rx
    path = tmp_path / "r.json"
    rx.main(["eval", "--path", str(run), "--num-envs", "256", "--push-speeds", "0,0.5,1,1.5", "--report", str(path)])
    out = capsys.readouterr().out
    assert "push recovery: one push after control step 80" in out
    r = json.loads(path.read_text())
    s = r["summary"]["push"]
    assert s["speeds"] == [0, 0.5, 1, 1.5] and s["directions_deg"] == [45.0 * i for i in range(8)] and s["push_step"] == 80
    assert len(s["cells"]) == 32 and sum(c["n"] for c in s["cells"]) == 256
    assert set(s["cells"][0]) == {"speed", "direction_deg", "n", "fell_before_push", "alive_at_push", "survived", "survival"}
    assert len(r["per_env"]["push_speed"]) == len(r["per_env"]["push_dir_deg"]) == 256
    assert r["per_env"]["push_speed"][8] == 0.5 and r["per_env"]["push_dir_deg"][9] == 45.0
    for extra, message in ((["--num-envs", "15", "--push-speeds", "0,1"], "16 cells"),
                           (["--num-envs", "64", "--push-speeds", "1", "--push-at", "10"], "after control step 400")):
        with pytest.raises(SystemExit, match=message):
            rx.main(["eval", "--path", str(run), *extra])


def test_op_rejects_bad_tensors():
    env = _env("jvrc_walk", 64, 8)
    env.reset()
    from learninghumanoidwalking_b200 import _lib
    O, h = _lib.ops(), env._h.value
    before = env.state_r.clone()
    d = torch.ones(8, 2, dtype=torch.float64, device=env.device)
    for bad, message in ((d.float(), "d has dtype"), (d[:4], "d has shape"), (d.cpu(), "must be a CUDA tensor"),
                         (d.t().contiguous().t(), "must be contiguous")):
        with pytest.raises(RuntimeError, match=message):
            O.sim_push(h, env.state_r, env.state_i, 0, 0, None, 0.0, 1, bad)
    with pytest.raises(RuntimeError, match="either d"):
        O.sim_push(h, env.state_r, env.state_i, 0, 0, env.ended, 1.0, 1, d)
    with pytest.raises(RuntimeError, match="ended has dtype"):
        O.sim_push(h, env.state_r, env.state_i, 0, 0, env.ended.float(), 1.0, 1, None)
    with pytest.raises(RuntimeError, match="finite and non-negative"):
        O.sim_push(h, env.state_r, env.state_i, 0, 0, env.ended, float("nan"), 1, None)
    with pytest.raises(RuntimeError, match="at least one control step"):
        O.sim_push(h, env.state_r, env.state_i, 0, 0, env.ended, 1.0, 0, None)
    assert torch.equal(env.state_r, before)
    env.close()
