"""The stair curriculum on the device (DESIGN.md §7.8): lhw_sim_step_stairs / lhw_sim_reset_stairs against the host body (levels and
integer words exactly, the pose to rounding), the ops' refusals, the flag off launching exactly the plain kernels, eager, graph-replayed
and step_slice-halved roll-outs agreeing bit for bit, a `train --snapshot` run resuming with its levels, and `train --stair-curriculum`
then `eval --footsteps` end to end."""
import pickle

import numpy as np
import pytest
import torch

from test_gpu_command import _actions, _graph_stepper
from test_stair_curriculum import TK, StairEmu, _flat

pytestmark = pytest.mark.gpu


def _env(precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model="jvrc_step", precision=precision, **kw)


@pytest.mark.parametrize("precision", [64, 32])
def test_device_equals_host_body(precision):
    """256 envs on a 5-level curriculum (levels set to -1 .. 5), max_traj_len 20, 40 autoreset steps: before every step the device
    records and levels are copied to the host body, and both take the step.  Levels, done / ended, the integer words (but the
    solver's count) and the plan words agree exactly.  At fp64 the pose and observation agree to rounding (the device fuses
    multiply-adds); at fp32 one step of contact and Newton solve amplifies that rounding past a useful bound, so only the exact
    words are compared there, and the reset (no physics step) is compared to 1e-4 as in §7.7.  Then an explicit reset of a
    mid-episode batch, the same way."""
    n, seed, K = 256, 3, 5
    env = _env(precision, n, seed=seed, max_traj_len=20, stair_curriculum=0.04)
    assert env.stair_levels == K
    host = StairEmu(_flat(precision), precision, n, seed, 0)
    env.stair_level.copy_(torch.arange(n, device=env.device, dtype=torch.int32) % (K + 2) - 1)
    env.reset()
    g = torch.Generator(device=env.device).manual_seed(1)
    close = lambda x, y, tol=1e-8: precision == 32 or np.abs(x - y).max() < tol
    moved = 0
    for t in range(40):
        host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
        level = env.stair_level.cpu().numpy().copy()
        lv0 = level.copy()
        a = _actions(env, g)
        hobs, _, _, _, hdone, hended, _, _ = host.step_stairs(a.cpu().numpy(), level, K, max_traj_len=20)
        env.step(a)
        assert np.array_equal(env.stair_level.cpu().numpy(), level), t
        assert np.array_equal(env.done.cpu().numpy(), hdone) and np.array_equal(env.ended.cpu().numpy(), hended), t
        assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7]), t
        sr = env.state_r.cpu().numpy()
        assert np.array_equal(sr[:, TK:TK + 3], host.sr[:, TK:TK + 3]), t
        assert close(sr, host.sr) and close(env.obs.cpu().numpy(), hobs), t
        moved += int((level != lv0).sum())
    assert moved > 0
    host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
    level = env.stair_level.cpu().numpy().copy()
    hobs = host.reset_stairs(level, K)
    env.reset(torch.ones(n, dtype=torch.int32))
    assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7])
    assert np.array_equal(env.state_r.cpu().numpy()[:, TK:TK + 3], host.sr[:, TK:TK + 3])
    tol = 1e-8 if precision == 64 else 1e-4
    assert np.abs(env.state_r.cpu().numpy() - host.sr).max() < tol and np.abs(env.obs.cpu().numpy() - hobs).max() < tol
    env.close()


def test_ops_refuse_bad_tensors_and_variants():
    from learninghumanoidwalking_b200 import _lib
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = _env(64, 8, seed=1, stair_curriculum=0.1)
    env.reset()
    h, dev = env._h.value, env.device
    a = torch.zeros(8, env.act_dim, dtype=env.dtype, device=dev)

    def step(e, level, k, handle=None):
        _lib.ops().sim_step_stairs(handle or e._h.value, e.state_r, e.state_i, 1, 0, a, 400, True, e.obs, e.term_obs, e.reward,
                                   e.rew_terms, e.done, e.ended, e.ep_len, e.ep_rew, level, k)

    def reset(e, level, k):
        _lib.ops().sim_reset_stairs(e._h.value, e.state_r, e.state_i, 1, 0, None, False, e.obs, level, k)

    good = env.stair_level
    for level, k, msg in [(good.cpu(), 11, "CUDA tensor"), (good.long(), 11, "dtype"), (good[:4], 11, "shape"),
                          (torch.zeros(16, dtype=torch.int32, device=dev)[::2], 11, "contiguous"), (good, 1, "n_levels"),
                          (good, 22, "n_levels")]:
        with pytest.raises(RuntimeError, match=msg):
            step(env, level, k)
        with pytest.raises(RuntimeError, match=msg):
            reset(env, level, k)
    for name in ("jvrc_walk", "h1", "jvrc_walk_terrain", "h1_walk"):
        other = BatchedHumanoidEnv(8, model=name, precision=64)
        other.reset()
        lv = torch.zeros(8, dtype=torch.int32, device=dev)
        with pytest.raises(RuntimeError, match=f"lhw_sim_reset_stairs: {name} has no stair curriculum"):
            reset(other, lv, 11)
        with pytest.raises(RuntimeError, match=f"lhw_sim_step_stairs: {name} has no stair curriculum"):
            _lib.ops().sim_step_stairs(other._h.value, other.state_r, other.state_i, 1, 0,
                                       torch.zeros(8, other.act_dim, dtype=other.dtype, device=dev), 400, True, other.obs, other.term_obs,
                                       other.reward, other.rew_terms, other.done, other.ended, other.ep_len, other.ep_rew, lv, 11)
        other.close()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_flag_off_is_the_plain_env(precision):
    """stair_curriculum=0 is the env as it was: no level tensor, one launch per step and per reset, and 300 autoreset steps bit for
    bit equal to an env built without the argument."""
    from learninghumanoidwalking_b200 import _lib
    L = _lib.lib()
    a, b = _env(precision, 512, seed=2, iteration_count=7000), _env(precision, 512, seed=2, iteration_count=7000, stair_curriculum=0.0)
    assert b.stair_level is None and b.stair_levels == 0
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
    a.close()
    b.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_eager_graph_and_halves_agree(precision):
    """Three copies of a curriculum batch (0.05 m, levels starting at 0 .. 5) under the same actions for 400 autoreset steps of
    max_traj_len 50: stepped eagerly, through a replayed CUDA graph, and as two step_slice halves.  Records, outputs and levels are
    bit-identical after every step; the levels move."""
    n = 512
    envs = {k: _env(precision, n, seed=6, max_traj_len=50, stair_curriculum=0.05) for k in ("eager", "graph", "halves")}
    for e in envs.values():
        e.stair_level.copy_(torch.arange(n, device=e.device, dtype=torch.int32) % 6)
        e.reset()
    start = envs["eager"].stair_level.clone()
    gens = {k: torch.Generator(device=e.device).manual_seed(7) for k, e in envs.items()}
    graph_step = _graph_stepper(envs["graph"], gens["graph"])
    for t in range(400):
        envs["eager"].step(_actions(envs["eager"], gens["eager"]))
        graph_step()
        a = _actions(envs["halves"], gens["halves"])
        envs["halves"].step_slice(0, n // 2, a[:n // 2].contiguous())
        envs["halves"].step_slice(n // 2, n, a[n // 2:].contiguous())
        e = envs["eager"]
        for k in ("graph", "halves"):
            o = envs[k]
            assert torch.equal(o.state_r, e.state_r) and torch.equal(o.state_i, e.state_i) and torch.equal(o.obs, e.obs), (k, t)
            assert torch.equal(o.stair_level, e.stair_level) and torch.equal(o.reward, e.reward), (k, t)
    assert not torch.equal(envs["eager"].stair_level, start)
    for x in envs.values():
        x.close()


TRAIN = ["--env", "jvrc_step", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3",
         "--eval-freq", "2", "--snapshot", "--stair-curriculum", "0.05"]


def test_resume_carries_the_levels(tmp_path):
    """`train --snapshot --stair-curriculum 0.05` for 4 iterations against 3 iterations then `resume --n-itr 4`: the same final
    snapshot, records and stair levels included, and the same checkpoints.  A curriculum run whose snapshot has no levels is
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
    assert torch.equal(sa["stair_level"], sb["stair_level"]) and sa["stair_level"].dtype == torch.int32
    plain = [x if x != "0.05" else "0" for x in TRAIN]
    rx.main(["train", "--logdir", str(tmp_path / "c"), "--n-itr", "2"] + plain)
    (run_c,) = list((tmp_path / "c").iterdir())
    assert "stair_level" not in torch.load(run_c / "snapshot" / "itr_1" / "rank_0.pt", weights_only=True)
    with open(run_c / "experiment.pkl", "rb") as f:
        args = pickle.load(f)
    args.stair_curriculum = 0.05
    with open(run_c / "experiment.pkl", "wb") as f:
        pickle.dump(args, f)
    with pytest.raises(SnapshotError, match="no stair levels"):
        rx.main(["resume", "--path", str(run_c), "--n-itr", "3"])


def test_train_then_eval_footsteps(tmp_path, capsys):
    import run_experiment as rx
    rx.main(["train", "--env", "jvrc_step", "--stair-curriculum", "0.15", "--logdir", str(tmp_path / "logs"), "--num-procs", "64",
             "--n-itr", "2", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    out = capsys.readouterr().out
    assert "Stair curriculum: levels of 0.01 m up to 0.15 m" in out
    assert out.count("Mean stair height") == 2 and out.count("Top stair level") == 2
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "256", "--footsteps", "forward:0,0.05,0.1,0.15"])
    out = capsys.readouterr().out
    assert "forward:0.15" in out
