"""Resumable training on the GPU: a run stopped after its snapshot and continued with PPO.restore / `run_experiment.py resume`
is the same run, bit for bit, as one that never stopped (weights, Adam moments, every environment's record, the logged
statistics, the checkpoints and the TensorBoard scalars)."""
import math
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOGGED = ("ep_rew", "ep_len", "actor_loss", "entropy", "critic_loss", "kl", "mirror", "clip_frac", "eval_rew", "eval_len")

CASES = {
    "jvrc_walk_fp32": dict(model="jvrc_walk", precision=32),
    "jvrc_walk_fp64": dict(model="jvrc_walk", precision=64),
    "h1": dict(model="h1", precision=64),                          # randomised dynamics, pushes and noise live in the record
    "jvrc_step": dict(model="jvrc_step", precision=64),            # step-height curriculum driven by the iteration
    "jvrc_walk_terrain": dict(model="jvrc_walk_terrain", precision=64),
    "learn_std": dict(model="jvrc_walk", precision=32, learn_std=True),
    "nccl_exchange": dict(model="jvrc_walk", precision=32, exchange="0"),   # LHW_FUSED_EXCHANGE=0: Adam step in FusedClipAdam.step_dev
}


def _args(logdir, **kw):
    d = dict(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=256, epochs=1,
             max_traj_len=50, num_procs=64, max_grad_norm=0.05, mirror_coeff=0.4, eval_freq=2, recurrent=False,
             imitate_coeff=0.0, std_dev=0.223, learn_std=False, logdir=str(logdir), steps_per_env=20)
    d.update(kw)
    return SimpleNamespace(**d)


def _env_fn(model, precision):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(64, model=model, precision=precision, seed=7)
    probe = base()
    r = probe.robot
    probe.close()
    if not hasattr(r, "mirrored_obs"):      # H1 has no mirror lists (the reference trains it without SymmetricEnv)
        return base
    return lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)


def _close(ppo):
    ppo.env.close()
    if ppo._comm is not None:
        ppo._comm.close()


def _same(a, b):
    return (math.isnan(a) and math.isnan(b)) or a == b


def _state_dicts_equal(p, q):
    a, b = torch.load(p, weights_only=False).state_dict(), torch.load(q, weights_only=False).state_dict()
    return list(a) == list(b) and all(torch.equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("case", list(CASES))
def test_resumed_run_is_bit_identical_to_the_straight_run(tmp_path, monkeypatch, case):
    from learninghumanoidwalking_b200.rl import PPO
    c = CASES[case]
    monkeypatch.setenv("LHW_FUSED_EXCHANGE", c.get("exchange", "1"))
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    env_fn = _env_fn(c["model"], c["precision"])
    kw = dict(learn_std=c.get("learn_std", False))
    # run A: 4 iterations straight, no snapshots
    a = PPO(env_fn, _args(tmp_path / "a", **kw), seed=11)
    log_a = a.train(None, 4, verbose=False)
    fin_a = [t.clone() for t in (a._flat_param, a._flat_m, a._flat_v, a.env.state_r, a.env.state_i)]
    steps_a = (a.actor_optimizer.step_count, a.critic_optimizer.step_count, a.total_steps, a._best_eval)
    _close(a)
    assert not (tmp_path / "a" / "snapshot").exists()
    # run B: 2 iterations with snapshots (iterations 0 and 1), stopped; a new PPO restores the snapshot and trains to 4
    b = PPO(env_fn, _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    log_b = b.train(None, 2, verbose=False)
    _close(b)
    del b
    b = PPO(env_fn, _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    assert b.restore(tmp_path / "b") == 1
    log_b += b.train(None, 4, verbose=False, start_itr=2)
    fin_b = [b._flat_param, b._flat_m, b._flat_v, b.env.state_r, b.env.state_i]
    for name, x, y in zip(("params", "exp_avg", "exp_avg_sq", "state_r", "state_i"), fin_a, fin_b):
        assert torch.equal(x, y), name
    assert (b.actor_optimizer.step_count, b.critic_optimizer.step_count, b.total_steps, b._best_eval) == steps_a
    assert [e["itr"] for e in log_b] == [0, 1, 2, 3]
    for ea, eb in zip(log_a[2:], log_b[2:]):
        for k in LOGGED:
            if k in ea or k in eb:
                assert _same(ea[k], eb[k]), (ea["itr"], k, ea[k], eb[k])
    for name in ("actor_3.pt", "critic_3.pt", "actor.pt", "critic.pt"):
        assert _state_dicts_equal(tmp_path / "a" / name, tmp_path / "b" / name), name
    snap = tmp_path / "b" / "snapshot"
    assert sorted(p.name for p in snap.iterdir()) == ["itr_3", "latest.json"]
    _close(b)


def _tree(path):
    return {str(p.relative_to(path)): (p.stat().st_size, p.stat().st_mtime_ns) for p in sorted(path.rglob("*"))}


def _compare_runs(run_a, run_b, world):
    """Same checkpoints (equal state dicts) and the same final snapshot in two run directories."""
    pts = lambda d: sorted(p.name for p in d.iterdir() if p.suffix == ".pt")
    assert pts(run_a) == pts(run_b) == ["actor.pt", "actor_0.pt", "actor_1.pt", "actor_3.pt", "critic.pt", "critic_0.pt",
                                        "critic_1.pt", "critic_3.pt"]
    for name in pts(run_a):
        assert _state_dicts_equal(run_a / name, run_b / name), name
    load = lambda d, f: torch.load(d / "snapshot" / "itr_3" / f, weights_only=True)
    la, lb = load(run_a, "learner.pt"), load(run_b, "learner.pt")
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert torch.equal(la[k], lb[k]), k
    assert (la["step_count"], la["adam_step_dev"], la["total_steps"], la["best_eval"]) == \
           (lb["step_count"], lb["adam_step_dev"], lb["total_steps"], lb["best_eval"])
    assert lb["elapsed"] > 0 and lb["args"]["n_itr"] == 4
    for r in range(world):
        sa, sb = load(run_a, f"rank_{r}.pt"), load(run_b, f"rank_{r}.pt")
        for k in ("state_r", "state_i"):
            assert torch.equal(sa[k], sb[k]), (r, k)
        assert torch.equal(sa["worker"]["current_state"], sb["worker"]["current_state"])
        assert torch.equal(sa["worker"]["gen"], sb["worker"]["gen"])


def _cli(*argv):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "run_experiment.py")] + list(argv), capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout


TRAIN = ["--env", "jvrc_walk", "--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1",
         "--seed", "3", "--eval-freq", "2", "--snapshot"]


def test_run_experiment_resume_continues_the_run(tmp_path):
    """`train --snapshot` stopped after iteration 2 (its last snapshot is of iteration 1) and `resume --n-itr 4` against a
    straight 4-iteration run: the same checkpoints and final snapshot; TensorBoard holds every step once (the stopped run's
    iteration-2 scalars are purged); resuming the finished run again has nothing to do and changes no file."""
    import run_experiment as rx
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    rx.main(["train", "--logdir", str(tmp_path / "a"), "--n-itr", "4"] + TRAIN)
    rx.main(["train", "--logdir", str(tmp_path / "b"), "--n-itr", "3"] + TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    out = _cli("resume", "--path", str(run_b), "--n-itr", "4")       # a new process, as after a real stop
    assert f"Resuming {run_b} after iteration 1." in out
    _compare_runs(run_a, run_b, 1)
    acc_a, acc_b = EventAccumulator(str(run_a)), EventAccumulator(str(run_b))
    acc_a.Reload()
    acc_b.Reload()
    assert set(acc_a.Tags()["scalars"]) == set(acc_b.Tags()["scalars"])
    for tag in acc_a.Tags()["scalars"]:
        sa, sb = acc_a.Scalars(tag), acc_b.Scalars(tag)
        assert [s.step for s in sb] == [s.step for s in sa] == ([0, 1, 3] if tag.startswith("Eval/") else [0, 1, 2, 3]), tag
        if not tag.startswith("Time/"):
            assert all(_same(x.value, y.value) for x, y in zip(sa, sb)), tag
    before = _tree(tmp_path)
    assert "Nothing to do" in _cli("resume", "--path", str(run_b), "--n-itr", "4")
    assert _tree(tmp_path) == before


def test_two_rank_resume_is_bit_identical(tmp_path):
    """The same through torchrun at world 2: every rank restores its own shard, and the replicas continue as one run."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")

    def run(*argv):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
               "--master-port", "29671", os.path.join(ROOT, "run_experiment.py")] + list(argv)
        out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, LHW_TENSORBOARD="0"))
        assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]

    run("train", "--logdir", str(tmp_path / "a"), "--n-itr", "4", *TRAIN)
    run("train", "--logdir", str(tmp_path / "b"), "--n-itr", "3", *TRAIN)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    run("resume", "--path", str(run_b), "--n-itr", "4")
    _compare_runs(run_a, run_b, 2)
