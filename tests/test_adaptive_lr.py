"""The KL-adaptive learning rate (`train --schedule adaptive`, DESIGN.md §7.3) on the host: the float64 rule, the rank mean,
the command line and its refusals, and runs recorded before the schedule existed.  The device side is
tests/test_gpu_adaptive_lr.py."""
import argparse
import math
import os
import pickle
import sys
from types import SimpleNamespace

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from learninghumanoidwalking_b200.rl import schedule  # noqa: E402
from learninghumanoidwalking_b200.rl.schedule import LR_MAX, LR_MIN, adapt_lr, rank_mean_kl  # noqa: E402

D = 0.01


@pytest.mark.parametrize("lr, kl, want", [
    (3e-4, 0.05, 3e-4 / 1.5),              # above 2 desired: decrease
    (3e-4, 2 * D, 3e-4),                   # exactly 2 desired: unchanged (strict >)
    (3e-4, math.nextafter(2 * D, 1), 3e-4 / 1.5),
    (3e-4, D, 3e-4),                       # inside the band
    (3e-4, D / 2, 3e-4),                   # exactly desired / 2: unchanged (strict <)
    (3e-4, math.nextafter(D / 2, 0), 3e-4 * 1.5),
    (3e-4, 1e-4, 3e-4 * 1.5),              # below desired / 2: increase
    (3e-4, 0.0, 3e-4),                     # rsl_rl's kl > 0 on the increase branch
    (3e-4, -1e-3, 3e-4),                   # negative (the estimator's rounding can give one)
    (3e-4, float("nan"), 3e-4),            # NaN: every comparison fails
    (3e-4, float("inf"), 3e-4 / 1.5),
    (1.2e-5, 1.0, LR_MIN),                 # clamp below
    (LR_MIN, 1.0, LR_MIN),
    (8e-3, 1e-4, LR_MAX),                  # clamp above
    (LR_MAX, 1e-4, LR_MAX),
])
def test_rule_on_a_table_of_kl_values(lr, kl, want):
    got = adapt_lr(lr, kl, D)
    assert got == want and isinstance(got, float), (lr, kl, got, want)


def test_rule_repeats_to_the_clamps_and_back():
    lr = 3e-4
    for _ in range(40):
        lr = adapt_lr(lr, 1.0, D)
    assert lr == LR_MIN
    for _ in range(40):
        lr = adapt_lr(lr, 1e-6, D)
    assert lr == LR_MAX


def test_rank_mean_is_a_float64_sum_in_rank_order():
    kls = np.array([0.1, 1e-8, 0.3, 7e-3], dtype=np.float32)
    s = 0.0
    for k in kls:
        s += float(k)
    assert rank_mean_kl(kls) == s / 4
    assert rank_mean_kl([np.float32(0.02)]) == float(np.float32(0.02))
    assert math.isnan(rank_mean_kl([0.1, float("nan")]))


def test_schedule_of_and_check():
    assert schedule.schedule_of(SimpleNamespace()) == ("fixed", 0.01)
    assert schedule.schedule_of(SimpleNamespace(schedule="adaptive", desired_kl=0.02)) == ("adaptive", 0.02)
    assert schedule.schedule_of(SimpleNamespace(schedule="adaptive", desired_kl=0.0)) == ("adaptive", 0.0)
    schedule.check("fixed", 0.0)                # the fixed schedule ignores --desired-kl
    schedule.check("adaptive", 1e-3)
    for kl in (0.0, -0.01, float("nan")):
        with pytest.raises(ValueError, match="desired-kl must be > 0"):
            schedule.check("adaptive", kl)
    with pytest.raises(ValueError, match="unknown learning-rate schedule"):
        schedule.check("linear", 0.01)


def _rx():
    import importlib.util
    spec = importlib.util.spec_from_file_location("lhw_run_experiment_adaptive", os.path.join(ROOT, "run_experiment.py"))
    rx = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(rx)
    return rx


def _parse(rx, *argv):
    p = argparse.ArgumentParser()
    for flag, kw in rx.TRAIN_FLAGS:
        p.add_argument(flag, **kw)
    return p.parse_args(["--env", "jvrc_walk", *argv])


def test_flags_parse_with_fixed_defaults():
    rx = _rx()
    a = _parse(rx)
    assert (a.schedule, a.desired_kl, a.lr) == ("fixed", 0.01, 3e-4)
    a = _parse(rx, "--schedule", "adaptive", "--desired-kl", "0.02", "--lr", "1e-3")
    assert (a.schedule, a.desired_kl, a.lr) == ("adaptive", 0.02, 1e-3)
    with pytest.raises(SystemExit):
        _parse(rx, "--schedule", "linear")


@pytest.mark.parametrize("argv, env, match", [
    (("--schedule", "adaptive", "--desired-kl", "0"), {}, "desired-kl must be > 0"),
    (("--schedule", "adaptive", "--desired-kl", "-0.01"), {}, "desired-kl must be > 0"),
    (("--schedule", "adaptive"), {"LHW_FUSED_EXCHANGE": "0"}, "LHW_FUSED_EXCHANGE=0"),
])
def test_train_refuses_before_any_run_directory_exists(tmp_path, monkeypatch, argv, env, match):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rx = _rx()
    with pytest.raises(SystemExit, match=match):
        rx.main(["train", "--env", "jvrc_walk", "--logdir", str(tmp_path / "logs"), *argv])
    assert not (tmp_path / "logs").exists()


def test_fixed_schedule_is_not_refused_on_the_baseline_exchange(monkeypatch):
    monkeypatch.setenv("LHW_FUSED_EXCHANGE", "0")
    rx = _rx()
    rx.check_schedule(_parse(rx))
    rx.check_schedule(_parse(rx, "--desired-kl", "0"))     # ignored by the fixed schedule


def test_experiment_pkl_without_the_keys_resumes_as_fixed(tmp_path, monkeypatch):
    """An experiment.pkl written before the schedule existed: `resume` reads it as a fixed-rate run (and so does PPO)."""
    rx = _rx()
    old = _parse(rx)
    del old.schedule, old.desired_kl
    with open(tmp_path / "experiment.pkl", "wb") as f:
        pickle.dump(old, f)
    with open(tmp_path / "experiment.pkl", "rb") as f:
        run_args = pickle.load(f)
    assert not hasattr(run_args, "schedule") and schedule.schedule_of(run_args) == ("fixed", 0.01)
    monkeypatch.setenv("LHW_FUSED_EXCHANGE", "0")     # would refuse an adaptive run
    rx.check_schedule(run_args)
    # resume gets as far as the snapshot (none here) without tripping over the missing keys
    with pytest.raises(SystemExit, match="no snapshot"):
        rx.main(["resume", "--path", str(tmp_path)])


def test_hand_assigned_optimisers_are_refused_under_the_adaptive_schedule():
    import torch
    from learninghumanoidwalking_b200.rl.ppo import PPO
    ppo = PPO.__new__(PPO)
    net = torch.nn.Linear(2, 2)
    ppo.__dict__.update(schedule="adaptive", desired_kl=0.01, _comm=object(), actor_optimizer=torch.optim.Adam(net.parameters()),
                        critic_optimizer=torch.optim.Adam(net.parameters()))
    with pytest.raises(ValueError, match="hand-assigned torch optimisers"):
        ppo._check_schedule()
    from learninghumanoidwalking_b200.rl.optim import FusedClipAdam
    ppo.actor_optimizer = ppo.critic_optimizer = FusedClipAdam.__new__(FusedClipAdam)
    ppo._check_schedule()
    ppo._comm = None
    with pytest.raises(ValueError, match="LHW_FUSED_EXCHANGE=0"):
        ppo._check_schedule()
    ppo.schedule = "fixed"
    ppo._check_schedule()


def test_ppo_refuses_a_bad_desired_kl_before_touching_the_device():
    from learninghumanoidwalking_b200.rl.ppo import PPO
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=64, epochs=1,
                           max_traj_len=10, num_procs=4, max_grad_norm=0.5, mirror_coeff=0.0, schedule="adaptive", desired_kl=-1.0)
    with pytest.raises(ValueError, match="desired-kl must be > 0"):
        PPO(lambda: None, args)
