"""Learning-rate schedules of `run_experiment.py train --schedule` (DESIGN.md §7.3).

"fixed" (the default, the reference's): Adam at `--lr` throughout.
"adaptive": rsl_rl's KL-adaptive rate, updated after every minibatch's loss and used by that same optimiser step.  The rate
lives in device memory and the fused exchange updates it (csrc/comm_kernels.cu); `adapt_lr` and `rank_mean_kl` are the same
float64 arithmetic on the host, bit for bit, for tests and for reading a run.
"""
from __future__ import annotations

import math

import numpy as np

SCHEDULES = ("fixed", "adaptive")
DEFAULT_DESIRED_KL = 0.01
LR_MIN, LR_MAX, LR_FACTOR = 1e-5, 1e-2, 1.5


def adapt_lr(lr: float, kl: float, desired_kl: float) -> float:
    """One step of the rule: kl > 2 desired -> lr / 1.5 (at least 1e-5); 0 < kl < desired / 2 -> lr * 1.5 (at most 1e-2);
    otherwise, and for a NaN kl, lr unchanged."""
    lr, kl, desired_kl = float(lr), float(kl), float(desired_kl)
    if kl > 2.0 * desired_kl:
        return max(LR_MIN, lr / LR_FACTOR)
    if kl > 0.0 and kl < desired_kl / 2.0:
        return min(LR_MAX, lr * LR_FACTOR)
    return lr


def rank_mean_kl(kls) -> float:
    """The mean the exchange takes over the ranks' float32 KL words: a float64 sum in rank order, divided by the world size."""
    s = 0.0
    for k in kls:
        s += float(np.float32(k))
    return s / len(kls)


def schedule_of(args) -> tuple[str, float]:
    """(schedule, desired_kl) of a run's arguments; arguments without them (an earlier run's experiment.pkl) are "fixed"."""
    kl = getattr(args, "desired_kl", None)
    return getattr(args, "schedule", None) or "fixed", float(DEFAULT_DESIRED_KL if kl is None else kl)


def check(schedule: str, desired_kl: float) -> None:
    """ValueError naming the reason for a schedule this build cannot run."""
    if schedule not in SCHEDULES:
        raise ValueError(f"unknown learning-rate schedule {schedule!r} (this build has: {', '.join(SCHEDULES)})")
    if schedule == "adaptive" and not (math.isfinite(desired_kl) and desired_kl > 0):
        raise ValueError(f"--desired-kl must be > 0 for the adaptive schedule, got {desired_kl}")
