"""The fp32 kernel source held to the fp64 kernel source ONE control step at a time, on the CPU emulation (tests/emu).

Free-running fp32 / fp64 comparisons can only hold an envelope (a walking robot is chaotic).  Here a fp64 driver advances a
closed-loop trajectory; before every step its record is rounded to fp32 and loaded into both the fp32 emulation and a fp64
shadow, both take the step with the same fp32 action, and the two are compared (tools/fp32_local_error.py).  Bounds sit near
fp32 rounding; a step above them passes only if fp64 copies perturbed at fp32-rounding size spread as far (a contact decision
taken within rounding distance of the ground, DESIGN.md §parity).  Flags, integer state and target counters must be equal."""
import numpy as np
import pytest

from tools import fp32_local_error as L

N_ENVS, STEPS = 8, 120
EXEMPT_SHARE = 0.01      # measured 0 .. 0.6 % of env-steps


@pytest.mark.parametrize("model", L.VARIANTS)
def test_fp32_one_step_error_against_fp64_from_the_same_state(model):
    res = L.run(L.EmulationBackend(model, N_ENVS, seed=3, first_id=7), model, STEPS, regime="noisy")
    n = res["env_steps"]
    print(f"\n[fp32 local error] {model}: {n} env-steps, {res['ended']} ended ({res['falls']} falls), exempt {len(res['exempt'])}")
    for r in res["exempt"]:
        print("   exempt step %d env %d: %s fp32 %.1e, fp64 copies %.1e" % r)
    # the run covers what it claims to: falls, truncations + auto-resets, and (where the variant has them) parameter events
    assert res["falls"] > 0 and res["ended"] > 0
    if model != "h1":
        assert res["ended"] > res["falls"], "no truncation"
    if model in ("h1", "jvrc_step", "jvrc_walk_terrain"):
        assert res["param_events"] > 0
    assert not res["mismatch"], res["mismatch"][:5]
    assert not res["fail"], "fp32 steps above the bounds that fp64 perturbed at rounding size does not reproduce: " + \
        "; ".join("step %d env %d %s fp32 %.1e fp64 copies %.1e" % r for r in res["fail"][:5])
    assert len(res["exempt"]) <= EXEMPT_SHARE * n, len(res["exempt"])
    # the bulk sits at fp32 rounding (measured medians 1e-7 .. 3e-6)
    for q, bound in (("qpos", 1e-6), ("qvel", 1e-5), ("obs", 1e-5), ("reward", 1e-5), ("rew_terms", 1e-5)):
        assert np.median(res["errors"][q]) < bound, (q, np.median(res["errors"][q]))


def test_fp32_one_step_error_at_zero_action():
    """The standing regime (a = 0, contact-heavy steady state) for the walking model."""
    res = L.run(L.EmulationBackend("jvrc_walk", 4, seed=5, first_id=0), "jvrc_walk", 80, regime="zero")
    assert not res["mismatch"] and not res["fail"], (res["mismatch"][:3], res["fail"][:3])
    assert len(res["exempt"]) <= EXEMPT_SHARE * res["env_steps"]
