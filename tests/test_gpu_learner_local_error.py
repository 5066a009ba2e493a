"""The CUDA learner held to a float64 PPO update (tools/learner_local_error.py), one optimiser step at a time and over whole
production-size iterations.

Per-step tier: every case of the table in DESIGN.md §2 runs 7 re-synchronised steps through PPO._update_step on real rollout
data (3 eager warm-ups, then the captured graph: capture + 4 replays), with lr / eps / clip / entropy and mirror coefficients
away from FusedClipAdam's defaults and max_grad_norm chosen from the measured norms for the case's clip regime.
Whole-iteration tier: PPO.train at run_experiment.py's default learner flags, two iterations (the second replays only graphs
captured in the first), against the float64 learner phase recomputed from the worker's buffer."""
import numpy as np
import pytest
import torch

from tools.learner_local_error import BOUNDS, CASES, gae64, per_step_case, run_iterations, switches

pytestmark = pytest.mark.gpu

REGIMES = {"both": (True, True), "neither": (False, False), "critic": (False, True), "actor": (True, False)}


@pytest.mark.parametrize("case", list(CASES))
def test_each_optimiser_step_matches_the_float64_update(case):
    kw, env = CASES[case]
    with switches(env):
        res, max_norm = per_step_case(**kw)
    assert len(res) >= 6 and all(e["B"] == kw["B"] and e["near"] == 0 for e in res)
    assert [e["graph"] for e in res] == [False] * 3 + [True] * (len(res) - 3)     # eager warm-ups, then capture + replays
    assert max(e["scalars"][6] for e in res) > 0                                   # some ratios left the clip range
    assert all(e["clipped"] == REGIMES[kw["regime"]] for e in res), [(e["norms"], max_norm) for e in res]
    for q in BOUNDS:
        worst = max(range(len(res)), key=lambda k: res[k][q])
        assert res[worst][q] <= 1.0, (q, worst, res[worst][q] * BOUNDS[q], BOUNDS[q])


def test_the_cases_cover_every_clip_regime():
    assert {kw["regime"] for kw, _ in CASES.values()} >= {"both", "neither", "critic"}


def test_vectorised_gae_is_the_oracle_on_the_device():
    from oracle.ppo_oracle import gae_rollout
    rng = np.random.RandomState(0)
    T, N = 400, 4096
    rew, val = rng.uniform(-1, 1, (T, N)), rng.uniform(-2, 2, (T, N))
    ended = (rng.rand(T, N) < 0.02).astype(np.int32)
    boot, last = rng.uniform(-2, 2, (T, N)) * (rng.rand(T, N) < 0.5), rng.uniform(-2, 2, N)
    d = lambda a: torch.as_tensor(a, device="cuda")
    got = gae64(d(rew), d(val), d(ended), d(boot), d(last), 0.99, 0.95).cpu().numpy()
    sub = slice(0, 4096, 61)
    assert np.abs(got[:, sub] - gae_rollout(rew[:, sub], val[:, sub], ended[:, sub], boot[:, sub], last[sub], 0.99, 0.95)).max() < 1e-12


# whole-iteration bounds.  returns: relative to max(1, |ref|); the lhw_gae launch takes gamma and lambda as float, which costs up
# to 3.1e-7 of the measured 3.3e-7, and against the float64 recursion with the fp32-rounded coefficients it stays within 6e-8.
# adv: absolute; stats: the logged iteration means, relative to max(1, |ref|).  The parameters and moments of a free-running
# iteration drift apart as far as float64 runs whose starting parameters differ by fp32 rounding (the controls), so they are
# held to three times the larger drift of two controls.
ITER_BOUNDS = dict(returns=1e-6, returns_vs_f32_coeffs=2e-7, adv=1e-5, stats=3e-3)


@pytest.mark.parametrize("model,kw", [("jvrc_walk", dict(n_envs=4096, steps=400)), ("h1", dict(n_envs=1024, steps=100))])
def test_whole_iterations_match_the_float64_learner_phase(model, kw):
    out = run_iterations(model=model, n_itr=2, **kw)
    assert [e["steps"] for e in out] == [225, 225]
    assert out[0]["graph"] is not None and out[1]["graph"] == out[0]["graph"]      # iteration 2 replays iteration 1's graph
    for e in out:
        assert e["idx_equal"] and e["gather_equal"]
        for q, b in ITER_BOUNDS.items():
            v = max(e[q]) if isinstance(e[q], list) else e[q]
            assert v <= b, (e["itr"], q, v, b, e["stats_got"], e["stats_ref"])
        for q in ("param_step", "exp_avg", "exp_avg_sq"):
            assert e[q] <= 3 * e["control_" + q], (e["itr"], q, e[q], e["control_" + q])
