"""One-control-step error of the fp32 step kernel against the fp64 kernel, re-synchronised every step.

Comparing fp32 and fp64 runs that evolve freely says little: a walking robot is chaotic, any rounding difference grows, and
only a loose envelope can hold.  Here both precisions take ONE control step from the same state, and then both are put back
on a common trajectory before the next step:

  D   fp64 driver at the model's own solver tolerance; it alone advances the trajectory (closed loop through D's observation)
  E   fp32 kernel (solver tolerance 1e-6) loaded with D's record rounded to fp32
  S   fp64 shadow loaded with the SAME fp32-rounded record
  E and S take one control step with the same fp32 action, and E is compared with S.

The state record has the same layout in both precisions, so re-synchronising is a copy.  The bulk of the one-step errors sits
near fp32 rounding (about 1e-5 relative in qvel), so BOUNDS below sit 300x under the free-running envelopes of the older fp32
tests.  A step above a bound is classified by a perturbation control: P re-runs fp64 from COPIES copies of the rounded record
whose qpos / qvel are multiplied by (1 + U(-EPS, EPS)) -- the size of the fp32 rounding of the state and of the forward
kinematics.  If the copies spread by at least FRAC of the fp32 error, the step is ill-conditioned (the dynamics of one
control step are discontinuous there: a foot corner starts or stops touching within rounding distance of the ground, see
DESIGN.md) and exempt; anything else is a defect.  done, ended, the integer state (phase, mode, traj_len, ep_len, rng_ctr,
have_prev, status) and the SteppingTask's target counters must be equal, with no exemption.

Two back ends share that logic: the CPU emulation of the kernel source (tests/emu, compiled for the host) and the device
kernels through BatchedHumanoidEnv.  `python tools/fp32_local_error.py` prints the emulation's distribution table (DESIGN.md);
`--device` the device's (needs a GPU).
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

VARIANTS = ("jvrc_walk", "h1", "jvrc_step", "jvrc_walk_terrain")
# per-env bounds on one control step: relative to max(1, |fp64 value|) for vectors, absolute for rewards
# (qacc_warm, the solver's warm start, is a solution at the fp32 solver tolerance: it only decides where the next solve starts)
BOUNDS = dict(qpos=1e-4, qvel=1e-4, obs=1e-4, term_obs=1e-4, record=1e-4, qacc_warm=1e-2, reward=1e-4, rew_terms=1e-4, ep_rew=1e-4)
# perturbation of qpos / qvel in the control, relative: 40 fp32 units in the last place, five times the p99 of the fp32 one-step
# qpos error.  A contact decision that fp32 takes on a corner within ~1e-7 m of the ground can happen on the last of the 25
# substeps, and smaller perturbations of the control step's START do not reliably move that corner across (DESIGN.md)
EPS = 40 * 2.0 ** -24
COPIES = 4
FRAC = 0.1                # a step is exempt when the fp64 copies spread by at least this fraction of the fp32 error
MAX_TRAJ_LEN = 40         # short episodes: truncations and auto-resets every run
F32_TOLERANCE = 1e-6      # the fp32 kernel's solver tolerance (BatchedHumanoidEnv's default for precision 32)


def layout(nq, nv, nu, nr, model):
    """Slices of the real state record (csrc/sim_core.h Persist): qpos, qvel, the rest of the dynamic record, and for the
    SteppingTask the target counters tk (small integers held exactly in the record's last 5 words)."""
    rest_end = nq + 2 * nv + 5 * nu + 4
    return dict(qpos=slice(0, nq), qvel=slice(nq, nq + nv), qacc_warm=slice(nq + nv, nq + 2 * nv), record=slice(nq + 2 * nv, rest_end),
                tk=slice(nr - 5, nr) if model == "jvrc_step" else None)


def _rel(x, y):
    x, y = np.asarray(x, np.float64), np.asarray(y, np.float64)
    return np.abs(x - y).max(axis=-1) / np.maximum(1.0, np.abs(y).max(axis=-1))


def errors(e, s, lay):
    """Per-env errors of step output e against s (dicts of numpy arrays, see the back ends), NaN where not applicable."""
    ended = s["ended"].astype(bool)
    out = dict(qpos=_rel(e["sr"][:, lay["qpos"]], s["sr"][:, lay["qpos"]]),
               qvel=_rel(e["sr"][:, lay["qvel"]], s["sr"][:, lay["qvel"]]),
               qacc_warm=_rel(e["sr"][:, lay["qacc_warm"]], s["sr"][:, lay["qacc_warm"]]),
               record=_rel(e["sr"][:, lay["record"]], s["sr"][:, lay["record"]]),
               obs=_rel(e["obs"], s["obs"]),
               reward=np.abs(e["reward"].astype(np.float64) - s["reward"]),
               rew_terms=np.abs(e["rew_terms"].astype(np.float64) - s["rew_terms"]).max(axis=-1))
    out["term_obs"] = np.where(ended, _rel(e["term_obs"], s["term_obs"]), np.nan)
    out["ep_rew"] = np.where(ended, _rel(e["ep_rew"][:, None], s["ep_rew"][:, None]), np.nan)
    return out


def exact_mismatch(e, s, lay):
    """Per-env: True where a quantity that must be equal differs (flags, integer state, episode length, target counters)."""
    ended = s["ended"].astype(bool)
    bad = (e["done"] != s["done"]) | (e["ended"] != s["ended"]) | (e["si"][:, :7] != s["si"][:, :7]).any(axis=1)
    bad |= ended & (e["ep_len"] != s["ep_len"])
    if lay["tk"] is not None:
        bad |= (e["sr"][:, lay["tk"]].astype(np.float64) != s["sr"][:, lay["tk"]]).any(axis=1)
    return bad


class EmulationBackend:
    """The kernel source compiled for the host (tests/emu): the arithmetic the device executes, lane by lane."""

    def __init__(self, model, n, seed, first_id):
        sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests", "emu")) if p not in sys.path]
        from emu_variants import Emu    # every variant of the kernel source, h1_walk included
        from learninghumanoidwalking_b200.model import load_model, pack_model
        mj = load_model(model)
        f64, f32 = pack_model(mj), pack_model(mj, tolerance=F32_TOLERANCE)
        self.D, self.S, self.P = (Emu(f64, 64, n, seed=seed, first_id=first_id) for _ in range(3))
        self.E = Emu(f32, 32, n, seed=seed, first_id=first_id)
        self.nq, self.nv, self.nu, self.nobs, self.nr = self.D.nq, self.D.nv, self.D.nu, self.D.nobs, self.D.nr

    def reset(self):
        return self.D.reset().astype(np.float64)

    def driver_record(self):
        return self.D.sr, self.D.si

    def load(self, which, sr, si):
        x = getattr(self, which)
        x.sr[:] = sr.astype(x.dt)
        x.si[:] = si

    def step(self, which, a, max_traj_len):
        x = getattr(self, which)
        o = x.step(a, max_traj_len=max_traj_len)
        return dict(obs=o[0], term_obs=o[1], rew_terms=o[2], reward=o[3], done=o[4].copy(), ended=o[5].copy(), ep_len=o[6],
                    ep_rew=o[7], sr=x.sr.copy(), si=x.si.copy())


class DeviceBackend:
    """The compiled kernels through the C-ABI (BatchedHumanoidEnv), one env object per role."""

    def __init__(self, model, n, seed, first_id, max_traj_len=MAX_TRAJ_LEN):
        import torch
        sys.path[:0] = [p for p in (ROOT, os.path.join(ROOT, "tests", "emu")) if p not in sys.path]
        from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
        self.torch = torch
        mk = lambda p: BatchedHumanoidEnv(n, model=model, precision=p, seed=seed, first_env_id=first_id, max_traj_len=max_traj_len)
        self.D, self.S, self.P, self.E = mk(64), mk(64), mk(64), mk(32)
        for x in (self.S, self.P, self.E):
            x.reset()                 # clears _fresh; the records are overwritten before every step
        self.nq, self.nv, self.nu, self.nobs = self.D.nq, self.D.nv, self.D.act_dim, self.D.obs_dim
        self.nr = self.D.state_r.shape[1]

    def reset(self):
        return self.D.reset().double().cpu().numpy()

    def driver_record(self):
        return self.D.state_r.cpu().numpy(), self.D.state_i.cpu().numpy()

    def load(self, which, sr, si):
        x = getattr(self, which)
        x.state_r.copy_(self.torch.from_numpy(np.ascontiguousarray(sr)).to(x.state_r.dtype))
        x.state_i.copy_(self.torch.from_numpy(np.ascontiguousarray(si)))

    def step(self, which, a, max_traj_len):
        x = getattr(self, which)
        assert x.max_traj_len == max_traj_len
        x.step(self.torch.from_numpy(np.ascontiguousarray(a)).to(device=x.device, dtype=x.dtype))
        c = lambda t: t.cpu().numpy()
        return dict(obs=c(x.obs), term_obs=c(x.term_obs), rew_terms=c(x.rew_terms), reward=c(x.reward), done=c(x.done),
                    ended=c(x.ended), ep_len=c(x.ep_len), ep_rew=c(x.ep_rew), sr=c(x.state_r), si=c(x.state_i))

    def close(self):
        for x in (self.D, self.S, self.P, self.E):
            x.close()


def noisy_policy(nobs, nu, rng):
    """A fixed tanh policy plus N(0, 0.3^2) exploration noise (the early-training regime: falls, resets)."""
    W = rng.normal(size=(nobs, nu)) / np.sqrt(nobs)
    return lambda obs: 0.3 * np.tanh(obs @ W / 10) + rng.normal(size=(obs.shape[0], nu)) * 0.3


def trained_policy(model, rng, sigma=0.05):
    """The actor of a finished jvrc_walk training run (tests/golden/trained_actor_jvrc_walk.pt) plus a little noise."""
    import torch
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    actor = torch.load(os.path.join(ROOT, "tests", "golden", f"trained_actor_{model}.pt"), map_location="cpu",
                       weights_only=False).double()
    actor.eval()

    def pol(obs):
        with torch.no_grad():
            a = actor(torch.from_numpy(np.ascontiguousarray(obs, dtype=np.float64)), deterministic=True).numpy()
        return a + rng.normal(size=a.shape) * sigma
    return pol


def run(backend, model, steps, regime="noisy", max_traj_len=MAX_TRAJ_LEN, rng_seed=0, eps=EPS, copies=COPIES, frac=FRAC,
        compare_source=None):
    """Drive `steps` re-synchronised control steps.  Returns a dict: per-quantity error arrays (bulk, every env-step),
    `exempt` and `fail` lists of (step, env, quantity, fp32 error, fp64 spread), `mismatch` (exact quantities), counts, and
    `param_events`: env-steps without an episode end that changed the record's parameter tail (H1 randomisation and pushes,
    SteppingTask target switches, terrain re-poses).
    `compare_source`: an EmulationBackend of the same variant; its fp32 emulation takes the same step from the same record,
    and the device's fp32 outputs are compared with it (`source` errors)."""
    rng, prng = np.random.RandomState(rng_seed), np.random.RandomState(rng_seed + 9)
    obs = backend.reset()
    n, nu = obs.shape[0], backend.nu
    pol = (lambda o: np.zeros((o.shape[0], nu))) if regime == "zero" else \
        trained_policy(model, rng) if regime == "trained" else noisy_policy(backend.nobs, nu, rng)
    lay = layout(backend.nq, backend.nv, nu, backend.nr, model)
    res = dict(errors={k: [] for k in BOUNDS}, exempt=[], fail=[], mismatch=[], ended=0, falls=0, env_steps=0, param_events=0,
               source={k: [] for k in BOUNDS})
    pq = slice(0, backend.nq + backend.nv)
    for k in range(steps):
        a = pol(obs).astype(np.float32)
        sr, si = backend.driver_record()
        R = sr.astype(np.float32)
        backend.load("E", R, si)
        backend.load("S", R.astype(np.float64), si)
        e = backend.step("E", a, max_traj_len)
        s = backend.step("S", a.astype(np.float64), max_traj_len)
        if compare_source is not None:
            compare_source.load("E", R, si)
            c = compare_source.step("E", a, max_traj_len)
            for q, v in errors(e, c, lay).items():
                res["source"][q].append(v)
            res["mismatch"] += [(k, i, "source") for i in np.nonzero(exact_mismatch(e, c, lay))[0]]
        obs = backend.step("D", a.astype(np.float64), max_traj_len)["obs"].astype(np.float64)
        err = errors(e, s, lay)
        for q, v in err.items():
            res["errors"][q].append(v)
        res["mismatch"] += [(k, i, "exact") for i in np.nonzero(exact_mismatch(e, s, lay))[0]]
        res["ended"] += int(s["ended"].sum())
        res["falls"] += int(s["done"].sum())
        tail = slice(lay["record"].stop, backend.nr)
        res["param_events"] += int((~s["ended"].astype(bool) & (s["sr"][:, tail] != R[:, tail]).any(axis=1)).sum())
        res["env_steps"] += n
        over = {q: np.nan_to_num(v, nan=0.0) > BOUNDS[q] for q, v in err.items()}
        flagged = np.nonzero(np.any(np.stack(list(over.values())), axis=0))[0]
        if flagged.size:
            spread = {q: np.zeros(n) for q in BOUNDS}
            for _ in range(copies):
                Rp = R.astype(np.float64)
                Rp[:, pq] *= 1 + eps * prng.uniform(-1, 1, size=Rp[:, pq].shape)
                backend.load("P", Rp, si)
                p = backend.step("P", a.astype(np.float64), max_traj_len)
                for q, v in errors(p, s, lay).items():
                    spread[q] = np.maximum(spread[q], np.nan_to_num(v, nan=0.0))
            for i in flagged:
                qs = [q for q in BOUNDS if over[q][i]]
                worst = max(qs, key=lambda q: err[q][i] / BOUNDS[q])
                rec = (k, int(i), worst, float(err[worst][i]), float(spread[worst][i]))
                ok = all(spread[q][i] >= frac * err[q][i] for q in qs)
                res["exempt" if ok else "fail"].append(rec)
    for key in ("errors", "source"):
        res[key] = {q: np.concatenate(v) if v else np.zeros(0) for q, v in res[key].items()}
    return res


def table_rows(name, res, key="errors"):
    rows = []
    for q in ("qpos", "qvel", "obs", "reward", "rew_terms", "term_obs"):
        v = res[key][q]
        v = v[np.isfinite(v)]
        if v.size:
            rows.append(f"| {name} | {q} | {np.median(v):.1e} | {np.percentile(v, 99):.1e} | {np.percentile(v, 99.9):.1e} | "
                        f"{v.max():.1e} | {v.size} |")
    return rows


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--device", action="store_true", help="the device kernels (needs a GPU) instead of the CPU emulation")
    ap.add_argument("--envs", type=int, default=None)
    ap.add_argument("--steps", type=int, default=None)
    ap.add_argument("--regime", default="noisy", choices=("zero", "noisy", "trained"))
    ap.add_argument("--variants", default=",".join(VARIANTS))
    args = ap.parse_args()
    n = args.envs or (100 if args.device else 8)
    steps = args.steps or (300 if args.device else 120)
    print("| variant | quantity | median | p99 | p99.9 | max | env-steps |\n|---|---|---|---|---|---|---|")
    notes = []
    for name in args.variants.split(","):
        be = DeviceBackend(name, n, seed=3, first_id=7) if args.device else EmulationBackend(name, n, seed=3, first_id=7)
        res = run(be, name, steps, regime=args.regime)
        print("\n".join(table_rows(name, res)))
        notes.append(f"{name}: {res['env_steps']} env-steps, {res['ended']} ended ({res['falls']} falls), {res['param_events']} parameter events, exempt {len(res['exempt'])}, "
                     f"failing {len(res['fail'])}, exact mismatches {len(res['mismatch'])}")
        for r in res["exempt"] + res["fail"]:
            notes.append(f"  {'exempt' if r in res['exempt'] else 'FAIL  '} step {r[0]} env {r[1]}: {r[2]} fp32 {r[3]:.1e}, fp64 copies {r[4]:.1e}")
        if args.device:
            be.close()
    print("\n".join(notes))


if __name__ == "__main__":
    main()
