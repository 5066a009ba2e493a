"""Error of the CUDA learner against a float64 PPO update, one optimiser step at a time and over whole iterations.

The learner that trains is PPO._update_step on the flat parameter buffer of PPO.make_optimizers(): the fused loss kernel,
lhw_linear_wgrad, and the fused exchange (clip + Adam for both networks) replayed from a captured CUDA graph.  Its unit tests
check each kernel alone; this tool checks their composition against an independent float64 update:

  L   the CUDA learner (fp32), stepped through PPO._update_step with the minibatch in ppo._mb (gather_minibatch), as train does
  S   a float64 shadow: float64 copies of policy, old policy and critic with hand-made torch.optim.Adam + clip_grad_norm_,
      stepped by the NON-fused branch of PPO.update_actor_critic (pinned to the reference's method by
      tests/test_ppo_update_golden.py; S itself by tests/test_learner_shadow.py).  While S runs, _lib.ops() raises and
      LHW_FUSED_LOSS=0: no lhw kernel is reached.

Per-step tier: before every step S is re-synchronised from L (flat parameters split into the actor then the critic segment,
both Adam moments, the Adam step number, the old policy; fp32 -> fp64 is exact), both take the same minibatch and errors cannot
accumulate.  Compared: the 7 returned scalars, the raw gradient of every parameter tensor (L: ppo._flat_grad, which the clip +
Adam kernels only read; S: recorded before clip_grad_norm_), the actor and critic pre-clip norms, and after the step the moments
and the parameters.  Adam divides by sqrt(v) per element, so an element whose gradient is small (relative to the fp32 rounding
of its sum over the minibatch) turns a tiny gradient difference into a large step difference.  The gradient is therefore bounded
directly, and the parameters and moments are held to a third computation: the float64 optimiser (the same torch clip + Adam as
S) applied to L's own gradient.  That isolates the clip + Adam kernels, their hyper-parameters and the actor / critic split.
The minibatches skip samples at a kink of the loss (a clip boundary or a ReLU, Shadow.near_kink), where fp32 and float64 may
legitimately take different branches.

Whole-iteration tier: PPO.train one iteration at a time; after each, the float64 reference recomputes the learner phase from the
worker's buffer: GAE over every environment (gae64, vectorised over environments), the unbiased advantage normalisation, the same
minibatch_indices call, gathers by plain indexing and all optimiser steps of S, free-running within the iteration.  A control
repeats the float64 phase from parameters perturbed by fp32 rounding: free-running runs drift apart that far on their own.

Imitation (opt-in, `--imitation`, IMITATION_CASES): the CUDA learner trains with a teacher (`train --imitate`, DESIGN §7.2),
and S carries a float64 copy of the same teacher behind the same projector, so that its non-fused branch computes the
reference's term (rl/algos/ppo.py:361-368).  Without a teacher S is the shadow above, unchanged.

Adaptive learning rate (opt-in, `--adaptive`, ADAPTIVE_CASES): the CUDA learner runs `--schedule adaptive` (DESIGN §7.3).  The
old policy is re-offset before every step, alternately far and near, so that the minibatch KL crosses both thresholds of a
desired_kl chosen from a probe.  After each step the device rate must equal the float64 rule (rl/schedule.py) applied to the
CUDA learner's own KL, bit for bit, and both shadows step with that rate.

`python tools/learner_local_error.py` prints the distribution tables (needs a GPU); `--rehearse` runs the float64 parts on the
CPU at a tiny size.
"""
from __future__ import annotations

import argparse
import contextlib
import os
import sys
import tempfile
import time
from copy import deepcopy
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

# per-step bounds (calibrated on an H100, DESIGN.md §2): scalars relative to max(1, |ref|); gradients per tensor, ||d||_2 relative
# to ||ref||_2 and max|d| relative to max|ref|; norms relative; moments relative per tensor norm; parameters (in units of the
# allowance) |dp| <= ulp32(p) + PARAM_LR * lr.  The moment bound is 2e-5, not 1e-5: the clip + Adam kernels take beta2 as a
# float, and 1 - 0.999f is 1.29e-5 (relative) short of 0.001, which exp_avg_sq carries whole.
BOUNDS = dict(scalar=1e-5, grad_l2=1e-5, grad_max=1e-4, norm=1e-5, moment=2e-5, param=1.0)
PARAM_LR = 1e-4
# a sample this close (relative) to a kink of the loss (clip boundary, ReLU) may take another branch in fp32 (Shadow.near_kink)
KINK_MARGIN = 1e-5


@contextlib.contextmanager
def no_lhw():
    """While the shadow steps: every torch.ops.lhw entry point raises, and the loss takes the torch graph.  (lhw_linear_wgrad
    is reached through _lib.ops() too; lhw_launch_count does not count it, so it cannot serve as the guard.)"""
    from learninghumanoidwalking_b200 import _lib
    real, env = _lib.ops, os.environ.get("LHW_FUSED_LOSS")

    def refuse():
        raise AssertionError("the float64 shadow reached a torch.ops.lhw entry point")
    _lib.ops = refuse
    os.environ["LHW_FUSED_LOSS"] = "0"
    try:
        yield
    finally:
        _lib.ops = real
        if env is None:
            os.environ.pop("LHW_FUSED_LOSS", None)
        else:
            os.environ["LHW_FUSED_LOSS"] = env


def mirror_fns(sym, dtype, device):
    """SymmetricEnv's clock-aware observation mirror and action mirror as matmuls in `dtype` (its matrices are float32, and
    their entries are 0 / +-1, so the float64 versions are exact)."""
    if sym is None:
        return None, None
    mo = sym.obs_mirror_clock_matrix.to(device, dtype)
    ma = sym.act_mirror_matrix.to(device, dtype)
    return (lambda o: o @ mo), (lambda a: a @ ma)


class Shadow:
    """float64 policy, old policy and critic with hand-made torch Adam: the reference's optimiser sequence
    (rl/algos/ppo.py:389-396) through PPO.update_actor_critic's non-fused branch."""

    def __init__(self, policy, old_policy, critic, hyper, sym=None, device="cpu", dtype=torch.float64, teacher=None,
                 projector=None, imitate_coeff=0.0):
        """teacher / projector / imitate_coeff: the imitation term (PPO.base_policy, .imitation_projector), with a copy of the
        teacher in `dtype`; without a teacher the shadow has no imitation attributes at all, as before."""
        from learninghumanoidwalking_b200.rl.ppo import PPO
        self.dtype, self.device = dtype, torch.device(device)
        cast = lambda m: deepcopy(m).to(self.device, dtype)
        self.policy, self.old_policy, self.critic = cast(policy), cast(old_policy), cast(critic)
        mk = lambda net: torch.optim.Adam(net.parameters(), lr=hyper["lr"], eps=hyper["eps"], foreach=False)
        self.ppo = PPO.__new__(PPO)
        self.ppo.__dict__.update(policy=self.policy, old_policy=self.old_policy, critic=self.critic, clip=hyper["clip"],
                                 ent_coeff=hyper["ent_coeff"], mirror_coeff=hyper["mirror_coeff"], imitate_coeff=0.0,
                                 grad_clip=hyper["max_grad_norm"], _comm=None, world=1,
                                 actor_optimizer=mk(self.policy), critic_optimizer=mk(self.critic))
        if teacher is not None:
            self.ppo.__dict__.update(base_policy=cast(teacher).eval().requires_grad_(False), imitation_projector=projector,
                                     imitate_coeff=float(imitate_coeff))
        self.mirror = mirror_fns(sym, dtype, self.device)

    def params(self):
        return list(self.policy.parameters()) + list(self.critic.parameters())

    def load(self, flat, m, v, step, old_policy=None):
        """Parameters, moments and completed Adam steps from flat vectors (actor segment, then critic segment)."""
        off = 0
        for net, opt in ((self.policy, self.ppo.actor_optimizer), (self.critic, self.ppo.critic_optimizer)):
            for p in net.parameters():
                k = p.numel()
                sl = lambda t: t[off:off + k].view_as(p).to(self.device, self.dtype).clone()
                with torch.no_grad():
                    p.copy_(sl(flat))
                opt.state[p] = dict(step=torch.tensor(float(step)), exp_avg=sl(m), exp_avg_sq=sl(v))
                off += k
        assert off == flat.numel()
        if old_policy is not None:
            with torch.no_grad():
                for q, r in zip(self.old_policy.parameters(), old_policy.parameters()):
                    q.copy_(r)
                self.old_policy.obs_mean.copy_(old_policy.obs_mean)
                self.old_policy.obs_std.copy_(old_policy.obs_std)

    def flat(self, what):
        if what == "param":
            return torch.cat([p.detach().reshape(-1) for p in self.params()])
        opt = lambda p: self.ppo.actor_optimizer if p in set(self.policy.parameters()) else self.ppo.critic_optimizer
        return torch.cat([opt(p).state[p][what].reshape(-1) for p in self.params()])

    def step(self, obs, act, ret, adv):
        """One update_actor_critic; returns (7 scalars, raw gradients per tensor, (actor, critic) pre-clip norms)."""
        real, rec = torch.nn.utils.clip_grad_norm_, []

        def spy(params, max_norm, *a, **k):
            params = list(params)
            grads = [p.grad.detach().clone() for p in params]
            n = real(params, max_norm, *a, **k)
            rec.append((grads, float(n)))
            return n
        c = lambda t: t.to(self.device, self.dtype)
        torch.nn.utils.clip_grad_norm_ = spy
        try:
            with no_lhw():
                out = self.ppo.update_actor_critic(c(obs), c(act), c(ret), c(adv), 1, mirror_observation=self.mirror[0],
                                                   mirror_action=self.mirror[1])
        finally:
            torch.nn.utils.clip_grad_norm_ = real
        assert len(rec) == 2
        return [float(x) for x in out], rec[0][0] + rec[1][0], (rec[0][1], rec[1][1])

    def optimise(self, grads):
        """clip_grad_norm_ x2 + Adam x2 on given gradients (no loss): the float64 optimiser on another learner's gradient."""
        for p, g in zip(self.params(), grads):
            p.grad = g.to(self.device, self.dtype).reshape(p.shape).clone()
        with no_lhw():
            torch.nn.utils.clip_grad_norm_(self.policy.parameters(), self.ppo.grad_clip)
            torch.nn.utils.clip_grad_norm_(self.critic.parameters(), self.ppo.grad_clip)
            self.ppo.actor_optimizer.step()
            self.ppo.critic_optimizer.step()

    @torch.no_grad()
    def near_kink(self, obs, act):
        """Per sample: the loss is within fp32 rounding of one of its kinks, where fp32 and float64 may take different branches.
        Either the float64 ratio lies within KINK_MARGIN of 1 +- clip (one such sample moves clip_frac by 1/B and the actor
        gradient by its whole contribution), or a ReLU pre-activation z of the differentiated passes (policy on the
        observations and on their mirror images, critic) lies within KINK_MARGIN * (|W| |x| + |b|) of zero (its unit's
        gradient for that sample is there or not)."""
        c = lambda t: t.to(self.device, self.dtype)
        obs, act = c(obs), c(act)
        lp = self.policy.distribution(obs).log_prob(act).sum(-1)
        olp = self.old_policy.distribution(obs).log_prob(act).sum(-1)
        near = ((lp - olp).exp().sub(1).abs() - self.ppo.clip).abs() < KINK_MARGIN
        passes = [(self.policy, self.policy.actor_layers, obs), (self.critic, self.critic.critic_layers, obs)]
        if self.mirror[0] is not None:
            passes.append((self.policy, self.policy.actor_layers, self.mirror[0](obs)))
        for net, layers, x in passes:
            x = (x - net.obs_mean) / net.obs_std
            for layer in layers:
                z = layer(x)
                scale = x.abs() @ layer.weight.abs().t() + layer.bias.abs()
                near |= (z.abs() < KINK_MARGIN * scale).any(-1)
                x = torch.relu(z)
        return near


def hyper_of(ppo):
    return dict(lr=ppo.lr, eps=ppo.eps, clip=ppo.clip, ent_coeff=ppo.ent_coeff, mirror_coeff=ppo.mirror_coeff,
                max_grad_norm=ppo.grad_clip)


def sym_of(env):
    return env if hasattr(env, "obs_mirror_clock_matrix") else None


# ---------------------------------------------------------------------------------------------------------------- the CUDA side
def adam_steps(ppo) -> int:
    if ppo._comm is not None:
        return ppo._comm.status()[0]
    return int(ppo.actor_optimizer.step_dev.item())


def preclip_norms(ppo):
    if ppo._comm is not None:
        return ppo._comm.status()[1]
    return float(ppo.actor_optimizer.total_norm().item()), float(ppo.critic_optimizer.total_norm().item())


def cuda_grads(ppo):
    """The raw gradient the exchange consumed, per parameter tensor: the clip + Adam kernels read ppo._flat_grad and write
    their clipped gradient elsewhere, so after the step it still holds the unclipped one."""
    sizes = [p.numel() for net in (ppo.policy, ppo.critic) for p in net.parameters()]
    return [g.clone() for g in torch.split(ppo._flat_grad.detach(), sizes)]


def ulp32(x):
    x = x.double().abs()
    return torch.where(x > 0, 2.0 ** (torch.floor(torch.log2(torch.clamp(x, min=1e-38))) - 23), torch.full_like(x, 2.0 ** -149))


def _rel(d, ref):
    r = float(ref)
    return float(d) / r if r > 0 else (0.0 if float(d) == 0 else float("inf"))


def compare_step(ppo, sh, sh_opt, ob, ab, rb, db, obs_mirr, act_mirr):
    """One re-synchronised optimiser step of the CUDA learner `ppo` and of the shadows; returns the errors of this step, each
    divided by its bound (<= 1 passes), plus diagnostics.  Under the adaptive schedule the shadows take the rate the device
    computed for this step, and the record holds it (lr0 -> lr1) with the rule's value for the learner's KL (lr_rule)."""
    from learninghumanoidwalking_b200.rl.schedule import adapt_lr
    adaptive = getattr(ppo, "schedule", "fixed") == "adaptive"
    flat0, m0, v0 = ppo._flat_param.clone(), ppo._flat_m.clone(), ppo._flat_v.clone()
    step0 = adam_steps(ppo)
    assert ppo.actor_optimizer.step_count == ppo.critic_optimizer.step_count == step0
    sh.load(flat0, m0, v0, step0, ppo.old_policy)
    near = int(sh.near_kink(ob, ab).sum())
    lr0 = ppo._comm.get_lr() if adaptive else ppo.lr
    out = ppo._update_step(ob, ab, rb, db, obs_mirr, act_mirr).double().cpu()
    torch.cuda.synchronize()
    assert adam_steps(ppo) == step0 + 1
    lr = ppo._comm.get_lr() if adaptive else ppo.lr
    for s in (sh, sh_opt):
        for opt in (s.ppo.actor_optimizer, s.ppo.critic_optimizer):
            opt.param_groups[0]["lr"] = lr
    g_cuda, n_cuda = cuda_grads(ppo), preclip_norms(ppo)
    ref, g_ref, n_ref = sh.step(ob, ab, rb, db)
    sh_opt.load(flat0, m0, v0, step0)
    sh_opt.optimise(g_cuda)
    e = dict(near=near, norms=n_cuda, norms_ref=n_ref, clipped=tuple(n > ppo.grad_clip for n in n_cuda), scalars=out.tolist())
    if adaptive:     # out[3] is the learner's float32 KL, widened exactly
        e.update(lr0=lr0, lr1=lr, kl=float(out[3]), kl_ref=ref[3], lr_rule=adapt_lr(lr0, float(out[3]), ppo.desired_kl))
    e["scalar"] = max(abs(float(out[k]) - ref[k]) / max(1.0, abs(ref[k])) for k in range(7)) / BOUNDS["scalar"]
    g_ref = [g.reshape(-1) for g in g_ref]
    l2 = [_rel((a.double() - b).norm(), b.norm()) for a, b in zip(g_cuda, g_ref)]
    e["grad_l2"] = max(l2) / BOUNDS["grad_l2"]
    e["grad_max"] = max(_rel((a.double() - b).abs().max(), b.abs().max()) for a, b in zip(g_cuda, g_ref)) / BOUNDS["grad_max"]
    e["grad_l2_per_tensor"] = [float(f"{x:.1e}") for x in l2]
    e["norm"] = max(abs(a - b) / b for a, b in zip(n_cuda, n_ref)) / BOUNDS["norm"]
    sizes = [p.numel() for p in sh.params()]
    seg = lambda t: torch.split(t.double().to(sh.device), sizes)
    mom = {sh: 0.0, sh_opt: 0.0}
    for name, mine in (("exp_avg", ppo._flat_m), ("exp_avg_sq", ppo._flat_v)):
        for ref_sh in (sh, sh_opt):
            for a, b in zip(seg(mine), seg(ref_sh.flat(name))):
                mom[ref_sh] = max(mom[ref_sh], _rel((a - b).norm(), b.norm()))
    e["moment"] = mom[sh_opt] / BOUNDS["moment"]
    e["moment_vs_shadow"] = mom[sh]
    p_new, p_opt, p_ref = ppo._flat_param.double().to(sh.device), sh_opt.flat("param"), sh.flat("param")
    allowed = ulp32(p_opt) + PARAM_LR * lr
    e["param"] = float(((p_new - p_opt).abs() / allowed).max()) / BOUNDS["param"]
    e["param_vs_shadow_lr"] = float((p_new - p_ref).abs().max()) / lr      # reported: S's own step, not bounded
    return e


def offset_mean_(policy, seed, scale=0.01):
    """Offset a policy's mean output by N(0, scale^2) per action, in place: by about a tenth of the action noise, so that a share
    of the ratios between this policy and an unmoved copy leaves the clip range."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    with torch.no_grad():
        b = policy.means.bias
        b.add_((scale * torch.randn(b.shape, generator=g, dtype=torch.float64)).to(b.device, b.dtype))


def reoffset_(old, policy, seed, scale):
    """old = policy with its mean output offset by N(0, scale^2) per action, in place (a captured graph keeps its addresses)."""
    with torch.no_grad():
        for q, p in zip(old.parameters(), policy.parameters()):
            q.copy_(p)
    offset_mean_(old, seed, scale)


def choose_desired_kl(kls, far):
    """desired_kl that puts every probed step with far[k] above 2 desired_kl and every other below desired_kl / 2, at the
    geometric middle of the gap."""
    hi = min(k for k, f in zip(kls, far) if f)
    lo = max(k for k, f in zip(kls, far) if not f)
    assert hi > 8 * lo > 0, f"the probed KLs do not straddle a factor-4 band with margin: {kls}"
    return float(np.sqrt(hi * lo))


def choose_max_norm(norms, regime):
    """max_grad_norm that puts every probed step in `regime` ("both" / "neither" / "actor" / "critic" clipped) with a factor-2
    margin; norms: [(actor, critic)] over the steps to come."""
    a, c = np.array([n[0] for n in norms]), np.array([n[1] for n in norms])
    if regime == "both":
        return float(0.5 * min(a.min(), c.min()))
    if regime == "neither":
        return float(2.0 * max(a.max(), c.max()))
    lo, hi = (a, c) if regime == "critic" else (c, a)      # "critic": only the critic's norm is above the bound
    assert 2 * lo.max() < hi.min(), f"no max_grad_norm clips the {regime} alone: {norms}"
    return float(np.sqrt(lo.max() * hi.min()))


def teacher_file(env):
    """A saved actor for `--imitate`: the trained jvrc_walk actor of tests/golden (no experiment.pkl: the identity by width), or
    for "h1" a 35-input actor with outputs of a trained policy's size, written next to an experiment.pkl naming h1 (the
    h1 -> h1_walk projector)."""
    if env == "jvrc_walk":
        return os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")
    assert env == "h1", env
    import pickle
    from learninghumanoidwalking_b200.rl.policies import Gaussian_FF_Actor, export_module
    d = os.path.join(tempfile.gettempdir(), "lhw_learner_local_error", "h1_teacher")
    os.makedirs(d, exist_ok=True)
    g = torch.Generator().manual_seed(123)
    actor = Gaussian_FF_Actor(35, 10)
    with torch.no_grad():
        for p in actor.parameters():
            p.copy_(torch.randn(p.shape, generator=g) / p.shape[-1] ** 0.5 if p.dim() > 1 else torch.zeros(p.shape))
    path = os.path.join(d, "actor_0.pt")
    torch.save(export_module(actor), path)
    with open(os.path.join(d, "experiment.pkl"), "wb") as f:
        pickle.dump(SimpleNamespace(env="h1"), f)
    return path


def per_step_case(model="jvrc_walk", B=21845, n_envs=4096, steps_per_env=44, steps=7, regime="critic", learn_std=False,
                  mirror=True, seed=0, hyper=None, imitate=None, imitate_coeff=2.0, kl_scales=None):
    """Build the CUDA learner on a sampled batch of `model`, choose max_grad_norm for `regime`, run `steps` re-synchronised steps
    through _update_step (3 eager warm-ups, then the captured graph).  LHW_* switches come from the caller's environment.
    imitate: the env of a teacher (teacher_file) to train with, at imitate_coeff; the shadows then carry its float64 copy.
    kl_scales: the adaptive schedule: before step k the old policy is the policy offset by kl_scales[k] (reoffset_), and
    desired_kl is chosen from a probe so that the far steps (the larger scale) decrease the rate and the others increase it.
    Returns (list of per-step error dicts, max_grad_norm)."""
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    h = dict(lr=2e-4, eps=1e-6, clip=0.15, entropy_coeff=0.01, mirror_coeff=0.3, std_dev=0.2)
    h.update(hyper or {})
    base = lambda: BatchedHumanoidEnv(n_envs, model=model, precision=32, seed=seed)
    env_fn = base
    if mirror:
        probe = base()
        r = probe.robot
        probe.close()
        env_fn = lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)
    args = SimpleNamespace(gamma=0.99, lam=0.95, lr=h["lr"], eps=h["eps"], entropy_coeff=h["entropy_coeff"], clip=h["clip"],
                           minibatch_size=B, epochs=1, max_traj_len=400, num_procs=n_envs, max_grad_norm=0.5,
                           mirror_coeff=h["mirror_coeff"] if mirror else 0.0, std_dev=h["std_dev"], learn_std=learn_std,
                           steps_per_env=steps_per_env, eval_batches=0, eval_at_start=False, logdir="/tmp/lhw_learner_local_error")
    if imitate is not None:
        args.imitate, args.imitate_coeff = teacher_file(imitate), imitate_coeff
    if kl_scales is not None:
        assert len(kl_scales) == steps
        args.schedule, args.desired_kl = "adaptive", 0.01     # desired_kl is chosen below
    ppo = PPO(env_fn, args, seed=seed)
    teach = dict(teacher=ppo.base_policy, projector=ppo.imitation_projector, imitate_coeff=ppo.imitate_coeff) \
        if imitate is not None else {}
    batch = ppo.sample_parallel_with_workers()
    obs, act = batch.states, batch.actions
    ret = batch.returns.contiguous()
    adv = ppo.normalize_advantages(ret, batch.values.contiguous(), from_rollout=True)
    n, C = obs.shape[0], B + 64 + B // 8         # C candidates per step: B samples and spares for the ill-conditioned ones
    assert n >= C * steps
    perm = torch.randperm(n, generator=torch.Generator().manual_seed(seed + 1))[:C * steps].view(steps, C).to(ppo.device)
    scale = [3.0 if k % 2 else 1.0 for k in range(steps)]      # larger advantages on every other step: more clipped ratios
    old = deepcopy(ppo.policy)
    offset_mean_(old, seed)
    sym = sym_of(ppo.env)
    probe = Shadow(ppo.policy, old, ppo.critic, hyper_of(ppo), sym, device=ppo.device, **teach)
    def first(cand, sh):
        i = cand[~sh.near_kink(obs[cand], act[cand])][:B]
        assert i.numel() == B, f"only {i.numel()} of {C} candidates are away from the loss's kinks"
        return i
    norms, kls = [], []
    for k, (c, s) in enumerate(zip(perm, scale)):
        if kl_scales is not None:
            reoffset_(probe.old_policy, probe.policy, seed + k, kl_scales[k])
        i = first(c, probe)
        out, _, n = probe.step(obs[i], act[i], ret[i], adv[i] * s)
        norms.append(n)
        kls.append(out[3])
    ppo.grad_clip = choose_max_norm(norms, regime)
    if kl_scales is not None:
        ppo.desired_kl = choose_desired_kl(kls, [x == max(kl_scales) for x in kl_scales])
    ppo.make_optimizers()
    offset_mean_(ppo.old_policy, seed)
    sh = Shadow(ppo.policy, ppo.old_policy, ppo.critic, hyper_of(ppo), sym, device=ppo.device, **teach)
    sh_opt = Shadow(ppo.policy, ppo.old_policy, ppo.critic, hyper_of(ppo), sym, device=ppo.device, **teach)
    obs_mirr = getattr(ppo.env, "mirror_clock_observation", None) if mirror else None
    act_mirr = getattr(ppo.env, "mirror_action", None) if mirror else None
    res = []
    for k, (cand, s) in enumerate(zip(perm, scale)):
        if kl_scales is not None:
            reoffset_(ppo.old_policy, ppo.policy, seed + k, kl_scales[k])
        # the minibatch skips the samples at a kink of the loss (Shadow.near_kink): there the two precisions may legitimately
        # take different branches, and one such sample moves a gradient far more than rounding does
        sh.load(ppo._flat_param, ppo._flat_m, ppo._flat_v, adam_steps(ppo), ppo.old_policy)
        i = first(cand, sh)
        assert i.numel() == B
        ob, ab, rb, db = ppo.gather_minibatch(obs, act, ret, (adv * s).contiguous(), i)
        e = compare_step(ppo, sh, sh_opt, ob, ab, rb, db, obs_mirr, act_mirr)
        e["graph"], e["B"], e["skipped"] = ppo._ug is not None, ob.shape[0], int(sh.near_kink(obs[cand], act[cand]).sum())
        if imitate is not None:   # the minibatch's taught samples (the projector's mask; all of them without one)
            e["taught"] = B if ppo.imitation_projector(ob)[1] is None else int(ppo.imitation_projector(ob)[1].sum())
        res.append(e)
    ppo.env.close()
    return res, ppo.grad_clip


# ---------------------------------------------------------------------------------------------------------- whole-iteration tier
def gae64(rewards, values, ended, boot, last_val, gamma, lam):
    """ppo_oracle.gae_rollout vectorised over environments (float64, time-major [T, N]): the backward recursion with the
    trajectory cut where ended[t] (bootstrap boot[t]) and the open tail bootstrapped with last_val."""
    r, v, b = (torch.as_tensor(x, dtype=torch.float64) for x in (rewards, values, boot))
    e = torch.as_tensor(ended).bool()
    T = r.shape[0]
    ret = torch.empty_like(r)
    g = torch.zeros_like(r[0])
    nxt = torch.as_tensor(last_val, dtype=torch.float64).to(r.device).clone()
    for t in range(T - 1, -1, -1):
        nv = torch.where(e[t], b[t], nxt)
        g = torch.where(e[t], torch.zeros_like(g), g)
        g = r[t] + gamma * nv - v[t] + gamma * lam * g
        ret[t] = g + v[t]
        nxt = v[t]
    return ret


def iteration_reference(ppo, state0, sym, obs_mirr_present=True, perturb=0.0, perturb_seed=1):
    """The float64 learner phase of the iteration the worker's buffer holds, from its own inputs; state0: (flat, m, v, step)
    of the CUDA learner before the iteration.  perturb > 0: the starting parameters multiplied by 1 + U(-perturb, perturb)
    (the control: how far float64 runs that start within fp32 rounding of each other drift apart).
    Returns dict(returns, adv, stats, flat, m, v, idx)."""
    buf = ppo.workers[0]._buf
    dev = ppo.device
    ret = gae64(buf.rewards, buf.values, buf.ended, buf.boot, buf.last_val, float(ppo.gamma), float(ppo.lam))
    envmaj = lambda x: x.transpose(0, 1).reshape(buf.T * buf.N, *x.shape[2:])
    ret_f, val_f = envmaj(ret).unsqueeze(-1), envmaj(buf.values.double()).unsqueeze(-1)
    d = ret_f - val_f
    adv = (d - d.mean()) / (d.std() + ppo.eps)
    obs, act = envmaj(buf.states), envmaj(buf.actions)
    sh = Shadow(ppo.policy, ppo.policy, ppo.critic, hyper_of(ppo), sym, device=dev)
    flat, m, v, step = state0
    if perturb:
        g = torch.Generator(device="cpu").manual_seed(perturb_seed)
        flat = flat.double() * (1 + perturb * (2 * torch.rand(flat.shape, generator=g, dtype=torch.float64) - 1)).to(flat.device)
    sh.load(flat, m, v, step)
    with torch.no_grad():       # old_policy = the policy at the start of the iteration
        for q, p in zip(sh.old_policy.parameters(), sh.policy.parameters()):
            q.copy_(p)
    if not obs_mirr_present:
        sh.mirror = (None, None)
    stats, idxs = [], []
    n = obs.shape[0]
    for epoch in range(ppo.epochs):
        for idx in ppo.minibatch_indices(n, ppo.iteration_count, epoch):
            idxs.append(idx)
            stats.append(sh.step(obs[idx], act[idx], ret_f[idx], adv[idx])[0])
    return dict(returns=ret, adv=adv, stats=np.mean(np.array(stats), axis=0), flat=sh.flat("param"), m=sh.flat("exp_avg"),
                v=sh.flat("exp_avg_sq"), idx=idxs)


def run_iterations(model="jvrc_walk", n_envs=4096, steps=400, n_itr=2, seed=0, **over):
    """PPO.train at run_experiment.py's default learner flags, one iteration per call (graphs persist across calls), each
    iteration compared with its float64 recomputation.  Returns a list of per-iteration dicts of errors."""
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(n_envs, model=model, precision=32, seed=seed, max_traj_len=steps)
    probe = base()
    r = probe.robot
    mirror = hasattr(r, "mirrored_obs")
    probe.close()
    env_fn = (lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)) \
        if mirror else base
    a = dict(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=64, epochs=3,
             max_traj_len=steps, num_procs=n_envs, max_grad_norm=0.5, mirror_coeff=0.4, std_dev=0.223, learn_std=False,
             steps_per_env=None, minibatch_scale="auto", eval_batches=0, eval_at_start=False, eval_freq=100,
             logdir="/tmp/lhw_learner_local_error")
    a.update(over)
    ppo = PPO(env_fn, SimpleNamespace(**a), seed=seed)
    ppo.make_optimizers()
    # the policy moves in place after make_optimizers(), as PPO.restore moves it: the first iteration's old_policy sync then
    # has work to do (in a straight run from make_optimizers() old_policy is already the policy, and a misplaced sync is a no-op)
    offset_mean_(ppo.policy, seed)
    sym = sym_of(ppo.env)
    seen = {}
    real_norm, real_gather = ppo.normalize_advantages, ppo.gather_minibatch

    def norm_spy(returns, values, from_rollout=False):
        out = real_norm(returns, values, from_rollout=from_rollout)
        seen["adv"], seen["ret"], seen["idx"], seen["gather_ok"] = out.clone(), returns.clone(), [], True
        return out

    def gather_spy(o, a_, r_, d_, idx):
        res = real_gather(o, a_, r_, d_, idx)
        seen["idx"].append(idx.clone())
        seen["gather_ok"] &= all(torch.equal(x, y[idx]) for x, y in zip(res, (o, a_, r_, d_)))
        return res
    ppo.normalize_advantages, ppo.gather_minibatch = norm_spy, gather_spy
    out = []
    for itr in range(n_itr):
        state0 = (ppo._flat_param.clone(), ppo._flat_m.clone(), ppo._flat_v.clone(), adam_steps(ppo))
        with switches({"LHW_TENSORBOARD": "0"}):
            log = ppo.train(None, itr + 1, verbose=False, start_itr=itr)[-1]
        ref = iteration_reference(ppo, state0, sym, obs_mirr_present=mirror and bool(ppo.mirror_coeff))
        # two controls: how far one free-running float64 run drifts is itself a random quantity
        ctls = [iteration_reference(ppo, state0, sym, obs_mirr_present=mirror and bool(ppo.mirror_coeff), perturb=2.0 ** -24,
                                    perturb_seed=k) for k in (1, 2)]
        buf = ppo.workers[0]._buf
        ret_ref = ref["returns"]
        # lhw_gae takes gamma and lambda as float: the float64 recursion with the fp32-rounded coefficients isolates that cost
        ret_c = gae64(buf.rewards, buf.values, buf.ended, buf.boot, buf.last_val, float(np.float32(ppo.gamma)), float(np.float32(ppo.lam)))
        e_coef = float(((ret_c - ret_ref).abs() / ret_ref.abs().clamp(min=1.0)).max())
        e = dict(itr=itr, steps=len(ref["idx"]), graph=None if ppo._ug is None else id(ppo._ug[0]))
        e["returns"] = float(((buf.returns.double() - ret_ref).abs() / ret_ref.abs().clamp(min=1.0)).max())
        e["returns_vs_f32_coeffs"] = float(((buf.returns.double() - ret_c).abs() / ret_c.abs().clamp(min=1.0)).max())
        e["returns_coeff_cost"] = e_coef
        e["adv"] = float((seen["adv"].double() - ref["adv"]).abs().max())
        e["idx_equal"] = len(seen["idx"]) == len(ref["idx"]) and all(torch.equal(x, y) for x, y in zip(seen["idx"], ref["idx"]))
        e["gather_equal"] = bool(seen["gather_ok"])
        got = [log[k] for k in ("actor_loss", "entropy", "critic_loss", "kl", "mirror")] + [log["clip_frac"]]
        want = [ref["stats"][k] for k in (0, 1, 2, 3, 4, 6)]
        e["stats"] = [abs(x - y) / max(1.0, abs(y)) for x, y in zip(got, want)]
        e["stats_got"], e["stats_ref"] = got, want
        sizes = [p.numel() for p in list(ppo.policy.parameters()) + list(ppo.critic.parameters())]
        per_tensor = lambda a, b: max(_rel((x.double() - y).norm(), y.norm()) for x, y in zip(torch.split(a, sizes), torch.split(b, sizes)))
        for name, mine, key in (("exp_avg", ppo._flat_m, "m"), ("exp_avg_sq", ppo._flat_v, "v")):
            e[name] = per_tensor(mine, ref[key])
            e["control_" + name] = max(per_tensor(ctl[key], ref[key]) for ctl in ctls)
        e["control_param_step"] = max(_rel((x - y).norm(), (y - z.double()).norm()) for ctl in ctls for x, y, z in
                                      zip(torch.split(ctl["flat"], sizes), torch.split(ref["flat"], sizes), torch.split(state0[0], sizes)))
        e["control_stats"] = [max(abs(c["stats"][k] - y) / max(1.0, abs(y)) for c in ctls) for k, y in enumerate(ref["stats"])]
        e["param_step"] = max(_rel((x.double() - y).norm(), (y - z.double()).norm()) for x, y, z in
                              zip(torch.split(ppo._flat_param, sizes), torch.split(ref["flat"], sizes), torch.split(state0[0], sizes)))
        out.append(e)
    ppo.env.close()
    return out


# ------------------------------------------------------------------------------------------------------------------ reporting
def table_rows(name, res):
    rows = []
    for q in ("scalar", "grad_l2", "grad_max", "norm", "moment", "param"):
        v = np.array([e[q] * BOUNDS[q] for e in res])
        rows.append(f"| {name} | {q} | {np.median(v):.1e} | {np.percentile(v, 99):.1e} | {v.max():.1e} | {BOUNDS[q]:.0e} |")
    return rows


CASES = {
    # name: (per_step_case keywords, LHW_* switches)
    "jvrc_walk_B21845": (dict(model="jvrc_walk", B=21845, regime="critic"), {}),
    "jvrc_walk_B300": (dict(model="jvrc_walk", B=300, regime="both", n_envs=1024, steps_per_env=8), {}),
    "jvrc_walk_B1": (dict(model="jvrc_walk", B=1, regime="neither", n_envs=64, steps_per_env=8), {}),
    "jvrc_step_B21845": (dict(model="jvrc_step", B=21845, regime="both"), {}),
    "h1_B21845": (dict(model="h1", B=21845, regime="neither", mirror=False), {}),
    "learn_std_B4097": (dict(model="jvrc_walk", B=4097, regime="critic", learn_std=True, n_envs=1024, steps_per_env=32), {}),
    "fallbacks_B4097": (dict(model="jvrc_walk", B=4097, regime="both", n_envs=1024, steps_per_env=32),
                        {"LHW_FUSED_LOSS": "0", "LHW_WGRAD_KERNEL": "0"}),
    "baseline_exchange_B4097": (dict(model="jvrc_walk", B=4097, regime="critic", n_envs=1024, steps_per_env=32),
                                {"LHW_FUSED_EXCHANGE": "0"}),
}


# opt-in (--imitation): the learner with a teacher, the jvrc_walk identity pair and h1 -> h1_walk (the standing projector)
IMITATION_CASES = {
    "imitate_jvrc_walk_B21845": (dict(model="jvrc_walk", B=21845, regime="both", imitate="jvrc_walk"), {}),
    "imitate_h1_to_h1_walk_B21845": (dict(model="h1_walk", B=21845, regime="neither", imitate="h1"), {}),
}


# opt-in (--adaptive): `--schedule adaptive`; the old policy alternates far / near, so the rate goes down and up again
ADAPTIVE_CASES = {
    "adaptive_jvrc_walk_B21845": (dict(model="jvrc_walk", B=21845, regime="both",
                                       kl_scales=[0.03, 0.003, 0.03, 0.003, 0.003, 0.03, 0.003]), {}),
    "adaptive_learn_std_B4097": (dict(model="jvrc_walk", B=4097, regime="both", learn_std=True, n_envs=1024, steps_per_env=32,
                                      kl_scales=[0.03, 0.003, 0.03, 0.003, 0.003, 0.03, 0.003]), {}),
}


@contextlib.contextmanager
def switches(env):
    old = {k: os.environ.get(k) for k in env}
    os.environ.update(env)
    try:
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def rehearse():
    """The float64 parts on the CPU at a tiny size: gae64 against ppo_oracle.gae_rollout, and a shadow step under the guard
    against the same step in float32 (both through update_actor_critic's torch branch)."""
    from learninghumanoidwalking_b200.rl.policies import FF_V, Gaussian_FF_Actor
    from oracle.ppo_oracle import gae_rollout
    rng = np.random.RandomState(0)
    T, N = 30, 9
    rew, val = rng.uniform(-1, 1, (T, N)), rng.uniform(-2, 2, (T, N))
    ended = (rng.rand(T, N) < 0.1).astype(np.int32)
    boot, last = rng.uniform(-2, 2, (T, N)) * (rng.rand(T, N) < 0.5), rng.uniform(-2, 2, N)
    gerr = float(np.abs(gae64(rew, val, ended, boot, last, 0.99, 0.95).numpy() - gae_rollout(rew, val, ended, boot, last, 0.99, 0.95)).max())
    torch.manual_seed(0)
    pol, cri = Gaussian_FF_Actor(37, 12, init_std=0.2), FF_V(37)
    old = deepcopy(pol)
    offset_mean_(old, 0)
    hyper = dict(lr=2e-4, eps=1e-6, clip=0.15, ent_coeff=0.01, mirror_coeff=0.0, max_grad_norm=0.05)
    s64, s32 = Shadow(pol, old, cri, hyper), Shadow(pol, old, cri, hyper, dtype=torch.float32)
    B = 64
    obs, act = torch.randn(B, 37), torch.randn(B, 12) * 0.2
    ret, adv = torch.randn(B, 1), torch.randn(B, 1)
    out64, g64, n64 = s64.step(obs, act, ret, adv)
    out32, g32, n32 = s32.step(obs, act, ret, adv)
    serr = max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(out32, out64))
    nerr = max(abs(a - b) / b for a, b in zip(n32, n64))
    return dict(gae=gerr, scalars=serr, norms=nerr, grads=len(g64))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--rehearse", action="store_true", help="the float64 parts on the CPU at a tiny size")
    ap.add_argument("--cases", default=",".join(CASES))
    ap.add_argument("--iterations", default="jvrc_walk,h1", help="whole-iteration tier variants ('' skips it)")
    ap.add_argument("--imitation", action="store_true", help="also the per-step cases with a teacher (IMITATION_CASES)")
    ap.add_argument("--adaptive", action="store_true", help="also the per-step cases of the adaptive schedule (ADAPTIVE_CASES)")
    args = ap.parse_args()
    if args.rehearse:
        print(rehearse())
        return
    print("| case | quantity | median | p99 | max | bound |\n|---|---|---|---|---|---|")
    notes = []
    names = [c for c in args.cases.split(",") if c] + (list(IMITATION_CASES) if args.imitation else []) \
        + (list(ADAPTIVE_CASES) if args.adaptive else [])
    for name in names:
        kw, env = {**CASES, **IMITATION_CASES, **ADAPTIVE_CASES}[name]
        t0 = time.time()
        with switches(env):
            res, mn = per_step_case(**kw)
        print("\n".join(table_rows(name, res)), f"({time.time() - t0:.0f} s)", flush=True)
        notes.append(f"{name}: max_grad_norm {mn:.4g}, norms {[tuple(round(x, 5) for x in e['norms']) for e in res]}, clipped "
                     f"{[e['clipped'] for e in res]}, clip_frac {[round(e['scalars'][6], 4) for e in res]}, skipped {[e['skipped'] for e in res]}, "
                     f"near {[e['near'] for e in res]}, graph {[e['graph'] for e in res]}, "
                     f"param vs S / lr {max(e['param_vs_shadow_lr'] for e in res):.2e}, "
                     f"moments vs S {max(e['moment_vs_shadow'] for e in res):.1e}, "
                     f"grad l2 per tensor {[e['grad_l2_per_tensor'] for e in res]}"
                     + (", kl " + str([round(e["kl"], 6) for e in res]) + ", lr " + str([e["lr1"] for e in res]) if "lr1" in res[0] else ""))
    print("\n".join(notes), flush=True)
    for name in [c for c in args.iterations.split(",") if c]:
        kw = dict(model="jvrc_walk") if name == "jvrc_walk" else dict(model="h1", n_envs=1024, steps=100)
        t0 = time.time()
        for e in run_iterations(**kw):
            print(name, {k: (v if not isinstance(v, float) else float(f"{v:.3e}")) for k, v in e.items()}, flush=True)
        print(f"{name}: {time.time() - t0:.0f} s", flush=True)


if __name__ == "__main__":
    main()
