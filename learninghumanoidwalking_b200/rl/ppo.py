"""PPO (clip objective) with the reference's learner API (rl/algos/ppo.py): PPO(env_fn, args, seed),
.train(env_fn, n_itr), .sample_parallel_with_workers(deterministic) -> BatchData,
.update_actor_critic(obs, act, ret, adv, mask, mirror_observation, mirror_action) -> 7-tuple,
.actor_optimizer / .critic_optimizer.

What changes underneath (the hot path of BASELINE.json):
  * sampling: one DeviceRolloutWorker over a BatchedHumanoidEnv with num_procs environments (no Ray, no host
    round trip inside a control step);
  * GAE, advantage normalisation, minibatch gathers and clip+Adam are CUDA launches on device tensors;
  * multi-GPU: env copies shard by index across ranks; ONE NCCL all-reduce of the flat (actor+critic) gradient
    per optimiser step, clipping computed on the reduced gradient, advantage statistics all-reduced (2 doubles).
The loss graph itself stays torch autograd + cuBLAS (north-star: "the small MLP policy left to cuBLAS").
"""
from __future__ import annotations

import datetime
import time
from copy import deepcopy
from pathlib import Path

import torch
import torch.distributed as dist
from torch.nn import functional as F

from .. import _lib
from .optim import FusedClipAdam
from . import schedule, snapshot
from .policies import FF_V, Gaussian_FF_Actor
from .snapshot import SnapshotError, plain_args
from .storage import BatchData
from .workers import DeviceRolloutWorker

# per-env tensors an env may own beside its records (None when off), which a snapshot shard then holds too: the name, what it is
# and the training flag that turns it on
_PER_ENV = {"stair_level": ("stair levels", "--stair-curriculum"), "action_delay": ("action delays", "--action-delay"),
            "payload": ("payloads", "--payload-mass"), "motor_strength": ("motor strengths", "--motor-strength"),
            "sensor": ("sensor errors", "--sensor-noise / --sensor-bias")}


class _FusedPPOLoss(torch.autograd.Function):
    """The loss tail of update_actor_critic (rl/algos/ppo.py:302-386) as ONE launch (csrc/ppo_kernels.cu: ppo_loss_kernel): the 7
    scalars and d total / d (policy mean, mirrored actions, values) come out of the forward pass; backward hands those gradients
    to autograd, which then only runs the MLP backward passes (cuBLAS)."""

    @staticmethod
    def forward(ctx, mu, values, mirr, old_mu, act, adv, ret, stds, clip, mirror_coeff, ent_coeff, bufs, imitation=None):
        g_mu, g_mirr, g_val, partials, ticket, out8 = bufs
        if imitation is None:
            _lib.ops().ppo_loss(mu, old_mu, act, adv, ret, values, mirr, stds, clip, mirror_coeff, ent_coeff, g_mu,
                                g_mirr if mirr is not None else None, g_val, partials, ticket, out8)
        else:   # (teacher actions [B,A], mask [B,1] or None, imitate_coeff): the imitation term in the same launch
            teacher_mu, imask, imitate_coeff = imitation
            _lib.ops().ppo_loss_imitation(mu, old_mu, act, adv, ret, values, mirr, stds, teacher_mu, imask, clip, mirror_coeff,
                                          ent_coeff, imitate_coeff, g_mu, g_mirr if mirr is not None else None, g_val, partials,
                                          ticket, out8)
        ctx.bufs, ctx.has_mirr = (g_mu, g_mirr, g_val), mirr is not None
        return out8[7]

    @staticmethod
    def backward(ctx, gout):
        g_mu, g_mirr, g_val = ctx.bufs
        return (g_mu * gout, g_val * gout, (g_mirr * gout) if ctx.has_mirr else None) + (None,) * 10


def get_worker_seed(master_seed: int, worker_id: int, offset: int = 0) -> int:
    """rl/utils/seeding.py:34-52 (the rank plays the worker's role)."""
    return (master_seed * 1_000_003 + offset * 10_007 + worker_id) % (2 ** 32 - 1)


class PPO:
    def __init__(self, env_fn, args, seed=None):
        self.seed = seed
        self.gamma, self.lam, self.lr, self.eps = args.gamma, args.lam, args.lr, args.eps
        self.ent_coeff, self.clip = args.entropy_coeff, args.clip
        self.minibatch_size, self.epochs = args.minibatch_size, args.epochs
        self.max_traj_len, self.n_proc = args.max_traj_len, args.num_procs
        self.grad_clip, self.mirror_coeff = args.max_grad_norm, args.mirror_coeff
        self.eval_freq = getattr(args, "eval_freq", 100)
        self.eval_batches = getattr(args, "eval_batches", 5)     # evaluate(num_batches=5) in the reference
        self.eval_at_start = getattr(args, "eval_at_start", True)  # the reference evaluates (and checkpoints) at iteration 0
        self.imitate_coeff = getattr(args, "imitate_coeff", 0.0)
        # `--schedule adaptive`: the KL-adaptive rate of DESIGN.md §7.3, held in device memory by the fused exchange
        self.schedule, self.desired_kl = schedule.schedule_of(args)
        schedule.check(self.schedule, self.desired_kl)
        # opt-in: TF32 tensor-core GEMMs for the MLPs (the reference trains in fp32 with torch's default allow_tf32 = False, and
        # so does this build unless asked otherwise; at minibatches >= 32k the update is GEMM bound)
        if getattr(args, "tf32", False):
            torch.backends.cuda.matmul.allow_tf32 = True
        if getattr(args, "recurrent", False):
            raise NotImplementedError("recurrent policies are outside the accelerated path (SURVEY.md §2 row 5)")
        self.recurrent = False
        self.steps_per_env = getattr(args, "steps_per_env", None) or self.max_traj_len
        self.total_steps, self.iteration_count = 0, 0
        self.save_path = Path(getattr(args, "logdir", "/tmp/lhw_b200_logs"))
        # opt-in (`train --snapshot`): the whole training state at every checkpoint point, for `run_experiment.py resume`
        self.write_snapshots = bool(getattr(args, "snapshot", False))
        self._run_args = plain_args(args)
        self._elapsed0 = 0.0                    # training time of the run before a restore()
        self.world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
        self.rank = dist.get_rank() if self.world > 1 else 0

        if not torch.cuda.is_available():
            raise _lib.LhwError("PPO needs a CUDA device (no CPU fallback on the hot path)")
        env = env_fn()
        self.env = env
        self.device = env.device
        obs_dim, action_dim = env.observation_space.shape[0], env.action_space.shape[0]
        # every rank builds identical initial weights (same seed), like N workers deep-copying one template
        if seed is not None:
            torch.manual_seed(seed)
        policy = Gaussian_FF_Actor(obs_dim, action_dim, init_std=args.std_dev, learn_std=getattr(args, "learn_std", False))
        critic = FF_V(obs_dim)
        with torch.no_grad():   # fixed normalisation from the env (rl/algos/ppo.py:94-113)
            policy.obs_mean = torch.tensor(env.obs_mean, dtype=torch.float32)
            policy.obs_std = torch.tensor(env.obs_std, dtype=torch.float32)
            critic.obs_mean, critic.obs_std = policy.obs_mean, policy.obs_std
        self.obs_rms = None
        self.policy = policy.to(self.device)
        self.critic = critic.to(self.device)
        self.old_policy = deepcopy(self.policy)
        self.base_policy, self.imitation_projector = None, None
        if getattr(args, "imitate", None):
            # the teacher (rl/imitation.py): every rank holds its own frozen copy; its parameters stay out of the flat buffer
            from . import imitation
            teacher, self.imitate_env, self.imitation_projector = imitation.check_teacher(
                args.imitate, self._inner_env().model_name, getattr(args, "imitate_env", None))
            self.base_policy = imitation.to_device(teacher, self.device)
        self.env_fn = env_fn
        wseed = get_worker_seed(seed if seed is not None else 0, self.rank)
        self.workers = [DeviceRolloutWorker(env, self.policy, self.critic, seed=wseed, worker_id=self.rank)]
        self.batch_size = env.num_envs * self.steps_per_env
        # `minibatch_size` counts this rank's samples.  minibatch_scale="auto" (run_experiment.py's default) keeps the
        # reference's number of optimiser steps per iteration instead of its absolute minibatch: the reference's default
        # geometry is 12 workers x 400 steps = 4800 samples in minibatches of 64 (225 updates per iteration over 3 epochs,
        # run_experiment.py:159-172); with N device environments the batch is N x steps_per_env, and 64-sample minibatches
        # would mean tens of thousands of launch-bound updates per iteration.  The minibatch grows with the batch.
        if getattr(args, "minibatch_scale", "off") == "auto" and self.batch_size > 12 * 400:
            self.minibatch_size = max(self.minibatch_size, int(round(self.minibatch_size * self.batch_size / (12 * 400))))
        if self.world > 1:
            # every rank must issue the same number of gradient exchanges per iteration: equal shards only
            cnt = torch.tensor([env.num_envs, -env.num_envs], device=self.device)
            dist.all_reduce(cnt, op=dist.ReduceOp.MAX)
            if int(cnt[0]) != -int(cnt[1]):
                raise ValueError(f"ranks hold different numbers of environments ({-int(cnt[1])}..{int(cnt[0])}): "
                                 "num_procs must be a multiple of the world size")
        self.actor_optimizer = self.critic_optimizer = None
        self._comm = None
        L = _lib.lib()
        self._adv_stats = torch.zeros(L.lhw_adv_stats_words(), dtype=torch.float64, device=self.device)
        self._mb = None
        self._ug, self._ug_calls = None, 0      # CUDA graph of one optimiser step (see _update_step)
        self._best_eval = float("-inf")         # ModelCheckpointer._best_metric (rl/utils/checkpointer.py:33)

    def load_pretrained(self, actor, critic):
        """`--continued` (rl/algos/ppo.py:69-82): take the weights and the embedded observation normalisation of a saved
        actor / critic pair (this build's or a reference checkout's — same state-dict keys); like the reference, the action
        noise `stds` is NOT restored but re-initialised from `--std-dev`, and neither optimiser state nor the iteration
        counter come back.  In place: captured graphs and the flat parameter buffer keep their addresses."""
        with torch.no_grad():
            for mine, theirs in ((self.policy, actor), (self.critic, critic)):
                sd = {k: v for k, v in theirs.state_dict().items() if k != "stds"}
                missing, unexpected = mine.load_state_dict(sd, strict=False)
                if unexpected or [k for k in missing if k != "stds"]:
                    raise ValueError(f"checkpoint does not fit the network: missing {missing}, unexpected {unexpected}")
                for name in ("obs_mean", "obs_std"):
                    v = getattr(theirs, name, None)
                    if torch.is_tensor(v):
                        getattr(mine, name).copy_(v.to(self.device, torch.float32))
            self.old_policy.load_state_dict(self.policy.state_dict())
            self.old_policy.obs_mean.copy_(self.policy.obs_mean)
            self.old_policy.obs_std.copy_(self.policy.obs_std)

    # ------------------------------------------------------------------ snapshots (rl/snapshot.py): resume a run bit for bit
    def _inner_env(self):
        """The batched env itself, not a SymmetricEnv wrapper around it (attribute writes must reach the env)."""
        return self.env.__dict__.get("env", self.env)

    def _fused_optimizers(self):
        a_opt, c_opt = self.actor_optimizer, self.critic_optimizer
        if not (isinstance(a_opt, FusedClipAdam) and isinstance(c_opt, FusedClipAdam)):
            raise SnapshotError("snapshots cover the optimisers of make_optimizers() (FusedClipAdam over the flat buffer) only")
        return a_opt, c_opt

    def snapshot_learner(self, itr: int, elapsed: float) -> dict:
        """The learner's part of the snapshot at the end of iteration `itr`: identical on every rank, written by rank 0."""
        a_opt, c_opt = self._fused_optimizers()
        if self._comm is not None:      # the fused exchange keeps one Adam step number for both networks in device memory
            dev = [self._comm.status()[0]] * 2
        else:
            dev = [int(a_opt.step_dev.item()), int(c_opt.step_dev.item())]
        cpu = lambda t: t.detach().cpu().clone()
        return dict(format=snapshot.FORMAT, itr=int(itr), world=self.world, args=self._run_args,
                    flat_param=cpu(self._flat_param), exp_avg=cpu(self._flat_m), exp_avg_sq=cpu(self._flat_v),
                    step_count=[a_opt.step_count, c_opt.step_count], adam_step_dev=dev,
                    obs_norm={f"{net}.{name}": cpu(getattr(getattr(self, net), name))
                              for net in ("policy", "critic") for name in ("obs_mean", "obs_std")},
                    best_eval=float(self._best_eval), total_steps=int(self.total_steps), elapsed=float(elapsed),
                    **self._schedule_state())

    def _schedule_state(self) -> dict:
        """The adaptive schedule's device rate (its float64 bits) for a snapshot; nothing under the fixed schedule."""
        if getattr(self, "schedule", "fixed") != "adaptive":
            return {}
        return dict(adaptive_lr=torch.tensor([self._comm.get_lr()], dtype=torch.float64))

    def snapshot_shard(self, itr: int) -> dict:
        """This rank's part of the snapshot: its environments' records and its sampler's state."""
        env = self._inner_env()
        return dict(format=snapshot.FORMAT, itr=int(itr), rank=self.rank, world=self.world, first_env_id=env.first_env_id,
                    num_envs=env.num_envs, model=env.model_name, precision=env.precision, seed=env.seed,
                    state_r=env.state_r.cpu(), state_i=env.state_i.cpu(), fresh=bool(env._fresh),
                    worker=self.workers[0].state_dict(), cpu_rng=torch.get_rng_state(),
                    **{name: getattr(env, name).cpu() for name in _PER_ENV if getattr(env, name, None) is not None})

    def restore(self, run_dir) -> int:
        """Load the last complete snapshot of `run_dir` into this freshly built PPO and its environment and return the iteration
        k it was taken at: `train(env_fn, n_itr, start_itr=k + 1)` then continues the run bit for bit.  A snapshot of another
        world size, num_procs, env, precision, shard or format is refused with a SnapshotError before anything is loaded.
        Runs make_optimizers() first if it has not run yet (it re-homes the parameters); captured graphs keep their addresses:
        everything is copied in place."""
        env = self._inner_env()
        _, learner, shard = snapshot.load(run_dir, self.rank, self.world,
                                          dict(env=env.model_name, precision=env.precision, num_procs=self.n_proc))
        for key, mine in (("first_env_id", env.first_env_id), ("num_envs", env.num_envs), ("seed", env.seed)):
            if shard.get(key) != mine:
                raise SnapshotError(f"{key} mismatch: the rank-{self.rank} shard has {key}={shard.get(key)}, this run has {mine}")
        if self.actor_optimizer is None:
            self.make_optimizers()
        a_opt, c_opt = self._fused_optimizers()
        for name, have, want in (("flat_param", learner["flat_param"], self._flat_param), ("exp_avg", learner["exp_avg"], self._flat_m),
                                 ("exp_avg_sq", learner["exp_avg_sq"], self._flat_v), ("state_r", shard["state_r"], env.state_r),
                                 ("state_i", shard["state_i"], env.state_i)):
            if have.shape != want.shape or have.dtype != want.dtype:
                raise SnapshotError(f"{name} of the snapshot is {tuple(have.shape)} {have.dtype}, this run has "
                                    f"{tuple(want.shape)} {want.dtype}")
        per_env = {name: getattr(env, name) for name in _PER_ENV if getattr(env, name, None) is not None}
        for name, mine in per_env.items():
            if name not in shard:
                raise SnapshotError(f"the snapshot holds no {_PER_ENV[name][0]} (was it written by a run without {_PER_ENV[name][1]}?)")
            if shard[name].shape != mine.shape or shard[name].dtype != mine.dtype:
                raise SnapshotError(f"{name} of the snapshot is {tuple(shard[name].shape)} {shard[name].dtype}, "
                                    f"this run has {tuple(mine.shape)} {mine.dtype}")
        with torch.no_grad():
            self._flat_param.copy_(learner["flat_param"])
            self._flat_m.copy_(learner["exp_avg"])
            self._flat_v.copy_(learner["exp_avg_sq"])
            for key, v in learner["obs_norm"].items():
                net, name = key.split(".")
                getattr(getattr(self, net), name).copy_(v)
            env.state_r.copy_(shard["state_r"])
            env.state_i.copy_(shard["state_i"])
            for name, mine in per_env.items():
                mine.copy_(shard[name])
        env._fresh = bool(shard["fresh"])
        a_opt.step_count, c_opt.step_count = learner["step_count"]
        if getattr(self, "schedule", "fixed") == "adaptive":
            if "adaptive_lr" not in learner:
                raise SnapshotError("the snapshot holds no learning rate of the adaptive schedule (was it written by a fixed-rate run?)")
            self._comm.set_lr(float(learner["adaptive_lr"][0]))
        if self._comm is not None:
            self._comm.set_step(learner["adam_step_dev"][0])
        else:
            a_opt.step_dev.fill_(learner["adam_step_dev"][0])
            c_opt.step_dev.fill_(learner["adam_step_dev"][1])
        self.workers[0].load_state_dict(shard["worker"])
        self._best_eval, self.total_steps = learner["best_eval"], learner["total_steps"]
        self._elapsed0 = learner["elapsed"]
        self.iteration_count = learner["itr"]
        torch.set_rng_state(shard["cpu_rng"])
        torch.cuda.synchronize(self.device)
        return learner["itr"]

    # ------------------------------------------------------------------ sampling (rl/algos/ppo.py:215-297)
    def sample_parallel_with_workers(self, deterministic=False) -> BatchData:
        w = self.workers[0]
        w.sync_state(iteration_count=self.iteration_count)
        return w.sample(self.gamma, self.lam, self.steps_per_env, self.max_traj_len, deterministic)

    # ------------------------------------------------------------------ one optimiser step (rl/algos/ppo.py:299-406)
    def _fused_loss_ok(self, obs_batch, mask) -> bool:
        import os
        return (os.environ.get("LHW_FUSED_LOSS", "1") != "0" and obs_batch.is_cuda and isinstance(mask, (int, float)) and mask == 1
                and not getattr(self.policy, "learn_std", False) and isinstance(self.policy, Gaussian_FF_Actor)
                and (self.imitate_coeff == 0.0 or getattr(self, "base_policy", None) is not None))

    def _loss_fused(self, obs_batch, action_batch, return_batch, advantage_batch, mirror_observation, mirror_action):
        """total loss (with the backward graph attached) and the 7 scalars, the elementwise part in one launch."""
        B, A = action_batch.shape
        bufs = getattr(self, "_loss_bufs", None)
        if bufs is None or bufs[0].shape != (B, A):
            f32 = dict(dtype=torch.float32, device=obs_batch.device)
            bufs = self._loss_bufs = (torch.empty(B, A, **f32), torch.empty(B, A, **f32), torch.empty(B, 1, **f32),
                                      torch.zeros(_lib.lib().lhw_ppo_loss_partial_words(B), dtype=torch.float64, device=obs_batch.device),
                                      torch.zeros(1, dtype=torch.int32, device=obs_batch.device), torch.zeros(8, **f32))
        mirr = None
        if mirror_observation is not None and mirror_action is not None:
            # the policy on the observations and on their mirror images in ONE pass (twice the rows per GEMM, half the launches)
            both = self.policy(torch.cat((obs_batch, mirror_observation(obs_batch)), 0), deterministic=True)
            mu = both[:B]
            mirr = mirror_action(both[B:]).contiguous()
        else:
            mu = self.policy(obs_batch, deterministic=True)
        with torch.no_grad():
            old_mu = self.old_policy(obs_batch, deterministic=True)
        imitation = None
        if getattr(self, "base_policy", None) is not None:
            teacher_mu, imask = self._teacher_actions(obs_batch)
            imitation = (teacher_mu.float().contiguous(), None if imask is None else imask.float().contiguous(), float(self.imitate_coeff))
        values = self.critic(obs_batch)
        stds = self.policy.stds if torch.is_tensor(self.policy.stds) else torch.as_tensor(self.policy.stds)
        total = _FusedPPOLoss.apply(mu, values, mirr, old_mu, action_batch, advantage_batch, return_batch,
                                    stds.to(mu.device, torch.float32), float(self.clip), float(self.mirror_coeff), float(self.ent_coeff), bufs,
                                    imitation)
        out = bufs[5].clone()       # the buffer is rewritten by the next update; callers may hold on to the scalars
        return total, tuple(out[k] for k in range(7))

    def _teacher_actions(self, obs_batch):
        """(teacher actions, mask or None) for a minibatch, without a graph; both loss paths take them from here."""
        if getattr(self, "imitation_projector", None) is None:
            raise ValueError("imitation needs an imitation_projector that maps the student's observations to the teacher's")
        with torch.no_grad():
            teacher_obs, imask = self.imitation_projector(obs_batch)
            return self.base_policy(teacher_obs, deterministic=True), imask

    def update_actor_critic(self, obs_batch, action_batch, return_batch, advantage_batch, mask,
                            mirror_observation=None, mirror_action=None):
        if self._fused_loss_ok(obs_batch, mask):
            total_loss, scalars = self._loss_fused(obs_batch, action_batch, return_batch, advantage_batch, mirror_observation,
                                                   mirror_action)
            return self._optimizer_step(total_loss, scalars)
        pdf = self.policy.distribution(obs_batch)
        log_probs = pdf.log_prob(action_batch).sum(-1, keepdim=True)
        with torch.no_grad():
            old_log_probs = self.old_policy.distribution(obs_batch).log_prob(action_batch).sum(-1, keepdim=True)
        ratio = (log_probs - old_log_probs).exp()
        cpi_loss = ratio * advantage_batch * mask
        clip_loss = ratio.clamp(1.0 - self.clip, 1.0 + self.clip) * advantage_batch * mask
        actor_loss = -torch.min(cpi_loss, clip_loss).mean()
        clip_fraction = torch.mean((torch.abs(ratio.detach() - 1) > self.clip).float())
        values = self.critic(obs_batch)
        critic_loss = F.mse_loss(return_batch, values)
        entropy_penalty = -(pdf.entropy() * mask).mean()
        deterministic_actions = pdf.mean
        if mirror_observation is not None and mirror_action is not None:
            mirror_actions = mirror_action(self.policy(mirror_observation(obs_batch)))
            mirror_loss = (deterministic_actions - mirror_actions).pow(2).mean()
        else:
            mirror_loss = torch.zeros_like(actor_loss)
        if getattr(self, "base_policy", None) is not None:
            # rl/algos/ppo.py:361-368: the teacher's deterministic actions on the projected observations (rl/imitation.py)
            base_actions, imask = self._teacher_actions(obs_batch)
            sq = (base_actions - deterministic_actions).pow(2)
            imitation_loss = (sq if imask is None else sq * imask).mean()
        else:
            imitation_loss = torch.zeros_like(actor_loss)
        with torch.no_grad():
            approx_kl_div = torch.mean((ratio - 1) - (log_probs - old_log_probs))
        total_loss = (actor_loss + self.mirror_coeff * mirror_loss + self.imitate_coeff * imitation_loss
                      + self.ent_coeff * entropy_penalty + critic_loss)
        return self._optimizer_step(total_loss, (actor_loss, entropy_penalty, critic_loss, approx_kl_div, mirror_loss, imitation_loss,
                                                 clip_fraction))

    def _optimizer_step(self, total_loss, scalars):
        """backward + the exchange / clip / Adam step (rl/algos/ppo.py:389-396); returns the 7 scalars detached."""
        self.actor_optimizer.zero_grad()
        self.critic_optimizer.zero_grad()
        total_loss.backward()
        a_opt, c_opt = self.actor_optimizer, self.critic_optimizer
        if self._comm is not None and isinstance(a_opt, FusedClipAdam) and isinstance(c_opt, FusedClipAdam):
            # the one exchange step of the path, fused: peer-memory all-reduce + 2x clip_grad_norm_ + 2x Adam in three
            # graph-capturable launches (csrc/comm_kernels.cu); at world 1 the same launches without the flag traffic
            a_opt.step_count += 1
            c_opt.step_count += 1
            g = a_opt.param_groups[0]
            if getattr(self, "schedule", "fixed") == "adaptive":
                # scalar 3, the minibatch's "Mean KL Div", drives the device rate; the same launches eager and in the graph
                self._comm.fused_step_adaptive(self._flat_param, self._flat_m, self._flat_v, self._n_actor,
                                               scalars[3].detach().float().reshape(1), self.desired_kl, g["betas"], g["eps"],
                                               g["max_norm"])
            else:
                self._comm.fused_step(self._flat_param, self._flat_m, self._flat_v, self._n_actor, g["lr"], g["betas"], g["eps"],
                                      g["max_norm"])
        elif getattr(self, "schedule", "fixed") == "adaptive":
            self._check_schedule()
        elif isinstance(a_opt, FusedClipAdam) and isinstance(c_opt, FusedClipAdam):
            if self.world > 1:  # baseline path: NCCL all-reduce of the flat gradient, then clip+Adam launches
                dist.all_reduce(self._flat_grad, op=dist.ReduceOp.SUM)
            a_opt.step()
            c_opt.step()
        else:  # hand-made torch optimisers (tests/test_training.py:140-141): the reference's own sequence
            torch.nn.utils.clip_grad_norm_(self.policy.parameters(), self.grad_clip)
            torch.nn.utils.clip_grad_norm_(self.critic.parameters(), self.grad_clip)
            a_opt.step()
            c_opt.step()
        # detached: a caller holding on to the losses must not keep this step's autograd graph (and its AccumulateGrad nodes)
        # alive into the next one, which may be captured into a CUDA graph
        return tuple(t.detach() for t in scalars)

    # ------------------------------------------------------------------ one minibatch update, replayed from a CUDA graph
    def _update_step(self, ob, ab, rb, db, obs_mirr, act_mirr) -> torch.Tensor:
        """update_actor_critic on the static minibatch buffers; returns the 7 scalars as one device vector.
        An update is ~600 small launches (three MLP forwards, autograd backward, clip + Adam); at the reference's minibatch
        sizes it is launch bound (2.5 ms of host time for 1.9 ms of kernels at 4096 samples, far worse at the default 64).
        After a few eager steps (cuBLAS / autograd warm-up — they are real updates) the whole step — losses, backward,
        gradient norms, clip + Adam with the step counter in device memory — is captured once and replayed.
        Every rank captures and replays the same step: the fused exchange (peer-memory all-reduce + clip + Adam) is three
        ordinary launches whose epoch / step counters live in device memory.  LHW_UPDATE_GRAPH=0 keeps the eager loop."""
        import os
        # the NCCL baseline (LHW_FUSED_EXCHANGE=0) on several ranks stays eager: a captured graph that holds NCCL work kept the
        # process group from shutting down (observed: destroy_process_group never returned); it is the baseline, not the path
        eager = ((self.world > 1 and self._comm is None) or os.environ.get("LHW_UPDATE_GRAPH", "1") == "0" or self._mb is None
                 or ob is not self._mb[0]
                 or not isinstance(self.actor_optimizer, FusedClipAdam) or not isinstance(self.critic_optimizer, FusedClipAdam))
        if not eager and self._ug is not None and self._ug[2] == ob.data_ptr():
            self._ug[0].replay()
            self.actor_optimizer.step_count += 1
            self.critic_optimizer.step_count += 1
            return self._ug[1]
        if eager:
            scalars = self.update_actor_critic(ob, ab, rb, db, 1, mirror_observation=obs_mirr, mirror_action=act_mirr)
            return torch.stack([s.detach().float() for s in scalars])
        if self._ug_calls < 3:
            # warm-up on a side stream, as graph capture will run on one (cuBLAS workspaces, autograd buffers)
            self._ug_calls += 1
            cur, side = torch.cuda.current_stream(self.device), torch.cuda.Stream(device=self.device)
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                scalars = self.update_actor_critic(ob, ab, rb, db, 1, mirror_observation=obs_mirr, mirror_action=act_mirr)
                out = torch.stack([s.detach().float() for s in scalars])
            cur.wait_stream(side)
            out.record_stream(cur)
            return out
        torch.cuda.synchronize(self.device)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            scalars = self.update_actor_critic(ob, ab, rb, db, 1, mirror_observation=obs_mirr, mirror_action=act_mirr)
            out = torch.stack([s.detach().float() for s in scalars])
        # capture does not execute, and the host-side counters it bumped belong to the replay below
        self.actor_optimizer.step_count -= 1
        self.critic_optimizer.step_count -= 1
        self._ug = (g, out, ob.data_ptr())
        return self._update_step(ob, ab, rb, db, obs_mirr, act_mirr)

    def make_optimizers(self):
        """Adam(lr, eps) for actor and critic (rl/algos/ppo.py:429-430) as fused clip+Adam over one flat buffer."""
        import os
        from .comm import PeerComm
        from .optim import flatten_modules_
        n_total = sum(p.numel() for m in (self.policy, self.critic) for p in m.parameters())
        # the fused exchange (peer all-reduce + clip + Adam, three launches) is the path at every world size;
        # LHW_FUSED_EXCHANGE=0 selects the baseline: NCCL all-reduce + lhw_grad_sumsq / lhw_clip_adam_dev per network
        fused = os.environ.get("LHW_FUSED_EXCHANGE", "1") != "0"
        if self._comm is not None:
            self._comm.close()
        self._comm = PeerComm(n_total, self.device) if fused else None
        flat, grad, segs = flatten_modules_([self.policy, self.critic], None if self._comm is None else self._comm.grad)
        self._flat_param, self._flat_grad = flat, grad
        self._flat_m, self._flat_v = torch.zeros_like(flat), torch.zeros_like(flat)
        self._n_actor = segs[0][1]
        sl = lambda t, k: t[segs[k][0]:segs[k][1]]
        self.actor_optimizer = FusedClipAdam(self.policy, lr=self.lr, eps=self.eps, max_norm=self.grad_clip,
                                             views=(sl(flat, 0), sl(grad, 0), sl(self._flat_m, 0), sl(self._flat_v, 0)))
        self.critic_optimizer = FusedClipAdam(self.critic, lr=self.lr, eps=self.eps, max_norm=self.grad_clip,
                                              views=(sl(flat, 1), sl(grad, 1), sl(self._flat_m, 1), sl(self._flat_v, 1)))
        self.actor_optimizer.world = self.critic_optimizer.world = self.world
        if getattr(self, "schedule", "fixed") == "adaptive":
            self._check_schedule()
            self._comm.set_lr(self.lr)      # `--lr` is the starting rate (so also after `--continued`)
        if self.world > 1:
            # replicas start from rank 0's weights whatever the seeding of the ranks was
            dist.broadcast(self._flat_param, src=0)
        # old_policy must not alias the flat buffer
        self.old_policy = deepcopy(self.policy)
        # the parameters have just been re-homed into the flat buffer: every captured graph (rollout step, optimiser step)
        # still holds the OLD parameter addresses -> drop them, they are re-captured on next use
        for w in self.workers:
            w.invalidate_graphs()
        self._ug, self._ug_calls = None, 0

    def _check_schedule(self):
        """The adaptive schedule lives on the fused exchange only: refuse the baseline exchange and hand-assigned optimisers."""
        if getattr(self, "schedule", "fixed") != "adaptive":
            return
        if not (isinstance(self.actor_optimizer, FusedClipAdam) and isinstance(self.critic_optimizer, FusedClipAdam)):
            raise ValueError("--schedule adaptive drives the fused exchange's device rate; hand-assigned torch optimisers "
                             "would ignore it (use make_optimizers())")
        if self._comm is None:
            raise ValueError("--schedule adaptive needs the fused exchange, which holds the rate in device memory; "
                             "LHW_FUSED_EXCHANGE=0 selects the baseline exchange, which has no adaptive schedule")

    # ------------------------------------------------------------------ device data path helpers
    def normalize_advantages(self, returns: torch.Tensor, values: torch.Tensor, from_rollout: bool = False) -> torch.Tensor:
        """rl/algos/ppo.py:484-485 on device; statistics are global across ranks.  from_rollout=True: `returns` / `values` are
        the batch the device worker has just produced, whose GAE launch already left the advantage's (sum, sumsq) behind —
        the normalisation is then a single 12 B/sample pass."""
        O = _lib.ops()
        n = returns.numel()
        adv = torch.empty_like(returns)
        buf = getattr(self.workers[0], "_buf", None) if getattr(self, "workers", None) else None
        if from_rollout and buf is not None and buf.T * buf.N == n:
            # (sum, sumsq) of returns - values were produced by the GAE launch of this very batch: no statistics pass
            O.adv_stats_from_gae(buf.adv_partials, buf.N, self._adv_stats)
        else:
            O.adv_stats(returns, values, self._adv_stats)
        if self.world > 1:
            dist.all_reduce(self._adv_stats[0:2], op=dist.ReduceOp.SUM)
        # equal shards are enforced in __init__, so the global count is n * world
        O.adv_apply(returns, values, adv, self._adv_stats, n * self.world, self.eps)
        return adv

    def gather_minibatch(self, obs, act, ret, adv, idx: torch.Tensor):
        B = idx.numel()
        if self._mb is None or self._mb[0].shape[0] != B:
            f32 = dict(dtype=torch.float32, device=self.device)
            self._mb = (torch.empty(B, obs.shape[1], **f32), torch.empty(B, act.shape[1], **f32),
                        torch.empty(B, 1, **f32), torch.empty(B, 1, **f32))
        o, a, r, d = self._mb
        _lib.ops().gather_minibatch(obs, act, ret, adv, idx, o, a, r, d)
        return o, a, r, d

    def minibatch_indices(self, num_samples: int, itr: int, epoch: int):
        """SubsetRandomSampler + BatchSampler(drop_last=True) with the reference's seeding
        (rl/algos/ppo.py:504-517): generator seeded seed + itr*epochs + epoch, identical on every rank."""
        g = None
        if self.seed is not None:
            g = torch.Generator()
            g.manual_seed(self.seed + itr * self.epochs + epoch)
        perm = torch.randperm(num_samples, generator=g)
        mb = self.minibatch_size or num_samples
        nb = num_samples // mb
        return perm[: nb * mb].view(nb, mb).to(self.device, non_blocking=True)

    # ------------------------------------------------------------------ evaluation + checkpoints (rl/algos/ppo.py:408-426)
    def evaluate(self, env_fn, nets, itr, num_batches=5):
        """num_batches deterministic batches from the persistent workers (episodes carry on from the training batch, as in the
        reference); the mean reward / length of the episodes that completed, over all ranks; `actor_{itr}.pt` / `critic_{itr}.pt`
        always, the un-suffixed `actor.pt` / `critic.pt` when the mean reward improved (ModelCheckpointer.save_if_best,
        rl/utils/checkpointer.py:54-83).  Returns (eval_batches, mean_reward, mean_length); no completed episode -> nan, which
        never counts as an improvement."""
        for net in nets.values():
            net.eval()
        eval_batches = [self.sample_parallel_with_workers(deterministic=True) for _ in range(num_batches)]
        tot = torch.zeros(3, dtype=torch.float64, device=self.device)
        for b in eval_batches:
            tot[0] += b.ep_rewards.double().sum()
            tot[1] += b.ep_lens.double().sum()
            tot[2] += b.ep_rewards.numel()
        if self.world > 1:
            dist.all_reduce(tot)
        rew_sum, len_sum, n_ep = tot.tolist()
        mean_rew = rew_sum / n_ep if n_ep else float("nan")
        mean_len = len_sum / n_ep if n_ep else float("nan")
        if self.rank == 0:
            self.save(itr)
            if mean_rew > self._best_eval:
                self._best_eval = mean_rew
                self.save(None)
        return eval_batches, mean_rew, mean_len

    # ------------------------------------------------------------------ training loop (rl/algos/ppo.py:428-641)
    def train(self, env_fn, n_itr, verbose=True, start_itr=0):
        """Iterations start_itr .. n_itr - 1.  start_itr > 0 continues a run restored from its snapshot at start_itr - 1:
        elapsed time and fps carry on, and the TensorBoard scalars the stopped run logged from start_itr on are dropped."""
        if self.actor_optimizer is None:
            self.make_optimizers()
        self._check_schedule()
        env = self.env
        obs_mirr = getattr(env, "mirror_clock_observation", None) if self.mirror_coeff else None
        act_mirr = getattr(env, "mirror_action", None) if self.mirror_coeff else None
        train_start = time.time() - getattr(self, "_elapsed0", 0.0)
        log = []
        writer = self._tensorboard_writer(purge_step=start_itr or None) if self.rank == 0 else None
        for itr in range(start_itr, n_itr):
            if verbose and self.rank == 0:
                print(f"********** Iteration {itr} ************")
            self.policy.train()
            self.critic.train()
            self.iteration_count = itr
            t0 = time.time()
            batch = self.sample_parallel_with_workers()
            observations, actions = batch.states, batch.actions
            returns, values = batch.returns.contiguous(), batch.values.contiguous()
            num_samples = observations.shape[0]
            torch.cuda.synchronize(self.device)
            sample_time = time.time() - t0
            if verbose and self.rank == 0:
                print(f"Sampling took {sample_time:.2f}s for {num_samples * self.world} steps.")
            advantages = self.normalize_advantages(returns, values, from_rollout=True)
            self.total_steps += num_samples * self.world
            self.old_policy.load_state_dict(self.policy.state_dict())
            # in place: a captured update graph holds the addresses of these tensors
            self.old_policy.obs_mean.copy_(self.policy.obs_mean)
            self.old_policy.obs_std.copy_(self.policy.obs_std)
            t1 = time.time()
            stats = torch.zeros(7, device=self.device)
            n_updates = 0
            for epoch in range(self.epochs):
                for idx in self.minibatch_indices(num_samples, itr, epoch):
                    ob, ab, rb, db = self.gather_minibatch(observations, actions, returns, advantages, idx)
                    stats += self._update_step(ob, ab, rb, db, obs_mirr, act_mirr)
                    n_updates += 1
            stats = (stats / max(1, n_updates)).tolist()   # the only host sync of the optimisation phase
            if getattr(self, "_comm", None) is not None:
                self._comm.status()    # raises if a peer missed a gradient exchange (bounded spin in the kernels)
            adaptive = getattr(self, "schedule", "fixed") == "adaptive"
            lr_now = self._comm.get_lr() if adaptive else None     # the stream has just been synchronised
            stairs = self._stair_stats()     # (mean stair height, fraction at the top level) or None
            optimize_time = time.time() - t1
            total_time = time.time() - train_start
            fps = self.total_steps / total_time
            ep_rew = float(batch.ep_rewards.mean()) if batch.ep_rewards.numel() else float("nan")
            ep_len = float(batch.ep_lens.float().mean()) if batch.ep_lens.numel() else float("nan")
            log.append(dict(itr=itr, sample_time=sample_time, optimize_time=optimize_time, fps=fps, ep_rew=ep_rew, ep_len=ep_len,
                            actor_loss=stats[0], entropy=stats[1], critic_loss=stats[2], kl=stats[3], mirror=stats[4],
                            clip_frac=stats[6]))
            if adaptive:
                log[-1]["lr"] = lr_now
            if stairs is not None:
                log[-1].update(mean_stair_height=stairs[0], top_stair_fraction=stairs[1])
            if verbose and self.rank == 0:
                print(f"Optimizer took: {optimize_time:.2f}s")
                print("-" * 37)
                for k, v in (("Mean Eprew", ep_rew), ("Mean Eplen", ep_len), ("Actor loss", stats[0]), ("Critic loss", stats[2]),
                             ("Mirror loss", stats[4]), ("Imitation loss", stats[5]), ("Mean KL Div", stats[3]),
                             ("Mean Entropy", stats[1]), ("Clip Fraction", stats[6]),
                             ("Mean noise std", float(torch.as_tensor(self.policy.stds).mean())),
                             *((("Learning rate", lr_now),) if adaptive else ()),
                             *((("Mean stair height", stairs[0]), ("Top stair level", stairs[1])) if stairs is not None else ())):
                    print(f"| {k:>15} | {v:>15.5g} |")
                print("-" * 37)
                eta = round((n_itr - itr) * total_time / (itr + 1))
                print(f"Total time elapsed: {total_time:.2f}s. Total steps: {self.total_steps} "
                      f"(fps={fps:.2f}. iter-avg={total_time / (itr + 1):.2f}s. ETA={datetime.timedelta(seconds=eta)})")
            if writer is not None:   # the reference's TensorBoard tags (rl/utils/logger.py:71-115)
                for tag, v in (("Loss/actor", stats[0]), ("Loss/critic", stats[2]), ("Loss/mirror", stats[4]),
                               ("Loss/imitation", stats[5]), ("Train/mean_reward", ep_rew), ("Train/mean_episode_length", ep_len),
                               ("Train/mean_noise_std", float(torch.as_tensor(self.policy.stds).mean())), ("Time/fps", fps),
                               ("Time/sample_time", sample_time), ("Time/optimize_time", optimize_time),
                               ("Time/total_elapsed", total_time), *((("Train/learning_rate", lr_now),) if adaptive else ()),
                               *((("Train/mean_stair_height", stairs[0]), ("Train/top_stair_fraction", stairs[1]))
                                 if stairs is not None else ())):
                    writer.add_scalar(tag, v, itr)
            if (itr == 0 and getattr(self, "eval_at_start", True)) or (itr + 1) % self.eval_freq == 0:     # rl/algos/ppo.py:597-615
                t2 = time.time()
                _, eval_rew, eval_len = self.evaluate(env_fn, {"actor": self.policy, "critic": self.critic}, itr,
                                                      num_batches=self.eval_batches)
                log[-1].update(eval_rew=eval_rew, eval_len=eval_len)
                if verbose and self.rank == 0:
                    print("====EVALUATE EPISODE====")
                    print(f"(Episode length:{eval_len:.3f}. Reward:{eval_rew:.3f}. Time taken:{time.time() - t2:.2f}s)")
                if writer is not None:
                    writer.add_scalar("Eval/mean_reward", eval_rew, itr)
                    writer.add_scalar("Eval/mean_episode_length", eval_len, itr)
                if getattr(self, "write_snapshots", False):      # after the evaluation batches: they advance the environments too
                    if writer is not None:
                        writer.flush()
                    snapshot.write(self, itr, time.time() - train_start)
        if writer is not None:
            writer.flush()
            writer.close()
        return log

    def _stair_stats(self):
        """The stair curriculum's state over every env of every rank (DESIGN.md §7.8): (mean of 0.01 L, fraction of envs at the
        top level K - 1), or None without the curriculum.  One small copy to the host, after the iteration's host sync."""
        env = self._inner_env()
        level = getattr(env, "stair_level", None)
        if level is None:
            return None
        top = env.stair_levels - 1
        lv = level.clamp(0, top)   # as the kernels read it
        t = torch.stack([lv.sum(dtype=torch.float64), (lv == top).sum(dtype=torch.float64),
                         torch.tensor(float(lv.numel()), dtype=torch.float64, device=lv.device)])
        if self.world > 1:
            dist.all_reduce(t, op=dist.ReduceOp.SUM)
        s, n_top, n = t.tolist()
        return 0.01 * s / n, n_top / n

    def _tensorboard_writer(self, purge_step=None):
        """TrainingLogger (rl/utils/logger.py:24-45): a SummaryWriter on the run directory; None if tensorboard is absent
        or LHW_TENSORBOARD=0.  purge_step: a resumed run hides the events of steps >= purge_step from the earlier files."""
        import os
        if os.environ.get("LHW_TENSORBOARD", "1") == "0":
            return None
        try:
            from torch.utils.tensorboard import SummaryWriter
        except Exception:
            return None
        self.save_path.mkdir(parents=True, exist_ok=True)
        return SummaryWriter(str(self.save_path), flush_secs=10, purge_step=purge_step)

    def save(self, itr):
        """actor_{itr}.pt / critic_{itr}.pt as whole pickled modules; itr None = the un-suffixed "best" pair
        (rl/utils/checkpointer.py:36-83)."""
        self.save_path.mkdir(parents=True, exist_ok=True)
        suffix = "" if itr is None else f"_{itr}"
        from .policies import export_module
        # self-contained CPU copies under the reference's class path (rl.policies.actor.Gaussian_FF_Actor / rl.policies.critic.FF_V):
        # loadable by a reference checkout's `run_experiment.py eval` / `--continued` (rl/policies/__init__.py)
        torch.save(export_module(self.policy), self.save_path / f"actor{suffix}.pt")
        torch.save(export_module(self.critic), self.save_path / f"critic{suffix}.pt")
