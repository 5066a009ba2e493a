"""DeviceRolloutWorker — replaces the N Ray actors of rl/workers/rollout_worker.py with one device-resident
vectorised sampler: N environments advance together, one CUDA launch per control step, policy / critic
inference batched on the same device (cuBLAS), transitions written straight into device rollout buffers.

Semantics kept from RolloutWorker.sample (rl/workers/rollout_worker.py:98-199), per environment:
  * exactly `max_steps` transitions per call; episodes persist across calls (state, traj_len, episode stats);
  * an episode ends on done or when traj_len reaches max_traj_len (truncation); `dones` stores done OR truncated;
  * bootstrap on an ended episode = (not done) * critic(next_state) with next_state the PRE-reset observation;
  * a path still open when the buffer fills bootstraps with critic(current state);
  * only completed episodes contribute ep_lens / ep_rewards.
"""
from __future__ import annotations

import torch

from .storage import BatchData, DeviceRolloutBuffer


class DeviceRolloutWorker:
    def __init__(self, env, policy, critic, seed: int | None = None, worker_id: int = 0):
        self.env, self.policy, self.critic = env, policy, critic
        self.worker_id = worker_id
        self.device = env.device
        self.gen = torch.Generator(device=self.device)
        self.gen.manual_seed(0 if seed is None else int(seed))
        self.current_state = None      # [N, obs_dim] float32; None before the first reset
        self._buf = None
        self._graphs = {}
        self.total_steps = 0

    def invalidate_graphs(self):
        """Drop the captured control-step graphs (they hold the addresses of the policy / critic parameters and of the
        rollout buffers): call after anything that re-homes those tensors, e.g. PPO.make_optimizers()."""
        self._graphs = {}

    def state_dict(self) -> dict:
        """What the next sample() depends on besides the env's records and the networks (rl/snapshot.py)."""
        cs = self.current_state
        return dict(current_state=None if cs is None else cs.cpu(), gen=self.gen.get_state(), total_steps=int(self.total_steps))

    def load_state_dict(self, sd: dict) -> None:
        """Inverse of state_dict(); in place where a captured graph may hold the address of current_state."""
        cs = sd["current_state"]
        if cs is None:
            self.current_state = None
        elif self.current_state is not None and self.current_state.shape == cs.shape:
            self.current_state.copy_(cs)
        else:
            self.current_state = cs.to(self.device).clone()
            self._noise = torch.zeros(0, cs.shape[0], self.env.act_dim, device=self.device)   # sample() sizes it
            self._graphs = {}
        self.gen.set_state(sd["gen"])
        self.total_steps = int(sd["total_steps"])

    def sync_state(self, policy_state_dict=None, critic_state_dict=None, obs_mean=None, obs_std=None, iteration_count=0):
        """The learner and the sampler share the same modules on the same device: nothing to ship.  Kept so the
        call site of rl/algos/ppo.py:238-242 works unchanged; state dicts are loaded if given."""
        if policy_state_dict is not None:
            self.policy.load_state_dict(policy_state_dict)
        if critic_state_dict is not None:
            self.critic.load_state_dict(critic_state_dict)
        if obs_mean is not None:
            self.policy.obs_mean = self.critic.obs_mean = obs_mean
        if obs_std is not None:
            self.policy.obs_std = self.critic.obs_std = obs_std
        self.env.robot.iteration_count = iteration_count

    # ------------------------------------------------------------------ one control step of the rollout loop
    def _parts(self, N: int):
        """The batch as one part, or as two halves (LHW_ROLLOUT_PARTS, default 2) that advance independently on their own streams:
        a control step of one half does not wait for the other half's, so the tail of one half's step launch (4096 fp64
        environments are 1.7 resident waves) and its MLP / buffer kernels overlap the other half's step kernel.  Every
        per-environment result is unchanged (an environment's trajectory does not depend on what it is launched with);
        LHW_ROLLOUT_SPLIT=0 keeps one part."""
        import os
        k = 1 if os.environ.get("LHW_ROLLOUT_SPLIT", "1") == "0" else int(os.environ.get("LHW_ROLLOUT_PARTS", "2"))
        if k <= 1 or N < 512 * k:
            return [(0, N)]
        cuts = [N * i // k for i in range(k + 1)]
        return [(cuts[i], cuts[i + 1]) for i in range(k)]

    def _step_body(self, buf, part, state, noise, t_idx, deterministic):
        """policy -> action -> critic -> env.step -> bootstrap -> buffer writes for the environments [lo, hi) of `part`, all on
        device tensors; `t_idx` is a 1-element device index so the same code can be replayed from a CUDA graph (no host-side
        loop counter).  `state` is the [hi - lo, obs] view of the worker's current observations."""
        env = self.env
        lo, hi = part
        V = lambda t: t[:, lo:hi]          # the part's columns of a time-major [T, N, ...] buffer
        mu = self.policy(state, deterministic=True)
        action = mu if deterministic else mu + self.policy.stds * V(noise).index_select(0, t_idx)[0]
        V(buf.states).index_copy_(0, t_idx, state.unsqueeze(0))
        V(buf.actions).index_copy_(0, t_idx, action.unsqueeze(0))
        V(buf.values).index_copy_(0, t_idx, self.critic(state).squeeze(-1).unsqueeze(0))
        obs, reward, done, ended = env.step_slice(lo, hi, action if env.dtype == torch.float32 else action.double())
        V(buf.rewards).index_copy_(0, t_idx, reward.float().unsqueeze(0))
        V(buf.ended).index_copy_(0, t_idx, ended.unsqueeze(0))
        V(buf.ep_len).index_copy_(0, t_idx, env.ep_len[lo:hi].unsqueeze(0))
        V(buf.ep_rew).index_copy_(0, t_idx, env.ep_rew[lo:hi].float().unsqueeze(0))
        # truncation bootstrap: (not done) * critic(pre-reset next_state) where the episode ended
        v_term = self.critic(env.term_obs[lo:hi].float()).squeeze(-1)
        V(buf.boot).index_copy_(0, t_idx, torch.where((ended != 0) & (done == 0), v_term, torch.zeros_like(v_term)).unsqueeze(0))
        state.copy_(obs.float())
        t_idx.add_(1)

    @torch.no_grad()
    def sample(self, gamma, lam, max_steps, max_traj_len, deterministic=False, env_major=True) -> BatchData:
        import os
        env = self.env
        N, T = env.num_envs, int(max_steps)
        # the truncation length lives on the batched env itself, not on a SymmetricEnv wrapper around it
        inner = env.__dict__.get("env", None)
        (inner if inner is not None else env).max_traj_len = int(max_traj_len)
        if self._buf is None or self._buf.T != T or self._buf.N != N:
            self._buf = DeviceRolloutBuffer(T, N, env.obs_dim, env.act_dim, self.device, gamma, lam)
            self._graphs = {}
        buf = self._buf
        buf.gamma, buf.lam = gamma, lam
        parts = self._parts(N)
        if self.current_state is None:
            self.current_state = env.reset().float().clone()
            self._noise = torch.zeros(T, N, env.act_dim, device=self.device)
        if getattr(self, "_t_idx", None) is None or len(self._t_idx) != len(parts):
            self._t_idx = [torch.zeros(1, dtype=torch.long, device=self.device) for _ in parts]
            self._streams = [torch.cuda.Stream(device=self.device) for _ in parts]
        if self._noise.shape[0] != T:
            self._noise = torch.zeros(T, N, env.act_dim, device=self.device)
        noise = self._noise
        states = [self.current_state[lo:hi] for lo, hi in parts]
        for t in self._t_idx:
            t.zero_()
        if not deterministic:
            noise.copy_(torch.randn(noise.shape, device=self.device, generator=self.gen))
        cur = torch.cuda.current_stream(self.device)
        use_graph = os.environ.get("LHW_ROLLOUT_GRAPH", "1") != "0"
        if use_graph:
            key = (bool(deterministic), int(max_traj_len), len(parts))
            graphs = self._graphs.get(key)
            first = 0
            if graphs is None:
                # warm-up on the side streams (cuBLAS workspaces, constant-memory upload), then capture ONE control step per part
                graphs = []
                for p, part in enumerate(parts):
                    s = self._streams[p]
                    s.wait_stream(cur)
                    with torch.cuda.stream(s):
                        self._step_body(buf, part, states[p], noise, self._t_idx[p], deterministic)
                    cur.wait_stream(s)
                first = 1
                if T > 1:
                    for p, part in enumerate(parts):
                        g = torch.cuda.CUDAGraph()
                        with torch.cuda.graph(g, stream=self._streams[p]):
                            self._step_body(buf, part, states[p], noise, self._t_idx[p], deterministic)
                        graphs.append(g)
                    self._graphs[key] = graphs   # capturing does not execute: warm-up did step 0, replays do the rest
            env.bind()   # make sure THIS env's model constants are the resident ones before replaying launches
            if graphs:
                for p, g in enumerate(graphs):     # each part runs its T steps on its own stream; they only meet at the end
                    s = self._streams[p]
                    s.wait_stream(cur)
                    with torch.cuda.stream(s):
                        for _ in range(first, T):
                            g.replay()
                for s in self._streams:
                    cur.wait_stream(s)
        else:
            for _ in range(T):
                for p, part in enumerate(parts):
                    self._step_body(buf, part, states[p], noise, self._t_idx[p], deterministic)
        buf.last_val.copy_(self.critic(self.current_state).squeeze(-1))
        buf.finish()
        self.total_steps += T * N
        return buf.get_data(env_major=env_major)
