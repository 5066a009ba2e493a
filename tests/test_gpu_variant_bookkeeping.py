"""Sims of every robot / task variant at both precisions alive in one process (csrc/sim_kernels.cu: one SimOf per sim, one
constant-bank object per variant and precision) step exactly as they do alone, whatever order their launches come in."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
MODELS = ("jvrc_walk", "h1", "jvrc_step", "jvrc_walk_terrain")
N, STEPS = 16, 10
RISING = [3000 + 800 * k for k in range(STEPS)]      # curriculum step heights 0, 0.01, ..., 0.09
FALLING = [11000 - 800 * k for k in range(STEPS)]    # 0.1, 0.09, ..., 0.01


def _env(model, precision, yaml=None):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(N, model=model, precision=precision, seed=7, path_to_yaml=yaml)


def _advance(env, k, heights):
    """Control step k of one sim: (jvrc_step) the curriculum height of iteration heights[k], a reset of env k % N, then a
    step under seeded actions.  Returns copies of the outputs and of the state record."""
    if env.model_name == "jvrc_step":
        env.robot.iteration_count = heights[k]
    env.reset(None if k == 0 else torch.arange(N) == k % N)
    a = 0.3 * torch.randn(N, env.act_dim, generator=torch.Generator().manual_seed(k), dtype=torch.float64)
    obs, rew, done, _ = env.step(a.to(env.device, env.dtype))
    return [t.clone() for t in (obs, rew, done, env.state_r, env.state_i)]


def _alone(model, precision, heights=RISING, yaml=None):
    env = _env(model, precision, yaml)
    out = [_advance(env, k, heights) for k in range(STEPS)]
    env.close()
    return out


def _same(x, y):
    return all(torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(x, y))


def test_every_variant_and_precision_interleaved_steps_as_alone():
    """The two jvrc_step sims of each precision share a constant-bank object and get different step heights between steps."""
    specs = [(m, p, RISING) for m in MODELS for p in (64, 32)] + [("jvrc_step", p, FALLING) for p in (64, 32)]
    alone = [_alone(m, p, h) for m, p, h in specs]
    envs = [_env(m, p) for m, p, _ in specs]
    for k in range(STEPS):
        for i, (m, p, h) in enumerate(specs):
            assert _same(_advance(envs[i], k, h), alone[i][k]), (m, p, k)
    for env in envs:
        env.close()
    for p in (64, 32):   # the curriculum really changed the footstep plans
        assert not _same(alone[specs.index(("jvrc_step", p, RISING))][-1], alone[specs.index(("jvrc_step", p, FALLING))][-1])


def test_sim_replaced_by_one_with_other_constants_steps_with_its_own(tmp_path):
    """Half-way, the fp32 jvrc_walk sim is destroyed and a new one with softer PD gains from a YAML takes its place (possibly at
    the freed address): from its first step on it must use its own constants, and the other sims theirs."""
    soft = tmp_path / "soft.yaml"
    soft.write_text("kp: [100, 100, 100, 125, 40, 40, 100, 100, 100, 125, 40, 40]\n")
    specs = [(m, p) for m in MODELS for p in (64, 32)]
    alone = [_alone(m, p) for m, p in specs]
    alone_soft = _alone("jvrc_walk", 32, yaml=soft)
    assert not _same(alone_soft[1], alone[specs.index(("jvrc_walk", 32))][1])   # the YAML really changed the dynamics
    envs = [_env(m, p) for m, p in specs]
    swap, half = specs.index(("jvrc_walk", 32)), STEPS // 2
    for k in range(STEPS):
        if k == half:
            envs[swap].close()
            envs[swap] = _env("jvrc_walk", 32, soft)
        for i, (m, p) in enumerate(specs):
            if i == swap and k >= half:
                assert _same(_advance(envs[i], k - half, RISING), alone_soft[k - half]), ("replacement", k)
            else:
                assert _same(_advance(envs[i], k, RISING), alone[i][k]), (m, p, k)
    for env in envs:
        env.close()
