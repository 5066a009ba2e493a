"""Imitation of a saved actor (rl/imitation.py, the imitation term of PPO.update_actor_critic, `train --imitate`), CPU tier:
the projectors on the kernel source's h1_walk observations, the supported and refused (teacher, student) pairs, the loss and
its gradient against float64 numpy and torch autograd, and the command line refusing a bad teacher before a run directory
exists.  The CUDA kernel is held to the same formula by tests/test_gpu_imitation.py."""
import os
import pickle
from argparse import Namespace

import numpy as np
import pytest
import torch

ENVS = ("jvrc_walk", "jvrc_walk_terrain", "jvrc_step", "h1", "h1_walk")


def _attrs(name):
    from learninghumanoidwalking_b200.envs.batched_env import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.model import load_model, pack_model
    env = BatchedHumanoidEnv.__new__(BatchedHumanoidEnv)
    env._iteration_count = float("inf")
    mj = load_model(name)
    env._setup_reference_attributes(name, mj["cfg"])
    return env, 2 * (int(pack_model(mj)[0]) % 100)


def test_env_widths_match_the_environments():
    from learninghumanoidwalking_b200.rl.imitation import ENV_DIMS
    assert set(ENV_DIMS) == set(ENVS)
    for name in ENVS:
        env, n_act = _attrs(name)
        assert ENV_DIMS[name] == (len(env.obs_mean), n_act), name
    # h1_walk's observation starts with h1's robot-state words, normalised the same way
    h1, _ = _attrs("h1")
    hw, _ = _attrs("h1_walk")
    assert np.array_equal(hw.obs_mean[:35], h1.obs_mean) and np.array_equal(hw.obs_std[:35], h1.obs_std)


def test_h1_walk_projector_masks_the_standing_samples_of_the_kernel_source():
    """The h1 -> h1_walk projector on observations of the kernel source (host emulation): over 150 closed-loop steps x 16
    environments with mode switches, the mask is mode == STANDING of the state record and the teacher reads the robot words."""
    from emu_variants import Emu
    from learninghumanoidwalking_b200.model import load_model, pack_model
    from learninghumanoidwalking_b200.rl.imitation import make_projector
    proj = make_projector("h1", "h1_walk", 35, 10, 43, 10)
    N, STANDING = 16, 0
    e = Emu(pack_model(load_model("h1_walk")), 64, N, seed=11, first_id=5)
    obs = e.reset()
    rng = np.random.RandomState(2)
    seen, switches, mode = set(), 0, e.si[:, 1].copy()
    for t in range(150):
        if t:
            obs = e.step(rng.normal(size=(N, 10)) * 0.3, max_traj_len=60)[0]
        tobs, mask = proj(torch.as_tensor(obs))
        assert mask.shape == (N, 1) and tobs.shape == (N, 35)
        assert np.array_equal(mask[:, 0].numpy(), (e.si[:, 1] == STANDING).astype(np.float64)), t
        assert np.array_equal(tobs.numpy(), obs[:, :35])
        seen |= set(mask[:, 0].tolist())
        switches += int((e.si[:, 1] != mode).sum())
        mode = e.si[:, 1].copy()
    assert seen == {0.0, 1.0} and switches > 0


def test_identity_pairs_and_refused_pairs():
    from learninghumanoidwalking_b200.rl.imitation import ENV_DIMS, IdentityProjector, make_projector
    x = torch.randn(5, 37)
    for t, s in (("jvrc_walk", "jvrc_walk"), ("jvrc_walk", "jvrc_walk_terrain"), ("jvrc_walk_terrain", "jvrc_walk"),
                 ("jvrc_step", "jvrc_step"), ("h1", "h1"), ("h1_walk", "h1_walk"), (None, "jvrc_walk")):
        so, sa = ENV_DIMS[s]
        p = make_projector(t, s, so, sa, so, sa)
        assert isinstance(p, IdentityProjector)
        o, m = p(x)
        assert o is x and m is None
    for t, s in (("jvrc_walk", "jvrc_step"), ("h1_walk", "h1"), ("jvrc_step", "jvrc_walk"), ("h1", "jvrc_walk")):
        (to, ta), (so, sa) = ENV_DIMS[t], ENV_DIMS[s]
        with pytest.raises(ValueError) as e:
            make_projector(t, s, to, ta, so, sa)
        assert t in str(e.value) and s in str(e.value)
    with pytest.raises(ValueError, match="action widths") as e:      # jvrc -> h1_walk: 12 actions against 10
        make_projector("jvrc_walk", "h1_walk", 37, 12, 43, 10)
    assert "jvrc_walk" in str(e.value) and "h1_walk" in str(e.value)
    with pytest.raises(ValueError) as e:      # no experiment.pkl, and the teacher reads 35 words where the student has 37
        make_projector(None, "jvrc_walk", 35, 12, 37, 12)
    assert "unknown env" in str(e.value) and "jvrc_walk" in str(e.value)


class _LeafActor(torch.nn.Module):
    """A policy whose mean IS a parameter [B, A] (float64): d total / d mu is then that parameter's gradient."""

    def __init__(self, mu, std):
        super().__init__()
        self.mu = torch.nn.Parameter(mu.clone())
        self.stds = torch.full((mu.shape[1],), std, dtype=torch.float64)
        self.learn_std = False

    def forward(self, state, deterministic=True):
        return self.mu

    def distribution(self, state):
        return torch.distributions.Normal(self.mu, self.stds, validate_args=False)


def _holder(coeff, mask_kind, B=40, A=10, seed=0):
    """PPO.update_actor_critic's attributes on a bare instance (as tests/test_ppo_update_golden.py builds it), float64, with a
    teacher behind the h1 -> h1_walk projector; lr 0 and no clipping, so the step leaves the raw gradients in place."""
    from learninghumanoidwalking_b200.rl.imitation import H1StandingProjector
    from learninghumanoidwalking_b200.rl.policies import FF_V, Gaussian_FF_Actor
    from learninghumanoidwalking_b200.rl.ppo import PPO
    g = torch.Generator().manual_seed(seed)
    obs = torch.randn(B, 43, generator=g, dtype=torch.float64)
    obs[:, 37:40] = 0.0
    standing = {"ones": torch.ones(B), "mixed": (torch.arange(B) % 3 == 0).double(), "empty": torch.zeros(B)}[mask_kind]
    obs[:, 39] = standing
    mu = 0.3 * torch.randn(B, A, generator=g, dtype=torch.float64)
    policy = _LeafActor(mu, 0.223)
    old_policy = _LeafActor(mu + 0.05 * torch.randn(B, A, generator=g, dtype=torch.float64), 0.223)
    torch.manual_seed(seed)
    critic = FF_V(43).double()
    teacher = Gaussian_FF_Actor(35, A).double().requires_grad_(False)
    with torch.no_grad():
        teacher.means.weight.normal_(0, 0.3, generator=g)
    ppo = PPO.__new__(PPO)
    ppo.__dict__.update(policy=policy, old_policy=old_policy, critic=critic, clip=0.2, ent_coeff=0.01, mirror_coeff=0.4,
                        imitate_coeff=coeff, grad_clip=1e12, _comm=None, world=1, base_policy=teacher,
                        imitation_projector=H1StandingProjector() if mask_kind != "ones" else None,
                        actor_optimizer=torch.optim.SGD(policy.parameters(), lr=0.0),
                        critic_optimizer=torch.optim.SGD(critic.parameters(), lr=0.0))
    if mask_kind == "ones":    # an all-ones mask: the identity projector on a teacher that reads the first 35 words
        ppo.imitation_projector = lambda o: (o[:, :35], None)
    act = mu + 0.223 * torch.randn(B, A, generator=g, dtype=torch.float64)
    ret, adv = torch.randn(B, 1, generator=g, dtype=torch.float64), torch.randn(B, 1, generator=g, dtype=torch.float64)
    with torch.no_grad():
        tau = teacher(obs[:, :35]).numpy()
    return ppo, (obs, act, ret, adv), mu.numpy(), tau, standing.double().numpy()


@pytest.mark.parametrize("mask_kind", ["ones", "mixed", "empty"])
def test_imitation_term_matches_numpy_and_autograd(mask_kind):
    from learninghumanoidwalking_b200.rl.ppo import PPO
    B, A, c = 40, 10, 0.7
    grads, outs = {}, {}
    for coeff in (c, 0.0):
        ppo, batch, mu, tau, m = _holder(coeff, mask_kind)
        outs[coeff] = [float(x) for x in PPO.update_actor_critic(ppo, *batch, 1)]
        grads[coeff] = ppo.policy.mu.grad.clone()
    # float64 numpy: imitation = mean over B*A of m_b (mu - tau)^2, d/dmu = 2 m_b (mu - tau) / (B*A)
    d = mu - tau
    loss = (m[:, None] * d * d).sum() / (B * A)
    g_imit = c * 2 * m[:, None] * d / (B * A)
    assert abs(outs[c][5] - loss) < 1e-12 * max(1.0, loss)
    assert outs[0.0][5] == outs[c][5]            # computed and reported whatever the coefficient
    assert np.abs((grads[c] - grads[0.0]).numpy() - g_imit).max() < 1e-13
    # torch autograd of the reference's formulation, (base_actions - pdf.mean).pow(2) weighted by the mask, then .mean()
    mu_t = torch.tensor(mu, requires_grad=True)
    (c * ((torch.tensor(tau) - mu_t).pow(2) * torch.tensor(m)[:, None]).mean()).backward()
    assert torch.allclose(grads[c] - grads[0.0], mu_t.grad, rtol=0, atol=1e-13)
    if mask_kind == "empty":
        assert outs[c][5] == 0.0 and torch.equal(grads[c], grads[0.0])
    else:
        assert outs[c][5] > 0 and (grads[c] - grads[0.0]).abs().max() > 0
    if mask_kind == "mixed":     # only the standing samples are taught
        assert (grads[c] - grads[0.0])[m == 0].abs().max() == 0


def test_a_teacher_without_a_projector_is_refused():
    from learninghumanoidwalking_b200.rl.ppo import PPO
    ppo, batch, *_ = _holder(1.0, "mixed")
    ppo.imitation_projector = None
    with pytest.raises(ValueError, match="projector"):
        PPO.update_actor_critic(ppo, *batch, 1)


@pytest.mark.skipif(not os.environ.get("LHW_REFERENCE"), reason="LHW_REFERENCE does not name a reference checkout")
def test_imitation_term_matches_the_reference_method():
    """The same batch through the reference's own update_actor_critic (rl/algos/ppo.py:361-368), called unbound on the holder
    as tools/gen_golden_ppo.py does; the reference checkout wins where the two differ."""
    import sys
    import types
    from learninghumanoidwalking_b200.rl.ppo import PPO
    sys.modules.setdefault("ray", types.ModuleType("ray"))
    sys.path.insert(0, os.environ["LHW_REFERENCE"])
    try:
        from rl.algos import ppo as refppo
        for kind in ("ones", "mixed", "empty"):
            ppo, batch, *_ = _holder(0.7, kind)
            mine = [float(x) for x in PPO.update_actor_critic(ppo, *batch, 1)]
            ppo, batch, *_ = _holder(0.7, kind)
            ppo.recurrent = False
            theirs = [float(x) for x in refppo.PPO.update_actor_critic(ppo, *batch, 1)]
            assert abs(mine[5] - theirs[5]) < 1e-12 * max(1.0, abs(theirs[5])), (kind, mine[5], theirs[5])
    finally:
        sys.path.remove(os.environ["LHW_REFERENCE"])


def _teacher_file(tmp_path, env, obs_dim, act_dim, run="teacher_run"):
    from learninghumanoidwalking_b200.rl.policies import Gaussian_FF_Actor, export_module
    d = tmp_path / run
    d.mkdir()
    torch.save(export_module(Gaussian_FF_Actor(obs_dim, act_dim)), d / "actor_3.pt")
    with open(d / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env=env), f)
    return d / "actor_3.pt"


def test_check_teacher_reads_the_teacher_env(tmp_path):
    from learninghumanoidwalking_b200.rl.imitation import H1StandingProjector, IdentityProjector, check_teacher
    path = _teacher_file(tmp_path, "h1", 35, 10)
    module, env, proj = check_teacher(path, "h1_walk")
    assert env == "h1" and isinstance(proj, H1StandingProjector) and module.means.out_features == 10
    assert isinstance(check_teacher(path, "h1")[2], IdentityProjector)
    path = _teacher_file(tmp_path, "h1_walk", 43, 10, "walker")
    with pytest.raises(ValueError, match="h1_walk") as e:
        check_teacher(path, "h1")     # an h1_walk teacher would read task words an h1 student does not have
    assert str(path) in str(e.value)


def test_train_refuses_a_bad_teacher_before_any_run_directory(tmp_path):
    import run_experiment as rx
    logdir = tmp_path / "logs"
    with pytest.raises(SystemExit, match="does not exist") as e:
        rx.main(["train", "--env", "h1_walk", "--logdir", str(logdir), "--n-itr", "1", "--imitate", str(tmp_path / "nope.pt")])
    assert "nope.pt" in str(e.value) and "h1_walk" in str(e.value)
    path = _teacher_file(tmp_path, "jvrc_walk", 37, 12)
    with pytest.raises(SystemExit) as e:
        rx.main(["train", "--env", "jvrc_step", "--logdir", str(logdir), "--n-itr", "1", "--imitate", str(path), "--imitate-coeff", "1"])
    assert "jvrc_walk" in str(e.value) and "jvrc_step" in str(e.value) and str(path) in str(e.value)
    assert not logdir.exists()
    with pytest.raises(NotImplementedError):       # recurrent policies stay outside the build
        rx.main(["train", "--env", "jvrc_walk", "--logdir", str(logdir), "--n-itr", "1", "--recurrent"])


def test_a_run_directory_teacher_copy_names_the_teacher_env(tmp_path):
    """A student run's teacher.pt sits next to the student's experiment.pkl: its env is the recorded imitate_env."""
    from learninghumanoidwalking_b200.rl.imitation import H1StandingProjector, TEACHER_FILE, check_teacher, teacher_env_of
    from learninghumanoidwalking_b200.rl.policies import Gaussian_FF_Actor, export_module
    run = tmp_path / "student_run"
    run.mkdir()
    torch.save(export_module(Gaussian_FF_Actor(35, 10)), run / TEACHER_FILE)
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="h1_walk", imitate="/elsewhere/actor_1.pt", imitate_env="h1"), f)
    assert teacher_env_of(run / TEACHER_FILE) == "h1"
    assert isinstance(check_teacher(run / TEACHER_FILE, "h1_walk")[2], H1StandingProjector)
    with open(run / "experiment.pkl", "wb") as f:       # a teacher of unknown env: not the student's env either
        pickle.dump(Namespace(env="h1_walk", imitate="/elsewhere/actor_1.pt", imitate_env=None), f)
    assert teacher_env_of(run / TEACHER_FILE) is None


def test_float64_shadow_carries_the_teacher():
    """tools/learner_local_error.py's Shadow with a teacher: float64 and float32 agree, its imitation scalar is the formula,
    and without a teacher the shadow has no imitation attributes (its default path is the one it always was)."""
    from learninghumanoidwalking_b200.rl.imitation import H1StandingProjector
    from learninghumanoidwalking_b200.rl.policies import FF_V, Gaussian_FF_Actor
    from tools.learner_local_error import Shadow, offset_mean_
    torch.manual_seed(0)
    pol, cri, teacher = Gaussian_FF_Actor(43, 10, init_std=0.2), FF_V(43), Gaussian_FF_Actor(35, 10)
    with torch.no_grad():
        teacher.means.weight.mul_(30.0)
    old = Gaussian_FF_Actor(43, 10, init_std=0.2)
    old.load_state_dict(pol.state_dict())
    offset_mean_(old, 0)
    hyper = dict(lr=2e-4, eps=1e-6, clip=0.15, ent_coeff=0.01, mirror_coeff=0.0, max_grad_norm=0.05)
    B = 64
    obs = torch.randn(B, 43)
    obs[:, 37:40] = 0.0
    obs[::2, 39] = 1.0
    act, ret, adv = torch.randn(B, 10) * 0.2, torch.randn(B, 1), torch.randn(B, 1)
    kw = dict(teacher=teacher, projector=H1StandingProjector(), imitate_coeff=2.0)
    s64, s32 = Shadow(pol, old, cri, hyper, **kw), Shadow(pol, old, cri, hyper, dtype=torch.float32, **kw)
    assert s64.ppo.base_policy.means.weight.dtype == torch.float64 and not s64.ppo.base_policy.means.weight.requires_grad
    with torch.no_grad():
        mu, tau = pol(obs.double().float()).double(), teacher(obs[:, :35]).double()
    expect = float((((mu - tau) ** 2) * obs[:, 39:40].double()).mean())
    out64, g64, _ = s64.step(obs, act, ret, adv)
    out32, g32, _ = s32.step(obs, act, ret, adv)
    assert out64[5] > 0 and abs(out64[5] - expect) < 1e-6 * expect
    assert max(abs(a - b) / max(1.0, abs(b)) for a, b in zip(out32, out64)) < 1e-5
    plain = Shadow(pol, old, cri, hyper)
    assert "base_policy" not in plain.ppo.__dict__ and plain.ppo.imitate_coeff == 0.0
    assert plain.step(obs, act, ret, adv)[0][5] == 0.0
