"""The float64 shadow of tools/learner_local_error.py on the CPU.  tests/test_gpu_learner_local_error.py holds the CUDA learner
to that shadow; here the shadow's exact configuration (float64 networks, hand-made torch Adam, the non-fused branch of
PPO.update_actor_critic, every lhw entry point refused) is pinned to tests/golden/ppo_update.json, the vectors of the reference's
own PPO.update_actor_critic that tests/test_ppo_update_golden.py holds the float32 method to, and the tool's float64 parts run
end to end at a tiny size."""
import os
from copy import deepcopy

import numpy as np
import pytest
import torch

from test_ppo_update_golden import G, _batch, _formula_weights_


def test_float64_shadow_matches_the_reference_method():
    from learninghumanoidwalking_b200.envs.batched_env import BatchedHumanoidEnv  # noqa: F401  (import only: no CUDA needed)
    from learninghumanoidwalking_b200.rl.policies import FF_V, Gaussian_FF_Actor
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    from tools.learner_local_error import Shadow
    h = G["hyper"]
    # the networks, normalisation and mirror lists of test_update_actor_critic_matches_the_reference_method
    policy, critic = Gaussian_FF_Actor(37, 12, init_std=0.223, learn_std=False), FF_V(37)
    _formula_weights_(policy, 0.0)
    _formula_weights_(critic, 3.0)
    old_policy = deepcopy(policy)
    _formula_weights_(policy, 0.02)
    obs_mean = 0.1 * torch.sin(torch.arange(37, dtype=torch.float32))
    obs_std = 1.0 + 0.5 * torch.cos(torch.arange(37, dtype=torch.float32)) ** 2
    for net in (policy, old_policy, critic):
        net.obs_mean, net.obs_std = obs_mean, obs_std
    mirrored_obs = [-0.1, 1, -2, 3, -4, 11, -12, -13, 14, -15, 16, 5, -6, -7, 8, -9, 10,
                    23, -24, -25, 26, -27, 28, 17, -18, -19, 20, -21, 22] + list(range(29, 37))
    sym = SymmetricEnv(lambda: object(), mirrored_obs=mirrored_obs, mirrored_act=[6, -7, -8, 9, -10, 11, 0.1, -1, -2, 3, -4, 5],
                       clock_inds=[29, 30])
    sh = Shadow(policy, old_policy, critic, dict(lr=h["lr"], eps=h["eps"], clip=h["clip"], ent_coeff=h["ent_coeff"],
                                                 mirror_coeff=h["mirror_coeff"], max_grad_norm=h["grad_clip"]), sym)
    assert all(p.dtype == torch.float64 for p in sh.params())
    obs, act, ret, adv = _batch(h["B"])
    for ref in G["steps"]:
        got = sh.step(obs, act, ret, adv)[0]
        assert len(got) == 7
        for name, a, b in zip(G["names"], got, ref):
            assert abs(a - b) <= 2e-5 * max(1.0, abs(b)), (name, a, b)
    for module, digest in ((sh.policy, G["actor"]), (sh.critic, G["critic"])):
        for p, d in zip(module.parameters(), digest):
            p = p.detach()
            assert abs(float(p.sum()) - d["sum"]) < 1e-4 * max(1.0, d["abs"] * 1e-2)
            assert abs(float(p.abs().sum()) - d["abs"]) < 1e-5 * max(1.0, d["abs"])
            assert np.abs(p.reshape(-1)[:8].numpy() - np.array(d["head"])).max() < 2e-6


def test_learner_local_error_rehearsal_on_the_cpu():
    """The tool's float64 parts without a device: its vectorised GAE against ppo_oracle.gae_rollout, and a float64 shadow step
    under the lhw guard against the same step in float32."""
    from learninghumanoidwalking_b200 import _lib
    from tools.learner_local_error import no_lhw, rehearse
    r = rehearse()
    assert r["gae"] < 1e-12 and r["grads"] == 12
    assert r["scalars"] < 1e-5 and r["norms"] < 1e-5
    with no_lhw(), pytest.raises(AssertionError, match="lhw entry point"):
        _lib.ops()
    assert os.environ.get("LHW_FUSED_LOSS") != "0"
    assert _lib.ops.__name__ == "ops"      # the guard put the real entry point back
