"""The compiled fp64 kernel, whose Newton Hessian is assembled on the fp64 tensor cores (mma.sync m8n8k4), held
to its source compiled for the host (tests/emu), one control step at a time from the same record, for every variant.  The DMMA's
internal rounding order is not specified and the device contracts to FMA, so the two agree to fp64 rounding, not bit for bit."""
import os
import sys

import numpy as np
import pytest
import torch

from tools import fp32_local_error as L

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
VARIANTS = ("jvrc_walk", "h1", "jvrc_step", "jvrc_walk_terrain", "h1_walk")
N, STEPS, MAX_TRAJ_LEN = 64, 60, 40
BOUND = 1e-10          # relative to max(1, |value|), per env and control step, on qpos and qvel
OVER_SHARE = 0.02      # env-steps allowed above it: a contact decision within rounding distance of its threshold


@pytest.mark.parametrize("model", VARIANTS)
def test_fp64_device_kernel_matches_its_source(model):
    sys.path[:0] = [p for p in (os.path.join(HERE, "emu"),) if p not in sys.path]
    from emu_variants import Emu
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.model import load_model, pack_model
    env = BatchedHumanoidEnv(N, model=model, precision=64, seed=3, first_env_id=7, max_traj_len=MAX_TRAJ_LEN)
    src = Emu(pack_model(load_model(model)), 64, N, seed=3, first_id=7)
    try:
        env.reset()
        lay = L.layout(src.nq, src.nv, src.nu, src.nr, model)
        pol = L.noisy_policy(src.nobs, src.nu, np.random.RandomState(0))
        err = {"qpos": [], "qvel": []}
        for _ in range(STEPS):
            src.sr[:] = env.state_r.cpu().numpy()
            src.si[:] = env.state_i.cpu().numpy()
            a = pol(env.obs.cpu().numpy())
            env.step(torch.from_numpy(a).to(device=env.device, dtype=env.dtype))
            o = src.step(a, max_traj_len=MAX_TRAJ_LEN)
            assert (env.done.cpu().numpy() == o[4]).all() and (env.ended.cpu().numpy() == o[5]).all()
            dev = env.state_r.cpu().numpy()
            for q in err:
                err[q].append(L._rel(dev[:, lay[q]], src.sr[:, lay[q]]))
    finally:
        env.close()
    for q, e in err.items():
        e = np.concatenate(e)
        print(f"\n[fp64 device vs source] {model} {q}: median {np.median(e):.1e} max {e.max():.1e}")
        assert np.isfinite(e).all()
        assert np.median(e) < BOUND, (q, np.median(e))
        assert (e > BOUND).mean() <= OVER_SHARE, (q, (e > BOUND).mean())
