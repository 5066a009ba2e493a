"""The fp32 device kernel held to the fp64 device kernel ONE control step at a time (tools/fp32_local_error.py), plus the
diverged-environment path on the device.

Three BatchedHumanoidEnvs per role (fp64 driver, fp64 shadow, fp32) and a fp64 one for the perturbation control; the records are
copied in before every step.  100 environments give ragged lock-step blocks in both precisions (14 fp32 / 8 or 7 fp64 warps per
block).  Same bounds and classifier as the CPU tier (test_fp32_local_error.py)."""
import numpy as np
import pytest
import torch

from tools import fp32_local_error as L

pytestmark = pytest.mark.gpu

N_ENVS, STEPS = 100, 300
# exempt steps allowed, as a share of env-steps.  Standing still keeps foot corners resting AT the ground, where every substep
# takes a contact decision within rounding distance of the threshold (emulation: up to 8 % for jvrc_step at a = 0)
EXEMPT_SHARE = {"zero": 0.1, "noisy": 0.01, "trained": 0.01}
# At 30000 env-steps per case the control's four random copies do not always move the corner whose contact decision fp32 took
# within rounding distance of the ground (measured: a few per case, each a contact-set switch).  A defect shows on most steps
# (a reward coefficient off by 1e-3 in fp32 leaves most steps unexplained), so the unexplained share is bounded instead of zero.
# Standing still, the environments sit in nearly the same state, so one such decision repeats across many of them (measured
# 58 of 30000 for jvrc_step at a = 0, at most 17 elsewhere).
UNEXPLAINED_SHARE = {"zero": 3e-3, "noisy": 1e-3, "trained": 1e-3}


def _check(model, regime, res):
    n = res["env_steps"]
    print(f"\n[fp32 local error, device] {model}/{regime}: {n} env-steps, {res['ended']} ended ({res['falls']} falls), "
          f"exempt {len(res['exempt'])}, unexplained {len(res['fail'])}")
    for r in res["fail"]:
        print("   unexplained: step %d env %d %s fp32 %.1e fp64 copies %.1e" % r)
    for q in ("qpos", "qvel", "obs", "reward"):
        v = res["errors"][q]
        print(f"   {q:7s} median {np.median(v):.1e} p99 {np.percentile(v, 99):.1e} p99.9 {np.percentile(v, 99.9):.1e} max {v.max():.1e}")
    assert not res["mismatch"], res["mismatch"][:5]
    assert len(res["fail"]) <= UNEXPLAINED_SHARE[regime] * n, "; ".join("step %d env %d %s fp32 %.1e fp64 copies %.1e" % r for r in res["fail"][:5])
    assert len(res["exempt"]) + len(res["fail"]) <= EXEMPT_SHARE[regime] * n, (len(res["exempt"]), len(res["fail"]))
    for q, bound in (("qpos", 1e-6), ("qvel", 1e-5), ("obs", 1e-5), ("reward", 1e-5)):
        assert np.median(res["errors"][q]) < bound, (q, np.median(res["errors"][q]))


@pytest.mark.parametrize("regime", ["zero", "noisy"])
@pytest.mark.parametrize("model", L.VARIANTS)
def test_fp32_device_one_step_error_against_fp64(model, regime):
    be = L.DeviceBackend(model, N_ENVS, seed=3, first_id=7)
    try:
        res = L.run(be, model, STEPS, regime=regime)
    finally:
        be.close()
    _check(model, regime, res)
    if regime == "noisy":
        assert res["falls"] > 0
        if model != "h1":                # H1 under this policy falls before the 40-step truncation
            assert res["ended"] > res["falls"], "no truncation"


def test_fp32_device_one_step_error_under_the_trained_walking_policy():
    be = L.DeviceBackend("jvrc_walk", N_ENVS, seed=3, first_id=7)
    try:
        res = L.run(be, "jvrc_walk", STEPS, regime="trained")
    finally:
        be.close()
    _check("jvrc_walk", "trained", res)


@pytest.mark.parametrize("model", L.VARIANTS)
def test_fp32_device_kernel_matches_its_source(model):
    """The compiled fp32 kernel against the fp32 kernel source on the host (tests/emu), one step from the same record: equal up
    to FMA contraction and rsqrtf (the host computes 1/sqrtf), so the same bounds and classifier apply; flags and integer state
    are equal."""
    n = 32
    be, src = L.DeviceBackend(model, n, seed=3, first_id=7), L.EmulationBackend(model, n, seed=3, first_id=7)
    try:
        res = L.run(be, model, 60, regime="noisy", compare_source=src)
    finally:
        be.close()
    v = res["source"]
    print(f"\n[fp32 device vs source] {model}: " + "  ".join(f"{q} median {np.median(v[q]):.1e} max {np.nanmax(v[q]):.1e}"
                                                           for q in ("qpos", "qvel", "obs", "reward")))
    assert not res["mismatch"], res["mismatch"][:5]
    for q, bound in (("qpos", 1e-6), ("qvel", 1e-5), ("obs", 1e-5), ("reward", 1e-5)):
        assert np.median(v[q]) < bound, (q, np.median(v[q]))
    over = np.zeros(res["env_steps"], bool)
    for q in ("qpos", "qvel", "obs", "reward", "rew_terms", "record"):
        over |= np.nan_to_num(v[q]) > L.BOUNDS[q]
    assert over.mean() <= 0.02, over.mean()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("model", L.VARIANTS)
@pytest.mark.parametrize("poison", ["nan", "nan_pose", "runaway"])
def test_diverged_environment_on_the_device(model, precision, poison):
    """An environment whose state has gone non-finite or runaway, inside a lock-step block of healthy ones: it gets a status
    word and done = ended = 1; with auto-reset it comes back with the fresh episode's observation (the same as the kernel source
    gives from the same record) and status / traj_len cleared; its block neighbours are bit-identical to an unpoisoned run."""
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    n, bad = 16, 3                       # env 3 shares its block with envs 0..13 (fp32) / 0..7 (fp64)
    mk = lambda: BatchedHumanoidEnv(n, model=model, precision=precision, seed=9, first_env_id=4)
    env, clean = mk(), mk()
    env.reset(); clean.reset()
    g = torch.Generator(device="cuda").manual_seed(3)
    for _ in range(3):
        a = torch.randn(n, env.act_dim, device="cuda", generator=g, dtype=env.dtype) * 0.2
        env.step(a); clean.step(a)
    nq = env.nq
    if poison == "nan":
        env.state_r[bad, nq + 7] = float("nan")
    elif poison == "nan_pose":
        env.state_r[bad, 9] = float("nan")
    else:
        env.state_r[bad, nq + 6:nq + env.nv] = 1e13
    sr0, si0 = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
    csr0, csi0 = clean.state_r.clone(), clean.state_i.clone()
    a = torch.randn(n, env.act_dim, device="cuda", generator=g, dtype=env.dtype) * 0.2
    keep = [i for i in range(n) if i != bad]
    # (1) without auto-reset: the status word survives the launch
    env.step(a, autoreset=False)
    clean.step(a, autoreset=False)
    assert env.done[bad].item() == 1 and env.ended[bad].item() == 1
    assert env.status_flags()[bad].item() != 0
    assert torch.equal(env.state_r[keep], clean.state_r[keep]) and torch.equal(env.obs[keep], clean.obs[keep])
    assert torch.equal(env.reward[keep], clean.reward[keep]) and torch.equal(env.state_i[keep, :7], clean.state_i[keep, :7])
    # (2) with auto-reset, from the same poisoned record
    from learninghumanoidwalking_b200.model import pack_model
    from emu import Emu
    env.state_r.copy_(torch.from_numpy(sr0)); env.state_i.copy_(torch.from_numpy(si0))
    clean.state_r.copy_(csr0); clean.state_i.copy_(csi0)
    obs, rew, done, ended = env.step(a)
    assert done[bad].item() == 1 and ended[bad].item() == 1
    assert torch.isfinite(obs[bad]).all()
    assert env.status_flags()[bad].item() == 0 and env.state_i[bad, 2].item() == 0
    tol = 1e-5 if precision == 32 else 1e-9
    e = Emu(pack_model(env.mj, tolerance=1e-6 if precision == 32 else None), precision, 1, seed=9, first_id=4 + bad)
    e.sr[0], e.si[0] = sr0[bad], si0[bad]
    eo = e.step(a[bad:bad + 1].cpu().numpy())
    assert eo[4][0] == 1 and eo[5][0] == 1
    assert np.abs(obs[bad].double().cpu().numpy() - eo[0][0]).max() < tol
    co = clean.step(a)
    assert torch.equal(obs[keep], co[0][keep]) and torch.equal(env.state_r[keep], clean.state_r[keep])
    env.close(); clean.close()
