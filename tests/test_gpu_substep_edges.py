"""The device build of one physics substep (sim_core.h substep, through the harness tests/dev/substep_dev.cu) at crafted contact,
limit and friction-loss states, against the float64 oracle, with no exempt share: every case of tests/dev/substep_cases.py
reaches its branch and agrees with oracle/ after 1 and after frame_skip substeps.

- fp64 with the solver tolerance at 1e-14 (as tests/test_gpu_parity.py): qpos to 1e-11 and qvel to 1e-10 (the CPU tier's
  bounds), qacc to 1e-7 of max(1, max |ref|), act_force, grf, cz_min, foot and root velocities, the contact points of each foot
  (coplanar duplicates merged), status 0; M against Oracle.mass_matrix and qfs against the oracle's smooth force
  -bias - damping qvel + ctrl where the oracle can build them (not for the H1 variants, whose per-env masses the oracle's
  building blocks do not take).  P12 copies M before it adds the damping, and leaves qfs alone, so both are the last substep's.
- fp32 at the trainer's default tolerance (1e-6) against the oracle started from the fp32-rounded state: DESIGN §2's one-step bound,
  1e-4 relative on qpos, qvel and qacc, and the same contact points.
- The product's lock-step launch (8 or 7 warps per block at fp64, 14 at fp32) with the cases mixed in its blocks and a ragged last
  block equals the one-warp launch bit for bit.
- The shipped kernel (step_kernel_mw through torch.ops.lhw) takes one control step from every crafted state, held to orc_step."""
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "dev"))
import substep_cases as C  # noqa: E402

pytestmark = pytest.mark.gpu
VARIANTS = list(C.NAMES.values())
CASES = [(name, cid) for name in VARIANTS for cid in C.case_ids(name)]


@pytest.fixture(scope="module")
def devs():
    import torch
    torch.cuda.init()
    hs = {}
    yield lambda name, prec: hs.setdefault((name, prec), C.Harness(C.twin_flat(name, prec), prec, device=True))
    for h in hs.values():
        h.close()


@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("name,cid", CASES, ids=[f"{n}-{c}" for n, c in CASES])
def test_device_substep_against_the_oracle(devs, name, cid, prec):
    print(f"\n[device {name} fp{prec} {cid}] " + C.run_case(devs(name, prec), name, prec, cid))


@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_lock_step_blocks_equal_one_warp_blocks(devs, name, prec):
    """All of a variant's cases in one batch (different cases side by side in a block), launched with one warp per block and with
    the product's warps per block (the last block ragged): records and Work fields bit for bit."""
    H = devs(name, prec)
    code = C.CODE[name]
    states = [s for cid in C.case_ids(name) for s in C.case_states(name, prec, cid)[0]]
    wpb = C.product_warps(prec, code)
    while len(states) % wpb == 0 or len(states) < wpb + 1:
        states = states + states[:1]
    sr, si, ctrl = C.records(code, prec, states)
    for nsub in (1, int(C.model(name)[0]["cfg"]["frame_skip"])):
        a = H.run(sr, si, ctrl, nsub, 1)
        b = H.run(sr, si, ctrl, nsub, wpb)
        assert np.array_equal(a[0].view(np.uint8), b[0].view(np.uint8)) and np.array_equal(a[1], b[1])
        for wa, wb in zip(a[2], b[2]):
            fa, fb = H.fields(wa), H.fields(wb)
            for k in ("qpos", "qvel", "qacc", "qfs", "M", "ncon", "lside", "grf", "foot_vel", "root_vlin"):
                assert np.array_equal(np.asarray(fa[k]).view(np.uint8), np.asarray(fb[k]).view(np.uint8)), (name, prec, nsub, k)
            cpf = C.CPF[code]
            for ch in range(2):   # the slots in use (the others keep whatever the shared memory held)
                used = slice(ch * cpf, ch * cpf + int(fa["ncon"][ch]))
                assert np.array_equal(fa["cpos"][used].view(np.uint8), fb["cpos"][used].view(np.uint8)), (name, prec, nsub, "cpos")


@pytest.mark.parametrize("prec", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_shipped_kernel_control_step_at_the_crafted_states(name, prec):
    """The shipped kernel at the same states: every crafted state written into a BatchedHumanoidEnv as the start of an episode, one
    control step through torch.ops.lhw (step_kernel_mw, the product's warps per block, auto-reset on), held to the oracle's
    orc_step from the same (at fp32: fp32-rounded) state.  fp64 (tolerance 1e-14): obs, reward, qpos and qvel to 1e-7 of
    max(1, |ref|), the bound of tests/test_gpu_parity.py; fp32 (the trainer's tolerance): DESIGN §2's one-step bound, 1e-4.
    done must be equal."""
    import torch
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    states, acts = C.control_step_states(name, prec)
    n = len(states)
    sr, si = C.kernel_records(name, prec, states)
    env = BatchedHumanoidEnv(n, model=name, precision=prec, seed=C.SEED, first_env_id=0, max_traj_len=400,
                             tolerance=1e-14 if prec == 64 else None)
    env.reset()
    env.state_r.copy_(torch.as_tensor(sr, dtype=env.dtype))
    env.state_i.copy_(torch.as_tensor(si))
    obs, rew, done, _ = env.step(torch.as_tensor(acts, device="cuda", dtype=env.dtype))
    torch.cuda.synchronize()
    oo, orew, od, oq, ov = C.oracle_control_step(name, states, acts)
    rel = lambda a, b: float(np.max(np.abs(a - b) / np.maximum(1.0, np.abs(b))))
    nq, nv = oq.shape[1], ov.shape[1]
    rec = env.state_r.double().cpu().numpy()
    err = dict(obs=rel(obs.double().cpu().numpy(), oo), reward=rel(rew.double().cpu().numpy(), orew),
               qpos=rel(rec[:, :nq], oq), qvel=rel(rec[:, nq:nq + nv], ov))
    env.close()
    assert (done.cpu().numpy() == od).all(), (done.cpu().numpy(), od)
    bound = 1e-7 if prec == 64 else 1e-4
    print(f"\n[shipped {name} fp{prec}, {n} states] " + " ".join(f"{k} {v / bound:.2g}" for k, v in err.items()))
    assert all(v <= bound for v in err.values()), err
