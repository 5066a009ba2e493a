"""h1_walk on the device (Cfg<5, 3>: the H1 robot with the WalkingTask): fp64 kernel against oracle/, fp32 one control step at a
time, rendered images against the host build, all five variants interleaved, and train / resume / eval through run_experiment.py."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tools import fp32_local_error as L

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NQ, NV, NU = 17, 16, 10


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def test_h1_walk_fp64_closed_loop_matches_oracle():
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from h1_walk_oracle import H1WalkOracle
    o, n = H1WalkOracle(tolerance=1e-14), 16
    env = BatchedHumanoidEnv(n, model="h1_walk", precision=64, seed=21, first_env_id=7, max_traj_len=60, tolerance=1e-14)
    assert env.obs_dim == 43 and env.act_dim == NU
    envs = o.make_envs(n, seed=21, first_id=7)
    assert _rel(env.reset().cpu().numpy(), o.batch_reset(envs, n)) < 1e-9
    rng = np.random.RandomState(0)
    n_end = n_fall = 0
    pushed, worst = False, 0.0
    for k in range(300):
        a = rng.normal(size=(n, NU)) * 0.3
        o_obs, o_tobs, o_terms, o_rew, o_done, o_end = o.batch_step(envs, n, a, max_traj_len=60)
        g_obs, g_rew, g_done, g_end = env.step(torch.as_tensor(a, device="cuda", dtype=env.dtype))
        assert (g_done.cpu().numpy() == o_done).all() and (g_end.cpu().numpy() == o_end).all(), f"step {k}"
        oq = np.stack([o.field(envs, i, "qpos")[:NQ] for i in range(n)])
        ov = np.stack([o.field(envs, i, "qvel")[:NV] for i in range(n)])
        worst = max(worst, _rel(g_obs.cpu().numpy(), o_obs), _rel(g_rew.cpu().numpy(), o_rew),
                    _rel(env.rew_terms.cpu().numpy(), o_terms), _rel(env.qpos.cpu().numpy(), oq), _rel(env.qvel.cpu().numpy(), ov))
        x = np.stack([o.field(envs, i, "xfrc") for i in range(n)])
        pushed |= bool(np.any(x))
        assert np.abs(env.state_r[:, -12:].cpu().numpy() - x).max() < 1e-12
        assert (env.state_i[:, 1].cpu().numpy() == np.stack([o.field(envs, i, "mode")[0] for i in range(n)])).all()
        m = o_end.astype(bool)
        if m.any():
            keep = ~np.isnan(o_tobs[m])     # the oracle's terminal observation has no torque words (the env has been reset since)
            assert _rel(env.term_obs.cpu().numpy()[m][keep], o_tobs[m][keep]) < 1e-7
        n_end += int(m.sum()); n_fall += int(o_done.sum())
    assert n_fall > 0 and n_end > n_fall and pushed
    assert worst < 1e-7, worst
    env.close()


@pytest.mark.parametrize("regime", ["zero", "noisy"])
def test_h1_walk_fp32_device_one_step_error_against_fp64(regime):
    be = L.DeviceBackend("h1_walk", 100, seed=3, first_id=7)
    try:
        res = L.run(be, "h1_walk", 300, regime=regime)
    finally:
        be.close()
    n = res["env_steps"]
    print(f"\n[fp32 local error, device] h1_walk/{regime}: {n} env-steps, {res['ended']} ended ({res['falls']} falls), "
          f"exempt {len(res['exempt'])}, unexplained {len(res['fail'])}")
    assert not res["mismatch"], res["mismatch"][:5]
    # the shares test_gpu_fp32_local_error.py allows the other variants
    assert len(res["fail"]) <= {"zero": 3e-3, "noisy": 1e-3}[regime] * n, res["fail"][:5]
    assert len(res["exempt"]) + len(res["fail"]) <= {"zero": 0.1, "noisy": 0.01}[regime] * n
    for q, bound in (("qpos", 1e-6), ("qvel", 1e-5), ("obs", 1e-5), ("reward", 1e-5)):
        assert np.median(res["errors"][q]) < bound, (q, np.median(res["errors"][q]))


@pytest.mark.parametrize("precision", [64, 32])
def test_h1_walk_device_images_match_host_build(precision):
    from emu_variants import RenderEmu
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.model import load_model, pack_model
    env = BatchedHumanoidEnv(8, model="h1_walk", precision=precision, seed=3)
    env.reset()
    g = torch.Generator(device=env.device).manual_seed(0)
    for _ in range(5):
        env.step(0.3 * torch.randn(8, env.act_dim, generator=g, device=env.device, dtype=env.dtype))
    dev = env.render_rgb(list(range(8)), 320, 240).cpu().numpy()
    host = RenderEmu(pack_model(load_model("h1_walk")), precision)
    sr, si = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
    for k in range(8):
        ref, _ = host.image(sr[k], si[k], 320, 240, (0.0, 0.0, 0.9, 3.0, 90.0, 15.0, 45.0))
        diff = np.abs(dev[k].astype(int) - ref.astype(int)).max(-1)
        assert (diff > 0).mean() <= 0.001 and diff.max() <= 2, (k, int((diff > 0).sum()), int(diff.max()))
    env.close()


def test_all_five_variants_interleaved_step_as_alone():
    """h1 and h1_walk sims of one precision take turns in the same constant-bank objects (sim_kernels.cu bank_tk)."""
    from test_gpu_variant_bookkeeping import MODELS, RISING, STEPS, _advance, _alone, _env, _same
    specs = [(m, p) for m in MODELS + ("h1_walk",) for p in (64, 32)]
    alone = [_alone(m, p) for m, p in specs]
    envs = [_env(m, p) for m, p in specs]
    for k in range(STEPS):
        for i, (m, p) in enumerate(specs):
            assert _same(_advance(envs[i], k, RISING), alone[i][k]), (m, p, k)
    for env in envs:
        env.close()


def _cli(*argv):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "run_experiment.py")] + list(argv), capture_output=True, text=True,
                         timeout=1200, env=dict(os.environ, LHW_TENSORBOARD="0"))
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout


def _weights(path):
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()      # the checkpoints pickle the reference's module names
    return torch.load(path, weights_only=False).state_dict()


def test_run_experiment_trains_h1_walk_with_the_mirror_loss(tmp_path):
    """`train --env h1_walk --num-procs 1024 --n-itr 2` wraps the env in SymmetricEnv (the mirror loss is on) and two runs with
    the same seed end with bit-identical weights."""
    runs = []
    for tag in ("a", "b"):
        out = _cli("train", "--env", "h1_walk", "--logdir", str(tmp_path / tag), "--num-procs", "1024", "--n-itr", "2", "--seed", "5")
        assert "Wrapping in SymmetricEnv." in out
        (run,) = list((tmp_path / tag).iterdir())
        runs.append(run)
    for name in ("actor.pt", "critic.pt"):
        sa, sb = _weights(runs[0] / name), _weights(runs[1] / name)
        assert list(sa) == list(sb) and all(torch.equal(sa[k], sb[k]) for k in sa), name


def test_run_experiment_resume_and_eval_h1_walk(tmp_path):
    """`resume` after 2 of 4 iterations ends bit-identical to the straight run, and `eval --out-dir` writes the roll-out video."""
    train = ["--env", "h1_walk", "--num-procs", "256", "--max-traj-len", "40", "--minibatch-size", "1024", "--epochs", "1",
             "--seed", "3", "--eval-freq", "2", "--snapshot"]
    _cli("train", "--logdir", str(tmp_path / "a"), "--n-itr", "4", *train)
    _cli("train", "--logdir", str(tmp_path / "b"), "--n-itr", "2", *train)
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    assert "Resuming" in _cli("resume", "--path", str(run_b), "--n-itr", "4")
    for name in ("actor.pt", "critic.pt", "actor_3.pt"):
        sa, sb = _weights(run_a / name), _weights(run_b / name)
        assert all(torch.equal(sa[k], sb[k]) for k in sa), name
    la = torch.load(run_a / "snapshot" / "itr_3" / "learner.pt", weights_only=True)
    lb = torch.load(run_b / "snapshot" / "itr_3" / "learner.pt", weights_only=True)
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert torch.equal(la[k], lb[k]), k
    out = tmp_path / "video"
    _cli("eval", "--logdir", str(tmp_path / "a"), "--ep-len", "2", "--out-dir", str(out))
    videos = list(out.iterdir())
    assert len(videos) == 1 and videos[0].suffix == ".mp4" and videos[0].stat().st_size > 1000
