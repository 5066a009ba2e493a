"""Imitation on the GPU: torch.ops.lhw.ppo_loss_imitation (csrc/ppo_kernels.cu, ppo_loss_kernel<true>) against the closed-form
oracle, the fused learner against the torch loss graph with a teacher, and `train --imitate` end to end: logging, the captured
update graph, the teacher copy in the run directory, a zero coefficient, learning from the teacher, resume and two ranks."""
import math
import os
import pickle
import re
import subprocess
import sys
from argparse import Namespace
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
JVRC_TEACHER = os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")   # no experiment.pkl: the identity by width


def _lib():
    from learninghumanoidwalking_b200 import _lib
    return _lib


def _oracle(mu, old_mu, act, adv, ret, val, mirr, stds, teacher, mask, clip, mirror_coeff, ent_coeff, imitate_coeff):
    """oracle/ppo_oracle.py: ppo_loss_and_grads plus the imitation term, float64: imitation = mean over B*A of
    m_b (mu - teacher)^2, total += imitate_coeff * imitation, g_mu += imitate_coeff * 2 m_b (mu - teacher) / (B*A)."""
    from oracle.ppo_oracle import ppo_loss_and_grads
    out8, g_mu, g_mirr, g_val = ppo_loss_and_grads(mu, old_mu, act, adv, ret, val, mirr, stds, clip, mirror_coeff, ent_coeff)
    B, A = mu.shape
    m = np.ones(B) if mask is None else np.asarray(mask, dtype=np.float64).reshape(-1)
    d = np.asarray(mu, dtype=np.float64) - np.asarray(teacher, dtype=np.float64)
    imitation = (m[:, None] * d * d).sum() / (B * A)
    out8 = out8.copy()
    out8[5] = imitation
    out8[7] += imitate_coeff * imitation
    return out8, g_mu + imitate_coeff * 2 * m[:, None] * d / (B * A), g_mirr, g_val


def _bufs(B, A):
    L = _lib()
    return (torch.empty(B, A, device="cuda"), torch.empty(B, A, device="cuda"), torch.empty(B, 1, device="cuda"),
            torch.zeros(L.lib().lhw_ppo_loss_partial_words(B), dtype=torch.float64, device="cuda"),
            torch.zeros(1, dtype=torch.int32, device="cuda"), torch.zeros(8, device="cuda"))


def test_ppo_loss_imitation_matches_the_closed_form_oracle():
    """Over B x A x mask x mirror, in the manner (and with the bounds) of test_gpu_ppo.py's ppo_loss check.  Where the mask is
    all zero or the coefficient is 0, g_mu / g_mirr / g_val equal ppo_loss's exactly."""
    L = _lib()
    rng = np.random.RandomState(5)
    d = lambda a: None if a is None else torch.as_tensor(np.ascontiguousarray(a), device="cuda")
    for B in (1, 255, 256, 257, 21845):
        for A in (10, 12):
            stds = np.full(A, 0.223, dtype=np.float32)
            mu = (rng.normal(size=(B, A)) * 0.2).astype(np.float32)
            old_mu = (mu + rng.normal(size=(B, A)) * 0.05).astype(np.float32)
            act = (old_mu + rng.normal(size=(B, A)) * 0.223).astype(np.float32)
            adv, ret, val = (rng.normal(size=(B, 1)).astype(np.float32) for _ in range(3))
            teacher = (mu + rng.normal(size=(B, A)) * 0.1).astype(np.float32)
            mixed = (rng.uniform(size=(B, 1)) < 0.4).astype(np.float32)
            mixed[0] = 1.0
            masks = {"none": None, "zero": np.zeros((B, 1), np.float32), "mixed": mixed}
            for with_mirr in (True, False):
                mirr = (mu + rng.normal(size=(B, A)) * 0.05).astype(np.float32) if with_mirr else None
                base = _bufs(B, A)
                L.ops().ppo_loss(d(mu), d(old_mu), d(act), d(adv), d(ret), d(val), d(mirr), d(stds), 0.2, 0.4, 0.01, base[0],
                                 base[1] if with_mirr else None, base[2], base[3], base[4], base[5])
                for kind, mask in masks.items():
                    for coeff in (1.5, 0.0):
                        g_mu, g_mirr, g_val, part, ticket, out8 = bufs = _bufs(B, A)
                        for _ in range(2):      # twice: the ticket counter must come back to zero
                            L.ops().ppo_loss_imitation(d(mu), d(old_mu), d(act), d(adv), d(ret), d(val), d(mirr), d(stds), d(teacher),
                                                       d(mask), 0.2, 0.4, 0.01, coeff, g_mu, g_mirr if with_mirr else None, g_val,
                                                       part, ticket, out8)
                        exp = _oracle(mu, old_mu, act, adv, ret, val, mirr, stds, teacher, mask, 0.2, 0.4, 0.01, coeff)
                        case = (B, A, kind, with_mirr, coeff)
                        assert int(ticket.item()) == 0, case
                        assert np.abs(out8.cpu().numpy() - exp[0]).max() < 2e-5, (case, out8, exp[0])
                        assert np.abs(g_mu.cpu().numpy() - exp[1]).max() < 1e-6 * max(1.0, np.abs(exp[1]).max() * B), case
                        assert np.abs(g_mu.cpu().numpy() - exp[1]).max() < 2e-5 * np.abs(exp[1]).max() + 1e-12, case
                        assert np.abs(g_val.cpu().numpy().reshape(-1) - exp[3]).max() < 2e-6 * np.abs(exp[3]).max() + 1e-12, case
                        if with_mirr:
                            assert np.abs(g_mirr.cpu().numpy() - exp[2]).max() < 2e-6 * np.abs(exp[2]).max() + 1e-12, case
                        if kind == "zero" or coeff == 0.0:
                            assert torch.equal(g_mu, base[0]) and torch.equal(g_val, base[2]), case
                            if with_mirr:
                                assert torch.equal(g_mirr, base[1]), case
                        if kind == "zero":
                            assert out8[5].item() == 0.0, case
                        else:
                            assert out8[5].item() > 0, case


def test_ppo_loss_imitation_rejects_bad_tensors():
    L = _lib()
    B, A = 300, 12
    x = torch.zeros(B, A, device="cuda")
    v = torch.zeros(B, 1, device="cuda")
    s = torch.full((A,), 0.2, device="cuda")
    g_mu, g_mirr, g_val, part, ticket, out8 = _bufs(B, A)
    call = lambda teacher, mask: L.ops().ppo_loss_imitation(x, x, x, v, v, v, None, s, teacher, mask, 0.2, 0.4, 0.0, 1.0, g_mu, None,
                                                            g_val, part, ticket, out8)
    call(x, v)
    for teacher, mask, msg in ((torch.zeros(B, A - 1, device="cuda"), None, "teacher_mu has shape"),
                               (torch.zeros(B, A, device="cuda", dtype=torch.float64), None, "teacher_mu has dtype"),
                               (torch.zeros(B, A), None, "teacher_mu must be a CUDA tensor"),
                               (x.t().contiguous().t(), None, "teacher_mu must be contiguous"),
                               (x, torch.zeros(B - 1, 1, device="cuda"), "mask must hold one value per sample"),
                               (x, torch.zeros(B, 1, device="cuda", dtype=torch.int32), "mask has dtype")):
        with pytest.raises(RuntimeError, match=msg):
            call(teacher, mask)
    with pytest.raises(RuntimeError, match="old_mu has shape"):      # ppo_loss's own checks come first
        L.ops().ppo_loss_imitation(x, x[:5], x, v, v, v, None, s, x, None, 0.2, 0.4, 0.0, 1.0, g_mu, None, g_val, part, ticket, out8)


# ------------------------------------------------------------------------------------------------------------ the learner
def _args(logdir, **kw):
    d = dict(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=256, epochs=1,
             max_traj_len=50, num_procs=64, max_grad_norm=0.05, mirror_coeff=0.4, eval_freq=2, recurrent=False,
             imitate_coeff=0.0, std_dev=0.223, learn_std=False, logdir=str(logdir), steps_per_env=20)
    d.update(kw)
    return SimpleNamespace(**d)


def _env_fn(model, seed=7):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(64, model=model, precision=32, seed=seed)
    probe = base()
    r = probe.robot
    probe.close()
    if not hasattr(r, "mirrored_obs"):
        return base
    return lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)


def _h1_teacher(tmp_path):
    """A saved h1 actor (random weights, h1's normalisation) next to an experiment.pkl that names its env."""
    from learninghumanoidwalking_b200.rl.policies import Gaussian_FF_Actor, export_module
    d = tmp_path / "h1_teacher"
    d.mkdir(exist_ok=True)
    torch.manual_seed(123)
    actor = Gaussian_FF_Actor(35, 10)
    with torch.no_grad():
        actor.means.weight.mul_(30.0)       # actions of the size a trained policy gives
    torch.save(export_module(actor), d / "actor_9.pt")
    with open(d / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="h1"), f)
    return str(d / "actor_9.pt")


def _close(ppo):
    ppo.env.close()
    if ppo._comm is not None:
        ppo._comm.close()


@pytest.mark.parametrize("pair", ["jvrc_walk", "h1_to_h1_walk"])
def test_fused_imitation_matches_the_torch_loss_graph(tmp_path, monkeypatch, pair):
    """LHW_FUSED_LOSS=1 (one launch of ppo_loss_kernel<true>) against =0 (the torch graph of update_actor_critic) with a
    teacher: the 7 scalars and the weights after one and two optimiser steps on rollout data."""
    from learninghumanoidwalking_b200.rl import PPO
    model, teacher = ("jvrc_walk", JVRC_TEACHER) if pair == "jvrc_walk" else ("h1_walk", _h1_teacher(tmp_path))
    res = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("LHW_FUSED_LOSS", mode)
        monkeypatch.setenv("LHW_UPDATE_GRAPH", "0")
        ppo = PPO(_env_fn(model, seed=8), _args(tmp_path, imitate=teacher, imitate_coeff=2.0), seed=8)
        assert ppo.base_policy is not None
        ppo.make_optimizers()
        batch = ppo.sample_parallel_with_workers()
        adv = ppo.normalize_advantages(batch.returns.contiguous(), batch.values.contiguous())
        env = ppo.env
        mo, ma = getattr(env, "mirror_clock_observation", None), getattr(env, "mirror_action", None)
        outs = []
        for k in range(2):
            sl = slice(300 * k, 300 * k + 300)
            o = ppo.update_actor_critic(batch.states[sl].contiguous(), batch.actions[sl].contiguous(), batch.returns[sl].contiguous(),
                                        (adv[sl] * (3.0 if k else 1.0)).contiguous(), 1, mirror_observation=mo, mirror_action=ma)
            outs.append(torch.stack([x.float() for x in o]).cpu())
        if pair != "jvrc_walk":
            standing = batch.states[:600, 39]
            assert 0 < standing.sum().item() < 600          # both kinds of samples are in the two minibatches
        res[mode] = (outs, ppo._flat_param.clone().cpu())
        _close(ppo)
    for a, b in zip(res["0"][0], res["1"][0]):
        assert (a - b).abs().max().item() < 2e-5 * max(1.0, a.abs().max().item()), (a, b)
        assert b[5] > 0
    assert (res["0"][1] - res["1"][1]).abs().max().item() < 2e-6


def _imitation_lines(out):
    return [float(v) for v in re.findall(r"\|\s+Imitation loss\s+\|\s+([\d.e+-]+|nan|inf)\s+\|", out)]


def test_zero_coefficient_computes_the_term_and_leaves_the_weights_alone(tmp_path, monkeypatch, capsys):
    """--imitate T --imitate-coeff 0 trains bit-identically to the same seeded run without --imitate, and still reports the
    imitation loss (> 0) it would have added."""
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    fin = {}
    for name, kw in (("plain", {}), ("zero", dict(imitate=JVRC_TEACHER, imitate_coeff=0.0))):
        ppo = PPO(_env_fn("jvrc_walk"), _args(tmp_path / name, eval_freq=100, **kw), seed=11)
        ppo.train(None, 2, verbose=True)
        assert ppo._ug is not None             # the update graph was captured (and replayed after it)
        fin[name] = [t.clone() for t in (ppo._flat_param, ppo._flat_m, ppo._flat_v)]
        _close(ppo)
        fin[name + "_out"] = _imitation_lines(capsys.readouterr().out)
    for x, y in zip(fin["plain"], fin["zero"]):
        assert torch.equal(x, y)
    assert fin["plain_out"] == [0.0, 0.0]
    assert len(fin["zero_out"]) == 2 and all(math.isfinite(v) and v > 0 for v in fin["zero_out"])


def test_the_student_learns_from_the_teacher(tmp_path, monkeypatch, capsys):
    """A fresh jvrc_walk student with the trained jvrc_walk actor as teacher and a large coefficient: the imitation loss falls.
    Measured on an H100 (see the bound): first and last of 8 iterations recorded next to it."""
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    ppo = PPO(_env_fn("jvrc_walk"), _args(tmp_path, eval_freq=100, imitate=JVRC_TEACHER, imitate_coeff=20.0, epochs=3, lr=3e-3),
              seed=5)
    ppo.train(None, 8, verbose=True)
    assert ppo._ug is not None
    _close(ppo)
    losses = _imitation_lines(capsys.readouterr().out)
    print("imitation loss per iteration:", losses)
    assert len(losses) == 8 and all(math.isfinite(v) for v in losses)
    # measured on an H100 80GB HBM3 (700 W): 0.02517, 0.02327, 0.01749, 0.01754, 0.02146, 0.01255, 0.01503, 0.01296 -- the loss
    # falls to ~0.5-0.6 of its start over the last two iterations; the bound leaves room for another card's rounding
    assert min(losses[-2:]) < 0.7 * losses[0], losses


def test_resumed_imitation_run_is_bit_identical(tmp_path, monkeypatch):
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    teacher = _h1_teacher(tmp_path)
    kw = dict(imitate=teacher, imitate_coeff=1.0)
    a = PPO(_env_fn("h1_walk"), _args(tmp_path / "a", **kw), seed=11)
    a.train(None, 4, verbose=False)
    assert a._ug is not None                # h1 -> h1_walk through the captured update graph
    fin_a = [t.clone() for t in (a._flat_param, a._flat_m, a._flat_v, a.env.state_r, a.env.state_i)]
    _close(a)
    b = PPO(_env_fn("h1_walk"), _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    b.train(None, 2, verbose=False)
    _close(b)
    del b
    b = PPO(_env_fn("h1_walk"), _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    assert b.restore(tmp_path / "b") == 1
    b.train(None, 4, verbose=False, start_itr=2)
    for x, y in zip(fin_a, (b._flat_param, b._flat_m, b._flat_v, b.env.state_r, b.env.state_i)):
        assert torch.equal(x, y)
    _close(b)


def _cli(*argv):
    out = subprocess.run([sys.executable, os.path.join(ROOT, "run_experiment.py")] + list(argv), capture_output=True, text=True,
                         timeout=900)
    assert out.returncode == 0, out.stdout[-2000:] + out.stderr[-3000:]
    return out.stdout


SMALL = ["--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"]


def test_train_h1_then_distil_it_into_h1_walk(tmp_path, capsys, monkeypatch):
    """`train --env h1` for 2 iterations, then `train --env h1_walk --imitate <its actor_1.pt> --imitate-coeff 1` (its update
    graph captured and replayed); the run's teacher.pt serves as a teacher again; then a `--snapshot` run of the same, stopped
    and resumed from the run directory alone (the teacher file moved away), equals the run that never stopped."""
    import run_experiment as rx
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    from learninghumanoidwalking_b200.rl import PPO
    rx.main(["train", "--env", "h1", "--logdir", str(tmp_path / "h1"), "--n-itr", "2"] + SMALL)
    (h1_run,) = list((tmp_path / "h1").iterdir())
    teacher = h1_run / "actor_1.pt"
    capsys.readouterr()
    trained, real_train = [], PPO.train

    def train_spy(self, *a, **k):
        trained.append(self)
        return real_train(self, *a, **k)
    monkeypatch.setattr(PPO, "train", train_spy)
    rx.main(["train", "--env", "h1_walk", "--logdir", str(tmp_path / "s"), "--n-itr", "2", "--imitate", str(teacher),
             "--imitate-coeff", "1"] + SMALL)
    monkeypatch.setattr(PPO, "train", real_train)
    out = capsys.readouterr().out
    (ppo,) = trained
    # 2 iterations x 2560 samples / 256 = 20 updates: 3 eager warm-ups, the capture (whose replay is the 4th), 16 replays
    assert ppo._ug is not None and ppo.actor_optimizer.step_count == 20 and ppo.base_policy is not None
    (run,) = list((tmp_path / "s").iterdir())
    losses = _imitation_lines(out)
    assert len(losses) == 2 and all(math.isfinite(v) and v > 0 for v in losses), losses
    acc = EventAccumulator(str(run))
    acc.Reload()
    tb = [s.value for s in acc.Scalars("Loss/imitation")]
    assert len(tb) == 2 and all(math.isfinite(v) and v > 0 for v in tb)
    assert (run / "teacher.pt").is_file() and rx.get_latest_actor(run).name == "actor_1.pt"
    args = pickle.load(open(run / "experiment.pkl", "rb"))
    assert args.imitate_env == "h1" and args.imitate == str(teacher)
    # the copy in the run directory is an h1 teacher too (its env is the run's imitate_env, not the run's own env)
    from learninghumanoidwalking_b200.rl.imitation import H1StandingProjector, check_teacher
    assert isinstance(check_teacher(run / "teacher.pt", "h1_walk")[2], H1StandingProjector)
    # resume: the straight run against one stopped after iteration 2 and resumed in a new process
    snap = SMALL + ["--snapshot", "--imitate-coeff", "1"]
    rx.main(["train", "--env", "h1_walk", "--logdir", str(tmp_path / "a"), "--n-itr", "4", "--imitate", str(teacher)] + snap)
    rx.main(["train", "--env", "h1_walk", "--logdir", str(tmp_path / "b"), "--n-itr", "3", "--imitate", str(teacher)] + snap)
    teacher.rename(tmp_path / "moved.pt")                  # resume needs nothing outside the run directory
    (run_a,), (run_b,) = list((tmp_path / "a").iterdir()), list((tmp_path / "b").iterdir())
    assert f"Resuming {run_b} after iteration 1." in _cli("resume", "--path", str(run_b), "--n-itr", "4")
    load = lambda d: torch.load(d / "snapshot" / "itr_3" / "learner.pt", weights_only=True)
    la, lb = load(run_a), load(run_b)
    for k in ("flat_param", "exp_avg", "exp_avg_sq"):
        assert torch.equal(la[k], lb[k]), k
    sd = lambda d: torch.load(d / "actor_3.pt", weights_only=False).state_dict()
    assert all(torch.equal(v, sd(run_b)[k]) for k, v in sd(run_a).items())


def test_two_rank_replicas_stay_identical_with_imitation(tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    script = tmp_path / "two_ranks.py"
    script.write_text(f"""
import sys
sys.path.insert(0, {ROOT!r})
from argparse import Namespace
import torch
import torch.distributed as dist
import run_experiment as rx
from learninghumanoidwalking_b200.rl import PPO
rank, world, local = rx._dist_setup()
args = Namespace(**{{**{vars(_args(tmp_path / 'logs', eval_freq=100))!r}, 'num_procs': 128, 'precision': 32, 'seed': 3,
                    'yaml': None, 'no_mirror': False, 'imitate': {JVRC_TEACHER!r}, 'imitate_coeff': 1.0}})
ppo = PPO(rx.make_env_fn(args, rank, world, local), args, seed=3)
ppo.train(None, 2, verbose=False)
got = [torch.empty_like(ppo._flat_param) for _ in range(world)]
dist.all_gather(got, ppo._flat_param)
assert ppo._ug is not None and torch.equal(got[0], got[1])
print("replicas equal")
ppo.env.close()
ppo._comm.close()
dist.destroy_process_group()
""")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29673", str(script)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, LHW_TENSORBOARD="0"))
    assert out.returncode == 0 and "replicas equal" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]


@pytest.mark.parametrize("case", ["imitate_jvrc_walk_B21845", "imitate_h1_to_h1_walk_B21845"])
def test_each_imitation_step_matches_the_float64_update(case):
    """tools/learner_local_error.py with a teacher: 7 re-synchronised production-size steps (3 eager, then the captured graph
    with the teacher's forward inside) against the float64 shadow carrying a float64 copy of the teacher behind the same
    projector, at the per-step bounds of tests/test_gpu_learner_local_error.py."""
    from tools.learner_local_error import BOUNDS, IMITATION_CASES, per_step_case, switches
    REGIMES = {"both": (True, True), "neither": (False, False)}
    kw, env = IMITATION_CASES[case]
    with switches(env):
        res, max_norm = per_step_case(**kw)
    assert len(res) >= 6 and all(e["B"] == kw["B"] and e["near"] == 0 for e in res)
    assert [e["graph"] for e in res] == [False] * 3 + [True] * (len(res) - 3)
    assert max(e["scalars"][6] for e in res) > 0
    assert all(e["scalars"][5] > 0 for e in res)                      # the term is there on every step
    if kw["imitate"] == "h1":                                         # the standing projector masks part of every minibatch
        assert all(0 < e["taught"] < e["B"] for e in res), [e["taught"] for e in res]
    assert all(e["clipped"] == REGIMES[kw["regime"]] for e in res), [(e["norms"], max_norm) for e in res]
    for q in BOUNDS:
        worst = max(range(len(res)), key=lambda k: res[k][q])
        assert res[worst][q] <= 1.0, (q, worst, res[worst][q] * BOUNDS[q], BOUNDS[q])
