"""The KL-adaptive learning rate on the device (`train --schedule adaptive`, DESIGN.md §7.3): the rule inside the fused exchange
against the float64 host rule bit for bit, each optimiser step against the float64 shadow, graph replay, resume, several ranks
and the entry point.  The host rule and the command line's refusals are tests/test_adaptive_lr.py."""
import math
import os
import struct
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 2.0 ** -7          # desired_kl with 2 D and D / 2 exact in float32: the KL word can sit exactly on each threshold


def _bits(x):
    return struct.pack("<d", x)


def _comm(n, seed):
    from learninghumanoidwalking_b200.rl.comm import PeerComm
    dev = torch.device("cuda", 0)
    c = PeerComm(n, dev)
    g = torch.Generator(device=dev).manual_seed(seed)
    p = torch.randn(n, device=dev, generator=g)
    return c, p, torch.zeros(n, device=dev), torch.zeros(n, device=dev)


def test_device_rule_is_the_host_rule_bit_for_bit():
    """Synthetic gradients and a scripted KL sequence through the adaptive exchange (eager, then from a captured graph).  After
    every step the device rate is adapt_lr of the previous one, and the parameters and moments equal those of the fixed-rate
    exchange given that new rate as its by-value `lr` in the same step: the rule runs before Adam, which takes (float)rate."""
    from learninghumanoidwalking_b200.rl.schedule import LR_MAX, LR_MIN, adapt_lr, rank_mean_kl
    n, n_actor = 10_001, 4_000
    A, pa, ma, va = _comm(n, 1)
    F, pf, mf, vf = _comm(n, 1)
    assert torch.equal(pa, pf)
    kl = torch.zeros(1, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(2)
    up, dn = math.nextafter(2 * D, 1), math.nextafter(D / 2, 0)     # both float32: 2 D and D / 2 are powers of two
    script = [(3e-4, [5 * D, 2 * D, up, D, D / 2, dn, 1e-6, 0.0, -1e-3, float("nan"), float("inf")]),
              (1.2e-5, [1.0, 1.0, 1.0]),                 # down to the lower clamp and held there
              (7e-3, [1e-6, 1e-6, 1e-6])]                # up to the upper clamp and held there
    seen = set()

    def step(x, graph=None):
        grad = torch.randn(n, device="cuda", generator=g) * 1e-2
        A.grad.copy_(grad)
        F.grad.copy_(grad)
        kl.fill_(x)
        lr0 = A.get_lr()
        if graph is None:
            A.fused_step_adaptive(pa, ma, va, n_actor, kl, D, (0.9, 0.999), 1e-5, 0.5)
        else:
            graph.replay()
        want = adapt_lr(lr0, rank_mean_kl([np.float32(x)]), D)
        got = A.get_lr()
        assert _bits(got) == _bits(want), (lr0, x, got, want)
        seen.add("down" if got < lr0 else "up" if got > lr0 else "same")
        F.fused_step(pf, mf, vf, n_actor, got, (0.9, 0.999), 1e-5, 0.5)
        torch.cuda.synchronize()
        for a, b in ((pa, pf), (ma, mf), (va, vf)):
            assert torch.equal(a, b), x
        return got

    ends = []
    for lr_start, kls in script:
        A.set_lr(lr_start)
        for x in kls:
            last = step(x)
        ends.append(last)
    assert ends[1:] == [LR_MIN, LR_MAX]
    assert seen == {"down", "up", "same"}
    # the same launches captured once and replayed: the rate is read from device memory on every replay
    A.set_lr(3e-4)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        A.fused_step_adaptive(pa, ma, va, n_actor, kl, D, (0.9, 0.999), 1e-5, 0.5)
    # capture does not run the step: the Adam step numbers of A and F still agree
    assert A.status()[0] == F.status()[0]
    for x in (5 * D, 5 * D, 1e-6, D, 1e-6):
        step(x, graph)
    A.close()
    F.close()


def test_adaptive_exchange_rejects_bad_tensors_before_any_launch():
    from learninghumanoidwalking_b200 import _lib
    O = _lib.ops()
    n = 1000
    A, p, m, v = _comm(n, 3)
    A.set_lr(3e-4)
    kl, lr = torch.zeros(1, device="cuda"), A.lr
    p0 = p.clone()
    bad = [(dict(kl=kl.double()), "kl has dtype"), (dict(kl=torch.zeros(2, device="cuda")), "kl has shape"),
           (dict(kl=kl.cpu()), "kl must be a CUDA tensor"), (dict(lr=lr.float()), "lr has dtype"),
           (dict(lr=torch.zeros(2, dtype=torch.float64, device="cuda")), "lr has shape"),
           (dict(lr=lr.cpu()), "lr must be a CUDA tensor"), (dict(desired_kl=0.0), "desired_kl must be > 0"),
           (dict(desired_kl=-1.0), "desired_kl must be > 0"), (dict(param=p[:-1]), "param has shape")]
    for over, match in bad:
        a = dict(param=p, kl=kl, lr=lr, desired_kl=0.01)
        a.update(over)
        with pytest.raises(RuntimeError, match=match):
            O.fused_exchange_adaptive(A._h.value, a["param"], m, v, 10, a["kl"], a["lr"], a["desired_kl"], 0.9, 0.999, 1e-5, 0.5)
    torch.cuda.synchronize()
    assert torch.equal(p, p0) and A.status()[0] == 0 and A.get_lr() == 3e-4
    with pytest.raises(_lib.LhwError):
        A.set_lr(0.0)
    A.close()


@pytest.mark.parametrize("case", ["adaptive_jvrc_walk_B21845", "adaptive_learn_std_B4097"])
def test_each_adaptive_step_matches_the_float64_update(case):
    """tools/learner_local_error.py under the adaptive schedule: 7 re-synchronised steps (3 eager, then the captured graph), the
    fused loss (and, with learn_std, the torch loss graph) feeding its KL to the exchange.  The rate after each step is the host
    rule on the learner's own KL, bit for bit, going down and up; the shadows step at that rate within the per-step bounds."""
    from tools.learner_local_error import ADAPTIVE_CASES, BOUNDS, per_step_case, switches
    REGIMES = {"both": (True, True), "critic": (False, True)}
    kw, env = ADAPTIVE_CASES[case]
    with switches(env):
        res, max_norm = per_step_case(**kw)
    assert len(res) == 7 and all(e["B"] == kw["B"] and e["near"] == 0 for e in res)
    assert [e["graph"] for e in res] == [False] * 3 + [True] * 4
    assert all(_bits(e["lr1"]) == _bits(e["lr_rule"]) for e in res), [(e["lr0"], e["kl"], e["lr1"], e["lr_rule"]) for e in res]
    assert any(e["lr1"] < e["lr0"] for e in res) and any(e["lr1"] > e["lr0"] for e in res), [(e["kl"], e["lr1"]) for e in res]
    assert all(e["clipped"] == REGIMES[kw["regime"]] for e in res), [(e["norms"], max_norm) for e in res]
    for q in BOUNDS:
        worst = max(range(len(res)), key=lambda k: res[k][q])
        assert res[worst][q] <= 1.0, (q, worst, res[worst][q] * BOUNDS[q], BOUNDS[q])


def test_fixed_cases_are_unchanged():
    from tools.learner_local_error import ADAPTIVE_CASES, CASES
    assert not set(CASES) & set(ADAPTIVE_CASES) and all("kl_scales" not in kw for kw, _ in CASES.values())


def _args(logdir, **kw):
    d = dict(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=256, epochs=1,
             max_traj_len=50, num_procs=64, max_grad_norm=0.05, mirror_coeff=0.4, eval_freq=2, recurrent=False,
             imitate_coeff=0.0, std_dev=0.223, learn_std=False, logdir=str(logdir), steps_per_env=20,
             schedule="adaptive", desired_kl=1e-6)
    d.update(kw)
    return SimpleNamespace(**d)


def _env_fn(model="jvrc_walk", seed=7):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    from learninghumanoidwalking_b200.rl.symmetric import SymmetricEnv
    base = lambda: BatchedHumanoidEnv(64, model=model, precision=32, seed=seed)
    probe = base()
    r = probe.robot
    probe.close()
    return lambda: SymmetricEnv(base, mirrored_obs=r.mirrored_obs, mirrored_act=r.mirrored_acts, clock_inds=r.clock_inds)


def _close(ppo):
    ppo.env.close()
    if ppo._comm is not None:
        ppo._comm.close()


def test_graph_replay_and_the_eager_loop_give_the_same_run(tmp_path, monkeypatch):
    """Two iterations with LHW_UPDATE_GRAPH=0 and with the captured update graph: the same weights, moments and rate.  In the
    eager loop every step's KL passes through Python, and the rate is the host rule folded over them."""
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.comm import PeerComm
    from learninghumanoidwalking_b200.rl.schedule import adapt_lr
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    kls, real = [], PeerComm.fused_step_adaptive

    def spy(self, param, exp_avg, exp_avg_sq, n_actor, kl, *a):
        kls.append(kl.clone())
        return real(self, param, exp_avg, exp_avg_sq, n_actor, kl, *a)
    fin = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("LHW_UPDATE_GRAPH", mode)
        monkeypatch.setattr(PeerComm, "fused_step_adaptive", spy if mode == "0" else real)
        ppo = PPO(_env_fn(), _args(tmp_path / mode, eval_batches=0, desired_kl=3e-3), seed=4)
        log = ppo.train(None, 2, verbose=False)
        assert (ppo._ug is not None) == (mode == "1")
        fin[mode] = [t.clone() for t in (ppo._flat_param, ppo._flat_m, ppo._flat_v)] + [ppo._comm.get_lr(), log]
        _close(ppo)
    assert len(kls) == 10
    want = 3e-4
    for k in kls:
        want = adapt_lr(want, float(k), 3e-3)
    diffs = [(fin["0"][k] - fin["1"][k]).abs().max().item() for k in range(3)]
    print("graph vs eager: rates", fin["0"][3], fin["1"][3], "max |d| param/m/v", diffs, "kl", [float(k) for k in kls])
    assert _bits(fin["0"][3]) == _bits(want) and want != 3e-4
    assert _bits(fin["1"][3]) == _bits(fin["0"][3]) and [e["lr"] for e in fin["1"][4]] == [e["lr"] for e in fin["0"][4]]
    for k in range(3):
        assert torch.equal(fin["0"][k], fin["1"][k]), diffs


def test_resumed_adaptive_run_is_bit_identical(tmp_path, monkeypatch):
    """Stopped after iteration 1 (its snapshot holds the device rate) and resumed: weights, moments and rate equal a run that
    never stopped.  desired_kl = 0.003 keeps the rate moving both ways instead of resting on a clamp."""
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    kw = dict(desired_kl=3e-3)
    a = PPO(_env_fn(), _args(tmp_path / "a", **kw), seed=11)
    log_a = a.train(None, 4, verbose=False)
    fin_a = [t.clone() for t in (a._flat_param, a._flat_m, a._flat_v)] + [a._comm.get_lr()]
    _close(a)
    b = PPO(_env_fn(), _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    b.train(None, 2, verbose=False)
    _close(b)
    del b
    learner = torch.load(tmp_path / "b" / "snapshot" / "itr_1" / "learner.pt", weights_only=True)
    assert learner["adaptive_lr"].dtype == torch.float64 and float(learner["adaptive_lr"][0]) == log_a[1]["lr"]
    b = PPO(_env_fn(), _args(tmp_path / "b", snapshot=True, **kw), seed=11)
    assert b.restore(tmp_path / "b") == 1
    log_b = b.train(None, 4, verbose=False, start_itr=2)
    for x, y in zip(fin_a[:3], (b._flat_param, b._flat_m, b._flat_v)):
        assert torch.equal(x, y)
    assert _bits(fin_a[3]) == _bits(b._comm.get_lr()) and [e["lr"] for e in log_b] == [e["lr"] for e in log_a[2:]]
    print("rates", [e["lr"] for e in log_a], "kl", [e["kl"] for e in log_a])
    _close(b)


def test_fixed_run_snapshot_has_no_rate_and_adaptive_refuses_it(tmp_path, monkeypatch):
    from learninghumanoidwalking_b200.rl import PPO
    from learninghumanoidwalking_b200.rl.snapshot import SnapshotError
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    a = PPO(_env_fn(), _args(tmp_path, snapshot=True, schedule="fixed"), seed=5)
    log = a.train(None, 2, verbose=False)
    _close(a)
    assert "lr" not in log[-1]
    learner = torch.load(tmp_path / "snapshot" / "itr_1" / "learner.pt", weights_only=True)
    assert "adaptive_lr" not in learner
    b = PPO(_env_fn(), _args(tmp_path, snapshot=True), seed=5)
    with pytest.raises(SnapshotError, match="no learning rate"):
        b.restore(tmp_path)
    _close(b)


def test_hand_assigned_optimisers_and_the_baseline_exchange_are_refused(tmp_path, monkeypatch):
    from learninghumanoidwalking_b200.rl import PPO
    monkeypatch.setenv("LHW_TENSORBOARD", "0")
    ppo = PPO(_env_fn(), _args(tmp_path), seed=1)
    ppo.actor_optimizer = torch.optim.Adam(ppo.policy.parameters(), lr=3e-4)
    ppo.critic_optimizer = torch.optim.Adam(ppo.critic.parameters(), lr=3e-4)
    with pytest.raises(ValueError, match="hand-assigned torch optimisers"):
        ppo.train(None, 1, verbose=False)
    _close(ppo)
    monkeypatch.setenv("LHW_FUSED_EXCHANGE", "0")
    ppo = PPO(_env_fn(), _args(tmp_path), seed=1)
    with pytest.raises(ValueError, match="LHW_FUSED_EXCHANGE=0"):
        ppo.train(None, 1, verbose=False)
    ppo.env.close()


SMALL = ["--num-procs", "64", "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"]


def test_entry_point_prints_and_logs_the_rate_only_when_adaptive(tmp_path, capsys):
    import pickle
    import re
    import run_experiment as rx
    from tensorboard.backend.event_processing.event_accumulator import EventAccumulator
    row = re.compile(r"\|\s+Learning rate\s+\|\s+([\d.e+-]+)\s+\|")
    for kind in ("adaptive", "fixed"):
        extra = ["--schedule", "adaptive", "--desired-kl", "0.005"] if kind == "adaptive" else []
        rx.main(["train", "--env", "jvrc_walk", "--logdir", str(tmp_path / kind), "--n-itr", "2"] + SMALL + extra)
        out = capsys.readouterr().out
        (run,) = list((tmp_path / kind).iterdir())
        acc = EventAccumulator(str(run))
        acc.Reload()
        args = pickle.load(open(run / "experiment.pkl", "rb"))
        if kind == "adaptive":
            rates = [float(x) for x in row.findall(out)]
            tb = [s.value for s in acc.Scalars("Train/learning_rate")]
            assert len(rates) == 2 and len(tb) == 2 and all(1e-5 <= r <= 1e-2 for r in rates), (rates, tb)
            assert (args.schedule, args.desired_kl) == ("adaptive", 0.005)
        else:
            assert not row.search(out) and "Train/learning_rate" not in acc.Tags()["scalars"]
            assert (args.schedule, args.desired_kl) == ("fixed", 0.01)


_RANKS = r'''
import os, sys
sys.path.insert(0, {root!r})
import numpy as np, torch, torch.distributed as dist
from types import SimpleNamespace
from learninghumanoidwalking_b200.rl.comm import PeerComm
from learninghumanoidwalking_b200.rl.schedule import adapt_lr, rank_mean_kl
local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank, world = dist.get_rank(), dist.get_world_size()
dev = torch.device("cuda", local)
n = 10001
c = PeerComm(n, dev)
c.set_lr(3e-4)
p, m, v = torch.zeros(n, device=dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
kl = torch.zeros(1, device=dev)
rng = np.random.RandomState(0)
lr = 3e-4
for step in range(12):
    kls = (rng.uniform(0, 0.03, world) * (10.0 if step % 3 == 0 else 1.0)).astype(np.float32)
    c.grad.fill_(1e-3 * (rank + 1))
    kl.fill_(float(kls[rank]))
    c.fused_step_adaptive(p, m, v, 5000, kl, 0.01, (0.9, 0.999), 1e-5, 0.5)
    lr = adapt_lr(lr, rank_mean_kl(kls), 0.01)
    got = c.get_lr()
    assert got == lr, (rank, step, got, lr)
c.status()
allp = [torch.empty_like(p) for _ in range(world)]
dist.all_gather(allp, p)
assert all(torch.equal(allp[0], q) for q in allp)
rates = [None] * world
dist.all_gather_object(rates, c.get_lr())
assert len(set(rates)) == 1
c.close()
# PPO under the adaptive schedule: the replicas, rate included, stay identical
from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
from learninghumanoidwalking_b200.rl import PPO
env_fn = lambda: BatchedHumanoidEnv(64, model="jvrc_walk", precision=32, seed=3, first_env_id=64 * rank, device=local)
a = SimpleNamespace(gamma=0.99, lam=0.95, lr=3e-4, eps=1e-5, entropy_coeff=0.0, clip=0.2, minibatch_size=256, epochs=1,
                    max_traj_len=50, num_procs=64 * world, max_grad_norm=0.05, mirror_coeff=0.0, eval_freq=10 ** 9,
                    eval_at_start=False, std_dev=0.223, learn_std=False, logdir="/tmp/lhw_adaptive_ranks", steps_per_env=20,
                    schedule="adaptive", desired_kl=3e-3)
ppo = PPO(env_fn, a, seed=3)
ppo.train(None, 2, verbose=False)
allp = [torch.empty_like(ppo._flat_param) for _ in range(world)]
dist.all_gather(allp, ppo._flat_param)
rates = [None] * world
dist.all_gather_object(rates, ppo._comm.get_lr())
assert all(torch.equal(allp[0], q) for q in allp) and len(set(rates)) == 1, rates
if rank == 0:
    print("replicas equal", rates[0])
ppo.env.close()
ppo._comm.close()
dist.destroy_process_group()
'''


@pytest.mark.parametrize("world", [2, 4, 8])
def test_ranks_agree_on_the_rate_of_the_rank_mean_kl(tmp_path, world):
    """Each rank publishes a different KL; every rank's rate is the host rule on their rank-order float64 mean, and PPO
    replicas (rate included) stay identical."""
    if torch.cuda.device_count() < world:
        pytest.skip(f"needs >= {world} GPUs")
    script = tmp_path / "ranks.py"
    script.write_text(_RANKS.format(root=ROOT))
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
           "--master-port", str(29690 + world), str(script)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=dict(os.environ, LHW_TENSORBOARD="0"))
    assert out.returncode == 0 and "replicas equal" in out.stdout, out.stdout[-2000:] + out.stderr[-3000:]
