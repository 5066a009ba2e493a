"""Evaluation statistics on the device (`eval --num-envs`, DESIGN.md §7.4): lhw_sim_eval_accumulate against a host
recomputation from the recorded roll-out, graph replay against an eager loop, the batched evaluation of one env against the
single-env `eval`, and the command line end to end."""
import json
import os

import numpy as np
import pytest
import torch

from test_eval_stats import DONE, LEN, RET, SEQLEN, TRACK, WORDS, recompute

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TRAINED = os.path.join(ROOT, "tests", "golden", "trained_actor_jvrc_walk.pt")
ERROR_SUMS = [TRACK + 4 * m + k for m in range(3) for k in (1, 2, 3)]


def _env(name, precision, n, max_traj_len, seed=5):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, seed=seed, max_traj_len=max_traj_len)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("env_name", ["jvrc_walk", "jvrc_walk_terrain", "h1_walk", "h1", "jvrc_step"])
def test_device_accumulators_equal_host_recomputation(env_name, precision):
    n, steps = 96, 10 if env_name == "h1" else 40
    env = _env(env_name, precision, n, steps)
    env.reset()
    acc = torch.zeros(n, WORDS, dtype=torch.float64, device=env.device)
    g = torch.Generator(device=env.device).manual_seed(1)
    scale = torch.where(torch.arange(n, device=env.device) % 2 == 0, 1.5, 0.02).to(env.dtype)[:, None]
    records = []
    for _ in range(steps):
        a = torch.randn(n, env.act_dim, generator=g, device=env.device).to(env.dtype) * scale
        env.step(a, autoreset=False)
        env.eval_accumulate(acc)
        records.append((env.state_r.cpu().numpy(), env.state_i.cpu().numpy(), env.reward.cpu().numpy(), env.rew_terms.cpu().numpy(),
                        env.done.cpu().numpy()))
    got = acc.cpu().numpy()
    want = recompute(env_name, 5 if env_name.startswith("h1") else 6, records, n)
    exact = [k for k in range(WORDS) if k not in ERROR_SUMS]   # counts, flags and plain float64 sums of step outputs
    assert np.array_equal(got[:, exact], want[:, exact]), np.abs(got - want)[:, exact].max()
    # the velocity errors: the device may contract a multiply-add that the host rounds twice
    np.testing.assert_allclose(got[:, ERROR_SUMS], want[:, ERROR_SUMS], rtol=1e-12, atol=1e-12)
    fell = got[:, DONE] != 0
    assert fell.any() and (~fell).any()
    if env_name == "jvrc_step":
        assert (got[:, SEQLEN] >= 1).all()
    else:
        assert np.array_equal(got[:, [TRACK, TRACK + 4, TRACK + 8]].sum(1), got[:, LEN])
    env.close()


def test_op_rejects_bad_tensors():
    env = _env("jvrc_walk", 64, 8, 40)
    env.reset()
    from learninghumanoidwalking_b200 import _lib
    O = _lib.ops()
    h = env._h.value
    ok = torch.zeros(8, WORDS, dtype=torch.float64, device=env.device)
    args = (env.state_r, env.state_i, env.reward, env.rew_terms, env.done)
    with pytest.raises(RuntimeError, match="acc has dtype"):
        O.sim_eval_accumulate(h, *args, ok.float())
    with pytest.raises(RuntimeError, match="acc has shape"):
        O.sim_eval_accumulate(h, *args, torch.zeros(8, WORDS + 1, dtype=torch.float64, device=env.device))
    with pytest.raises(RuntimeError, match="reward has dtype"):
        O.sim_eval_accumulate(h, env.state_r, env.state_i, env.reward.float(), env.rew_terms, env.done, ok)
    with pytest.raises(RuntimeError, match="must be a CUDA tensor"):
        O.sim_eval_accumulate(h, *args, ok.cpu())
    assert not ok.any()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_graph_replay_equals_eager_loop(precision):
    from learninghumanoidwalking_b200.rl import evaluation
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    policy = torch.load(TRAINED, weights_only=False).cuda().eval()
    out = []
    for graph in (True, False):
        env = _env("jvrc_walk", precision, 300, 120)
        out.append(evaluation.rollout(env, policy, 120, graph=graph).cpu())
        env.close()
    assert torch.equal(out[0], out[1])
    assert out[0][:, LEN].min() > 0 and out[0][:, RET].abs().sum() > 0


@pytest.fixture(scope="module")
def trained_run(tmp_path_factory):
    """A 2-iteration jvrc_walk run at the default horizon and without YAML (what the single-env `eval` assumes)."""
    import run_experiment as rx
    logdir = tmp_path_factory.mktemp("logs")
    rx.main(["train", "--env", "jvrc_walk", "--logdir", str(logdir), "--num-procs", "64", "--n-itr", "2", "--minibatch-size", "256",
             "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    (run,) = list(logdir.iterdir())
    return run


def test_one_env_equals_the_single_env_eval(trained_run, tmp_path):
    import run_experiment as rx
    episodes = rx.main(["eval", "--path", str(trained_run), "--ep-len", "10", "--seed", "7"])
    report = rx.main(["eval", "--path", str(trained_run), "--num-envs", "1", "--precision", "64", "--seed", "7"])
    assert report["max_traj_len"] == 400 and report["num_envs"] == 1
    first_len, first_ret = episodes[0]
    assert report["per_env"]["length"] == [first_len]
    assert report["per_env"]["return"] == [first_ret]
    assert report["per_env"]["fell"] == [len(episodes) > 1 or first_len < 400]


def test_command_line_report_and_refusals(trained_run, tmp_path, capsys):
    import run_experiment as rx
    path = tmp_path / "r.json"
    rx.main(["eval", "--path", str(trained_run), "--num-envs", "256", "--report", str(path), "--seed", "2"])
    out = capsys.readouterr().out
    assert "256 environments, one episode each, horizon 400 control steps" in out and "command tracking" in out
    r = json.loads(path.read_text())
    assert {"actor", "env", "precision", "seed", "num_envs", "max_traj_len", "summary", "per_env"} <= set(r)
    assert (r["env"], r["precision"], r["seed"], r["num_envs"], r["max_traj_len"]) == ("jvrc_walk", 64, 2, 256, 400)
    assert r["actor"].endswith("actor_1.pt")
    s = r["summary"]
    assert {"fall_fraction", "length", "return", "reward_terms", "tracking"} <= set(s)
    assert set(s["length"]) == {"mean", "min", "p5", "median"} and set(s["return"]) == {"mean", "std"}
    assert set(s["tracking"]) == {"STANDING", "INPLACE", "FORWARD"}
    assert sum(t["steps"] for t in s["tracking"].values()) == sum(r["per_env"]["length"])
    assert len(r["per_env"]["length"]) == 256 and len(r["per_env"]["reward_term_sums"]) == 10
    assert all(1 <= n <= 400 for n in r["per_env"]["length"])
    for extra, message in ((["--num-envs", "0"], "at least one environment"), (["--num-envs", "4", "--out-dir", str(tmp_path)], "cannot be combined")):
        with pytest.raises(SystemExit, match=message):
            rx.main(["eval", "--path", str(trained_run), *extra])
