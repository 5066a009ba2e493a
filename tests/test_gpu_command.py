"""Held walking commands on the device (DESIGN.md §7.6): lhw_sim_set_command against the host command body, the op's refusals,
uncommanded rows of a mixed batch against a batch that never got a command (eagerly, through graph replay and through the two
step_slice halves), held rows until their reset, the command sweep's accumulators, and `eval --command` end to end."""
import json
import pickle
import shutil
from argparse import Namespace

import numpy as np
import pytest
import torch

from test_command import HELD, _layout, _lib as _host_lib, set_command as host_set_command
from test_gpu_eval_stats import TRAINED

pytestmark = pytest.mark.gpu
WALKING = ["jvrc_walk", "jvrc_walk_terrain", "h1_walk"]


def _env(name, precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model=name, precision=precision, **kw)


def _actions(env, g, scale=0.5):
    return (torch.randn(env.num_envs, env.act_dim, generator=g, device=env.device) * scale).to(env.dtype)


def _command(n, seed=1):
    rng = np.random.RandomState(seed)
    mode = rng.randint(-1, 3, size=n).astype(np.int32)
    ref = rng.uniform(-0.5, 0.5, size=(n, 3))
    return mode, ref


class _HostRecords:
    """The device records copied to a host emulation's arrays (emu_variants.Emu has the layout the host bodies take)."""

    def __init__(self, env):
        self.n, self.nr, self.dt = env.num_envs, env.state_r.shape[1], np.float64 if env.precision == 64 else np.float32
        self.sr, self.si = env.state_r.cpu().numpy().copy(), env.state_i.cpu().numpy().copy()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", WALKING)
def test_device_command_equals_host_body(name, precision):
    from learninghumanoidwalking_b200.model import load_model, pack_model
    env = _env(name, precision, 256, seed=2)
    env.reset()
    g = torch.Generator(device=env.device).manual_seed(1)
    for _ in range(15):
        env.step(_actions(env, g))
    host = _HostRecords(env)
    obs = env.obs.cpu().numpy().copy()
    mode, ref = _command(env.num_envs)
    ref = ref.astype(host.dt)
    rc, given = host_set_command(_host_lib(), int(pack_model(load_model(name))[0]), precision, host, mode, ref, obs)
    assert rc == 0 and 0 < given.sum() < env.num_envs
    env.set_command(mode.tolist(), torch.as_tensor(ref))
    assert np.array_equal(env.state_r.cpu().numpy().view(np.uint8), host.sr.view(np.uint8))
    assert np.array_equal(env.state_i.cpu().numpy(), host.si)
    assert np.array_equal(env.obs.cpu().numpy().view(np.uint8), obs.view(np.uint8))
    assert (env.state_i.cpu().numpy()[given, 1] == mode[given] | HELD).all()
    env.close()


def test_op_rejects_bad_tensors_and_values():
    env = _env("jvrc_walk", 64, 8)
    env.reset()
    from learninghumanoidwalking_b200 import _lib
    O, h = _lib.ops(), env._h.value
    before_r, before_i, before_o = env.state_r.clone(), env.state_i.clone(), env.obs.clone()
    mode = torch.zeros(8, dtype=torch.int32, device=env.device)
    ref = torch.zeros(8, 3, dtype=torch.float64, device=env.device)
    for bad_mode, bad_ref, message in ((mode.long(), ref, "mode has dtype"), (mode[:4], ref, "mode has shape"),
                                       (mode.cpu(), ref, "must be a CUDA tensor"), (mode, ref.float(), "ref has dtype"),
                                       (mode, ref[:, :2].contiguous(), "ref has shape"), (mode, ref.t().contiguous().t(), "must be contiguous"),
                                       (mode + 3, ref, "mode must be -1"), (mode - 2, ref, "mode must be -1"),
                                       (mode, ref + float("nan"), "ref must be finite"), (mode, ref + float("inf"), "ref must be finite")):
        with pytest.raises(RuntimeError, match=message):
            O.sim_set_command(h, env.state_r, env.state_i, bad_mode, bad_ref, env.obs)
    with pytest.raises(RuntimeError, match="obs has shape"):
        O.sim_set_command(h, env.state_r, env.state_i, mode, ref, env.obs[:, :-1].contiguous())
    acc = torch.zeros(8, 5, dtype=torch.float64, device=env.device)
    for bad, message in ((acc.float(), "acc has dtype"), (acc[:, :4].contiguous(), "acc has shape"), (acc.cpu(), "must be a CUDA tensor")):
        with pytest.raises(RuntimeError, match=message):
            O.sim_command_accumulate(h, env.state_r, env.done, bad)
    assert torch.equal(env.state_r, before_r) and torch.equal(env.state_i, before_i) and torch.equal(env.obs, before_o)
    # the Python API refuses on the host, with the same rules
    for args, message in ((([3] * 8, np.zeros((8, 3))), "mode must be -1"), (([0] * 8, np.full((8, 3), np.nan)), "ref must be finite"),
                          (([0] * 4, np.zeros((4, 3))), "mode must hold 8"), (([0.5] * 8, np.zeros((8, 3))), "mode must hold 8")):
        with pytest.raises(ValueError, match=message):
            env.set_command(*args)
    env.close()
    for name in ("h1", "jvrc_step"):
        other = _env(name, 64, 8)
        other.reset()
        with pytest.raises(RuntimeError, match=f"{name} .*has no velocity command"):
            O.sim_set_command(other._h.value, other.state_r, other.state_i, mode, ref, other.obs)
        with pytest.raises(ValueError, match=f"{name} has no velocity command"):
            other.set_command([0] * 8, np.zeros((8, 3)))
        other.close()


def _graph_stepper(env, g):
    """Steps env through one captured CUDA graph of env.step (the first step eager, as the capture's warm-up)."""
    a = torch.zeros(env.num_envs, env.act_dim, dtype=env.dtype, device=env.device)
    state = dict(graph=None)
    cur = torch.cuda.current_stream(env.device)
    s = torch.cuda.Stream(device=env.device)

    def step():
        a.copy_(_actions(env, g))
        s.wait_stream(cur)
        with torch.cuda.stream(s):
            if state["graph"] is None:
                env.step(a)
                state["graph"] = torch.cuda.CUDAGraph()
                with torch.cuda.graph(state["graph"], stream=s):
                    env.step(a)
            else:
                env.bind()
                state["graph"].replay()
        cur.wait_stream(s)
    return step


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", WALKING)
def test_mixed_batch_untouched_rows_and_held_rows(name, precision):
    """Four copies of one batch under the same actions with autoreset on, for 400 steps: `plain` never gets a command; `eager`,
    `graph` (replayed CUDA graph) and `halves` (step_slice over two halves) get the same mixed command after their reset.  The
    three commanded copies are bit-identical; their rows given -1 equal `plain`'s rows bit for bit, records and outputs; a held
    row keeps its mode and reference until its episode ends, and carries no hold after its reset."""
    n = 512
    envs = {k: _env(name, precision, n, seed=5) for k in ("plain", "eager", "graph", "halves")}
    mode, ref = _command(n, seed=3)
    for k, e in envs.items():
        e.reset()
        if k != "plain":
            e.set_command(mode, ref)
    gens = {k: torch.Generator(device=e.device).manual_seed(7) for k, e in envs.items()}
    graph_step = _graph_stepper(envs["graph"], gens["graph"])
    free = torch.as_tensor(mode < 0, device=envs["plain"].device)
    held_live = torch.as_tensor(mode >= 0, device=free.device)
    want_word = torch.as_tensor(mode, device=free.device) | HELD
    mr = _layout(envs["plain"].act_dim)[1]
    ref_dev = torch.as_tensor(ref, device=free.device).to(envs["plain"].dtype)
    resets = held_steps = 0
    for t in range(400):
        envs["plain"].step(_actions(envs["plain"], gens["plain"]))
        envs["eager"].step(_actions(envs["eager"], gens["eager"]))
        graph_step()
        a = _actions(envs["halves"], gens["halves"])
        envs["halves"].step_slice(0, n // 2, a[:n // 2].contiguous())
        envs["halves"].step_slice(n // 2, n, a[n // 2:].contiguous())
        p, e = envs["plain"], envs["eager"]
        for k in ("graph", "halves"):
            o = envs[k]
            assert torch.equal(o.state_r, e.state_r) and torch.equal(o.state_i, e.state_i) and torch.equal(o.obs, e.obs), (k, t)
        assert torch.equal(e.state_r[free], p.state_r[free]) and torch.equal(e.state_i[free], p.state_i[free]), t
        for x, y in ((e.obs, p.obs), (e.reward, p.reward), (e.done, p.done), (e.ended, p.ended), (e.term_obs, p.term_obs)):
            assert torch.equal(x[free], y[free]), t
        ended = e.ended != 0
        held_live &= ~ended
        resets += int((ended & (torch.as_tensor(mode, device=free.device) >= 0)).sum())
        assert torch.equal(e.state_i[held_live, 1], want_word[held_live]), t
        assert torch.equal(e.state_r[held_live, mr:mr + 3], ref_dev[held_live]), t
        assert not (e.state_i[~held_live, 1] & HELD).any(), t
        held_steps += int(held_live.sum())
    # every commanded row ran held for a while and then ended; its reset left it unheld
    assert resets > 0 and held_steps > 10 * int((mode >= 0).sum()), (resets, held_steps)
    for x in envs.values():
        x.close()


def _random_actor(env):
    from learninghumanoidwalking_b200.rl import Gaussian_FF_Actor
    torch.manual_seed(0)
    return Gaussian_FF_Actor(env.obs_dim, env.act_dim, init_std=0.223).cuda().eval()


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", WALKING)
def test_sweep_accumulators(name, precision):
    """evaluation.rollout with held commands: for every env the tracking steps of its held mode equal its EV_LEN and those of the
    other modes are 0; graph replay equals the eager loop bit for bit; and the signed-velocity records equal a float64
    recomputation from the records of an eager loop of the same launches (the step counts and flags exactly, the velocity sums to
    1e-12: the device may contract a multiply-add that the host rounds twice)."""
    from learninghumanoidwalking_b200.rl import evaluation as ev
    n, steps = 384, 100
    cells = [("FORWARD", 0.0), ("FORWARD", 0.3), ("INPLACE", -0.4), ("INPLACE", 0.4), ("STANDING", 0.0)]
    mode, value = ev.command_grid(n, cells)
    command = (mode, ev.command_refs(mode, value))
    probe = _env(name, precision, n, seed=1, max_traj_len=steps)
    policy = _random_actor(probe)
    probe.close()
    out = {}
    for graph in (True, False):
        env = _env(name, precision, n, seed=1, max_traj_len=steps)
        acc, cacc = ev.rollout(env, policy, steps, graph=graph, command=command)
        out[graph] = (acc.cpu().numpy(), cacc.cpu().numpy())
        env.close()
    assert np.array_equal(out[True][0], out[False][0]) and np.array_equal(out[True][1], out[False][1])
    acc, cacc = out[True]
    for m in range(3):
        assert np.array_equal(acc[:, ev.TRACK + 4 * m], np.where(mode == m, acc[:, ev.LEN], 0)), m
    assert np.array_equal(cacc[:, ev.C_LEN], acc[:, ev.LEN]) and np.array_equal(cacc[:, ev.C_DONE], acc[:, ev.DONE])
    # the recomputation from an eager loop's records (the same launches as rollout(graph=False))
    env = _env(name, precision, n, seed=1, max_traj_len=steps)
    env.reset()
    env.set_command(*command)
    state = env.obs.float().clone()
    want = np.zeros((n, 5))
    nq = env.nq
    with torch.no_grad():
        for _ in range(steps):
            a = policy(state, deterministic=True)
            obs, _, done, _ = env.step(a if env.dtype == torch.float32 else a.double(), autoreset=False)
            state.copy_(obs.float())
            sr, dn = env.state_r.cpu().numpy().astype(np.float64), done.cpu().numpy()
            live = want[:, 4] == 0
            qw, x, y, z = sr[:, 3:7].T
            s = 2 / (qw * qw + x * x + y * y + z * z)
            X, Y, Z = x * s, y * s, z * s
            wX, wY, wZ, xX, xY, xZ, yY, yZ, zZ = qw * X, qw * Y, qw * Z, x * X, x * Y, x * Z, y * Y, y * Z, z * Z
            v0, v1, v2 = sr[:, nq], sr[:, nq + 1], sr[:, nq + 2]
            vf = (1 - (yY + zZ)) * v0 + (xY + wZ) * v1 + (xZ - wY) * v2
            vl = (xY - wZ) * v0 + (1 - (xX + zZ)) * v1 + (yZ + wX) * v2
            want[live, 0] += 1
            want[live, 1] += vf[live]
            want[live, 2] += vl[live]
            want[live, 3] += sr[live, nq + 5]
            want[live & (dn != 0), 4] = 1
    env.close()
    assert np.array_equal(cacc[:, [0, 4]], want[:, [0, 4]])
    np.testing.assert_allclose(cacc[:, 1:4], want[:, 1:4], rtol=1e-12, atol=1e-12)
    assert (cacc[:, 4] != 0).any() or steps == cacc[:, 0].min()


def _policy():
    from learninghumanoidwalking_b200.rl.policies import install_reference_aliases
    install_reference_aliases()
    return torch.load(TRAINED, weights_only=False).cuda().eval()


def test_command_line_on_the_trained_actor(tmp_path, capsys):
    """`eval --num-envs 256 --command forward:0,0.2,0.4 inplace:-0.4,0.4 standing --report r.json` and the single-env
    `eval --command forward:0.3` on the trained jvrc_walk actor."""
    run = tmp_path / "run"
    run.mkdir()
    shutil.copy(TRAINED, run / "actor.pt")
    with open(run / "experiment.pkl", "wb") as f:
        pickle.dump(Namespace(env="jvrc_walk", max_traj_len=400, yaml=None), f)
    import run_experiment as rx
    path = tmp_path / "r.json"
    rx.main(["eval", "--path", str(run), "--num-envs", "256", "--command", "forward:0,0.2,0.4", "inplace:-0.4,0.4", "standing",
             "--report", str(path)])
    out = capsys.readouterr().out
    assert "held commands" in out and "forward 0.2" in out and "inplace -0.4" in out
    r = json.loads(path.read_text())
    cells = r["summary"]["commands"]["cells"]
    assert [(c["mode"], c["value"]) for c in cells] == [("FORWARD", 0.0), ("FORWARD", 0.2), ("FORWARD", 0.4), ("INPLACE", -0.4),
                                                       ("INPLACE", 0.4), ("STANDING", 0.0)]
    assert [c["n"] for c in cells] == [43, 43, 43, 43, 42, 42]
    assert all(c["tracking"]["steps"] > 0 for c in cells)
    pe = r["per_env"]
    assert pe["command_mode"][:7] == ["FORWARD", "FORWARD", "FORWARD", "INPLACE", "INPLACE", "STANDING", "FORWARD"]
    assert pe["command_value"][1] == 0.2 and len(pe["v_fwd_sum"]) == len(pe["yaw_rate_sum"]) == len(pe["command_steps"]) == 256
    assert pe["command_steps"] == pe["length"]
    # the single-env roll-out holds its one command, re-applied after every reset
    episodes = rx.main(["eval", "--path", str(run), "--ep-len", "5", "--command", "forward:0.3"])
    assert sum(l for l, _ in episodes) == 200
    for extra, message in ((["--command", "forward:0.1,0.2"], "add --num-envs"),
                           (["--num-envs", "2", "--command", "forward:0,0.2", "standing"], "3 cells")):
        with pytest.raises(SystemExit, match=message):
            rx.main(["eval", "--path", str(run), *extra])
