"""Chosen stepping-stone plans on the device (DESIGN.md §7.7): lhw_sim_reset_footsteps against the host body (integer and plan
words exactly, the settled pose to rounding), the op's refusals,
untouched rows of a mixed batch against a batch that never got a plan (eagerly, through graph replay and through the two step_slice
halves), the drawn plan given back equal to reset(), a mid-episode copy of the records resuming bit for bit, and `train` then
`eval --footsteps` end to end."""
import json

import numpy as np
import pytest
import torch

from test_footsteps import CURVED, FORWARD, LATERAL, TK, FootEmu, _flat, _oracle, drawn_plan
from test_gpu_command import _actions, _graph_stepper

pytestmark = pytest.mark.gpu


def _env(precision, n, **kw):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    return BatchedHumanoidEnv(n, model="jvrc_step", precision=precision, **kw)


def _plans(n, seed=1):
    """A mixed set of plans: every type, heights up to 0.2 m, both sides, named and drawn curved plans, and rows given -1."""
    rng = np.random.RandomState(seed)
    mode = rng.randint(-1, 5, size=n).astype(np.int32)
    value = np.zeros(n)
    value[mode == FORWARD] = rng.uniform(-0.2, 0.2, size=(mode == FORWARD).sum())
    value[mode == LATERAL] = rng.choice([-1.0, 1.0], size=(mode == LATERAL).sum())
    value[mode == CURVED] = rng.randint(-1, 109, size=(mode == CURVED).sum())
    return mode, value


@pytest.mark.parametrize("precision", [64, 32])
def test_device_reset_footsteps_equals_host_body(precision):
    n, seed = 256, 2
    env = _env(precision, n, seed=seed, iteration_count=11000)
    host = FootEmu(_flat(precision, 11000), precision, n, seed, 0)
    env.reset()
    g = torch.Generator(device=env.device).manual_seed(1)
    for _ in range(15):
        env.step(_actions(env, g))
    host.sr[:], host.si[:] = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
    obs = env.obs.cpu().numpy().copy()
    mode, value = _plans(n)
    hobs = host.reset_footsteps(mode, value)
    hobs[mode < 0] = obs[mode < 0]
    env.reset_footsteps(mode, value)
    # the integer words but the solver's count and the plan words are the host body's exactly; the settled pose is the same computation, compiled with
    # the device's fused multiply-adds, so it agrees to rounding
    sr = env.state_r.cpu().numpy()
    assert np.array_equal(env.state_i.cpu().numpy()[:, :7], host.si[:, :7])     # [7]: the solver's iteration total
    assert np.array_equal(sr[:, TK:TK + 3], host.sr[:, TK:TK + 3])
    assert sr[mode < 0].tobytes() == host.sr[mode < 0].tobytes()
    tol = 1e-9 if precision == 64 else 1e-4
    assert np.abs(sr - host.sr).max() < tol and np.abs(env.obs.cpu().numpy() - hobs).max() < tol
    env.close()


def test_op_rejects_bad_tensors_and_values():
    from learninghumanoidwalking_b200 import _lib
    env = _env(64, 8, seed=1)
    env.reset()
    op, h = _lib.ops().sim_reset_footsteps, env._h.value
    dev = env.device
    good_m, good_v = torch.zeros(8, dtype=torch.int32, device=dev) - 1, torch.zeros(8, dtype=torch.float64, device=dev)

    def call(mode=None, value=None, state_r=None):
        op(h, env.state_r if state_r is None else state_r, env.state_i, 1, 0, good_m if mode is None else mode,
           good_v if value is None else value, False, env.obs)

    def mv(m, v):
        return (torch.full((8,), m, dtype=torch.int32, device=dev), torch.full((8,), v, dtype=torch.float64, device=dev))

    for kw, msg in [(dict(mode=good_m.cpu()), "CUDA tensor"), (dict(mode=good_m.long()), "dtype"), (dict(value=good_v.float()), "dtype"),
                    (dict(value=good_v[:4]), "shape"), (dict(state_r=env.state_r[:, :-1].contiguous()), "shape"),
                    (dict(mode=torch.full((8,), 5, dtype=torch.int32, device=dev)), "mode must be"),
                    (dict(zip(("mode", "value"), mv(4, float("nan")))), "finite"),
                    (dict(zip(("mode", "value"), mv(4, 0.25))), "FORWARD stair height"),
                    (dict(zip(("mode", "value"), mv(3, 0.5))), "LATERAL"),
                    (dict(zip(("mode", "value"), mv(0, 109))), "CURVED"), (dict(zip(("mode", "value"), mv(0, 2.5))), "CURVED"),
                    (dict(zip(("mode", "value"), mv(1, 1))), "STANDING or BACKWARD"),
                    (dict(zip(("mode", "value"), mv(2, -1))), "STANDING or BACKWARD")]:
        with pytest.raises(RuntimeError, match=msg):
            call(**kw)
    before = env.state_r.clone()
    call()    # every row -1: nothing changes
    assert torch.equal(before, env.state_r)
    with pytest.raises(ValueError, match="never been reset"):
        _env(64, 4, seed=1).reset_footsteps([4, 4, -1, 4], [0.1, 0.1, 0, 0.1])
    for name in ("jvrc_walk", "h1", "jvrc_walk_terrain", "h1_walk"):
        from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
        other = BatchedHumanoidEnv(8, model=name, precision=64)
        other.reset()
        with pytest.raises(RuntimeError, match=f"{name} has no footstep plan"):
            op(other._h.value, other.state_r, other.state_i, 1, 0, good_m, good_v, False, other.obs)
        with pytest.raises(ValueError, match=f"{name} has no footstep plan"):
            other.reset_footsteps([-1] * 8, [0] * 8)
        other.close()
    env.close()


@pytest.mark.parametrize("precision", [64, 32])
def test_mixed_batch_untouched_rows(precision):
    """Four copies of one batch under the same actions with autoreset on, for 400 steps: `plain` never gets a plan; `eager`,
    `graph` (replayed CUDA graph) and `halves` (step_slice over two halves) get the same mixed plans after their reset.  The three
    planned copies are bit-identical, and their rows given -1 equal `plain`'s bit for bit, records and outputs."""
    n = 512
    envs = {k: _env(precision, n, seed=5, iteration_count=7000) for k in ("plain", "eager", "graph", "halves")}
    mode, value = _plans(n, seed=3)
    for k, e in envs.items():
        e.reset()
        if k != "plain":
            e.reset_footsteps(mode, value)
    gens = {k: torch.Generator(device=e.device).manual_seed(7) for k, e in envs.items()}
    graph_step = _graph_stepper(envs["graph"], gens["graph"])
    free = torch.as_tensor(mode < 0, device=envs["plain"].device)
    ends = 0
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
        ends += int(e.ended[~free].sum())
    assert ends > 0
    for x in envs.values():
        x.close()


@pytest.mark.parametrize("height", [0.0, 0.1])
@pytest.mark.parametrize("precision", [64, 32])
def test_drawn_plan_given_back_equals_reset(precision, height):
    n, seed = 512, 9
    ic = 3000 + 8000 * height / 0.1
    a, b = _env(precision, n, seed=seed, iteration_count=ic), _env(precision, n, seed=seed, iteration_count=ic)
    o = _oracle()
    dt = np.float64 if precision == 64 else np.float32
    plan = [drawn_plan(o, seed, i, 1, height, dt) for i in range(n)]      # a fresh env's first reset: event counter 1
    a.reset()
    b.reset_footsteps([p[0] for p in plan], [p[1] for p in plan])
    assert torch.equal(a.state_r, b.state_r) and torch.equal(a.state_i, b.state_i) and torch.equal(a.obs, b.obs)
    a.close()
    b.close()


def test_mid_episode_copy_of_a_chosen_plan_resumes():
    """The plan lives in the record (mode word, seq, tk): records copied mid-episode into a new env continue bit for bit."""
    n = 256
    env, g = _env(64, n, seed=4), torch.Generator(device="cuda").manual_seed(3)
    env.reset()
    env.reset_footsteps(*_plans(n, seed=5))
    for _ in range(30):
        env.step(_actions(env, g))
    other = _env(64, n, seed=4)
    other.reset()
    other.state_r.copy_(env.state_r)
    other.state_i.copy_(env.state_i)
    g2 = torch.Generator(device="cuda").manual_seed(11)
    g.manual_seed(11)
    for t in range(100):
        env.step(_actions(env, g))
        other.step(_actions(other, g2))
        assert torch.equal(env.state_r, other.state_r) and torch.equal(env.state_i, other.state_i), t
        assert torch.equal(env.obs, other.obs) and torch.equal(env.reward, other.reward), t
    env.close()
    other.close()


def test_train_then_eval_footsteps(tmp_path, capsys):
    """`train --env jvrc_step --n-itr 2`, then `eval --num-envs 256 --footsteps ... --report` and the single-env roll-out with one
    plan (with its video when OpenCV is present)."""
    import run_experiment as rx
    rx.main(["train", "--env", "jvrc_step", "--logdir", str(tmp_path / "logs"), "--num-procs", "64", "--n-itr", "2",
             "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    path = tmp_path / "r.json"
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--num-envs", "256", "--footsteps", "forward:0,0.05,0.1,0.15",
             "lateral:left,right", "backward", "curved", "curved:3", "standing", "--report", str(path)])
    out = capsys.readouterr().out
    assert "chosen footstep plans" in out and "forward:0.15" in out and "lateral:right" in out
    r = json.loads(path.read_text())
    cells = r["summary"]["footsteps_sweep"]["cells"]
    assert [c["label"] for c in cells] == ["forward:0", "forward:0.05", "forward:0.1", "forward:0.15", "lateral:left", "lateral:right",
                                           "backward", "curved", "curved:3", "standing"]
    assert [c["n"] for c in cells] == [26] * 6 + [25] * 4
    for c in cells:
        assert set(c) == {"mode", "value", "label", "n", "fall_fraction", "mean_length", "mean_reached", "mean_sequence_length",
                          "completed_fraction", "return_mean"}
        assert 0 <= c["fall_fraction"] <= 1 and 0 <= c["completed_fraction"] <= 1
    pe = r["per_env"]
    assert pe["footstep_mode"][:11] == ["FORWARD"] * 4 + ["LATERAL"] * 2 + ["BACKWARD", "CURVED", "CURVED", "STANDING", "FORWARD"]
    assert pe["footstep_value"][3] == 0.15 and pe["footstep_value"][5] == -1.0 and len(pe["footstep_value"]) == 256
    episodes = rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--ep-len", "2", "--footsteps", "forward:0.1"])
    assert sum(l for l, _ in episodes) == 80
    cv2 = pytest.importorskip("cv2", reason="OpenCV (cv2) is needed to write the video")
    out_dir = tmp_path / "video"
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--ep-len", "2", "--footsteps", "forward:0.1", "--out-dir", str(out_dir)])
    videos = list(out_dir.iterdir())
    assert len(videos) == 1 and videos[0].suffix == ".mp4"
    cap = cv2.VideoCapture(str(videos[0]))
    ok, frame = cap.read()
    cap.release()
    assert ok and frame.shape == (480, 640, 3)
