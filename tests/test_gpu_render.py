"""torch.ops.lhw.sim_render / BatchedHumanoidEnv.render_rgb on the device: images equal to the host build of the same source
(tests/emu/render_emu.cpp), read-only, batched = single calls, each sim renders its own model, argument checks, and the
`eval --out-dir` video end to end."""
import numpy as np
import pytest
import torch

from learninghumanoidwalking_b200.model import load_model, pack_model
from render_emu import RenderEmu

pytestmark = pytest.mark.gpu
VARIANTS = ("jvrc_walk", "h1", "jvrc_step", "jvrc_walk_terrain")
W, H = 320, 240


def make_env(name, precision, n=8, steps=5):
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(n, model=name, precision=precision, seed=3)
    env.reset()
    g = torch.Generator(device=env.device).manual_seed(0)
    for _ in range(steps):
        env.step(0.3 * torch.randn(n, env.act_dim, generator=g, device=env.device, dtype=env.dtype))
    torch.cuda.synchronize()
    return env


def camera(env):
    return (0.0, 0.0, 0.9 if env.model_name == "h1" else 0.8, 3.0, 90.0, 15.0, 45.0)


@pytest.mark.parametrize("precision", [64, 32])
@pytest.mark.parametrize("name", VARIANTS)
def test_device_images_match_host_build(name, precision):
    env = make_env(name, precision)
    ids = list(range(env.num_envs))
    dev = env.render_rgb(ids, W, H).cpu().numpy()
    host = RenderEmu(pack_model(load_model(name)), precision)
    sr, si = env.state_r.cpu().numpy(), env.state_i.cpu().numpy()
    for k in ids:
        ref, _ = host.image(sr[k], si[k], W, H, camera(env))
        diff = np.abs(dev[k].astype(int) - ref.astype(int)).max(-1)
        assert (diff > 0).mean() <= 0.001 and diff.max() <= 2, (k, int((diff > 0).sum()), int(diff.max()))
    env.close()


def test_render_reads_state_only():
    env = make_env("jvrc_step", 32)
    before = (env.state_r.clone(), env.state_i.clone())
    a = torch.full((env.num_envs, env.act_dim), 0.1, device=env.device, dtype=env.dtype)
    twin = make_env("jvrc_step", 32)
    env.render_rgb(list(range(env.num_envs)), W, H)
    torch.cuda.synchronize()
    assert torch.equal(env.state_r, before[0]) and torch.equal(env.state_i, before[1])
    assert torch.equal(env.state_r, twin.state_r) and torch.equal(env.state_i, twin.state_i)
    env.step(a)
    twin.step(a)
    for x, y in ((env.obs, twin.obs), (env.reward, twin.reward), (env.done, twin.done), (env.state_r, twin.state_r),
                 (env.state_i, twin.state_i), (env.rew_terms, twin.rew_terms)):
        assert torch.equal(x, y)
    env.close()
    twin.close()


def test_batched_call_equals_single_calls():
    env = make_env("jvrc_walk", 64)
    many = env.render_rgb([3, 0, 7], W, H)
    for j, k in enumerate((3, 0, 7)):
        assert torch.equal(many[j], env.render_rgb((k,), W, H)[0])
    assert not torch.equal(many[0], many[1])
    env.close()


def test_each_sim_renders_its_own_model(monkeypatch):
    from learninghumanoidwalking_b200.envs import batched_env
    a = make_env("jvrc_walk", 32, n=2, steps=0)
    ref = a.render_rgb((0,), W, H).clone()
    heavy = load_model("jvrc_walk")
    for lk in heavy["links"]:
        lk["inertia"] = [4 * v for v in lk["inertia"]]        # boxes twice as large
    monkeypatch.setattr(batched_env, "load_model", lambda name: heavy)
    b = make_env("jvrc_walk", 32, n=2, steps=0)
    b.bind()                                                 # b's model now sits in the constant bank
    assert torch.equal(a.render_rgb((0,), W, H), ref)
    b.state_r.copy_(a.state_r)
    b.state_i.copy_(a.state_i)
    assert not torch.equal(b.render_rgb((0,), W, H), ref)
    assert torch.equal(a.render_rgb((0,), W, H), ref)
    a.close()
    b.close()


def test_op_rejects_bad_arguments_before_a_launch():
    from learninghumanoidwalking_b200 import _lib
    env = make_env("jvrc_walk", 32, n=4, steps=0)
    O, h = _lib.ops(), env._h.value
    ids = torch.zeros(1, dtype=torch.int32, device=env.device)
    rgb = torch.zeros(1, 32, 32, 3, dtype=torch.uint8, device=env.device)
    cam = (0.0, 0.0, 0.8, 3.0, 90.0, 15.0, 45.0)

    def call(state_r=env.state_r, state_i=env.state_i, ids=ids, w=32, hgt=32, cam=cam, rgb=rgb):
        O.sim_render(h, state_r, state_i, ids, w, hgt, *cam, rgb)

    torch.cuda.synchronize()
    launches = _lib.lib().lhw_launch_count()
    bad = [
        (dict(state_r=env.state_r.cpu()), "must be a CUDA tensor"),
        (dict(state_r=env.state_r.double()), "dtype"),
        (dict(state_r=env.state_r.t().contiguous().t()), "contiguous"),
        (dict(state_i=env.state_i[:2]), "shape"),
        (dict(ids=ids.long()), "dtype"),
        (dict(ids=torch.tensor([4], dtype=torch.int32, device=env.device)), "env_ids must lie in"),
        (dict(ids=torch.tensor([-1], dtype=torch.int32, device=env.device)), "env_ids must lie in"),
        (dict(rgb=rgb.float()), "dtype"),
        (dict(rgb=torch.zeros(1, 32, 33, 3, dtype=torch.uint8, device=env.device)), "shape"),
        (dict(rgb=torch.zeros(2, 32, 32, 3, dtype=torch.uint8, device=env.device)), "shape"),
        (dict(w=8), "16..4096"),
        (dict(hgt=5000), "16..4096"),
        (dict(cam=cam[:3] + (0.0,) + cam[4:]), "distance"),
        (dict(cam=cam[:6] + (180.0,)), "fovy"),
        (dict(cam=cam[:6] + (0.0,)), "fovy"),
    ]
    for kw, msg in bad:
        with pytest.raises(RuntimeError, match=msg):
            call(**kw)
    assert _lib.lib().lhw_launch_count() == launches
    call()
    assert _lib.lib().lhw_launch_count() == launches + 1
    env.close()


def test_eval_out_dir_writes_the_rollout_video(tmp_path):
    cv2 = pytest.importorskip("cv2", reason="OpenCV (cv2) is needed to decode the video")
    import run_experiment as rx
    rx.main(["train", "--env", "jvrc_walk", "--logdir", str(tmp_path / "logs"), "--num-procs", "64", "--n-itr", "2",
             "--max-traj-len", "40", "--minibatch-size", "256", "--epochs", "1", "--seed", "3", "--eval-freq", "2"])
    out = tmp_path / "video"
    rx.main(["eval", "--logdir", str(tmp_path / "logs"), "--ep-len", "2", "--out-dir", str(out)])
    run = rx.get_latest_run_dir(tmp_path / "logs")
    video = out / (rx.get_latest_actor(run).stem + ".mp4")
    assert sorted(p.name for p in out.iterdir()) == [video.name]
    cap = cv2.VideoCapture(str(video))
    frames = []
    while True:
        ok, f = cap.read()
        if not ok:
            break
        frames.append(f[..., ::-1])
    cap.release()
    assert len(frames) == 81 and frames[0].shape == (480, 640, 3)
    assert any(not np.array_equal(frames[0], f) for f in frames[1:])
    from learninghumanoidwalking_b200.envs import BatchedHumanoidEnv
    env = BatchedHumanoidEnv(1, model="jvrc_walk", precision=64, seed=0)
    env.reset()
    first = env.render_rgb((0,), 640, 480)[0].cpu().numpy().astype(float)
    assert np.abs(frames[0].astype(float) - first).mean() < 6.0      # mp4 is lossy
    env.close()
