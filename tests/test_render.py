"""The renderer's source (csrc/render_core.h), built for the host, against oracle/render_oracle.py and known answers: forward
kinematics, whole images of each robot / task, an empty checkerboard, one link's box on its projected rectangle, and the
shadow under the feet."""
import numpy as np
import pytest

from emu import Emu
from learninghumanoidwalking_b200.model import load_model, pack_model
from oracle import render_oracle as RO
from render_emu import RenderEmu
from tools.compile_model import kinematics

CAM = (0.0, 0.0, 0.8, 3.0, 90.0, 15.0, 45.0)     # BatchedHumanoidEnv.render_rgb's tracking camera (z 0.9 for h1)
W, H = 200, 150
VARIANTS = ("jvrc_walk", "h1", "jvrc_step", "jvrc_walk_terrain")


def cam_for(name):
    return (0.0, 0.0, 0.9 if name == "h1" else 0.8) + CAM[3:]


def record(name, precision=64, n=1, seed=0):
    e = Emu(pack_model(load_model(name)), precision=precision, n=n, seed=seed)
    e.reset()
    return e.sr, e.si


def forward_record(precision=64):
    """a jvrc_step record in FORWARD mode (floor dropped to -2, stairs)"""
    sr, si = record("jvrc_step", precision, n=32, seed=1)
    k = int(np.flatnonzero(si[:, 1] == RO.ST_FORWARD)[0])
    return sr[k], si[k]


@pytest.mark.parametrize("name", VARIANTS)
def test_forward_kinematics_matches_compile_model(name):
    mj = load_model(name)
    rng = np.random.default_rng(7)
    for precision in (64, 32):
        R = RenderEmu(pack_model(mj), precision)
        for _ in range(10):
            nu = len(mj["links"]) - 1
            quat = rng.normal(size=4)
            qpos = np.concatenate([rng.uniform(-2, 2, 3), quat / np.linalg.norm(quat), rng.uniform(-1.2, 1.2, nu)])
            if precision == 32:
                qpos = qpos.astype(np.float32).astype(np.float64)
            xpos, xmat = R.fk(qpos)
            xp, xm = kinematics(mj, qpos)
            np.testing.assert_allclose(xpos, xp, atol=1e-5)
            np.testing.assert_allclose(xmat, xm, atol=1e-5)


def _compare(img, ref, frac=0.002, levels=2):
    bad = np.abs(img.astype(int) - ref.astype(int)).max(axis=-1) > levels
    assert bad.mean() <= frac, f"{bad.sum()} of {bad.size} pixels differ by more than {levels} levels"


@pytest.mark.parametrize("case", ["jvrc_walk", "h1", "jvrc_step_forward", "jvrc_walk_terrain"])
def test_image_matches_oracle(case):
    name = "jvrc_step" if case == "jvrc_step_forward" else case
    mj = load_model(name)
    if case == "jvrc_step_forward":
        sr, si = forward_record()
        assert RO.record_parts(mj, sr, si)[2] == RO.ST_FORWARD
    else:
        sr, si = (a[0] for a in record(name))
    img, _ = RenderEmu(pack_model(mj), 64).image(sr, si, W, H, cam_for(name))
    ref = RO.render(mj, sr, si, W, H, cam_for(name))
    _compare(img, ref)
    link = RO.to_byte(np.array(RO.ALBEDO["link"]) * RO.AMBIENT)
    assert (img[..., 0] >= link[0]).sum() > 200 and (img[..., 0] > img[..., 2] + 40).sum() > 200, "the robot is not in the picture"
    if case == "jvrc_step_forward":
        slab_lit = RO.to_byte(np.array(RO.ALBEDO["slab"]) * (RO.AMBIENT + RO.DIFFUSE * RO.LIGHT[2]))
        assert (img == slab_lit).all(axis=-1).sum() > 100, "no slab top faces in view"


def test_robot_out_of_view_leaves_an_exact_checkerboard():
    mj = load_model("jvrc_walk")
    sr, si = (a[0].copy() for a in record("jvrc_walk"))
    sr[2] += 1e4
    img, _ = RenderEmu(pack_model(mj), 64).image(sr, si, W, H, CAM)
    lit = RO.AMBIENT + RO.DIFFUSE * RO.LIGHT[2]
    allowed = {tuple(RO.to_byte(RO.SKY))} | {tuple(RO.to_byte(np.array(RO.ALBEDO[k]) * lit)) for k in ("floor_a", "floor_b")}
    colours = {tuple(c) for c in img.reshape(-1, 3)}
    assert colours == allowed, colours ^ allowed
    ref = RO.render(mj, sr, si, W, H, CAM)
    assert (img == ref).all(axis=-1).mean() >= 0.999


def test_one_link_box_lands_on_its_projected_rectangle():
    mj = load_model("jvrc_walk")
    sr, si = (a[0] for a in record("jvrc_walk"))
    link = 4                                      # right shank
    img, _ = RenderEmu(pack_model(mj), 64).image(sr, si, W, H, CAM, only_box=link)
    mask = img[..., 0].astype(int) > 1.5 * img[..., 2].astype(int) + 1
    rows, cols = np.nonzero(mask)
    assert len(rows) > 20
    qpos, _, _ = RO.record_parts(mj, sr, si)
    c, R, h, _ = RO.scene(mj, qpos)[0][link]
    corners = [c + R @ (h * np.array(s)) for s in np.array(np.meshgrid([-1, 1], [-1, 1], [-1, 1])).reshape(3, -1).T]
    xs, ys = zip(*(RO.project(p, qpos[:2], CAM, W, H) for p in corners))
    assert abs(cols.min() - np.ceil(min(xs))) <= 1 and abs(cols.max() - np.floor(max(xs))) <= 1, (cols.min(), cols.max(), xs)
    assert abs(rows.min() - np.ceil(min(ys))) <= 1 and abs(rows.max() - np.floor(max(ys))) <= 1, (rows.min(), rows.max(), ys)


def test_floor_under_the_feet_is_darker_with_the_robot_present():
    mj = load_model("jvrc_walk")
    sr, si = (a[0].copy() for a in record("jvrc_walk"))
    R = RenderEmu(pack_model(mj), 64)
    img, boxes = R.image(sr, si, W, H, CAM)
    away = sr.copy()
    away[2] += 1e4
    empty, _ = R.image(away, si, W, H, CAM)
    nl = len(mj["links"])
    x, y = RO.project(boxes[nl, :3], sr[:2], CAM, W, H)        # the right foot's contact box
    lit, amb = RO.AMBIENT + RO.DIFFUSE * RO.LIGHT[2], RO.AMBIENT
    window = (slice(max(0, int(y) - 25), int(y) + 25), slice(max(0, int(x) - 25), int(x) + 25))
    shadowed = np.zeros(img.shape[:2], bool)
    for k in ("floor_a", "floor_b"):
        alb = np.array(RO.ALBEDO[k])
        shadowed |= (empty == RO.to_byte(alb * lit)).all(-1) & (img == RO.to_byte(alb * amb)).all(-1)
    assert shadowed[window].sum() >= 5, "no shadowed floor pixel near the feet"
