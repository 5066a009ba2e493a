"""Independent numpy restatement of the renderer (learninghumanoidwalking_b200/csrc/render_core.h) for the tests.

Same scene definition and shading formula as the header comment there, computed differently: float64 throughout, forward
kinematics from tools/compile_model.py:kinematics on the model JSON, principal axes by numpy.linalg.eigh, and its own
vectorised box / sphere / plane intersection over all pixels at once.  Test infrastructure only: the product never imports it.
"""
from __future__ import annotations

import numpy as np

from tools.compile_model import kinematics

# palette and light, restated from render_core.h
ALBEDO = {"floor_a": (0.78, 0.78, 0.76), "floor_b": (0.52, 0.54, 0.56), "link": (0.90, 0.58, 0.30),
          "contact": (0.25, 0.50, 0.90), "slab": (0.55, 0.62, 0.50)}
SKY = (0.60, 0.74, 0.90)
LIGHT = np.array([-0.36, -0.48, 0.80])
AMBIENT, DIFFUSE = 0.35, 0.65
SHADOW_BIAS, HIT_EPS, FLOOR_FAR, CHECKER, MIN_HALF = 1e-3, 1e-4, 50.0, 0.5, 0.005
NSLAB, ST_FORWARD = 20, 4


def to_byte(c):
    return np.minimum(255.0, np.floor(255.0 * np.asarray(c) + 0.5)).astype(np.uint8)


def record_parts(mj, sr, si):
    """qpos, the slab sequence [20, 4] (None without slabs) and the stepping mode of one environment's record."""
    nj = (len(mj["links"]) - 1) // 2
    nq, nv, nu = 7 + 2 * nj, 6 + 2 * nj, 2 * nj
    sr = np.asarray(sr, dtype=np.float64)
    seq = None
    if has_slabs(mj):
        off = nq + 2 * nv + 5 * nu + 4
        seq = sr[off:off + 4 * NSLAB].reshape(NSLAB, 4)
    return sr[:nq], seq, int(si[1])


def has_slabs(mj):
    return mj["name"] == "jvrc_step" or bool(mj.get("terrain"))


def inertia_box(lk):
    a = lk["inertia"]
    inertia = np.array([[a[0], a[3], a[4]], [a[3], a[1], a[5]], [a[4], a[5], a[2]]])
    lam, V = np.linalg.eigh(inertia)
    half = np.array([3.0 / (2.0 * lk["mass"]) * (lam[(k + 1) % 3] + lam[(k + 2) % 3] - lam[k]) for k in range(3)])
    return V, np.maximum(MIN_HALF, np.sqrt(np.maximum(0.0, half)))


def scene(mj, qpos, seq=None, mode=0):
    """boxes [(centre, rotation, half sizes, material)] in the test order, spheres [(centre, radius)], floor height."""
    xpos, xmat = kinematics(mj, np.asarray(qpos, dtype=np.float64))
    boxes, spheres = [], []
    for i, lk in enumerate(mj["links"]):
        V, h = inertia_box(lk)
        boxes.append((xpos[i] + xmat[i] @ np.array(lk["com"]), xmat[i] @ V, h, "link"))
    for g in mj["geoms"]:
        lk = g["link"]
        if g["type"] == "box":
            boxes.append((xpos[lk] + xmat[lk] @ np.array(g["pos"]), xmat[lk], np.array(g["size"], dtype=float), "contact"))
        else:
            spheres += [(xpos[lk] + xmat[lk] @ np.array(p), g["radius"]) for p in g["points"]]
    if has_slabs(mj):
        half = np.array(mj["stepping"]["slab_half"] if mj["name"] == "jvrc_step" else mj["terrain"]["strip_half"], dtype=float)
        for x, y, z, th in seq:
            c, s = np.cos(th), np.sin(th)
            boxes.append((np.array([x, y, z - half[2]]), np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]]), half, "slab"))
    floor_z = -2.0 if (mj["name"] == "jvrc_step" and mode == ST_FORWARD) else 0.0
    return boxes, spheres, floor_z


def camera(cam, width, height):
    dx, dy, z, dist, az, el, fovy = cam
    a, e = np.deg2rad(az), np.deg2rad(el)
    f = np.array([np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), -np.sin(e)])
    r = np.array([np.sin(a), -np.cos(a), 0.0])
    u = np.cross(r, f)
    th = np.tan(np.deg2rad(fovy) / 2)
    return f, r * th * width / height, u * th


def rays(root_xy, cam, width, height):
    """eye [3] and unit ray directions [H, W, 3]."""
    f, r, u = camera(cam, width, height)
    eye = np.array([root_xy[0] + cam[0], root_xy[1] + cam[1], cam[2]]) - cam[3] * f
    x = 2 * (np.arange(width) + 0.5) / width - 1
    y = 1 - 2 * (np.arange(height) + 0.5) / height
    d = f + x[None, :, None] * r + y[:, None, None] * u
    return eye, d / np.linalg.norm(d, axis=-1, keepdims=True)


def project(p, root_xy, cam, width, height):
    """pixel coordinates (column, row) of world point p (pixel centres at integers)."""
    f, r, u = camera(cam, width, height)
    eye = np.array([root_xy[0] + cam[0], root_xy[1] + cam[1], cam[2]]) - cam[3] * f
    w = np.asarray(p, dtype=float) - eye
    x, y = (w @ r) / (r @ r) / (w @ f), (w @ u) / (u @ u) / (w @ f)
    return (x + 1) * width / 2 - 0.5, (1 - y) * height / 2 - 0.5


def _box(o, d, c, R, h):
    """slab test; o, d broadcast to [N, 3]: (entry t, exit t, entry axis, sign of the entry normal)."""
    lo, ld = (o - c) @ R, d @ R
    lo, ld = np.broadcast_arrays(lo, ld)
    with np.errstate(divide="ignore", invalid="ignore"):
        t1, t2 = (-h - lo) / ld, (h - lo) / ld
    ta, tb = np.minimum(t1, t2), np.maximum(t1, t2)
    par = ld == 0
    inside = np.abs(lo) <= h
    ta = np.where(par, np.where(inside, -np.inf, np.inf), ta)
    tb = np.where(par, np.where(inside, np.inf, -np.inf), tb)
    ax = np.argmax(ta, axis=-1)
    tn = np.take_along_axis(ta, ax[..., None], -1)[..., 0]
    tf = tb.min(axis=-1)
    sg = -np.sign(np.take_along_axis(ld, ax[..., None], -1)[..., 0])
    return tn, tf, ax, sg


def render(mj, sr, si, width, height, cam):
    """One environment's record -> rgb [H, W, 3] uint8."""
    qpos, seq, mode = record_parts(mj, sr, si)
    boxes, spheres, floor_z = scene(mj, qpos, seq, mode)
    eye, d = rays(qpos[:2], cam, width, height)
    d = d.reshape(-1, 3)
    n_pix = len(d)
    best = np.full(n_pix, np.inf)
    mat = np.full(n_pix, "", dtype=object)
    nrm = np.zeros((n_pix, 3))

    def take(hit, t, n, m):
        upd = hit & (t < best - HIT_EPS)
        best[upd] = t[upd]
        nrm[upd] = n[upd] if np.ndim(n) == 2 else n
        mat[upd] = m

    robot = [b for b in boxes if b[3] != "slab"]
    slabs = [b for b in boxes if b[3] == "slab"]
    for c, R, h, m in robot:
        tn, tf, ax, sg = _box(eye, d, c, R, h)
        take((tn <= tf) & (tn > 0), tn, sg[:, None] * R.T[ax], m)
    for c, r in spheres:
        w = eye - c
        b = d @ w
        disc = b * b - (w @ w - r * r)
        t = -b - np.sqrt(np.maximum(disc, 0))
        take((disc >= 0) & (t > 0), t, (eye + t[:, None] * d - c) / r, "contact")
    for c, R, h, m in slabs:
        tn, tf, ax, sg = _box(eye, d, c, R, h)
        take((tn <= tf) & (tn > 0), tn, sg[:, None] * R.T[ax], m)
    if eye[2] > floor_z:
        with np.errstate(divide="ignore", invalid="ignore"):
            t = np.where(d[:, 2] < 0, (floor_z - eye[2]) / d[:, 2], np.inf)
        p = eye + np.where(np.isfinite(t), t, 0)[:, None] * d
        odd = (np.floor(p[:, 0] / CHECKER) + np.floor(p[:, 1] / CHECKER)).astype(np.int64) & 1
        hit = (d[:, 2] < 0) & (t <= FLOOR_FAR)
        upd = hit & (t < best - HIT_EPS)
        best[upd] = t[upd]
        nrm[upd] = (0.0, 0.0, 1.0)
        mat[upd & (odd == 0)] = "floor_a"
        mat[upd & (odd == 1)] = "floor_b"
    lam = np.maximum(0.0, nrm @ LIGHT)
    lit = (mat != "") & (lam > 0)
    o = eye + np.where(np.isfinite(best), best, 0)[:, None] * d + SHADOW_BIAS * nrm
    shadow = o[:, 2] < floor_z
    for c, R, h, _ in boxes:
        tn, tf, _, _ = _box(o, LIGHT, c, R, h)
        shadow |= np.maximum(tn, 0) <= tf
    for c, r in spheres:
        w = o - c
        b = w @ LIGHT
        disc = b * b - (np.einsum("ij,ij->i", w, w) - r * r)
        shadow |= (disc >= 0) & (-b + np.sqrt(np.maximum(disc, 0)) >= 0)
    lam = np.where(lit & ~shadow, lam, 0.0)
    out = np.empty((n_pix, 3))
    out[:] = SKY
    for m, alb in ALBEDO.items():
        sel = mat == m
        out[sel] = np.array(alb) * (AMBIENT + DIFFUSE * lam[sel])[:, None]
    return to_byte(out).reshape(height, width, 3)
