// render_core.h — ray-cast picture of one environment (host + device code, like sim_core.h).
//
// Replaces the reference's video path, rl/utils/eval.py:37-86 (EvaluateEnv.run: mujoco.Renderer offscreen frames of the
// roll-out).  The scene is built from the compiled model and one environment's HBM state record only: the renderer does
// its own forward kinematics and never touches the step kernel or its outputs.
//
// Scene (all fp32, whatever the simulator's precision):
//   * every link as its equivalent-inertia box (MuJoCo's inertia visualisation): centred at the link com, axes = the principal
//     axes of the link inertia (3x3 symmetric Jacobi), half extents h_a = sqrt(3 / (2 m) (I_b + I_c - I_a)), at least 5 mm.
//     H1 uses the nominal masses and inertias of the model, not the per-environment randomised ones;
//   * the contact geometry of the physics in a second colour: JVRC foot boxes (foot_pos / foot_size), H1 foot spheres
//     (foot_pts / foot_radius);
//   * slab variants (jvrc_step, terrain): all 20 slabs as the physics has them, parked ones included: box k centred at
//     (seq[k].x, seq[k].y, seq[k].z - slab_half.z), yawed by seq[k].theta, half sizes slab_half;
//   * the floor plane z = floor_z (-2 for jvrc_step in FORWARD mode, else 0) with a 0.5 m checkerboard, out to FLOOR_FAR
//     metres along the ray (beyond it the sky shows: the far checkerboard is finer than a pixel).
// Forward kinematics (serial, fp32, the formula of tools/compile_model.py:kinematics): root from qpos[0:7]; child i of
// parent p: R_i = R_p link_rot_i Rot(axis_i, q_i), p_i = p_p + R_p link_pos_i.
//
// Camera: pinhole from seven scalars (dx, dy, z, distance, azimuth, elevation, fovy; degrees).  Look-at point
// t = (root_x + dx, root_y + dy, z) with the root position read from the record, forward f = (ce ca, ce sa, -se)
// (a = azimuth, e = elevation: e > 0 looks down), eye = t - distance f, right r = (sa, -ca, 0), up u = r x f.  The ray of
// pixel (px, py) of a W x H image (row 0 at the top) points along f + x r + y u, normalised, with
// x = (2 (px + 0.5) / W - 1) tan(fovy / 2) W / H and y = (1 - 2 (py + 0.5) / H) tan(fovy / 2).
//
// Shading: closest hit; primitives are tested in the order robot link boxes, contact geometry, slabs, floor, and a later one
// replaces the hit so far only when it is nearer by more than HIT_EPS (coplanar faces: the earlier primitive wins).
//   colour c = albedo * (AMBIENT + DIFFUSE * max(0, n . L) * visible),
//   visible = 0 when the ray from p + SHADOW_BIAS n toward L meets any primitive (the floor included), else 1;
//   no hit: c = SKY.  Channel value = min(255, floor(255 c + 0.5)).  No anti-aliasing.
// The palette and the light live in render_albedo() / the constants below (oracle/render_oracle.py restates them).
#pragma once
#include <math.h>
#include <stdint.h>

#include "sim_core.h"

namespace lhw {
namespace render {

// ---------------------------------------------------------------- palette and light (the one place they are defined)
enum { MAT_FLOOR_A = 0, MAT_FLOOR_B = 1, MAT_LINK = 2, MAT_CONTACT = 3, MAT_SLAB = 4 };
LHW_DEV void render_albedo(int mat, float c[3]) {
  switch (mat) {
    case MAT_FLOOR_A: c[0] = 0.78f; c[1] = 0.78f; c[2] = 0.76f; break;
    case MAT_FLOOR_B: c[0] = 0.52f; c[1] = 0.54f; c[2] = 0.56f; break;
    case MAT_LINK: c[0] = 0.90f; c[1] = 0.58f; c[2] = 0.30f; break;
    case MAT_CONTACT: c[0] = 0.25f; c[1] = 0.50f; c[2] = 0.90f; break;
    default: c[0] = 0.55f; c[1] = 0.62f; c[2] = 0.50f; break;   // MAT_SLAB
  }
}
constexpr float SKY_R = 0.60f, SKY_G = 0.74f, SKY_B = 0.90f;
constexpr float LIGHT_X = -0.36f, LIGHT_Y = -0.48f, LIGHT_Z = 0.80f;   // unit vector toward the light
constexpr float AMBIENT = 0.35f, DIFFUSE = 0.65f;
constexpr float SHADOW_BIAS = 1e-3f, HIT_EPS = 1e-4f, FLOOR_FAR = 50.0f, CHECKER = 0.5f, MIN_HALF = 0.005f;

// ---------------------------------------------------------------- camera (host: from the seven scalars)
struct Camera {
  float fwd[3], right[3], up[3];   // right / up pre-scaled by tan(fovy/2) W/H and tan(fovy/2)
  float look[3];                   // (dx, dy, z): added to (root_x, root_y, 0)
  float dist;
};
inline Camera make_camera(double dx, double dy, double z, double distance, double azimuth, double elevation, double fovy,
                          int width, int height) {
  const double d2r = 3.14159265358979323846 / 180.0;
  const double ca = cos(azimuth * d2r), sa = sin(azimuth * d2r), ce = cos(elevation * d2r), se = sin(elevation * d2r);
  const double th = tan(0.5 * fovy * d2r), tw = th * width / height;
  const double f[3] = {ce * ca, ce * sa, -se}, r[3] = {sa, -ca, 0.0};
  const double u[3] = {r[1] * f[2] - r[2] * f[1], r[2] * f[0] - r[0] * f[2], r[0] * f[1] - r[1] * f[0]};
  Camera c;
  for (int k = 0; k < 3; k++) {
    c.fwd[k] = (float)f[k];
    c.right[k] = (float)(r[k] * tw);
    c.up[k] = (float)(u[k] * th);
  }
  c.look[0] = (float)dx; c.look[1] = (float)dy; c.look[2] = (float)z;
  c.dist = (float)distance;
  return c;
}

// ---------------------------------------------------------------- scene of one environment
template <int NJ, int TK> struct Scene {
  static constexpr int NL = 1 + 2 * NJ;
  static constexpr bool SPH = Cfg<NJ, TK>::SPHERES;
  static constexpr int NFOOT = SPH ? 0 : 2, NSL = Cfg<NJ, TK>::SLABS ? NSLAB : 0, NBOX = NL + NFOOT + NSL;
  static constexpr int NSPH = SPH ? 2 * Cfg<NJ, TK>::NPTS : 0;
  float bc[NBOX][3], br[NBOX][9], bh[NBOX][3];   // box centre, rotation (row-major, box frame -> world), half sizes
  float sc[NSPH ? NSPH : 1][4];                  // sphere centre, radius
  float eye[3], floor_z;
  // forward kinematics and the link-frame inertia boxes (scratch of the set-up)
  float xpos[NL][3], xmat[NL][9], lv[NL][9], lh[NL][3];
};

template <int NJ, int TK> LHW_DEV int box_material(int b) {
  return b < Scene<NJ, TK>::NL ? MAT_LINK : b < Scene<NJ, TK>::NL + Scene<NJ, TK>::NFOOT ? MAT_CONTACT : MAT_SLAB;
}

// serial forward kinematics from the record's qpos (the formula of tools/compile_model.py:kinematics), fp32
template <class real, int NJ, int TK>
LHW_DEV void scene_fk(const Model<real, NJ, TK>& m, const real* qpos, float xpos[][3], float xmat[][9]) {
  constexpr int NL = 1 + 2 * NJ;
  float q0 = (float)qpos[3], q1 = (float)qpos[4], q2 = (float)qpos[5], q3 = (float)qpos[6];
  const float n = 1.0f / sqrtf(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
  q0 *= n; q1 *= n; q2 *= n; q3 *= n;
  float* R = xmat[0];
  R[0] = 1 - 2 * (q2 * q2 + q3 * q3); R[1] = 2 * (q1 * q2 - q0 * q3); R[2] = 2 * (q1 * q3 + q0 * q2);
  R[3] = 2 * (q1 * q2 + q0 * q3); R[4] = 1 - 2 * (q1 * q1 + q3 * q3); R[5] = 2 * (q2 * q3 - q0 * q1);
  R[6] = 2 * (q1 * q3 - q0 * q2); R[7] = 2 * (q2 * q3 + q0 * q1); R[8] = 1 - 2 * (q1 * q1 + q2 * q2);
  for (int k = 0; k < 3; k++) xpos[0][k] = (float)qpos[k];
#pragma unroll 1
  for (int i = 1; i < NL; i++) {
    const int p = (i - 1) % NJ == 0 ? 0 : i - 1;
    const float* Rp = xmat[p];
    float s, c;
    sincosf((float)qpos[6 + i], &s, &c);
    const float a[3] = {(float)m.axis[i][0], (float)m.axis[i][1], (float)m.axis[i][2]};
    // Rot(a, q) = c I + s [a]x + (1 - c) a a^T
    const float K[9] = {0, -a[2], a[1], a[2], 0, -a[0], -a[1], a[0], 0};
    float J[9], LJ[9];
    for (int r = 0; r < 3; r++)
      for (int k = 0; k < 3; k++) J[3 * r + k] = (r == k ? c : 0.0f) + s * K[3 * r + k] + (1 - c) * a[r] * a[k];
    for (int r = 0; r < 3; r++)
      for (int k = 0; k < 3; k++)
        LJ[3 * r + k] = (float)m.link_rot[i][3 * r] * J[k] + (float)m.link_rot[i][3 * r + 1] * J[3 + k] +
                        (float)m.link_rot[i][3 * r + 2] * J[6 + k];
    for (int r = 0; r < 3; r++) {
      for (int k = 0; k < 3; k++) xmat[i][3 * r + k] = Rp[3 * r] * LJ[k] + Rp[3 * r + 1] * LJ[3 + k] + Rp[3 * r + 2] * LJ[6 + k];
      xpos[i][r] = xpos[p][r] + Rp[3 * r] * (float)m.link_pos[i][0] + Rp[3 * r + 1] * (float)m.link_pos[i][1] +
                   Rp[3 * r + 2] * (float)m.link_pos[i][2];
    }
  }
}

// link i's equivalent-inertia box in the link frame: principal axes V (columns) by cyclic Jacobi, half extents lh
template <class real, int NJ, int TK> LHW_DEV void scene_inertia_box(const Model<real, NJ, TK>& m, int i, float V[9], float lh[3]) {
  float A[3][3] = {{(float)m.inertia[i][0], (float)m.inertia[i][3], (float)m.inertia[i][4]},
                   {(float)m.inertia[i][3], (float)m.inertia[i][1], (float)m.inertia[i][5]},
                   {(float)m.inertia[i][4], (float)m.inertia[i][5], (float)m.inertia[i][2]}};
  for (int k = 0; k < 9; k++) V[k] = (k % 4 == 0) ? 1.0f : 0.0f;
#pragma unroll 1
  for (int sweep = 0; sweep < 6; sweep++) {
#pragma unroll 1
    for (int pr = 0; pr < 3; pr++) {
      const int p = pr == 2 ? 1 : 0, q = pr == 0 ? 1 : 2;
      const float apq = A[p][q];
      if (apq == 0.0f) continue;
      const float theta = (A[q][q] - A[p][p]) / (2 * apq);
      const float t = (theta >= 0 ? 1.0f : -1.0f) / (fabsf(theta) + sqrtf(theta * theta + 1));
      const float c = 1.0f / sqrtf(t * t + 1), s = t * c;
      for (int k = 0; k < 3; k++) {
        const float akp = A[k][p], akq = A[k][q];
        A[k][p] = c * akp - s * akq;
        A[k][q] = s * akp + c * akq;
      }
      for (int k = 0; k < 3; k++) {
        const float apk = A[p][k], aqk = A[q][k];
        A[p][k] = c * apk - s * aqk;
        A[q][k] = s * apk + c * aqk;
      }
      for (int k = 0; k < 3; k++) {
        const float vkp = V[3 * k + p], vkq = V[3 * k + q];
        V[3 * k + p] = c * vkp - s * vkq;
        V[3 * k + q] = s * vkp + c * vkq;
      }
    }
  }
  const float mass = (float)m.mass[i];
  for (int a = 0; a < 3; a++) {
    const float h2 = 3.0f / (2.0f * mass) * (A[(a + 1) % 3][(a + 1) % 3] + A[(a + 2) % 3][(a + 2) % 3] - A[a][a]);
    lh[a] = fmaxf(MIN_HALF, sqrtf(fmaxf(0.0f, h2)));
  }
}

// link i's box in the world (needs scene_fk and scene_inertia_box of link i)
template <class real, int NJ, int TK> LHW_DEV void scene_link(const Model<real, NJ, TK>& m, int i, Scene<NJ, TK>& s) {
  const float* R = s.xmat[i];
  const float c[3] = {(float)m.com[i][0], (float)m.com[i][1], (float)m.com[i][2]};
  for (int r = 0; r < 3; r++) {
    s.bc[i][r] = s.xpos[i][r] + R[3 * r] * c[0] + R[3 * r + 1] * c[1] + R[3 * r + 2] * c[2];
    for (int k = 0; k < 3; k++) s.br[i][3 * r + k] = R[3 * r] * s.lv[i][k] + R[3 * r + 1] * s.lv[i][3 + k] + R[3 * r + 2] * s.lv[i][6 + k];
    s.bh[i][r] = s.lh[i][r];
  }
}

// foot f's contact geometry: box NL + f (JVRC) or spheres f * NPTS ... (H1)
template <class real, int NJ, int TK> LHW_DEV void scene_foot(const Model<real, NJ, TK>& m, int f, Scene<NJ, TK>& s) {
  constexpr int NL = 1 + 2 * NJ, NPTS = Cfg<NJ, TK>::NPTS;
  const int lk = (f + 1) * NJ;
  const float* R = s.xmat[lk];
  if constexpr (Scene<NJ, TK>::SPH) {
    for (int k = 0; k < NPTS; k++) {
      float* o = s.sc[f * NPTS + k];
      const float v[3] = {(float)m.foot_pts[f][k][0], (float)m.foot_pts[f][k][1], (float)m.foot_pts[f][k][2]};
      for (int r = 0; r < 3; r++) o[r] = s.xpos[lk][r] + R[3 * r] * v[0] + R[3 * r + 1] * v[1] + R[3 * r + 2] * v[2];
      o[3] = (float)m.foot_radius[f];
    }
  } else {
    const int b = NL + f;
    const float v[3] = {(float)m.foot_pos[f][0], (float)m.foot_pos[f][1], (float)m.foot_pos[f][2]};
    for (int r = 0; r < 3; r++) {
      s.bc[b][r] = s.xpos[lk][r] + R[3 * r] * v[0] + R[3 * r + 1] * v[1] + R[3 * r + 2] * v[2];
      for (int k = 0; k < 3; k++) s.br[b][3 * r + k] = R[3 * r + k];
      s.bh[b][r] = (float)m.foot_size[f][r];
    }
  }
}

// slab k from the record's footstep sequence (slab variants only)
template <class real, int NJ, int TK> LHW_DEV void scene_slab(const Model<real, NJ, TK>& m, const real* sr, int k, Scene<NJ, TK>& s) {
  if constexpr (Cfg<NJ, TK>::SLABS) {
    constexpr int SEQ = Dims<real, NJ, TK>::NSTATE_R - Dims<real, NJ, TK>::NPARAM;   // seq[NSLAB][4] opens the parameter tail
    const real* q = sr + SEQ + 4 * k;
    const int b = Scene<NJ, TK>::NL + Scene<NJ, TK>::NFOOT + k;
    float sn, cs;
    sincosf((float)q[3], &sn, &cs);
    s.bc[b][0] = (float)q[0]; s.bc[b][1] = (float)q[1]; s.bc[b][2] = (float)q[2] - (float)m.slab_half[2];
    const float R[9] = {cs, -sn, 0, sn, cs, 0, 0, 0, 1};
    for (int e = 0; e < 9; e++) s.br[b][e] = R[e];
    for (int e = 0; e < 3; e++) s.bh[b][e] = (float)m.slab_half[e];
  }
}

// eye and floor height
template <class real, int NJ, int TK> LHW_DEV void scene_view(const real* sr, const int32_t* si, const Camera& cam, Scene<NJ, TK>& s) {
  const float t[3] = {(float)sr[0] + cam.look[0], (float)sr[1] + cam.look[1], cam.look[2]};
  for (int k = 0; k < 3; k++) s.eye[k] = t[k] - cam.dist * cam.fwd[k];
  s.floor_z = (Cfg<NJ, TK>::STEP && si[1] == ST_FORWARD) ? -2.0f : 0.0f;   // sim_core.h: floor dropped in FORWARD mode
}

// the whole set-up in one thread (host); the kernel runs the same pieces side by side
template <class real, int NJ, int TK>
LHW_DEV void build_scene(const Model<real, NJ, TK>& m, const real* sr, const int32_t* si, const Camera& cam, Scene<NJ, TK>& s) {
  constexpr int NL = 1 + 2 * NJ;
  scene_fk(m, sr, s.xpos, s.xmat);
  for (int i = 0; i < NL; i++) scene_inertia_box(m, i, s.lv[i], s.lh[i]);
  for (int i = 0; i < NL; i++) scene_link(m, i, s);
  for (int f = 0; f < 2; f++) scene_foot(m, f, s);
  for (int k = 0; k < Scene<NJ, TK>::NSL; k++) scene_slab(m, sr, k, s);
  scene_view(sr, si, cam, s);
}

// ---------------------------------------------------------------- ray queries
// box b: entry distance (> 0, camera outside) and the entry face's world normal; returns false on a miss
template <int NJ, int TK> LHW_DEV bool hit_box(const Scene<NJ, TK>& s, int b, const float o[3], const float d[3], float& t, float n[3]) {
  const float* R = s.br[b];
  const float w[3] = {o[0] - s.bc[b][0], o[1] - s.bc[b][1], o[2] - s.bc[b][2]};
  float tn = -INFINITY, tf = INFINITY;
  int ax = 0;
  float sg = 0;
  for (int a = 0; a < 3; a++) {
    const float lo = R[a] * w[0] + R[3 + a] * w[1] + R[6 + a] * w[2];
    const float ld = R[a] * d[0] + R[3 + a] * d[1] + R[6 + a] * d[2];
    const float h = s.bh[b][a];
    if (ld == 0.0f) {
      if (lo < -h || lo > h) return false;
      continue;
    }
    const float t1 = (-h - lo) / ld, t2 = (h - lo) / ld;
    const float ta = fminf(t1, t2), tb = fmaxf(t1, t2);
    if (ta > tn) { tn = ta; ax = a; sg = ld > 0 ? -1.0f : 1.0f; }
    if (tb < tf) tf = tb;
  }
  if (!(tn <= tf) || !(tn > 0)) return false;
  t = tn;
  for (int r = 0; r < 3; r++) n[r] = sg * R[3 * r + ax];
  return true;
}
// any intersection at t >= 0 (shadow rays)
template <int NJ, int TK> LHW_DEV bool meets_box(const Scene<NJ, TK>& s, int b, const float o[3], const float d[3]) {
  const float* R = s.br[b];
  const float w[3] = {o[0] - s.bc[b][0], o[1] - s.bc[b][1], o[2] - s.bc[b][2]};
  float tn = 0.0f, tf = INFINITY;
  for (int a = 0; a < 3; a++) {
    const float lo = R[a] * w[0] + R[3 + a] * w[1] + R[6 + a] * w[2];
    const float ld = R[a] * d[0] + R[3 + a] * d[1] + R[6 + a] * d[2];
    const float h = s.bh[b][a];
    if (ld == 0.0f) {
      if (lo < -h || lo > h) return false;
      continue;
    }
    const float t1 = (-h - lo) / ld, t2 = (h - lo) / ld;
    tn = fmaxf(tn, fminf(t1, t2));
    tf = fminf(tf, fmaxf(t1, t2));
  }
  return tn <= tf;
}
// sphere k: (entry distance, is the camera outside) as for boxes; `any` = intersection at t >= 0
template <int NJ, int TK> LHW_DEV bool hit_sphere(const Scene<NJ, TK>& s, int k, const float o[3], const float d[3], float& t, bool any) {
  const float* c = s.sc[k];
  const float w[3] = {o[0] - c[0], o[1] - c[1], o[2] - c[2]};
  const float b = w[0] * d[0] + w[1] * d[1] + w[2] * d[2];
  const float disc = b * b - (w[0] * w[0] + w[1] * w[1] + w[2] * w[2] - c[3] * c[3]);
  if (!(disc >= 0)) return false;
  const float q = sqrtf(disc);
  t = -b - q;
  return any ? (-b + q >= 0) : (t > 0);
}

template <int NJ, int TK> LHW_DEV bool occluded(const Scene<NJ, TK>& s, const float o[3], const float L[3]) {
  if (o[2] < s.floor_z) return true;   // the light is above every floor
#pragma unroll 1
  for (int b = 0; b < Scene<NJ, TK>::NBOX; b++)
    if (meets_box(s, b, o, L)) return true;
#pragma unroll 1
  for (int k = 0; k < Scene<NJ, TK>::NSPH; k++) {
    float t;
    if (hit_sphere(s, k, o, L, t, true)) return true;
  }
  return false;
}

LHW_DEV uint8_t to_byte(float c) { return (uint8_t)fminf(255.0f, floorf(255.0f * c + 0.5f)); }

// pixel (px, py) of a W x H image -> rgb
template <int NJ, int TK> LHW_DEV void shade_pixel(const Scene<NJ, TK>& s, const Camera& cam, int px, int py, int W, int H, uint8_t rgb[3]) {
  constexpr int NL = Scene<NJ, TK>::NL, NFOOT = Scene<NJ, TK>::NFOOT;
  const float x = 2.0f * ((float)px + 0.5f) / (float)W - 1.0f, y = 1.0f - 2.0f * ((float)py + 0.5f) / (float)H;
  float d[3];
  for (int k = 0; k < 3; k++) d[k] = cam.fwd[k] + x * cam.right[k] + y * cam.up[k];
  const float inv = 1.0f / sqrtf(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  for (int k = 0; k < 3; k++) d[k] *= inv;
  float best = INFINITY, n[3] = {0, 0, 1};
  int mat = -1;
  // robot link boxes, foot boxes (JVRC), foot spheres (H1), slabs, floor: a later primitive must be nearer by HIT_EPS
#pragma unroll 1
  for (int b = 0; b < NL + NFOOT; b++) {
    float t, nb[3];
    if (hit_box(s, b, s.eye, d, t, nb) && t < best - HIT_EPS) { best = t; mat = box_material<NJ, TK>(b); n[0] = nb[0]; n[1] = nb[1]; n[2] = nb[2]; }
  }
#pragma unroll 1
  for (int k = 0; k < Scene<NJ, TK>::NSPH; k++) {
    float t;
    if (hit_sphere(s, k, s.eye, d, t, false) && t < best - HIT_EPS) {
      best = t; mat = MAT_CONTACT;
      for (int r = 0; r < 3; r++) n[r] = (s.eye[r] + t * d[r] - s.sc[k][r]) / s.sc[k][3];
    }
  }
#pragma unroll 1
  for (int b = NL + NFOOT; b < Scene<NJ, TK>::NBOX; b++) {
    float t, nb[3];
    if (hit_box(s, b, s.eye, d, t, nb) && t < best - HIT_EPS) { best = t; mat = MAT_SLAB; n[0] = nb[0]; n[1] = nb[1]; n[2] = nb[2]; }
  }
  if (d[2] < 0 && s.eye[2] > s.floor_z) {
    const float t = (s.floor_z - s.eye[2]) / d[2];
    if (t <= FLOOR_FAR && t < best - HIT_EPS) {
      best = t; n[0] = 0; n[1] = 0; n[2] = 1;
      const float fx = s.eye[0] + t * d[0], fy = s.eye[1] + t * d[1];
      mat = (((int)floorf(fx / CHECKER) + (int)floorf(fy / CHECKER)) & 1) ? MAT_FLOOR_B : MAT_FLOOR_A;
    }
  }
  if (mat < 0) {
    rgb[0] = to_byte(SKY_R); rgb[1] = to_byte(SKY_G); rgb[2] = to_byte(SKY_B);
    return;
  }
  const float L[3] = {LIGHT_X, LIGHT_Y, LIGHT_Z};
  float lam = fmaxf(0.0f, n[0] * L[0] + n[1] * L[1] + n[2] * L[2]);
  if (lam > 0) {
    float o[3];
    for (int r = 0; r < 3; r++) o[r] = s.eye[r] + best * d[r] + SHADOW_BIAS * n[r];
    if (occluded(s, o, L)) lam = 0;
  }
  float alb[3];
  render_albedo(mat, alb);
  const float k = AMBIENT + DIFFUSE * lam;
  for (int r = 0; r < 3; r++) rgb[r] = to_byte(alb[r] * k);
}

}  // namespace render

#if defined(__CUDACC__)
// render_kernels.cu: n_ids images [n_ids, H, W, 3] uint8 of the environments env_ids (rows of state_r / state_i), with the
// model read from `d_model` (a sim's global-memory model twin)
template <class real, int NJ, int TK>
int render_launch(const Model<real, NJ, TK>* d_model, const real* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids,
                  int n_ids, int width, int height, const render::Camera& cam, uint8_t* rgb, cudaStream_t stream);
#endif

}  // namespace lhw
