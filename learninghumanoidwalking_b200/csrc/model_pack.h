// model_pack.h — host-side: fill lhw::Model<real,NJ> from the flat double array the Python host passes over the
// C-ABI (layout produced by learninghumanoidwalking_b200/model/loader.py:pack_model; keep in sync).
#pragma once
#include <math.h>
#include <string.h>

#include "sim_core.h"

namespace lhw {

// the compile-time variant that with_variant hands its callable
template <class R, int J, int T> struct Variant {
  using real = R;
  static constexpr int NJ = J, TK = T;
};

// calls f(Variant<real, NJ, TK>{}) for the variant whose code is `code` (sim_core.h LHW_FOR_EACH_VARIANT), with real = double
// at precision 64 and float otherwise.  Returns 0, or -1 without calling f when no variant has that code.
template <class F> int with_variant(int code, int precision, F&& f) {
#define LHW_VARIANT_CASE(J, T)                                                      \
  if (code == variant_code(J, T)) {                                                 \
    if (precision == 64) f(Variant<double, J, T>{}); else f(Variant<float, J, T>{}); \
    return 0;                                                                       \
  }
  LHW_FOR_EACH_VARIANT(LHW_VARIANT_CASE)
#undef LHW_VARIANT_CASE
  return -1;
}

// returns 0 on success, negative on malformed input
// the first word is the variant's code (sim_core.h variant_code: 6 jvrc_walk, 5 h1, 106 jvrc_step, 206 jvrc_walk_terrain).
// `plan_table` (STEP only): caller-owned buffer of MAXPLAN * PLAN_STRIDE reals that receives the footstep plans; the caller
// points m.plans at its device copy.
template <class real, int NJ, int TK> int fill_model(Model<real, NJ, TK>& m, const double* b, int n, real* plan_table = nullptr) {
  constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ;
  int p = 0;
  auto rd = [&]() -> double { return p < n ? b[p++] : (p++, 0.0); };
  memset(&m, 0, sizeof(m));
  if ((int)rd() != variant_code(NJ, TK)) return -1;
  for (int i = 0; i < NL; i++) {
    for (int k = 0; k < 3; k++) m.link_pos[i][k] = (real)rd();
    for (int k = 0; k < 9; k++) m.link_rot[i][k] = (real)rd();
    for (int k = 0; k < 3; k++) m.axis[i][k] = (real)rd();
    m.mass[i] = (real)rd();
    for (int k = 0; k < 3; k++) m.com[i][k] = (real)rd();
    for (int k = 0; k < 6; k++) m.inertia[i][k] = (real)rd();
  }
  for (int i = 0; i < NL; i++) {
    m.axis_id[i] = -1;
    bool ident = true;
    for (int k = 0; k < 9; k++) ident = ident && (double)m.link_rot[i][k] == ((k % 4 == 0) ? 1.0 : 0.0);
    for (int a = 0; a < 3 && ident && i > 0; a++)
      if ((double)m.axis[i][a] == 1.0 && (double)m.axis[i][(a + 1) % 3] == 0.0 && (double)m.axis[i][(a + 2) % 3] == 0.0) m.axis_id[i] = a;
  }
  m.any_damping = 0;
  for (int d = 0; d < NV; d++) {
    m.armature[d] = (real)rd();
    m.damping[d] = (real)rd();
    m.range_lo[d] = (real)rd();
    m.range_hi[d] = (real)rd();
    m.dof_invw[d] = (real)rd();
    if (m.damping[d] > 0) m.any_damping = 1;
  }
  for (int f = 0; f < 2; f++) {
    for (int k = 0; k < 3; k++) m.foot_pos[f][k] = (real)rd();
    for (int k = 0; k < 3; k++) m.foot_size[f][k] = (real)rd();
    m.foot_invw[f] = (real)rd();
  }
  const double h = rd();
  m.h = (real)h;
  for (int k = 0; k < 3; k++) m.grav[k] = (real)rd();
  double solref[2], solimp[5];
  for (int k = 0; k < 2; k++) solref[k] = rd();
  for (int k = 0; k < 5; k++) solimp[k] = rd();
  const double mu = rd(), impratio = rd(), meaninertia = rd(), tolerance = rd();
  m.max_iter = (int)rd();
  // MuJoCo mj_makeImpedance: refsafe clamps the time constant to 2 h; K, B from (timeconst, dampratio) and dmax
  double tau = solref[0] < 2 * h ? 2 * h : solref[0], zeta = solref[1];
  for (int k = 0; k < 2; k++) solimp[k] = solimp[k] < 0.0001 ? 0.0001 : (solimp[k] > 0.9999 ? 0.9999 : solimp[k]);
  const double dmax = solimp[1];
  m.K = (real)(1.0 / fmax(1e-15, dmax * dmax * tau * tau * zeta * zeta));
  m.B = (real)(2.0 / fmax(1e-15, dmax * tau));
  m.Kc = m.K; m.Bc = m.B;
  for (int k = 0; k < 5; k++) m.solimp[k] = (real)solimp[k];
  m.mu = (real)mu;
  m.mu_reg = (real)(mu * sqrt(1.0 / fmax(1e-15, impratio)));
  const double t = tolerance * meaninertia * (NV > 1 ? NV : 1);
  m.tol2 = (real)(t * t);
  for (int k = 0; k < NU; k++) m.kp[k] = (real)rd();
  for (int k = 0; k < NU; k++) m.kd[k] = (real)rd();
  for (int k = 0; k < NQ; k++) m.nominal[k] = (real)rd();
  m.smoothing = (real)rd();
  m.frame_skip = (int)rd();
  for (int k = 0; k < 3; k++) m.head[k] = (real)rd();
  const double total_mass = rd();
  m.fcap = (real)(total_mass * 9.8 * 0.5);  // tasks/rewards.py:129
  m.goal_height = (real)rd();
  m.period = (int)rd();
  if (m.period < (Cfg<NJ, TK>::STAND ? 0 : 1) || m.period > MAXPERIOD) return -2;
  for (int c = 0; c < 4; c++)
    for (int k = 0; k < m.period; k++) m.clock[c][k] = (real)rd();
  m.ncap = (int)rd();
  if (m.ncap < 0 || m.ncap > MAXCAP) return -5;
  for (int c = 0; c < m.ncap; c++) {
    m.cap_link[c] = (int)rd();
    for (int k = 0; k < 3; k++) m.cap_p0[c][k] = (real)rd();
    for (int k = 0; k < 3; k++) m.cap_p1[c][k] = (real)rd();
    m.cap_r[c] = (real)rd();
  }
  m.npair = (int)rd();
  if (m.npair < 0 || m.npair > MAXPAIR) return -6;
  for (int c = 0; c < m.npair; c++) { m.pair_a[c] = (unsigned char)rd(); m.pair_b[c] = (unsigned char)rd(); }
  // task / robot variant tail
  m.done_lo = (real)rd(); m.done_hi = (real)rd();
  for (int k = 0; k < 5; k++) m.obs_noise[k] = (real)rd();
  m.dynrand_interval = (int)rd(); m.perturb_interval = (int)rd();
  m.perturb_force = (real)rd(); m.perturb_torque = (real)rd(); m.init_noise = (real)rd();
  for (int f = 0; f < 2; f++) {
    const int npts = (int)rd();
    if (npts != (Cfg<NJ, TK>::SPHERES ? Cfg<NJ, TK>::NPTS : 0)) return -7;
    m.foot_radius[f] = (real)rd();
    for (int k = 0; k < npts; k++)
      for (int x = 0; x < 3; x++) m.foot_pts[f][k][x] = (real)rd();
  }
  m.pel_mass = (real)rd();
  for (int k = 0; k < 3; k++) m.pel_com[k] = (real)rd();
  for (int k = 0; k < 6; k++) m.pel_Ic[k] = (real)rd();
  m.rest_mass = (real)rd();
  for (int k = 0; k < 3; k++) m.rest_mc[k] = (real)rd();
  for (int k = 0; k < 6; k++) m.rest_Io[k] = (real)rd();
  for (int k = 0; k < 3; k++) m.torso_com[k] = (real)rd();
  m.pdrand_k = (real)rd();
  if constexpr (Cfg<NJ, TK>::TERRAIN) {
    for (int k = 0; k < 3; k++) m.slab_half[k] = (real)rd();
    m.side_tol = (real)rd(); m.terrain_pitch = (real)rd(); m.terrain_bump = (real)rd(); m.terrain_zlo = (real)rd();
    m.terrain_zhi = (real)rd(); m.terrain_xy = (real)rd(); m.terrain_interval = (int)rd();
    const double tc0 = rd(), zc = rd();
    m.side_faces = (int)rd();
    if (m.terrain_interval < 1) return -10;
    if (tc0 > 0) {   // the foot-ground contact pairs carry their own solref (mj_makeImpedance with refsafe)
      const double tc = tc0 < 2 * h ? 2 * h : tc0;
      m.Kc = (real)(1.0 / fmax(1e-15, dmax * dmax * tc * tc * zc * zc));
      m.Bc = (real)(2.0 / fmax(1e-15, dmax * tc));
    }
  }
  if constexpr (Cfg<NJ, TK>::SLABS) {
    for (int f = 0; f < 2; f++)
      m.foot_rad[f] = (real)(sqrt((double)m.foot_size[f][0] * m.foot_size[f][0] + (double)m.foot_size[f][1] * m.foot_size[f][1] +
                                  (double)m.foot_size[f][2] * m.foot_size[f][2]) * 1.0001 + 1e-6);
  }
  if constexpr (Cfg<NJ, TK>::STEP) {
    for (int f = 0; f < 2; f++)
      for (int k = 0; k < 3; k++) m.foot_site[f][k] = (real)rd();
    for (int k = 0; k < 3; k++) m.slab_half[k] = (real)rd();
    m.target_radius = (real)rd(); m.side_tol = (real)rd(); m.delay_frames = (int)rd(); m.step_height = (real)rd();
    m.slab_contacts_are_floor = (int)rd();
    m.side_faces = (int)rd();
    m.nplan = (int)rd();
    if (m.nplan < 1 || m.nplan > MAXPLAN || !plan_table) return -8;
    for (int i = 0; i < m.nplan; i++) {
      const int len = (int)rd();
      if (len < 1 || len > NSLAB) return -9;
      real* row = plan_table + (size_t)i * PLAN_STRIDE;
      row[0] = (real)len;
      for (int k = 0; k < 3 * len; k++) row[1 + k] = (real)rd();
    }
    m.plans = plan_table;
  }
  // assumption switches (model/*.json "assumptions"): bit 0 = explicit Euler instead of the implicit joint-damping solve
  const int aflags = (int)rd();
  m.explicit_euler = aflags & 1;
  if (p != n) return -3;
  return 0;
}

}  // namespace lhw
