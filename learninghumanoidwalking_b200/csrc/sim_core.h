// sim_core.h — one environment per warp: articulated-body forward dynamics, soft-contact Newton solve,
// PD actuation, reward / observation / termination / auto-reset, all inside one control step.
//
// Replaces (reference file:line, /root/reference):
//   envs/common/base_humanoid_env.py:199-227 (step), :247-276 (reset_model)
//   robots/robot_base.py:41-98 (_do_simulation: frame_skip x {PD torque, mj_step})
//   envs/common/robot_interface.py:493-546 (step_pd / set_motor_torque / step)
//   mujoco.mj_step (external, SURVEY.md Appendix A)
//   tasks/walking_task.py:85-205, tasks/rewards.py:9-174, tasks/observations.py:12-72,
//   envs/jvrc/jvrc_base.py:133-145, envs/jvrc/jvrc_walk.py:65-67
//   H1 standing variant (Cfg<5,0>): envs/h1/h1_base.py:91-117, tasks/standing_task.py:49-131,
//   envs/common/domain_randomization.py:10-56, base_humanoid_env.py:228-233, :247-338
//   JVRC stepping variant (Cfg<6,1>): envs/jvrc/jvrc_step.py:41-76, tasks/stepping_task.py:52-334 (footstep sequences,
//   stepping-stone slabs, target tracking, goal-step observation), utils/footstep_plans.txt
//   terrain extension (Cfg<6,2>): WalkingTask on re-posed terraces, ranges of tasks/walking_task.py:172-179 (not a reference env)
//   H1 walking variant (Cfg<5,3>): the robot of Cfg<5,0> with the WalkingTask of Cfg<6,0> (envs/h1/h1_walk.py; DESIGN.md §4.6)
//
// Execution model.  Every phase is a `LHW_LANES(l) { ... }` block: on the GPU each of the 32 lanes of the
// warp runs the body once with its own lane id and `LHW_SYNC()` is __syncwarp(); all inter-lane traffic goes
// through the per-warp shared-memory `Work` struct (or warp_sum shuffles).  With LHW_CPU_EMU defined the same
// source runs the 32 lanes sequentially on the host — that build exists ONLY for tests/ (it lets the CPU test
// tier check this exact arithmetic against oracle/); the product never uses it.
//
// Spatial algebra: all motion/force vectors are expressed in a world-aligned inertial frame whose origin `o`
// coincides with the root link origin at the current instant, so parent->child propagation needs no
// transforms (V_child = V_parent + S qd, composite inertias are plain sums).
// Tree: free root (dofs 0-2 world translation, 3-5 body-frame rotation) + two serial chains of NJ hinges.
// This gives the mass matrix an arrow structure [root | chain0 | chain1] with a zero chain0-chain1 block,
// which the factorisation exploits (two NJ x NJ Choleskys side by side + a 6x6 Schur complement).
#pragma once
#include <math.h>
#include <stdint.h>

// Model tables that are indexed by the LANE (per-link / per-dof constants of the per-substep phases) are read from a
// global-memory twin of the model (LDG through L1) instead of the constant bank, which serialises a warp's distinct addresses
// (few instructions, but a disproportionate share of the stall samples sat behind those LDCs).
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
#define LHW_GLD(m, field) __ldg(&(m).gm->field)
#else
#define LHW_GLD(m, field) ((m).field)
#endif

#if defined(__CUDACC__) && !defined(LHW_CPU_EMU)
#define LHW_DEV __device__ __forceinline__
#define LHW_DEVNI inline __device__ __noinline__   // inline: the header is included by more than one translation unit
#else
#define LHW_DEV inline
#define LHW_DEVNI inline
#endif

#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
#define LHW_LANES(l) for (int l = (int)(threadIdx.x & 31), _o = 1; _o; _o = 0)
#define LHW_LANES_ORDERED(l) LHW_LANES(l)
#define LHW_SYNC() __syncwarp()
#elif defined(LHW_EMU_REVERSE)
// host emulation with the lanes of a phase run in descending order: a phase whose lanes only touch their own data (or data
// finished before the preceding LHW_SYNC) gives bit-identical results in either order, so forward vs reverse is a race check
#define LHW_LANES(l) for (int l = 31; l >= 0; --l)
#define LHW_LANES_ORDERED(l) for (int l = 0; l < 32; ++l)   // phases whose emulation of a warp-wide prefix needs ascending lanes
#define LHW_SYNC() ((void)0)
#else
#define LHW_LANES(l) for (int l = 0; l < 32; ++l)
#define LHW_LANES_ORDERED(l) LHW_LANES(l)
#define LHW_SYNC() ((void)0)
#endif

// optional block-level rendez-vous once per substep (multi-warp blocks only): keeps the warps of a block in the same
// region of the code so they share instruction-cache fills
#ifndef LHW_BLOCK_SYNC
#define LHW_BLOCK_SYNC(on) ((void)0)
#endif
// Newton-step census (tools/newton_census.py): only the census build of the CPU emulation (tools/newton_census.cpp) defines
// this hook; the product compiles none of it.
// Events: 0 = solve starts, 1 = line-search evaluation number n (0 = at alpha 0), 2 = solve done (w.iters_total has the steps)
#ifndef LHW_NEWTON_HOOK
#define LHW_NEWTON_HOOK(event, w, n) ((void)0)
#endif
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
#define LHW_ASSUME_SHARED(p) __builtin_assume(__isShared(p))
#else
#define LHW_ASSUME_SHARED(p) ((void)0)
#endif

// exclusive prefix count over the lanes of a warp of (a + b), a and b in {0, 1}; `run` is a warp-uniform running total.
// In the CPU emulation the lanes run in order, so a plain running counter declared outside LHW_LANES does the same.
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
#define LHW_PREFIX2(a, b, run, pos)                                                                              \
  do {                                                                                                           \
    const unsigned _ma = __ballot_sync(0xffffffffu, (a)), _mb = __ballot_sync(0xffffffffu, (b));                 \
    const unsigned _lt = (1u << (threadIdx.x & 31)) - 1u;                                                        \
    (pos) = (run) + __popc(_ma & _lt) + __popc(_mb & _lt);                                                       \
    (run) += __popc(_ma) + __popc(_mb);                                                                          \
  } while (0)
#else
#define LHW_PREFIX2(a, b, run, pos) do { (pos) = (run); (run) += ((a) ? 1 : 0) + ((b) ? 1 : 0); } while (0)
#endif

// lane-strided loop over N items with a COMPILE-TIME trip count (the item guard vanishes when N is a multiple of 32)
#define LHW_STRIDED(it, l, N) \
  _Pragma("unroll") for (int _k = 0, it = (l); _k < ((N) + 31) / 32; _k++, it += 32) if ((N) % 32 == 0 || it < (N))

namespace lhw {

constexpr int NREW = 10;
constexpr int MAXPERIOD = 96;
constexpr int NSTATE_I = 8;    // int32 words per env in the integer state record
constexpr int MAXCAP = 16;     // self-collision capsules
constexpr int MAXPAIR = 64;

// robot / task variant, keyed by the chain length NJ.  Everything variant-specific below is `if constexpr` on these
// flags, so each instantiation only carries its own code.
template <int NJ, int TK> struct Cfg;
template <> struct Cfg<6, 0> {  // JVRC-1, WalkingTask: box feet (mjc_PlaneBox: at most 4 of the 8 corners per foot)
  static constexpr int CPF = 4, NPTS = 8, RFOOT = 0;
  static constexpr bool SPHERES = false, FLOSS = false, PERENV = false, STAND = false, H1OBS = false, STEP = false, SLABS = false, TERRAIN = false;
};
template <> struct Cfg<5, 0> {  // Unitree H1, StandingTask: 3 capsules per foot = 6 end spheres; dof friction loss;
  static constexpr int CPF = 6, NPTS = 6, RFOOT = 1;  // per-env randomised mass / com / damping / frictionloss; xfrc perturbations
  static constexpr bool SPHERES = true, FLOSS = true, PERENV = true, STAND = true, H1OBS = true, STEP = false, SLABS = false, TERRAIN = false;
};
template <> struct Cfg<6, 1> {  // JVRC-1, SteppingTask: box feet on the floor + 20 per-env stepping-stone slabs;
  static constexpr int CPF = 8, NPTS = 8, RFOOT = 0;  // per foot 4 corner slots (with multiplicity) + 4 sole-edge x slab-boundary slots
  static constexpr bool SPHERES = false, FLOSS = false, PERENV = false, STAND = false, H1OBS = false, STEP = true, SLABS = true, TERRAIN = false;
};
template <> struct Cfg<6, 2> {  // JVRC-1, WalkingTask on uneven / compliant terrain (extension, BASELINE configs[4]): 20 terraces
  static constexpr int CPF = 8, NPTS = 8, RFOOT = 0;  // = the slabs of the stepping stones, re-posed like the reference's manip_hfield hook
  static constexpr bool SPHERES = false, FLOSS = false, PERENV = false, STAND = false, H1OBS = false, STEP = false, SLABS = true, TERRAIN = true;
};
template <> struct Cfg<5, 3> {  // Unitree H1 (the robot of Cfg<5, 0>), WalkingTask (the task of Cfg<6, 0>)
  static constexpr int CPF = 6, NPTS = 6, RFOOT = 1;
  static constexpr bool SPHERES = true, FLOSS = true, PERENV = true, STAND = false, H1OBS = true, STEP = false, SLABS = false, TERRAIN = false;
};
// H1OBS: the observation starts with h1_base's robot state (+ motor torques) and carries uniform observation noise.
// RFOOT: the chain that ends in the right foot (JVRC-1 lists its right leg first, H1 its left leg)
// every (NJ, TK) above, once: the host code instantiates, dispatches and keeps its books from this list
#define LHW_FOR_EACH_VARIANT(X) X(6, 0) X(5, 0) X(6, 1) X(6, 2) X(5, 3)
// a variant's code, the first word of its flat model (model/loader.py): 6, 5, 106, 206, 305
constexpr int variant_code(int nj, int tk) { return nj + 100 * tk; }
constexpr int NSLAB = 20;          // stepping stones per env (envs/jvrc/gen_xml.py:147-153)
constexpr int NCORNER = 4;         // corner slots per foot (mjc_PlaneBox keeps at most 4)
constexpr int MAXPLAN = 128, PLAN_STRIDE = 1 + 3 * NSLAB;   // footstep plan table: [len, (x y theta) * len]
enum { ST_CURVED = 0, ST_STANDING = 1, ST_BACKWARD = 2, ST_LATERAL = 3, ST_FORWARD = 4 };  // tasks/stepping_task.py:268-271

enum { STANDING = 0, INPLACE = 1, FORWARD = 2 };
// WalkingTask variants: a mode held by lhw_sim_set_command (DESIGN.md §7.6) carries this bit in the int record's mode word.
// load_state splits the word into Work::mode and Work::hold and store_state joins them; every other reader masks it off.
constexpr int32_t MODE_HELD = 1 << 30;

// ---------------------------------------------------------------- math wrappers
// the transcendental ones are deliberately NOT inlined on the device: each inlined copy of exp/tan/atan2/pow/sincos
// is 100-400 SASS instructions and the kernel is instruction-cache bound, one shared copy each
LHW_DEV float m_sqrt(float x) { return sqrtf(x); }
LHW_DEV double m_sqrt(double x) { return sqrt(x); }
LHW_DEV float m_abs(float x) { return fabsf(x); }
LHW_DEV double m_abs(double x) { return fabs(x); }
LHW_DEVNI float m_exp(float x) { return expf(x); }
LHW_DEVNI double m_exp(double x) { return exp(x); }
LHW_DEVNI float m_tan(float x) { return tanf(x); }
LHW_DEVNI double m_tan(double x) { return tan(x); }
LHW_DEVNI float m_atan2(float y, float x) { return atan2f(y, x); }
LHW_DEVNI double m_atan2(double y, double x) { return atan2(y, x); }
LHW_DEVNI float m_pow(float x, float y) { return powf(x, y); }
LHW_DEVNI double m_pow(double x, double y) { return pow(x, y); }
LHW_DEVNI void m_sincos(float x, float* s, float* c) { sincosf(x, s, c); }
LHW_DEVNI void m_sincos(double x, double* s, double* c) { sincos(x, s, c); }
template <class T> LHW_DEV T m_min(T a, T b) { return a < b ? a : b; }
template <class T> LHW_DEV T m_max(T a, T b) { return a > b ? a : b; }

template <class real, class F> LHW_DEV real warp_sum(F f) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  real v = f((int)(threadIdx.x & 31));
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
#else
  real s = 0;
  for (int l = 0; l < 32; ++l) s += f(l);
  return s;
#endif
}

// fp64 tensor-core product on one 8x8 tile, a warp collective (called outside LHW_LANES, like warp_sum):
// D = C + sum_k A_k B_k over KS k-steps of mma.sync m8n8k4 .f64 (A_k 8x4 row-major, B_k 4x8 column-major).
// Fragment layout (PTX ISA, m8n8k4 .f64): lane l holds A_k[l >> 2][l & 3] = a(l, k), B_k[l & 3][l >> 2] = b(l, k) and
// C[l >> 2][2 (l & 3) + i] = c(l, i), i = 0, 1; store(l, i, v) receives D at that place.  a and b return 0 for padding.
// The CPU emulation builds the tiles from the same lambdas and sums C + products in k order; the DMMA's internal rounding
// order is not specified, so device and host agree to rounding, not bit for bit.
template <int KS, class FA, class FB, class FC, class FS> LHW_DEV void warp_mma_f64(FA a, FB b, FC c, FS store) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  const int l = (int)(threadIdx.x & 31);
  double d0 = c(l, 0), d1 = c(l, 1);
#pragma unroll
  for (int k = 0; k < KS; k++) {
    const double ak = a(l, k), bk = b(l, k);
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                 : "+d"(d0), "+d"(d1) : "d"(ak), "d"(bk));
  }
  store(l, 0, d0);
  store(l, 1, d1);
#else
  double A[KS][8][4], B[KS][4][8], D[8][8];
  for (int l = 0; l < 32; ++l) {
    for (int k = 0; k < KS; k++) {
      A[k][l >> 2][l & 3] = a(l, k);
      B[k][l & 3][l >> 2] = b(l, k);
    }
    for (int i = 0; i < 2; i++) D[l >> 2][2 * (l & 3) + i] = c(l, i);
  }
  for (int r = 0; r < 8; r++)
    for (int col = 0; col < 8; col++)
      for (int k = 0; k < KS; k++)
        for (int kk = 0; kk < 4; kk++) D[r][col] += A[k][r][kk] * B[k][kk][col];
  for (int l = 0; l < 32; ++l)
    for (int i = 0; i < 2; i++) store(l, i, D[l >> 2][2 * (l & 3) + i]);
#endif
}

// warp ballot of a per-lane predicate; bit helpers (the CPU emulation evaluates the predicate lane by lane)
template <class F> LHW_DEV unsigned warp_ballot(F f) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return __ballot_sync(0xffffffffu, f((int)(threadIdx.x & 31)));
#else
  unsigned m = 0;
  for (int l = 0; l < 32; ++l) m |= f(l) ? (1u << l) : 0u;
  return m;
#endif
}
LHW_DEV int bit_count(unsigned m) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return __popc(m);
#else
  return __builtin_popcount(m);
#endif
}
LHW_DEV int lowest_bit(unsigned m) {   // index of the lowest set bit (m != 0)
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return __ffs(m) - 1;
#else
  return __builtin_ctz(m);
#endif
}
LHW_DEV int nth_bit(unsigned m, int n) {   // index of the n-th (0-based) set bit, 32 if there is none
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  const unsigned r = __fns(m, 0, n + 1);
  return r == 0xffffffffu ? 32 : (int)r;
#else
  for (int i = 0; i < 32; i++)
    if (m & (1u << i)) { if (n == 0) return i; n--; }
  return 32;
#endif
}

// ---------------------------------------------------------------- rng: philox4x32-10, counter (event, stream, env)
LHW_DEV void philox(uint32_t seed, uint32_t env_id, uint32_t ctr, uint32_t stream, uint32_t out[4]) {
  uint32_t c0 = ctr, c1 = stream, c2 = env_id, c3 = 0x4c485742u;
  uint32_t k0 = seed, k1 = 0x9E3779B9u ^ (seed * 0x85EBCA6Bu + 1u);
#pragma unroll
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n1 = (uint32_t)p1, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1, n3 = (uint32_t)p0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
template <class real> LHW_DEV real u01(uint32_t u) { return (real)(u >> 8) * (real)(1.0 / 16777216.0); }
LHW_DEV int randint(uint32_t u, int n) { return (int)(((uint64_t)u * (uint64_t)n) >> 32); }

// ---------------------------------------------------------------- model constants (one per robot/task)
template <class real, int NJ, int TK> struct Model {
  static constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ, NA = 6 + NJ;
  static constexpr int NT = 21 + NJ * (NJ + 1) + 12 * NJ;  // structurally non-zero lower-triangle entries of H
  real link_pos[NL][3], link_rot[NL][9], axis[NL][3];
  real mass[NL], com[NL][3], inertia[NL][6];  // xx yy zz xy xz yz about com, link frame
  real armature[NV], damping[NV], range_lo[NV], range_hi[NV], dof_invw[NV];
  real foot_pos[2][3], foot_size[2][3], foot_invw[2];
  real foot_pts[2][Cfg<NJ, TK>::NPTS][3], foot_radius[2];  // SPHERES: sphere centres in the foot link frame
  real h, grav[3];
  real K, B, Kc, Bc, solimp[5], mu, mu_reg;  // mu_reg = mu * sqrt(1/impratio); Kc, Bc: foot-ground contacts (= K, B by default)
  real tol2;                         // (tolerance * meaninertia * nv)^2 : threshold on |grad|^2
  real kp[NU], kd[NU], nominal[NQ], smoothing;
  real head[3], fcap, goal_height;
  real clock[4][MAXPERIOD];  // r_frc r_vel l_frc l_vel
  int max_iter, frame_skip, period, any_damping;
  int explicit_euler;   // model switch (SURVEY App. A.1): 1 = integrate qacc as solved, no (M + h B) solve (default 0: MuJoCo's implicit joint damping)
  int ncap, npair, cap_link[MAXCAP];
  real cap_p0[MAXCAP][3], cap_p1[MAXCAP][3], cap_r[MAXCAP];
  unsigned char pair_a[MAXPAIR], pair_b[MAXPAIR];
  // task / robot variant constants (zero / unused where the variant has no such feature)
  real done_lo, done_hi, obs_noise[5], perturb_force, perturb_torque, init_noise;  // init_noise in radians
  int dynrand_interval, perturb_interval;
  real pdrand_k;   // RobotBase(pdrand_k): PD gains ~ U((1-k) g, (1+k) g) once per control step; 0 = off (reference default)
  real pel_mass, pel_com[3], pel_Ic[6], rest_mass, rest_mc[3], rest_Io[6], torso_com[3];  // root link = pelvis body + welded rest
  int axis_id[NL];  // 0/1/2: hinge axis is +e_x/+e_y/+e_z of the link frame AND link_rot is the identity (fast FK path); -1: general
  // SteppingTask (Cfg::STEP): force-sensor sites, slab half sizes, target logic, curriculum step height, footstep plans
  real foot_site[2][3], slab_half[3], target_radius, side_tol, step_height, foot_rad[2];   // foot_rad: box circumradius (+1e-6)
  // terrain extension (Cfg::TERRAIN): terrace pitch, bump range, pose ranges of the manip_hfield hook, re-pose interval
  real terrain_pitch, terrain_bump, terrain_zlo, terrain_zhi, terrain_xy;
  int terrain_interval;
  int delay_frames, nplan;
  int slab_contacts_are_floor;   // 0: reference behaviour (SURVEY C-2), foot-stone contacts invisible to GRF / contact z
  int side_faces;                // 1: slab side faces (stair risers) stop foot-box corners that are inside a slab; 0: they pass through
  const real* plans;   // [nplan][PLAN_STRIDE] in global memory (host memory in the CPU emulation)
  const Model* gm;     // the same record in global memory (device builds; unused by the CPU emulation)
};

// Out-of-line device routines must not read the model through a generic reference (that turns every constant-bank
// LDC into a generic load): the translation unit that owns the __constant__ object specialises this hook; the default
// (host emulation) just returns what it was given.
template <class real, int NJ, int TK> struct ModelHome {
  static LHW_DEV const Model<real, NJ, TK>& get(const Model<real, NJ, TK>& passed) { return passed; }
};
template <class real, int NJ, int TK> LHW_DEV const Model<real, NJ, TK>& model_ref(const Model<real, NJ, TK>& passed) {
  return ModelHome<real, NJ, TK>::get(passed);
}

template <class real, int NJ, int TK> struct Dims {
  static constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ, NA = 6 + NJ;
  // robot state (roll, pitch, root angular velocity, joint positions / velocities [, motor torques]), then the task's words
  static constexpr int NROBOT = Cfg<NJ, TK>::H1OBS ? 5 + 3 * NU : 5 + 2 * NU;
  static constexpr int NOBS = NROBOT + (Cfg<NJ, TK>::STAND ? 0 : Cfg<NJ, TK>::STEP ? 10 : 8);
  // real-valued state record per env (HBM, env-major so one warp streams its env's record contiguously)
  static constexpr int NPARAM = Cfg<NJ, TK>::PERENV ? NL + 3 * NL + 6 + 2 * NU + 3 + 12 : (Cfg<NJ, TK>::SLABS ? 4 * NSLAB + 5 : 0);
  static constexpr int NSTATE_R = NQ + NV + NV + 5 * NU + 3 + 1 + NPARAM;
};

// ---------------------------------------------------------------- arrow-packed symmetric matrix
// ordering [root | chain0 | chain1]; chain0-chain1 coupling is structurally zero and not stored
// 16-byte aligned (as is Work): lets the compiler fuse neighbouring shared-memory accesses into LDS.64 / LDS.128
template <class real, int NJ, int TK> struct alignas(16) Arrow {
  real r[6][6];      // root block (M: full symmetric; factor: lower triangle)
  real x[2][6][NJ];  // coupling  x[chain][root dof][chain dof]   (factor: X = B L^-T)
  real c[2][NJ][NJ]; // chain blocks (M: full symmetric; factor: lower triangle)
};

// ---------------------------------------------------------------- per-warp working set (shared memory)
// persistent state (mirrors the HBM record, same order); variants with per-env model parameters append them
template <class real, int NJ, int TK> struct Persist {
  static constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ;
  real qpos[NQ], qvel[NV], qacc_warm[NV], act_len[NU], act_vel[NU], prev_pred[NU], prev_action[NU], prev_torque[NU];
  real mode_ref[3], ep_rew;
};
template <class real, int NJ, int TK> struct PersistRand : Persist<real, NJ, TK> {
  static constexpr int NL = 1 + 2 * NJ, NU = 2 * NJ;
  real p_mass[NL], p_com[NL][3], p_inertia0[6];  // link masses / coms; root inertia about its com (xx yy zz xy xz yz)
  real p_damping[NU], p_floss[NU];
  real p_pelcom[3];                              // com of the pelvis BODY (point of application of xfrc[0])
  real xfrc[2][6];                               // world [force, torque] on the pelvis / torso bodies
};
// SteppingTask: the footstep sequence (= the slab poses: slab k's top face passes through seq[k]) and the task counters
template <class real, int NJ, int TK> struct PersistStep : Persist<real, NJ, TK> {
  real seq[NSLAB][4];   // x y z theta, world
  real tk[5];           // seq_len, t1, t2, target_reached, target_reached_frames (small integers, held exactly)
};
template <bool C, class A, class B> struct Select { typedef A type; };
template <class A, class B> struct Select<false, A, B> { typedef B type; };

template <class real, int NJ, int TK>
struct alignas(16) Work : Select<Cfg<NJ, TK>::PERENV, PersistRand<real, NJ, TK>,
                                 typename Select<Cfg<NJ, TK>::SLABS, PersistStep<real, NJ, TK>, Persist<real, NJ, TK>>::type>::type {
  static constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ, NA = 6 + NJ;
  static constexpr int CPF = Cfg<NJ, TK>::CPF, NCON = 2 * CPF, NEDGE = 4 * NCON, NPTS = Cfg<NJ, TK>::NPTS;
  static constexpr int NOBS = Dims<real, NJ, TK>::NOBS;
  static constexpr int NFL = Cfg<NJ, TK>::FLOSS ? NU : 1;
  static constexpr int NSL = Cfg<NJ, TK>::SLABS ? NSLAB : 1, NST = Cfg<NJ, TK>::SLABS ? 1 : 0;
  int phase, mode, traj_len, ep_len, have_prev, status;
  uint32_t rng_ctr, env_id;
  // ---- control-step scratch
  real target[NU], ctrl[NU], act_force[NU], kp_step[NU], kd_step[NU];
  // ---- kinematics / dynamics
  real sc[NU][2];
  real o[3], xr[NL][3], xmat[NL][9];
  real S[NV][6];
  real V[NL][6];
  Arrow<real, NJ, TK> M, H;
  real hdinv[NV];
  real qfs[NV], qacc[NV], Ma[NV], grad[NV], sdir[NV], Ms[NV], vec[NV];
  // ---- contacts (slot = foot*4 + k), expressed through the foot's spatial motion: J_contact = P(p) S_foot
  int ncon[2];
  // stepping stones: cos/sin of the slab yaws, per-corner multiplicity, crossing-slot distances
  real slab_cs[NSL][2], cmul[NST ? 16 : 1], xcd[NST ? NCON : 1];
  int ncorner[2], nside[2];
  // riser contacts (slab side faces): horizontal outward normal per slot, (0, 0) = the slot's normal is +z
  real cn[NST ? NCON : 1][2];
  real site[2][3], rquat[4], goal[8];   // lagged site_xpos / root xquat ; _goal_steps_{x,y,z,theta}
  real cpos[NCON][Cfg<NJ, TK>::SLABS ? 5 : 3], cD[NCON], cKid[NCON];   // SLABS: (px, py, pz, 1, 0), see pmap_sel
  real ejar[NEDGE];   // edge residuals J a - aref (P8 leaves aref here, P9 turns it into the residual in place)
  int lside[NU];
  real lD[NU], ljar[NU];
  real fD[NFL], flim[NFL], fjar[NFL];  // dof friction-loss rows: 1/R, floss * R (half width of the quadratic zone)
  // two scratch groups with disjoint lifetimes share storage: rigid-body quantities live from P2 to P8 (the last
  // reader is qfrc_smooth), the Newton quantities from P9 to P11
  union {
    struct {
      real inert[NL][10], comp[NL][10];
      real A[NL][6], F[NL][6];
      real ccd[2 * NPTS];   // signed distance of each candidate point (box corner / sphere), > 0: not a candidate
      int cslot[NCON];
      real cwp[NST ? 16 : 1][3];   // SLABS: foot-box corners relative to o
      real cside[NST ? 16 : 1], csn[NST ? 16 : 1][2];   // SLABS: per corner, inset behind the nearest side face of the first slab that
                                                        // holds it unsupported (< 0: none) and that face's outward normal
    };
    struct {
      real T[2][NA][6], Af[2][6][6], Ff[2][6], ya[2][6], ys[2][6];
      // contact-frame point map: rows = unit wrenches of (n, t1, t2) applied at the contact.  The slab variants (16 slots)
      // rebuild the entries from cpos instead (pmap3): dropping the table is what lets 14 fp64 environments share an SM
      real Pm[Cfg<NJ, TK>::SLABS ? 1 : NCON][3][6];
      real cF[NCON][3], cW[NCON][Cfg<NJ, TK>::SLABS ? 6 : 5];   // SLABS: + the (t1, t2) entry, non-zero for riser contacts only
      real ejv[NEDGE], ljv[NU], fjv[NFL];
    };
    real capE[MAXCAP][6];  // self-collision capsule end points; lives where T was (T is dead after the Hessian build)
    real obs[NOBS];        // the observation is packed at env level, when both scratch groups are dead
  };
  // ---- what mj_step leaves behind (pre-integration state of the last substep)
  real root_vlin[3], foot_vel[2][3], grf[2], cz_min, qacc_lag[3];
  real rew[NREW];
  int iters_total, selfcol, nfloor;   // nfloor: contacts the task's floor-contact queries see (last substep)
  int hold;   // WalkingTask variants: the mode and reference are held (MODE_HELD); it sits in the tail padding of every variant
};

// ---------------------------------------------------------------- small vector helpers
template <class real> LHW_DEV void cross(const real* a, const real* b, real* c) {
  real x = a[1] * b[2] - a[2] * b[1], y = a[2] * b[0] - a[0] * b[2], z = a[0] * b[1] - a[1] * b[0];
  c[0] = x; c[1] = y; c[2] = z;
}
template <class real> LHW_DEV real dot3(const real* a, const real* b) { return a[0] * b[0] + a[1] * b[1] + a[2] * b[2]; }
template <class real> LHW_DEV real dot6(const real* a, const real* b) {
  return a[0] * b[0] + a[1] * b[1] + a[2] * b[2] + a[3] * b[3] + a[4] * b[4] + a[5] * b[5];
}
template <class real> LHW_DEV void mv3(const real* R, const real* v, real* out) {
  real x = R[0] * v[0] + R[1] * v[1] + R[2] * v[2];
  real y = R[3] * v[0] + R[4] * v[1] + R[5] * v[2];
  real z = R[6] * v[0] + R[7] * v[1] + R[8] * v[2];
  out[0] = x; out[1] = y; out[2] = z;
}
// spatial inertia (m, h=m*c, Io) times motion vector [w; v] -> force [n; f]
template <class real> LHW_DEV void inert_mul(const real* I, const real* mvv, real* out) {
  const real m = I[0];
  const real* h = I + 1;
  const real* w = mvv;
  const real* v = mvv + 3;
  real hv[3], hw[3];
  cross(h, v, hv);
  cross(h, w, hw);
  out[0] = I[4] * w[0] + I[7] * w[1] + I[8] * w[2] + hv[0];
  out[1] = I[7] * w[0] + I[5] * w[1] + I[9] * w[2] + hv[1];
  out[2] = I[8] * w[0] + I[9] * w[1] + I[6] * w[2] + hv[2];
  out[3] = m * v[0] - hw[0];
  out[4] = m * v[1] - hw[1];
  out[5] = m * v[2] - hw[2];
}
// row of the it-th entry (row-major) of a lower triangle with at most 6 rows: 0,1,1,2,2,2,... packed 3 bits per entry
LHW_DEV int tri_row(int it) { return (int)((0x5B6DB2491B6D2448ull >> (3 * it)) & 7ull); }
template <int NJ> LHW_DEV int dof_link(int d) { return d < 6 ? 0 : d - 5; }
template <int NJ> LHW_DEV int loc2dof(int foot, int j) { return j < 6 ? j : 6 + foot * NJ + (j - 6); }
// fast reciprocal square root (pivot scaling); the product keeps 1/sqrt explicitly, never sqrt then divide
LHW_DEV float m_rsqrt(float x) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return rsqrtf(x);
#else
  return 1.0f / sqrtf(x);
#endif
}
LHW_DEV double m_rsqrt(double x) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  // single-precision seed (MUFU.RSQ) + one Newton step in double: relative error ~1.5 * (6e-8)^2 = 5e-15, a third of
  // the dependent-instruction chain of the library rsqrt(double); pivots and quaternion norms are far inside float range
  float y0;   // the bare MUFU.RSQ: rsqrtf() wraps it in a denormal-input rescale that these operands never need
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y0) : "f"((float)x));
  const double y = (double)y0;
  return y * (1.5 - 0.5 * x * y * y);
#else
  return 1.0 / sqrt(x);
#endif
}
// contact-frame velocity of the point p of a body moving with spatial motion y
template <class real> LHW_DEV void contact_u(const real* p, const real* y, real* u) {
  u[0] = y[5] + y[0] * p[1] - y[1] * p[0];
  u[1] = y[4] + y[2] * p[0] - y[0] * p[2];
  u[2] = -(y[3] + y[1] * p[2] - y[2] * p[1]);
}
// contact-frame velocity of a RISER contact (slab side face, horizontal outward normal (nx, ny)): frame n = (nx, ny, 0),
// t1 = +z, t2 = n x t1 = (ny, -nx, 0).  `u` comes in as contact_u gives it — the components of the world velocity along the
// canonical frame C0 = (+z, +y, -x) of every floor / top-face contact — and leaves as (n.v, t1.v, t2.v) = Q' u with
// Q = [[0, 1, 0], [ny, 0, -nx], [-nx, 0, -ny]] (the riser frame's vectors written in C0).  (0, 0) = a C0 contact: unchanged.
template <class real> LHW_DEV void riser_u(const real* cn, real* u) {
  const real nx = cn[0], ny = cn[1];
  if (nx != 0 || ny != 0) {
    const real a = u[0], b = u[1], c = u[2];
    u[0] = ny * b - nx * c;
    u[1] = a;
    u[2] = -nx * b - ny * c;
  }
}
// column a of the contact point map P(p) (see P9) without the table: with the contact record cp = (px, py, pz, 1, 0) the
// entries are P[r][a] = sgn[r] * cp[idx[r]]; idx / sgn depend on the lane's column only and are hoisted out of the contact loops
// sgn[r] is a sign-bit mask (0 or 0x80000000) applied with one integer XOR (sflip), not a multiply on the fp64 pipe
LHW_DEV void pmap_sel(int a, int idx[3], unsigned sgn[3]) {
  idx[0] = a == 0 ? 1 : a == 1 ? 0 : a == 5 ? 3 : 4;  sgn[0] = a == 1 ? 0x80000000u : 0u;
  idx[1] = a == 0 ? 2 : a == 2 ? 0 : a == 4 ? 3 : 4;  sgn[1] = a == 0 ? 0x80000000u : 0u;
  idx[2] = a == 1 ? 2 : a == 2 ? 1 : a == 3 ? 3 : 4;  sgn[2] = (a == 1 || a == 3) ? 0x80000000u : 0u;
}
LHW_DEV double sflip(double x, unsigned m) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return __hiloint2double(__double2hiint(x) ^ (int)m, __double2loint(x));
#else
  return m ? -x : x;
#endif
}
LHW_DEV float sflip(float x, unsigned m) {
#if defined(__CUDA_ARCH__) && !defined(LHW_CPU_EMU)
  return __int_as_float(__float_as_int(x) ^ (int)m);
#else
  return m ? -x : x;
#endif
}
// power-law impedance sigmoid of MuJoCo's getimpedance()
template <class real> LHW_DEVNI real impedance(const real* solimp, real dist) {
  const real d0 = solimp[0], dw = solimp[1], width = solimp[2], mid = solimp[3], power = solimp[4];
  const real x = m_abs(dist) / width;
  if (x >= 1) return dw;
  if (x <= 0) return d0;
  real y;
  if (power < (real)1.0000001) y = x;
  else if (power == (real)2) {
    if (x <= mid) { const real t = x / mid; y = t * t * mid; }
    else { const real t = (1 - x) / (1 - mid); y = 1 - t * t * (1 - mid); }
  } else if (x <= mid) y = m_pow(x / mid, power) * mid;
  else y = 1 - m_pow((1 - x) / (1 - mid), power) * (1 - mid);
  return d0 + y * (dw - d0);
}

// squared distance between the segments p1-q1 and p2-q2 (closest points by clamping)
template <class real> LHW_DEV real seg_seg_dist2(const real* p1, const real* q1, const real* p2, const real* q2) {
  real d1[3], d2[3], r[3];
#pragma unroll
  for (int x = 0; x < 3; x++) { d1[x] = q1[x] - p1[x]; d2[x] = q2[x] - p2[x]; r[x] = p1[x] - p2[x]; }
  const real a = dot3(d1, d1), e = dot3(d2, d2), f = dot3(d2, r), EPS = (real)1e-12;
  real s, t;
  if (a <= EPS && e <= EPS) { s = t = 0; }
  else if (a <= EPS) { s = 0; t = m_min(m_max(f / e, (real)0), (real)1); }
  else {
    const real c = dot3(d1, r);
    if (e <= EPS) { t = 0; s = m_min(m_max(-c / a, (real)0), (real)1); }
    else {
      const real b = dot3(d1, d2), den = a * e - b * b;
      s = den > EPS ? (b * f - c * e) / den : (real)0;
      s = m_min(m_max(s, (real)0), (real)1);
      t = (b * s + f) / e;
      if (t < 0) { t = 0; s = m_min(m_max(-c / a, (real)0), (real)1); }
      else if (t > 1) { t = 1; s = m_min(m_max((b - c) / a, (real)0), (real)1); }
    }
  }
  real dd = 0;
#pragma unroll
  for (int x = 0; x < 3; x++) { const real w_ = r[x] + d1[x] * s - d2[x] * t; dd += w_ * w_; }
  return dd;
}

// ================================================================= H x = b : arrow Cholesky with the forward
// substitution fused into the factorisation (the right-hand side rides along as one more "row")
// A_c = L_c L_c',  X_c = B_c L_c^-T,  C - sum_c X_c X_c' = L_C L_C'.  Reciprocal pivots in hdinv; the diagonal of
// the factor is never stored (nor read).  x (global dof order) is overwritten with the solution.
template <class real, int NJ, int TK> LHW_DEVNI void arrow_factor_solve(Work<real, NJ, TK>& w, real* x) {
  LHW_ASSUME_SHARED(&w);
  LHW_ASSUME_SHARED(x);
  Arrow<real, NJ, TK>& H = w.H;
  // column steps of both chains side by side.  lane = chain * 16 + row; rows 0..NJ-1: the chain block, NJ..NJ+5: the coupling
  // rows (X = B L^-T), NJ+6: the right-hand side (forward substitution).  All three kinds of row do the SAME arithmetic on
  // their own row pointer, so the step is one branch-free instruction stream (a per-kind if/else would run three times)
  // the three kinds of row live at three places of the same Work record: the lane's row is a word offset from &H.c[0][0][0],
  // chosen with integer selects (the pointer-valued ?: compiled to a jump table per column step), and a failed pivot is
  // only replaced here; it is reported once, from the stored reciprocal pivots, after the factorisation
  real* const hc0 = &H.c[0][0][0];
  const int ox = (int)(&H.x[0][0][0] - hc0), ob = (int)(x - hc0);
#pragma unroll
  for (int k = 0; k < NJ; k++) {
    LHW_LANES(l) {
      const int ch = l >> 4, r = l & 15;
      if (r < NJ + 7 && (r >= NJ || r >= k)) {
        const int o_c = (ch * NJ + r) * NJ, o_x = ox + (ch * 6 + r - NJ) * NJ, o_b = ob + 6 + ch * NJ;
        real* pr = hc0 + (r < NJ ? o_c : (r < NJ + 6 ? o_x : o_b));
        const real* pk = H.c[ch][k];
        real dk = pk[k], t = pr[k];
#pragma unroll
        for (int mm = 0; mm < k; mm++) {
          const real pkm = pk[mm];
          dk -= pkm * pkm;
          t -= pr[mm] * pkm;
        }
        dk = dk > 0 ? dk : (real)1e-30;
        const real inv = m_rsqrt(dk);
        if (r == k) w.hdinv[6 + ch * NJ + k] = inv;
        else pr[k] = t * inv;
      }
    }
    LHW_SYNC();
  }
  // Schur complement of the root block and of the root right-hand side
  // (21 entries of the root block + its 6 right-hand sides: the same 2 NJ-term sum against a different second operand)
  LHW_LANES(l) {
    if (l < 27) {
      const int r = l < 21 ? tri_row(l) : l - 21, c = l - r * (r + 1) / 2;
      real* dst = l < 21 ? &H.r[r][c] : x + r;
      const real* q = l < 21 ? &H.x[0][c][0] : x + 6;     // second operand and its stride from chain 0 to chain 1
      const int qs = l < 21 ? 6 * NJ : NJ;
      real acc = *dst;
#pragma unroll
      for (int ch = 0; ch < 2; ch++)
#pragma unroll
        for (int k = 0; k < NJ; k++) acc -= H.x[ch][r][k] * q[ch * qs + k];
      *dst = acc;
    }
  }
  LHW_SYNC();
#pragma unroll
  for (int k = 0; k < 6; k++) {
    LHW_LANES(l) {
      if (l < 7 && l >= k) {   // rows 0..5 of the Schur complement, row 6 = the root right-hand side: same arithmetic
        real* pr = hc0 + (l < 6 ? (int)(&H.r[0][0] - hc0) + 6 * l : ob);
        const real* pk = H.r[k];
        real dk = pk[k], t = pr[k];
#pragma unroll
        for (int mm = 0; mm < k; mm++) {
          const real pkm = pk[mm];
          dk -= pkm * pkm;
          t -= pr[mm] * pkm;
        }
        dk = dk > 0 ? dk : (real)1e-30;
        const real inv = m_rsqrt(dk);
        if (l == k) w.hdinv[k] = inv;
        else pr[k] = t * inv;
      }
    }
    LHW_SYNC();
  }
  // back substitution: root (one lane, fully unrolled), coupling, then both chains side by side
  LHW_LANES(l) {
    if (l == 0) {
      real z[6];
#pragma unroll
      for (int k = 5; k >= 0; k--) {
        real t = x[k];
#pragma unroll
        for (int mm = k + 1; mm < 6; mm++) t -= H.r[mm][k] * z[mm];
        z[k] = t * w.hdinv[k];
      }
#pragma unroll
      for (int k = 0; k < 6; k++) x[k] = z[k];
    }
  }
  LHW_SYNC();
  LHW_LANES(l) {
    const int ch = l >> 4, k = l & 15;
    if (k < NJ) {
      real t = x[6 + ch * NJ + k];
#pragma unroll
      for (int r = 0; r < 6; r++) t -= H.x[ch][r][k] * x[r];
      x[6 + ch * NJ + k] = t;
    }
    if (l < 6 + 2 * NJ && w.hdinv[l] >= m_rsqrt((real)1e-30)) w.status |= 2;   // a pivot was not positive (or NaN)
  }
  LHW_SYNC();
  LHW_LANES(l) {
    if (l < 2) {
      real z[NJ];
      real* pb = x + 6 + l * NJ;
#pragma unroll
      for (int k = NJ - 1; k >= 0; k--) {
        real t = pb[k];
#pragma unroll
        for (int mm = k + 1; mm < NJ; mm++) t -= H.c[l][mm][k] * z[mm];
        z[k] = t * w.hdinv[6 + l * NJ + k];
      }
#pragma unroll
      for (int k = 0; k < NJ; k++) pb[k] = z[k];
    }
  }
  LHW_SYNC();
}

// y = M x for the arrow-packed symmetric M (lane = dof), result written to out[dof]
template <class real, int NJ, int TK> LHW_DEV real arrow_row_dot(const Arrow<real, NJ, TK>& M, int d, const real* x) {
  real acc = 0;
  if (d < 6) {
#pragma unroll
    for (int j = 0; j < 6; j++) acc += M.r[d][j] * x[j];
#pragma unroll
    for (int ch = 0; ch < 2; ch++)
#pragma unroll
      for (int k = 0; k < NJ; k++) acc += M.x[ch][d][k] * x[6 + ch * NJ + k];
  } else {
    const int ch = (d - 6) / NJ, k = d - 6 - ch * NJ;
#pragma unroll
    for (int j = 0; j < 6; j++) acc += M.x[ch][j][k] * x[j];
#pragma unroll
    for (int kk = 0; kk < NJ; kk++) acc += M.c[ch][k][kk] * x[6 + ch * NJ + kk];
  }
  return acc;
}


// images of a dof-space vector x: outM = M x (lane = dof), outY[f] = S_foot x (lanes 20..31), then the pyramid-edge
// rows e_out = J_edge x - e_sub and limit rows l_out = side * x - l_sub (inactive rows get `fill`).  Used for the warm
// start (x = qacc, sub = aref, fill = 1) and for the search direction (x = s, sub = 0, fill = 0): one shared copy.
template <class real, int NJ, int TK>
LHW_DEVNI void constraint_images(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m_arg, const real* x, real* outM, real (*outY)[6],
                                 real* e_out, real* l_out, real* f_out, const real* e_sub, const real* l_sub,
                                 const real* f_sub, real fill) {
  constexpr int NV = 6 + 2 * NJ, NU = 2 * NJ, NA = 6 + NJ, CPF = Cfg<NJ, TK>::CPF, NEDGE = 8 * CPF;
  const Model<real, NJ, TK>& m = model_ref<real, NJ, TK>(m_arg);
  LHW_ASSUME_SHARED(&w); LHW_ASSUME_SHARED(x); LHW_ASSUME_SHARED(outM); LHW_ASSUME_SHARED(outY);
  LHW_ASSUME_SHARED(e_out); LHW_ASSUME_SHARED(l_out);
  if (e_sub) { LHW_ASSUME_SHARED(e_sub); LHW_ASSUME_SHARED(l_sub); }
  // M x (lanes 0..NV-1) and S_foot x (lanes 20..31) are the same shape of sum -- six root terms, then NJ terms of one chain
  // (root rows: of both chains) -- so they run as ONE instruction stream on per-lane coefficient pointers / strides; the three
  // lane roles as separate branches would be executed one after the other (same summation order as arrow_row_dot)
  LHW_LANES(l) {
    if (l < NV || l >= 20) {
      const int ch = l < NV ? (l < 6 ? 0 : (l - 6) / NJ) : (l - 20) / 6;           // chain (dof lanes) / foot (S_foot lanes)
      const int k = l < NV ? l - 6 - ch * NJ : (l - 20) - ch * 6;                    // chain dof / spatial component
      const real* pa = l < 6 ? &w.M.r[l][0] : (l < NV ? &w.M.x[ch][0][k] : &w.S[0][k]);
      const int sa = l < 6 ? 1 : (l < NV ? NJ : 6);
      const real* pb = l < 6 ? &w.M.x[0][l][0] : (l < NV ? &w.M.c[ch][k][0] : &w.S[6 + ch * NJ][k]);
      const int sb = l < NV ? 1 : 6;
      const real* xb = x + 6 + ch * NJ;
      real acc = 0;
#pragma unroll
      for (int j = 0; j < 6; j++) acc += pa[j * sa] * x[j];
#pragma unroll
      for (int kk = 0; kk < NJ; kk++) acc += pb[kk * sb] * xb[kk];
      if (l < 6) {
        const real* pc = &w.M.x[1][l][0];
#pragma unroll
        for (int kk = 0; kk < NJ; kk++) acc += pc[kk] * x[6 + NJ + kk];
      }
      real* dst = l < NV ? outM + l : &outY[ch][k];
      *dst = acc;
    }
  }
  LHW_SYNC();
  LHW_LANES(l) {
    LHW_STRIDED(ed, l, NEDGE) {
      const int s = ed >> 2, e = ed & 3, f = s / CPF;
      real v = fill;
      if (s - f * CPF < w.ncon[f]) {
        real u[3];
        contact_u(w.cpos[s], outY[f], u);
        if constexpr (Cfg<NJ, TK>::SLABS) riser_u(w.cn[s], u);
        v = u[0] + ((e & 1) ? -m.mu : m.mu) * u[1 + (e >> 1)] - (e_sub ? e_sub[ed] : (real)0);
      }
      e_out[ed] = v;
    }
    if (l < NU) {
      l_out[l] = w.lside[l] ? w.lside[l] * x[6 + l] - (l_sub ? l_sub[l] : (real)0) : fill;
      if constexpr (Cfg<NJ, TK>::FLOSS) f_out[l] = x[6 + l] - (f_sub ? f_sub[l] : (real)0);
    }
  }
  LHW_SYNC();
}

// force of a friction-loss row at residual x (MuJoCo PrimalUpdateConstraint): linear inside |x| < floss R, saturated outside
template <class real> LHW_DEV real floss_force(real D, real lim, real fl, real x, real* curv) {
  if (x <= -lim) { *curv = 0; return fl; }
  if (x >= lim) { *curv = 0; return -fl; }
  *curv = D;
  return -D * x;
}

// P10 (e, second half) and (f) of the fp64 kernels on the fp64 tensor cores (mma.sync m8n8k4): T_f = Af S_f, then
// H = M + sum_f S_f' T_f + the limit / friction-loss diagonal, on the arrow pattern.  Af must be complete (after an LHW_SYNC);
// H is complete after the next LHW_SYNC.  Out of line (like arrow_factor_solve), so that its fragment addressing does not add
// to substep's live registers.
// Padding: only the padded k of BOTH operands are zeroed.  The padded rows and columns of a tile repeat the block's last row or
// column and reach only entries of D that are never stored, so each lane needs one predicate for its fragments,
// (l & 3) < 2, and every read stays inside its block.
template <class real, int NJ, int TK> LHW_DEVNI void newton_hessian_f64(Work<real, NJ, TK>& w) {
  LHW_ASSUME_SHARED(&w);
  constexpr int NA = 6 + NJ;
  constexpr bool FLOSS = Cfg<NJ, TK>::FLOSS;
  const double* const S = &w.S[0][0];
  // k-step k of a 6-long sum: lane l holds term 4 k + (l & 3) of row / column l >> 2 of a row-major block of `rows` rows and
  // stride 6
  const auto frag6 = [](const double* p, int rows, int l, int k) {
    return k && (l & 3) >= 2 ? 0.0 : p[m_min(l >> 2, rows - 1) * 6 + (l & 3) + 4 * k];
  };
  // C fragment entry of a row-major rows x cols block
  const auto cfrag = [](const double* p, int rows, int cols, int l, int i) {
    return p[m_min(l >> 2, rows - 1) * cols + m_min(2 * (l & 3) + i, cols - 1)];
  };
  // T_f in two tiles per foot, the root dofs and the foot's chain dofs, 2 k-steps each; T_f = 0 without contacts.
  // T_f goes through w.T[foot][dof][component]: the C fragment of this product is not the B fragment of the next one
#pragma unroll
  for (int f = 0; f < 2; f++) {
    if (w.ncon[f]) {
#pragma unroll
      for (int n = 0; n < 2; n++)
        warp_mma_f64<2>([&](int l, int k) { return frag6(&w.Af[f][0][0], 6, l, k); },
                        [&](int l, int k) { return frag6(S + 6 * (n ? 6 + f * NJ : 0), n ? NJ : 6, l, k); },
                        [](int, int) { return 0.0; },
                        [&](int l, int i, double v) {
                          const int a = l >> 2, j = 2 * (l & 3) + i;
                          if (a < 6 && j < (n ? NJ : 6)) w.T[f][6 * n + j][a] = v;
                        });
    } else {
      LHW_LANES(l) { LHW_STRIDED(it, l, NA * 6) (&w.T[f][0][0])[it] = 0; }
    }
  }
  LHW_SYNC();
  // H as five tiles: the root block (both feet in one chain of 4 k-steps) and per chain the coupling block (root rows x chain
  // columns) and the chain block (2 k-steps each).  A fragments: S' of the root dofs (root and coupling tiles) or of the chain
  // dofs; B: T.  Only the lower triangles the factorisation reads are stored
  const double* const T = &w.T[0][0][0];
  const auto s_root = [&](int l, int k) { return frag6(S, 6, l, k & 1); };
  warp_mma_f64<4>(s_root, [&](int l, int k) { return frag6(T + (k >> 1) * NA * 6, 6, l, k & 1); },
                  [&](int l, int i) { return cfrag(&w.M.r[0][0], 6, 6, l, i); },
                  [&](int l, int i, double v) {
                    const int r = l >> 2, t = 2 * (l & 3) + i;
                    if (r < 6 && t <= r) w.H.r[r][t] = v;
                  });
#pragma unroll
  for (int ch = 0; ch < 2; ch++) {
    const auto t_chain = [&](int l, int k) { return frag6(T + (ch * NA + 6) * 6, NJ, l, k); };
    warp_mma_f64<2>(s_root, t_chain, [&](int l, int i) { return cfrag(&w.M.x[ch][0][0], 6, NJ, l, i); },
                    [&](int l, int i, double v) {
                      const int j = l >> 2, k = 2 * (l & 3) + i;
                      if (j < 6 && k < NJ) w.H.x[ch][j][k] = v;
                    });
    warp_mma_f64<2>([&](int l, int k) { return frag6(S + 6 * (6 + ch * NJ), NJ, l, k); }, t_chain,
                    [&](int l, int i) { return cfrag(&w.M.c[ch][0][0], NJ, NJ, l, i); },
                    [&](int l, int i, double v) {
                      const int k = l >> 2, t = 2 * (l & 3) + i;
                      if (k < NJ && t <= k) {
                        if (k == t && w.lside[ch * NJ + k] && w.ljar[ch * NJ + k] < 0) v += w.lD[ch * NJ + k];
                        if constexpr (FLOSS) {
                          if (k == t) {
                            const real xj = w.fjar[ch * NJ + k], lim = w.flim[ch * NJ + k];
                            if (xj > -lim && xj < lim) v += w.fD[ch * NJ + k];
                          }
                        }
                        w.H.c[ch][k][t] = v;
                      }
                    });
  }
}

// ================================================================= carried payload (lhw_sim_step_payload, DESIGN.md §7.10)
// A point mass m >= 0 kg rigidly attached to the root link at r, given in the root link's frame relative to the compiled model's
// root-link centre of mass com[0].  The payload step kernels read an env's four words (m, rx, ry, rz) once per control step and
// hand them to every substep.
template <class real> struct Payload { real m, r[3]; };

// the plain link-inertia build: no payload
template <class real, int NJ, int TK>
LHW_DEV void root_payload(const Work<real, NJ, TK>&, const Model<real, NJ, TK>&, int, const real*, real&, real*, real*) {}

// Link i's mass ms, its centre of mass c (rotated to world axes by R, before the link origin is added) and its inertia Ib about
// that centre (link frame) become the composite of the root link and the payload pl.  Only the root link (i == 0) carries one,
// and a payload of mass exactly 0 leaves the plain build's values alone, whatever its offset.  With p = com[0] + r and the root
// link's (ms, c, Ib) as the build has them (H1: the env's randomised p_mass[0], p_com[0], p_inertia0):
//   M' = ms + m,  c' = (ms c + m p) / M',  I' = Ib + ms (|c - c'|^2 E - (c - c')(c - c')^T) + m (|p - c'|^2 E - (p - c')(p - c')^T)
template <class real, int NJ, int TK>
LHW_DEV void root_payload(const Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, int i, const real* R, real& ms, real* c,
                          real* Ib, const Payload<real>& pl) {
  if (i != 0 || pl.m == 0) return;
  real cl[3], cc[3], d1[3], d2[3];
#pragma unroll
  for (int x = 0; x < 3; x++) {
    const real c0 = LHW_GLD(m, com[0][x]);
    if constexpr (Cfg<NJ, TK>::PERENV) cl[x] = w.p_com[0][x];
    else cl[x] = c0;
    const real p = c0 + pl.r[x];
    cc[x] = (ms * cl[x] + pl.m * p) / (ms + pl.m);
    d1[x] = cl[x] - cc[x];
    d2[x] = p - cc[x];
  }
  const real a1 = dot3(d1, d1), a2 = dot3(d2, d2);
  Ib[0] += ms * (a1 - d1[0] * d1[0]) + pl.m * (a2 - d2[0] * d2[0]);
  Ib[1] += ms * (a1 - d1[1] * d1[1]) + pl.m * (a2 - d2[1] * d2[1]);
  Ib[2] += ms * (a1 - d1[2] * d1[2]) + pl.m * (a2 - d2[2] * d2[2]);
  Ib[3] -= ms * d1[0] * d1[1] + pl.m * d2[0] * d2[1];
  Ib[4] -= ms * d1[0] * d1[2] + pl.m * d2[0] * d2[2];
  Ib[5] -= ms * d1[1] * d1[2] + pl.m * d2[1] * d2[2];
  ms += pl.m;
  mv3(R, cc, c);
}

// ================================================================= one physics substep (mujoco.mj_step)
// PL: empty (the plain step) or one Payload<real> (the root link carries it; root_payload above).  The pack keeps the plain
// instantiations' parameter list, and so their code, as it was.
template <class real, int NJ, int TK, class... PL>
LHW_DEVNI void substep(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m_arg, const bool last, const int block_sync = 0,
                       const bool chained = false, const PL... pl) {
  constexpr int NL = 1 + 2 * NJ, NV = 6 + 2 * NJ, NU = 2 * NJ, NA = 6 + NJ;
  constexpr int CPF = Cfg<NJ, TK>::CPF, NCON = 2 * CPF, NEDGE = 4 * NCON, NPTS = Cfg<NJ, TK>::NPTS;
  constexpr bool PERENV = Cfg<NJ, TK>::PERENV, FLOSS = Cfg<NJ, TK>::FLOSS;
  LHW_ASSUME_SHARED(&w);
  const Model<real, NJ, TK>& m = model_ref<real, NJ, TK>(m_arg);  // device: the __constant__ object itself (LDC), not a generic reference
  // ---------------- P1 forward kinematics.  (a) sin/cos of all joints side by side + root rotation
  LHW_LANES(l) {
    if (l < NU) {
      m_sincos(w.qpos[7 + l], &w.sc[l][0], &w.sc[l][1]);
    } else if (l == NU) {
      real q0 = w.qpos[3], q1 = w.qpos[4], q2 = w.qpos[5], q3 = w.qpos[6];
      const real n = m_rsqrt(q0 * q0 + q1 * q1 + q2 * q2 + q3 * q3);
      q0 *= n; q1 *= n; q2 *= n; q3 *= n;
      real* R = w.xmat[0];
      R[0] = 1 - 2 * (q2 * q2 + q3 * q3); R[1] = 2 * (q1 * q2 - q0 * q3); R[2] = 2 * (q1 * q3 + q0 * q2);
      R[3] = 2 * (q1 * q2 + q0 * q3); R[4] = 1 - 2 * (q1 * q1 + q3 * q3); R[5] = 2 * (q2 * q3 - q0 * q1);
      R[6] = 2 * (q1 * q3 - q0 * q2); R[7] = 2 * (q2 * q3 + q0 * q1); R[8] = 1 - 2 * (q1 * q1 + q2 * q2);
      w.o[0] = w.qpos[0]; w.o[1] = w.qpos[1]; w.o[2] = w.qpos[2];
      w.xr[0][0] = w.xr[0][1] = w.xr[0][2] = 0;
      if constexpr (Cfg<NJ, TK>::STEP) { w.rquat[0] = q0; w.rquat[1] = q1; w.rquat[2] = q2; w.rquat[3] = q3; }
    }
  }
  LHW_SYNC();
  // (b) both chains level by level; lane = chain*16 + matrix element (9 elements) ; elements 9..11 do the origin
#pragma unroll 1
  for (int k = 0; k < NJ; k++) {
    LHW_LANES(l) {
      const int ch = l >> 4, e = l & 15;
      if (e < 12) {
        const int i = 1 + ch * NJ + k, p = k == 0 ? 0 : i - 1;
        const real* Rp = w.xmat[p];
        if (e < 9) {
          const int r = e / 3, c = e - 3 * r;
          const real sn = w.sc[i - 1][0], cs = w.sc[i - 1][1];
          const int ax = LHW_GLD(m, axis_id[i]);
          if (ax >= 0) {
            // rotation about a coordinate axis of the parent-aligned frame: column `ax` is kept, the other two
            // columns rotate in their plane:  col_b' = cs col_b + sn col_c ,  col_c' = cs col_c - sn col_b  (b=ax+1, c=ax+2 cyclic)
            const int b = ax == 2 ? 0 : ax + 1, cc = ax == 0 ? 2 : ax - 1;
            real v = Rp[3 * r + c];
            if (c == b) v = cs * v + sn * Rp[3 * r + cc];
            else if (c == cc) v = cs * v - sn * Rp[3 * r + b];
            w.xmat[i][e] = v;
          } else {
            // column c of (link_rot * Rj):  Rj[:,c] = cos e_c + (1-cos) a_c a + sin (a x e_c)
            const real* a = m.axis[i];
            const real t = 1 - cs;
            real col[3] = {t * a[c] * a[0], t * a[c] * a[1], t * a[c] * a[2]};
            col[c] += cs;
            const int c1 = c == 2 ? 0 : c + 1, c2 = c == 0 ? 2 : c - 1;
            col[c1] += sn * a[c2];
            col[c2] -= sn * a[c1];
            const real* L0 = m.link_rot[i];
            const real b0 = L0[0] * col[0] + L0[1] * col[1] + L0[2] * col[2];
            const real b1 = L0[3] * col[0] + L0[4] * col[1] + L0[5] * col[2];
            const real b2 = L0[6] * col[0] + L0[7] * col[1] + L0[8] * col[2];
            w.xmat[i][e] = Rp[3 * r] * b0 + Rp[3 * r + 1] * b1 + Rp[3 * r + 2] * b2;
          }
        } else {
          const int r = e - 9;
          const real lp[3] = {LHW_GLD(m, link_pos[i][0]), LHW_GLD(m, link_pos[i][1]), LHW_GLD(m, link_pos[i][2])};
          w.xr[i][r] = w.xr[p][r] + Rp[3 * r] * lp[0] + Rp[3 * r + 1] * lp[1] + Rp[3 * r + 2] * lp[2];
        }
      }
    }
    LHW_SYNC();
  }
  // ---------------- P2 motion vectors S (per dof) and link spatial inertias about o (per link)
  LHW_LANES(l) {
    if (l < NV) {
      real* S = w.S[l];
      if (l < 3) {
#pragma unroll
        for (int c = 0; c < 6; c++) S[c] = 0;
        S[3 + l] = 1;
      } else if (l < 6) {
        const int k = l - 3;
        S[0] = w.xmat[0][k]; S[1] = w.xmat[0][3 + k]; S[2] = w.xmat[0][6 + k];
        S[3] = S[4] = S[5] = 0;
      } else {
        const int i = l - 5;
        const real ax3[3] = {LHW_GLD(m, axis[i][0]), LHW_GLD(m, axis[i][1]), LHW_GLD(m, axis[i][2])};
        mv3(w.xmat[i], ax3, S);
        cross(w.xr[i], S, S + 3);  // velocity at o of a rotation about the axis through xr: w x (o - p) = p x w
      }
    }
    if (l >= 32 - NL) {  // the other end of the warp builds the link inertias concurrently
      const int i = l - (32 - NL);
      const real* R = w.xmat[i];
      real c[3];
      real Ib[6];
#pragma unroll
      for (int x = 0; x < 6; x++) Ib[x] = LHW_GLD(m, inertia[i][x]);
      real ms;
      if constexpr (PERENV) {
        mv3(R, w.p_com[i], c);
        ms = w.p_mass[i];
        if (i == 0) {
#pragma unroll
          for (int x = 0; x < 6; x++) Ib[x] = w.p_inertia0[x];
        }
      } else {
        const real cm[3] = {LHW_GLD(m, com[i][0]), LHW_GLD(m, com[i][1]), LHW_GLD(m, com[i][2])};
        mv3(R, cm, c);
        ms = LHW_GLD(m, mass[i]);
      }
      root_payload(w, m, i, R, ms, c, Ib, pl...);
#pragma unroll
      for (int x = 0; x < 3; x++) c[x] += w.xr[i][x];
      const real B[9] = {Ib[0], Ib[3], Ib[4], Ib[3], Ib[1], Ib[5], Ib[4], Ib[5], Ib[2]};
      real T[9];
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int cc = 0; cc < 3; cc++) T[3 * r + cc] = R[3 * r] * B[cc] + R[3 * r + 1] * B[3 + cc] + R[3 * r + 2] * B[6 + cc];
      real Iw[6];  // xx yy zz xy xz yz
      const int ri[6] = {0, 1, 2, 0, 0, 1}, ci[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
      for (int e = 0; e < 6; e++)
        Iw[e] = T[3 * ri[e]] * R[3 * ci[e]] + T[3 * ri[e] + 1] * R[3 * ci[e] + 1] + T[3 * ri[e] + 2] * R[3 * ci[e] + 2];
      const real cc2 = dot3(c, c);
      real* I = w.inert[i];
      I[0] = ms; I[1] = ms * c[0]; I[2] = ms * c[1]; I[3] = ms * c[2];
      I[4] = Iw[0] + ms * (cc2 - c[0] * c[0]); I[5] = Iw[1] + ms * (cc2 - c[1] * c[1]); I[6] = Iw[2] + ms * (cc2 - c[2] * c[2]);
      I[7] = Iw[3] - ms * c[0] * c[1]; I[8] = Iw[4] - ms * c[0] * c[2]; I[9] = Iw[5] - ms * c[1] * c[2];
    }
  }
  LHW_SYNC();
  // ---------------- P3 composite inertias (suffix sums, lane = chain*10 + component) ; link velocities V
  // (prefix sums, lanes 20..31 = chain*6 + component) ; velocity-product terms need V first -> next phase
  LHW_LANES(l) {
    if (l < 20) {
      const int ch = l / 10, e = l - ch * 10;
      real acc = 0;
#pragma unroll
      for (int k = NJ - 1; k >= 0; k--) {
        const int i = 1 + ch * NJ + k;
        acc += w.inert[i][e];
        w.comp[i][e] = acc;
      }
    } else {
      const int ch = (l - 20) / 6, e = (l - 20) - ch * 6;
      real acc = e < 3 ? w.xmat[0][3 * e] * w.qvel[3] + w.xmat[0][3 * e + 1] * w.qvel[4] + w.xmat[0][3 * e + 2] * w.qvel[5]
                       : w.qvel[e - 3];
      if (ch == 0) w.V[0][e] = acc;
#pragma unroll
      for (int k = 0; k < NJ; k++) {
        const int i = 1 + ch * NJ + k;
        acc += w.S[5 + i][e] * w.qvel[5 + i];
        w.V[i][e] = acc;
      }
    }
  }
  LHW_SYNC();
  // ---------------- P4 root composite (lanes 0..9) ; per-joint velocity-product acceleration (V x S) qd (lanes 10..)
  LHW_LANES(l) {
    if (l < 10) w.comp[0][l] = w.inert[0][l] + w.comp[1][l] + w.comp[1 + NJ][l];
    else if (l < 10 + NU) {
      const int i = 1 + (l - 10);
      const real* Vi = w.V[i];
      const real* S = w.S[5 + i];
      const real qd = w.qvel[5 + i];
      real t1[3], t2[3], t3[3];
      cross(Vi, S, t1);          // w x w_s
      cross(Vi, S + 3, t2);      // w x v_s
      cross(Vi + 3, S, t3);      // v x w_s
#pragma unroll
      for (int c = 0; c < 3; c++) {
        w.A[i][c] = t1[c] * qd;
        w.A[i][3 + c] = (t2[c] + t3[c]) * qd;
      }
    } else if (l == 31) {
      const real* V0 = w.V[0];
      real t[3];
      cross(V0 + 3, V0, t);  // v_o x w : the rotational free-joint axes move with the body
      w.A[0][0] = w.A[0][1] = w.A[0][2] = 0;
#pragma unroll
      for (int c = 0; c < 3; c++) w.A[0][3 + c] = t[c] - m.grav[c];  // gravity folded in as base acceleration -g
    }
  }
  LHW_SYNC();
  // ---------------- P5 mass matrix (CRBA), lane = dof ; bias accelerations A (prefix sums, lanes 20..31)
  LHW_LANES(l) {
    if (l < NV) {
      real f[6];
      inert_mul(w.comp[dof_link<NJ>(l)], w.S[l], f);
      if (l < 6) {
#pragma unroll
        for (int j = 0; j < 6; j++)
          if (j <= l) {
            const real v = dot6(w.S[j], f);
            w.M.r[l][j] = v; w.M.r[j][l] = v;
          }
      } else {
        const int ch = (l - 6) / NJ, k = l - 6 - ch * NJ;
#pragma unroll
        for (int kk = 0; kk < NJ; kk++)
          if (kk <= k) {
            real v = dot6(w.S[6 + ch * NJ + kk], f);
            if (kk == k) v += LHW_GLD(m, armature[l]);
            w.M.c[ch][k][kk] = v; w.M.c[ch][kk][k] = v;
          }
#pragma unroll
        for (int j = 0; j < 6; j++) w.M.x[ch][j][k] = dot6(w.S[j], f);
      }
    } else if (l >= 20) {
      const int ch = (l - 20) / 6, e = (l - 20) - ch * 6;
      real acc = w.A[0][e];
#pragma unroll
      for (int k = 0; k < NJ; k++) {
        const int i = 1 + ch * NJ + k;
        acc += w.A[i][e];
        w.A[i][e] = acc;
      }
    }
  }
  LHW_SYNC();
  // stepping stones, broad phase: per foot the set of slabs whose footprint (grown by the foot box's circumradius) holds
  // the box centre and whose top face is within vertical reach; a superset of the slabs any corner / sole edge can touch,
  // so the narrow phases below give exactly what an exhaustive test over the 20 slabs gives
  unsigned near_slabs[2] = {0u, 0u};
  if constexpr (Cfg<NJ, TK>::SLABS) {
#pragma unroll
    for (int f = 0; f < 2; f++) {
      near_slabs[f] = warp_ballot([&](int l) -> bool {
        if (l >= NSLAB) return false;
        const int lk = (f + 1) * NJ;
        const real* R = w.xmat[lk];
        const real* fp = m.foot_pos[f];
        const real cx = w.o[0] + w.xr[lk][0] + R[0] * fp[0] + R[1] * fp[1] + R[2] * fp[2];
        const real cy = w.o[1] + w.xr[lk][1] + R[3] * fp[0] + R[4] * fp[1] + R[5] * fp[2];
        const real cz = w.o[2] + w.xr[lk][2] + R[6] * fp[0] + R[7] * fp[1] + R[8] * fp[2];
        const real rad = m.foot_rad[f];
        const real* sl = w.seq[l];
        if (!(cz - rad < sl[2]) || !(cz + rad > sl[2] - 2 * m.slab_half[2])) return false;
        const real c = w.slab_cs[l][0], sn = w.slab_cs[l][1];
        const real dx = cx - sl[0], dy = cy - sl[1];
        return m_abs(c * dx + sn * dy) <= m.slab_half[0] + rad && m_abs(-sn * dx + c * dy) <= m.slab_half[1] + rad;
      });
    }
  }
  // ---------------- P6 link forces f_i = I A + V x* (I V) (lane = link) ; foot-box corner candidates (lanes 16..31)
  LHW_LANES(l) {
    if (l < NL) {
      real IA[6], IV[6], t1[3], t2[3], t3[3];
      inert_mul(w.inert[l], w.A[l], IA);
      inert_mul(w.inert[l], w.V[l], IV);
      const real* V = w.V[l];
      cross(V, IV, t1);          // w x n
      cross(V + 3, IV + 3, t2);  // v x f
      cross(V, IV + 3, t3);      // w x f
#pragma unroll
      for (int c = 0; c < 3; c++) {
        w.F[l][c] = IA[c] + t1[c] + t2[c];
        w.F[l][3 + c] = IA[3 + c] + t3[c];
      }
    } else if (Cfg<NJ, TK>::SPHERES && l >= 16 && l < 16 + 2 * NPTS) {
      // mjc_PlaneCapsule = two mjc_PlaneSphere: dist = centre height - radius, contact iff dist < 0
      const int f = (l - 16) / NPTS, i = (l - 16) - f * NPTS, lk = (f + 1) * NJ;
      const real* R = w.xmat[lk];
      const real* pt = m.foot_pts[f][i];
      const real cd = w.o[2] + w.xr[lk][2] + R[6] * pt[0] + R[7] * pt[1] + R[8] * pt[2] - m.foot_radius[f];
      w.ccd[l - 16] = cd < 0 ? cd : (real)1;
    } else if (!Cfg<NJ, TK>::SPHERES && l >= 16) {
      // mjc_PlaneBox against the ground plane z = 0 (normal +z): one lane per (foot, corner); a corner is a contact
      // candidate when it is below the plane and on the plane side of the box centre
      const int f = (l - 16) >> 3, i = (l - 16) & 7, lk = (f + 1) * NJ;
      const real* R = w.xmat[lk];
      const real ld = R[6] * ((i & 1) ? m.foot_size[f][0] : -m.foot_size[f][0]) +
                      R[7] * ((i & 2) ? m.foot_size[f][1] : -m.foot_size[f][1]) +
                      R[8] * ((i & 4) ? m.foot_size[f][2] : -m.foot_size[f][2]);
      if constexpr (Cfg<NJ, TK>::SLABS) {
        // stepping stones: the corner rests on the HIGHEST surface under it (floor plane, or the top face of a slab whose
        // footprint contains it); surfaces at exactly that height each contribute an identical contact -> multiplicity
        real v[3], cr[3];
        v[0] = ((i & 1) ? m.foot_size[f][0] : -m.foot_size[f][0]) + m.foot_pos[f][0];
        v[1] = ((i & 2) ? m.foot_size[f][1] : -m.foot_size[f][1]) + m.foot_pos[f][1];
        v[2] = ((i & 4) ? m.foot_size[f][2] : -m.foot_size[f][2]) + m.foot_pos[f][2];
        mv3(R, v, cr);
#pragma unroll
        for (int x = 0; x < 3; x++) { cr[x] += w.xr[lk][x]; w.cwp[l - 16][x] = cr[x]; }
        const real ax = w.o[0] + cr[0], ay = w.o[1] + cr[1], az = w.o[2] + cr[2];
        const real floor_z = (Cfg<NJ, TK>::STEP && w.mode == ST_FORWARD) ? (real)-2 : (real)0;   // stepping_task.py:332-334
        real best = 0;
        int have = 0, mult = 0, with_floor = 0;
        real side_inset = -1, side_nx = 0, side_ny = 0;
        if (az - floor_z < 0) { best = floor_z; have = 1; mult = 1; with_floor = 1; }
#pragma unroll 1
        for (unsigned mk = near_slabs[f]; mk; mk &= mk - 1) {
          const int sidx = lowest_bit(mk);
          const real* sl = w.seq[sidx];
          const real d = az - sl[2];
          if (!(d < 0) || -d >= 2 * m.slab_half[2]) continue;
          const real c = w.slab_cs[sidx][0], sn = w.slab_cs[sidx][1];
          const real dx = ax - sl[0], dy = ay - sl[1];
          const real ix = m.slab_half[0] - m_abs(c * dx + sn * dy), iy = m.slab_half[1] - m_abs(-sn * dx + c * dy);
          if (ix < 0 || iy < 0) continue;
          const real inset = ix < iy ? ix : iy;
          if (-d > m.side_tol && -d > inset) {
            // inside the slab, too deep for its top face: the nearest SIDE face holds the corner (a stair riser); first such
            // slab in index order, x' faces win ties
            if (m.side_faces && side_inset < 0 && !(ld > 0)) {
              const real xs = c * dx + sn * dy, ys = -sn * dx + c * dy;
              real lx = 0, ly = 0;
              if (ix <= iy) lx = xs < 0 ? (real)-1 : (real)1; else ly = ys < 0 ? (real)-1 : (real)1;
              side_inset = inset;
              side_nx = c * lx - sn * ly;
              side_ny = sn * lx + c * ly;
            }
            continue;
          }
          if (!have || sl[2] > best) { best = sl[2]; have = 1; mult = 1; with_floor = 0; }
          else if (sl[2] == best) mult++;
        }
        w.ccd[l - 16] = (have && !(ld > 0)) ? az - best : (real)1;
        w.cmul[l - 16] = with_floor ? (real)mult : (real)-mult;   // sign: the floor plane is one of the `mult` supports
        w.cside[l - 16] = side_inset;
        w.csn[l - 16][0] = side_nx; w.csn[l - 16][1] = side_ny;
      } else {
      const real dist0 = w.o[2] + w.xr[lk][2] + R[6] * m.foot_pos[f][0] + R[7] * m.foot_pos[f][1] + R[8] * m.foot_pos[f][2];
      w.ccd[l - 16] = (dist0 + ld > 0 || ld > 0) ? (real)1 : dist0 + ld;
      }
    }
  }
  LHW_SYNC();
  // ---------------- P7 subtree forces (suffix sums, lane = chain*6 + comp) ; contact slots: the first (at most) 4
  // candidate corners of each foot in corner-index order, as mjc_PlaneBox returns them (lanes 12, 13)
  LHW_LANES(l) {
    if (l < 12) {
      const int ch = l / 6, e = l - ch * 6;
      real acc = 0;
#pragma unroll
      for (int k = NJ - 1; k >= 0; k--) {
        const int i = 1 + ch * NJ + k;
        acc += w.F[i][e];
        w.F[i][e] = acc;
      }
    } else if (l < 14) {
      const int f = l - 12;
      int cnt = 0;
#pragma unroll
      for (int i = 0; i < NPTS; i++)
        if (cnt < (Cfg<NJ, TK>::SLABS ? NCORNER : CPF) && !(w.ccd[f * NPTS + i] > 0)) { w.cslot[f * CPF + cnt] = i; cnt++; }
      w.ncorner[f] = cnt;
      if constexpr (Cfg<NJ, TK>::SLABS) {
        // riser contacts take the first of the foot's CPF - NCORNER extra slots, in corner order (the sole-edge crossings of
        // P7x fill what is left)
        int ns = 0;
#pragma unroll 1
        for (int i = 0; i < NPTS; i++) {
          const real ins = w.cside[f * NPTS + i];
          if (!(ins < 0) && ns < CPF - NCORNER) {
            const int s = f * CPF + cnt + ns;
            const real nx = w.csn[f * NPTS + i][0], ny = w.csn[f * NPTS + i][1];
            w.cpos[s][0] = w.cwp[f * 8 + i][0] + (real)0.5 * ins * nx;
            w.cpos[s][1] = w.cwp[f * 8 + i][1] + (real)0.5 * ins * ny;
            w.cpos[s][2] = w.cwp[f * 8 + i][2];
            w.xcd[s] = -ins;
            w.cn[s][0] = nx; w.cn[s][1] = ny;
            ns++;
          }
        }
        cnt += ns;
        w.nside[f] = ns;
      }
      w.ncon[f] = cnt;
    }
  }
  LHW_SYNC();
  if constexpr (Cfg<NJ, TK>::SLABS) {
    // ---------------- P7x sole-edge x slab-boundary crossings: the remaining vertices of (sole rectangle) clipped against
    // (slab footprint) -- the face-face manifold of a box-box test with the slab's top face as reference face.  One lane
    // per (slab, sole edge): Liang-Barsky clip of the edge against the footprint; an entry / exit parameter strictly
    // inside (0,1) is a polygon vertex.  Kept: the first CPF - NCORNER per foot in (slab, edge, entry-then-exit) order.
#pragma unroll 1
    for (int f = 0; f < 2; f++) {
      int run = w.nside[f];     // the extra slots the riser contacts of P7 already took
      const int ntask = 4 * bit_count(near_slabs[f]);
#pragma unroll 1
      for (int pass = 0; pass * 32 < ntask; pass++) {
        LHW_LANES_ORDERED(l) {   // LHW_PREFIX2 below
          const int t = pass * 32 + l;
          int he = 0, hx = 0;
          real pe[4], px[4];   // x, y, z relative to o, signed distance
          if (t < ntask) {
            const int sidx = nth_bit(near_slabs[f], t >> 2), ed = t & 3;
            const int ia = ed == 0 ? 0 : ed == 1 ? 1 : ed == 2 ? 3 : 2, ib = ed == 0 ? 1 : ed == 1 ? 3 : ed == 2 ? 2 : 0;
            const real* A = w.cwp[f * 8 + ia];
            const real* B = w.cwp[f * 8 + ib];
            const real* sl = w.seq[sidx];
            const real c = w.slab_cs[sidx][0], sn = w.slab_cs[sidx][1];
            const real Ax = w.o[0] + A[0] - sl[0], Ay = w.o[1] + A[1] - sl[1], Bx = w.o[0] + B[0] - sl[0], By = w.o[1] + B[1] - sl[1];
            const real ax = c * Ax + sn * Ay, ay = -sn * Ax + c * Ay, bx = c * Bx + sn * By, by = -sn * Bx + c * By;
            const real dx = bx - ax, dy = by - ay;
            real t0 = 0, t1 = 1;
            bool ok = true;
#pragma unroll
            for (int b = 0; b < 4; b++) {
              const real pp = b == 0 ? -dx : b == 1 ? dx : b == 2 ? -dy : dy;
              const real qq = b == 0 ? ax + m.slab_half[0] : b == 1 ? m.slab_half[0] - ax : b == 2 ? ay + m.slab_half[1] : m.slab_half[1] - ay;
              if (pp == 0) { if (qq < 0) ok = false; }
              else {
                const real r = qq / pp;
                if (pp < 0) { if (r > t1) ok = false; else if (r > t0) t0 = r; }
                else { if (r < t0) ok = false; else if (r < t1) t1 = r; }
              }
            }
            if (ok) {
#pragma unroll
              for (int side = 0; side < 2; side++) {
                const real tt = side == 0 ? t0 : t1;
                if (side == 0 ? !(t0 > 0) : !(t1 < 1)) continue;
                const real zr = A[2] + tt * (B[2] - A[2]);
                const real cd = (w.o[2] + zr) - sl[2];
                if (!(cd < 0) || -cd > m.side_tol) continue;
                real* o4 = side == 0 ? pe : px;
                o4[0] = A[0] + tt * (B[0] - A[0]); o4[1] = A[1] + tt * (B[1] - A[1]); o4[2] = zr - (real)0.5 * cd; o4[3] = cd;
                if (side == 0) he = 1; else hx = 1;
              }
            }
          }
          int pos;
          LHW_PREFIX2(he, hx, run, pos);
          if (he && pos < CPF - NCORNER) {
            const int sl_ = f * CPF + w.ncorner[f] + pos;
            w.cpos[sl_][0] = pe[0]; w.cpos[sl_][1] = pe[1]; w.cpos[sl_][2] = pe[2]; w.xcd[sl_] = pe[3];
            w.cn[sl_][0] = 0; w.cn[sl_][1] = 0;
          }
          if (hx && pos + he < CPF - NCORNER) {
            const int sl_ = f * CPF + w.ncorner[f] + pos + he;
            w.cpos[sl_][0] = px[0]; w.cpos[sl_][1] = px[1]; w.cpos[sl_][2] = px[2]; w.xcd[sl_] = px[3];
            w.cn[sl_][0] = 0; w.cn[sl_][1] = 0;
          }
        }
      }
      LHW_LANES(l) {
        if (l == 0) w.ncon[f] = w.ncorner[f] + (run < CPF - NCORNER ? run : CPF - NCORNER);
      }
    }
    LHW_SYNC();
  }
  // ---------------- P7b per contact slot: position, impedance, regulariser, reference stiffness (lane = slot)
  LHW_LANES(l) {
    if (l < NCON && l - (l / CPF) * CPF < w.ncon[l / CPF]) {
      const int f = l / CPF, lk = (f + 1) * NJ;
      real cd, mult = 1;
      if constexpr (Cfg<NJ, TK>::SLABS) {
        if (l - f * CPF < w.ncorner[f]) {
          const int i = w.cslot[l];
          cd = w.ccd[f * NPTS + i];
          mult = m_abs(w.cmul[f * NPTS + i]);
          w.cpos[l][0] = w.cwp[f * 8 + i][0]; w.cpos[l][1] = w.cwp[f * 8 + i][1];
          w.cpos[l][2] = w.cwp[f * 8 + i][2] - (real)0.5 * cd;
          w.cn[l][0] = 0; w.cn[l][1] = 0;
          // share of this slot's force that the task's floor-contact queries see (xcd is free for corner slots)
          w.xcd[l] = (!Cfg<NJ, TK>::STEP || m.slab_contacts_are_floor) ? (real)1 : (w.cmul[f * NPTS + i] > 0 ? (real)1 / mult : (real)0);
        } else {
          cd = w.xcd[l];   // riser / crossing slot: position, distance and normal already written by P7 / P7x
          w.xcd[l] = (!Cfg<NJ, TK>::STEP || m.slab_contacts_are_floor) ? (real)1 : (real)0;
        }
        w.cpos[l][3] = 1; w.cpos[l][4] = 0;
      } else {
      const int i = w.cslot[l];
      cd = w.ccd[f * NPTS + i];
      real v[3], corner[3];
      if constexpr (Cfg<NJ, TK>::SPHERES) {
        v[0] = m.foot_pts[f][i][0]; v[1] = m.foot_pts[f][i][1]; v[2] = m.foot_pts[f][i][2];
      } else {
        v[0] = ((i & 1) ? m.foot_size[f][0] : -m.foot_size[f][0]) + m.foot_pos[f][0];
        v[1] = ((i & 2) ? m.foot_size[f][1] : -m.foot_size[f][1]) + m.foot_pos[f][1];
        v[2] = ((i & 4) ? m.foot_size[f][2] : -m.foot_size[f][2]) + m.foot_pos[f][2];
      }
      mv3(w.xmat[lk], v, corner);
      w.cpos[l][0] = corner[0] + w.xr[lk][0];
      w.cpos[l][1] = corner[1] + w.xr[lk][1];
      // contact point: half way through the penetration (box corner), resp. sphere centre - n (r + dist/2)
      w.cpos[l][2] = corner[2] + w.xr[lk][2] - (Cfg<NJ, TK>::SPHERES ? m.foot_radius[f] + (real)0.5 * cd : (real)0.5 * cd);
      }
      const real imp = impedance(m.solimp, cd);
      const real Rn = m_max((real)1e-15, (1 - imp) / imp * (m.foot_invw[f] * (1 + m.mu * m.mu)));
      w.cD[l] = mult / (2 * m.mu_reg * m.mu_reg * Rn);
      w.cKid[l] = m.Kc * imp * cd;
    }
  }
  LHW_SYNC();
  // ---------------- P8 pyramid-edge reference accelerations (lane = edge; foot spatial velocity from P3) ;
  // qfrc_smooth + warm start (lane = dof) ; joint limits (lanes 18..18+NU)
  LHW_LANES(l) {
    LHW_STRIDED(ed, l, NEDGE) {
      const int s = ed >> 2, e = ed & 3, f = s / CPF;
      if (s - f * CPF < w.ncon[f]) {
        real u[3];
        contact_u(w.cpos[s], w.V[(f + 1) * NJ], u);
        if constexpr (Cfg<NJ, TK>::SLABS) riser_u(w.cn[s], u);
        const real vel = u[0] + ((e & 1) ? -m.mu : m.mu) * u[1 + (e >> 1)];
        w.ejar[ed] = -m.Bc * vel - w.cKid[s];
      }
    }
    if (l < NV) {
      const int lk = dof_link<NJ>(l);
      real Ft[6];
      if (lk == 0) {
#pragma unroll
        for (int c = 0; c < 6; c++) Ft[c] = w.F[0][c] + w.F[1][c] + w.F[1 + NJ][c];
      } else {
#pragma unroll
        for (int c = 0; c < 6; c++) Ft[c] = w.F[lk][c];
      }
      real q;
      if constexpr (PERENV) {
        q = -(l >= 6 ? w.p_damping[l - 6] : m.damping[l]) * w.qvel[l] - dot6(w.S[l], Ft);
        if (l < 6) {
          // xfrc_applied on the pelvis / torso bodies (both inside the root link): J_com' [f; tau], root dofs only
#pragma unroll
          for (int b = 0; b < 2; b++) {
            const real* fx = w.xfrc[b];
            if (l < 3) q += fx[l];
            else {
              real r[3], rxf[3];
              mv3(w.xmat[0], b == 0 ? w.p_pelcom : m.torso_com, r);
              cross(r, fx, rxf);
              const int k = l - 3;
              q += w.xmat[0][k] * (fx[3] + rxf[0]) + w.xmat[0][3 + k] * (fx[4] + rxf[1]) + w.xmat[0][6 + k] * (fx[5] + rxf[2]);
            }
          }
        }
      } else {
        q = -LHW_GLD(m, damping[l]) * w.qvel[l] - dot6(w.S[l], Ft);
      }
      if (l >= 6) q += w.ctrl[l - 6];
      w.qfs[l] = q;
      // warm start: the last solution, extrapolated linearly from the one before it (in vec since P12) once the control step
      // has had a substep; a_k + (a_k - a_{k-1}) starts the solve inside the final active set more often, so fewer substeps
      // take a second Newton step -- and a lock-step block pays the largest count among its warps (DESIGN.md §4.1)
      w.qacc[l] = chained ? 2 * w.qacc_warm[l] - w.vec[l] : w.qacc_warm[l];
    } else if (l < NV + NU) {
      const int u = l - NV, d = 6 + u;
      const real q = w.qpos[7 + u];
      const real dlo = q - LHW_GLD(m, range_lo[d]), dhi = LHW_GLD(m, range_hi[d]) - q;
      int side = 0;
      real dist = 0;
      if (dlo < 0) { side = 1; dist = dlo; }
      else if (dhi < 0) { side = -1; dist = dhi; }
      w.lside[u] = side;
      if (side) {
        const real imp = impedance(m.solimp, dist);
        w.lD[u] = (real)1 / m_max((real)1e-15, (1 - imp) / imp * m.dof_invw[d]);
        w.ljar[u] = -m.B * (side * w.qvel[d]) - m.K * imp * dist;
      }
      if constexpr (FLOSS) {
        // dof friction loss: J = e_d, pos = 0 -> impedance solimp[0], aref = -B vel
        const real imp = m.solimp[0];
        const real Rf = m_max((real)1e-15, (1 - imp) / imp * m.dof_invw[d]);
        w.fD[u] = (real)1 / Rf;
        w.flim[u] = w.p_floss[u] * Rf;
        w.fjar[u] = -m.B * w.qvel[d];
      }
    }
  }
  LHW_SYNC();
  LHW_BLOCK_SYNC(block_sync & 2);  // optional second rendez-vous of the block's warps, before the solver
  // ---------------- P9 Newton start: contact point maps Pm, then Ma = M a, ya = S_foot a and the row residuals
  if constexpr (!Cfg<NJ, TK>::SLABS)
  LHW_LANES(l) {
    if (l < NCON && l - (l / CPF) * CPF < w.ncon[l / CPF]) {
      // rows of P: spatial wrench [p x e ; e] of a unit force along e = n (+z), t1 (+y), t2 (-x) applied at p
      const real px = w.cpos[l][0], py = w.cpos[l][1], pz = w.cpos[l][2];
      real* P = &w.Pm[l][0][0];
      P[0] = py;  P[1] = -px; P[2] = 0;   P[3] = 0;  P[4] = 0; P[5] = 1;
      P[6] = -pz; P[7] = 0;   P[8] = px;  P[9] = 0;  P[10] = 1; P[11] = 0;
      P[12] = 0;  P[13] = -pz; P[14] = py; P[15] = -1; P[16] = 0; P[17] = 0;
    }
  }
  // (the reference accelerations sit in ejar / ljar / fjar since P8: subtracted in place, every lane its own entries)
  constraint_images<real, NJ, TK>(w, m, w.qacc, w.Ma, w.ya, w.ejar, w.ljar, w.fjar, w.ejar, w.ljar, w.fjar, (real)1);

  // ---------------- P10 primal Newton on  1/2 (a-a_s)' M (a-a_s) + sum_r 1/2 D_r min(0, J_r a - aref_r)^2
  // residuals (Ma, ejar, ljar) are carried incrementally: x += alpha * (direction image)
  bool converged = false;
  LHW_NEWTON_HOOK(0, w, 0);
  for (int iter = 0; iter <= m.max_iter && !converged; iter++) {
    // (a) per contact: force in the contact frame and the 3x3 weight  W = sum_active D w w'  (lane = contact);
    // active set = sign of the carried residuals (inactive slots carry jar = 1)
    LHW_LANES(l) {
      if (l < NCON && l - (l / CPF) * CPF < w.ncon[l / CPF]) {
        const real* jr = w.ejar + 4 * l;
        const real D = w.cD[l], mu = m.mu;
        const int a0 = jr[0] < 0, a1 = jr[1] < 0, a2 = jr[2] < 0, a3 = jr[3] < 0;
        const real f0 = a0 ? -D * jr[0] : (real)0, f1 = a1 ? -D * jr[1] : (real)0;
        const real f2 = a2 ? -D * jr[2] : (real)0, f3 = a3 ? -D * jr[3] : (real)0;
        w.cF[l][0] = f0 + f1 + f2 + f3;
        w.cF[l][1] = mu * (f0 - f1);
        w.cF[l][2] = mu * (f2 - f3);
        w.cW[l][0] = D * (a0 + a1 + a2 + a3);
        w.cW[l][1] = D * mu * (a0 - a1);
        w.cW[l][2] = D * mu * (a2 - a3);
        w.cW[l][3] = D * mu * mu * (a0 + a1);
        w.cW[l][4] = D * mu * mu * (a2 + a3);
        if constexpr (Cfg<NJ, TK>::SLABS) {
          w.cW[l][5] = 0;
          const real nx = w.cn[l][0], ny = w.cn[l][1];
          if (nx != 0 || ny != 0) {
            // everything downstream (Ff, Af) works in the canonical frame C0 = (+z, +y, -x): f0 = Q f, W0 = Q W Q' with the riser
            // frame's vectors as the columns of Q (see riser_u)
            const real Q[3][3] = {{0, 1, 0}, {ny, 0, -nx}, {-nx, 0, -ny}};
            const real fc[3] = {w.cF[l][0], w.cF[l][1], w.cF[l][2]};
            const real Wc[3][3] = {{w.cW[l][0], w.cW[l][1], w.cW[l][2]}, {w.cW[l][1], w.cW[l][3], 0}, {w.cW[l][2], 0, w.cW[l][4]}};
            real QW[3][3], W0[3][3];
#pragma unroll
            for (int r = 0; r < 3; r++) {
              w.cF[l][r] = Q[r][0] * fc[0] + Q[r][1] * fc[1] + Q[r][2] * fc[2];
#pragma unroll
              for (int c = 0; c < 3; c++) QW[r][c] = Q[r][0] * Wc[0][c] + Q[r][1] * Wc[1][c] + Q[r][2] * Wc[2][c];
            }
#pragma unroll
            for (int r = 0; r < 3; r++)
#pragma unroll
              for (int c = 0; c < 3; c++) W0[r][c] = QW[r][0] * Q[c][0] + QW[r][1] * Q[c][1] + QW[r][2] * Q[c][2];
            w.cW[l][0] = W0[0][0]; w.cW[l][1] = W0[0][1]; w.cW[l][2] = W0[0][2];
            w.cW[l][3] = W0[1][1]; w.cW[l][4] = W0[2][2]; w.cW[l][5] = W0[1][2];
          }
        }
      }
    }
    LHW_SYNC();
    // (c) per foot: wrench Ff = sum P' cF  (lane = foot*6 + component)
    LHW_LANES(l) {
      if (l < 12) {
        const int f = l / 6, a = l - f * 6;
        real acc = 0;
        int ia[3];
        unsigned sa[3];
        pmap_sel(a, ia, sa);
        for (int k = 0; k < w.ncon[f]; k++) {
          const real* cf = w.cF[f * CPF + k];
          if constexpr (Cfg<NJ, TK>::SLABS) {
            const real* cp = w.cpos[f * CPF + k];
            acc += sflip(cp[ia[0]], sa[0]) * cf[0] + sflip(cp[ia[1]], sa[1]) * cf[1] + sflip(cp[ia[2]], sa[2]) * cf[2];
          } else {
            const real* P = &w.Pm[f * CPF + k][0][0];
            acc += P[a] * cf[0] + P[6 + a] * cf[1] + P[12 + a] * cf[2];
          }
        }
        w.Ff[f][a] = acc;
      }
    }
    LHW_SYNC();
    // (d) gradient (lane = dof)
    LHW_LANES(l) {
      if (l < NV) {
        real g = w.Ma[l] - w.qfs[l];
        const real gf = dot6(w.S[l], w.Ff[l < 6 ? 0 : (l - 6) / NJ]);    // one stream for root and chain dofs
        if (l < 6) g -= gf + dot6(w.S[l], w.Ff[1]);
        else {
          g -= gf;
          if (w.lside[l - 6] && w.ljar[l - 6] < 0) g -= w.lside[l - 6] * (-w.lD[l - 6] * w.ljar[l - 6]);
          if constexpr (FLOSS) {
            real cv;
            g -= floss_force(w.fD[l - 6], w.flim[l - 6], w.p_floss[l - 6], w.fjar[l - 6], &cv);
          }
        }
        w.grad[l] = g;
        w.sdir[l] = -g;
      }
    }
    LHW_SYNC();
    const real g2 = warp_sum<real>([&](int l) { return l < NV ? w.grad[l] * w.grad[l] : (real)0; });
    if (g2 < m.tol2 || iter == m.max_iter) { converged = true; break; }
    // (e) a Newton step is needed: spatial weight per foot  Af = sum P' W P  (2 x 21 items, mirrored) ...
    LHW_LANES(l) {
      for (int it = l; it < 42; it += 32) {
        const int f = it / 21;
        const int a = tri_row(it - f * 21), b = it - f * 21 - a * (a + 1) / 2;
        real acc = 0;
        int ia[3], ib[3];
        unsigned sa[3], sb[3];
        pmap_sel(a, ia, sa);
        pmap_sel(b, ib, sb);
        for (int k = 0; k < w.ncon[f]; k++) {
          const int s = f * CPF + k;
          const real* W = w.cW[s];
          real a0, a1, a2, b0, b1, b2;
          if constexpr (Cfg<NJ, TK>::SLABS) {
            const real* cp = w.cpos[s];
            a0 = sflip(cp[ia[0]], sa[0]); a1 = sflip(cp[ia[1]], sa[1]); a2 = sflip(cp[ia[2]], sa[2]);
            b0 = sflip(cp[ib[0]], sb[0]); b1 = sflip(cp[ib[1]], sb[1]); b2 = sflip(cp[ib[2]], sb[2]);
          } else {
            const real* P = &w.Pm[s][0][0];
            a0 = P[a]; a1 = P[6 + a]; a2 = P[12 + a]; b0 = P[b]; b1 = P[6 + b]; b2 = P[12 + b];
          }
          if constexpr (Cfg<NJ, TK>::SLABS)
            acc += a0 * (W[0] * b0 + W[1] * b1 + W[2] * b2) + a1 * (W[1] * b0 + W[3] * b1 + W[5] * b2) + a2 * (W[2] * b0 + W[5] * b1 + W[4] * b2);
          else
            acc += a0 * (W[0] * b0 + W[1] * b1 + W[2] * b2) + a1 * (W[1] * b0 + W[3] * b1) + a2 * (W[2] * b0 + W[4] * b2);
        }
        w.Af[f][a][b] = acc;
        w.Af[f][b][a] = acc;
      }
    }
    LHW_SYNC();
    if constexpr (sizeof(real) == 8) {
      newton_hessian_f64<real, NJ, TK>(w);
    } else {
    // ... and T_f = Af S_f (per foot, per ancestor dof, per component)
    LHW_LANES(l) {
      for (int it = l; it < 2 * NA * 6; it += 32) {
        const int f = it / (NA * 6), r = it - f * (NA * 6), j = r / 6, a = r - j * 6;
        const real* S = w.S[loc2dof<NJ>(f, j)];
        const real* Af = w.Af[f][a];
        real acc = 0;
#pragma unroll
        for (int b = 0; b < 6; b++) acc += Af[b] * S[b];
        w.T[f][j][a] = w.ncon[f] ? acc : (real)0;
      }
    }
    LHW_SYNC();
    // (f) H = M + S' Af S + diag(limit D) on the arrow pattern (21 + 2*36 + 2*21 items)
    // (21 root + 2 x 6 NJ coupling + 2 x NJ(NJ+1)/2 chain items; a pass of 32 lanes is almost always of ONE kind, so per-kind
    // branches cost nothing here -- a single stream on per-item pointers was measured 12 % MORE instructions for this phase)
    LHW_LANES(l) {
      for (int it = l; it < 21 + 2 * 6 * NJ + NJ * (NJ + 1); it += 32) {
        if (it < 21) {
          const int r = tri_row(it), t = it - r * (r + 1) / 2;
          w.H.r[r][t] = w.M.r[r][t] + dot6(w.S[r], w.T[0][t]) + dot6(w.S[r], w.T[1][t]);
        } else if (it < 21 + 2 * 6 * NJ) {
          const int q = it - 21, ch = q / (6 * NJ), rr = q - ch * 6 * NJ, j = rr / NJ, k = rr - j * NJ;
          w.H.x[ch][j][k] = w.M.x[ch][j][k] + dot6(w.S[6 + ch * NJ + k], w.T[ch][j]);
        } else {
          const int q = it - 21 - 2 * 6 * NJ, ch = q / (NJ * (NJ + 1) / 2), rr = q - ch * (NJ * (NJ + 1) / 2);
          const int k = tri_row(rr), t = rr - k * (k + 1) / 2;
          real acc = w.M.c[ch][k][t] + dot6(w.S[6 + ch * NJ + k], w.T[ch][6 + t]);
          if (k == t && w.lside[ch * NJ + k] && w.ljar[ch * NJ + k] < 0) acc += w.lD[ch * NJ + k];
          if constexpr (FLOSS) {
            if (k == t) {
              const real xj = w.fjar[ch * NJ + k], lim = w.flim[ch * NJ + k];
              if (xj > -lim && xj < lim) acc += w.fD[ch * NJ + k];
            }
          }
          w.H.c[ch][k][t] = acc;
        }
      }
    }
    }
    LHW_SYNC();
    arrow_factor_solve<real, NJ, TK>(w, w.sdir);
    // (g) images of the search direction: M s, foot spatial accelerations, edge / limit rates
    constraint_images<real, NJ, TK>(w, m, w.sdir, w.Ms, w.ys, w.ejv, w.ljv, w.fjv, (const real*)nullptr, (const real*)nullptr,
                                (const real*)nullptr, (real)0);
    const real sMs = warp_sum<real>([&](int l) { return l < NV ? w.sdir[l] * w.Ms[l] : (real)0; });
    const real sg = warp_sum<real>([&](int l) { return l < NV ? w.sdir[l] * (w.Ma[l] - w.qfs[l]) : (real)0; });
    // (h) exact line search: phi'(alpha) is continuous, piecewise linear, increasing; safeguarded 1-D Newton
    const real LS_TOL = sizeof(real) == 8 ? (real)2e-14 : (real)1e-5;
    real alpha = 1, lo = 0, hi = -1, d_at0 = 0;
    for (int ls = 0; ls < 40; ls++) {
      LHW_NEWTON_HOOK(1, w, ls);
      const real al = ls == 0 ? (real)0 : alpha;
      const real cd = warp_sum<real>([&](int l) {
        real acc = 0;
        LHW_STRIDED(ed, l, NEDGE) {
          const real x = w.ejar[ed] + al * w.ejv[ed];   // inactive slots: jar = 1, jv = 0
          if (x < 0) acc += w.cD[ed >> 2] * x * w.ejv[ed];
        }
        if (l < NU) {
          const real xl = w.ljar[l] + al * w.ljv[l];
          if (xl < 0) acc += w.lD[l] * xl * w.ljv[l];
          if constexpr (FLOSS) {
            real cv;
            acc -= floss_force(w.fD[l], w.flim[l], w.p_floss[l], w.fjar[l] + al * w.fjv[l], &cv) * w.fjv[l];
          }
        }
        return acc;
      });
      const real d = al * sMs + sg + cd;
      if (ls == 0) {
        d_at0 = d;
        if (!(d < 0)) { alpha = 0; break; }  // not a descent direction: at the roundoff floor
        continue;                            // first trial: the full Newton step alpha = 1
      }
      // done when phi' is zero relative to phi'(0), or to the size of the terms that cancel in it (the roundoff floor: a warm
      // start close to the solution has a tiny phi'(0), and trials below that floor only chase rounding)
      if (m_abs(d) <= LS_TOL * m_max(m_abs(d_at0), al * sMs + m_abs(sg) + m_abs(cd))) break;
      const real cdd = warp_sum<real>([&](int l) {
        real acc = 0;
        LHW_STRIDED(ed, l, NEDGE)
          if (w.ejar[ed] + al * w.ejv[ed] < 0) acc += w.cD[ed >> 2] * w.ejv[ed] * w.ejv[ed];
        if (l < NU && w.ljar[l] + al * w.ljv[l] < 0) acc += w.lD[l] * w.ljv[l] * w.ljv[l];
        if constexpr (FLOSS) {
          if (l < NU) {
            real cv;
            floss_force(w.fD[l], w.flim[l], w.p_floss[l], w.fjar[l] + al * w.fjv[l], &cv);
            acc += cv * w.fjv[l] * w.fjv[l];
          }
        }
        return acc;
      });
      if (d < 0) lo = al; else hi = al;
      real an = al - d / (sMs + cdd);
      if (an <= lo || (hi > 0 && an >= hi)) an = hi > 0 ? (real)0.5 * (lo + hi) : 2 * al;
      if (an == al) break;
      alpha = an;
    }
    LHW_LANES(l) {
      if (l < NV) {
        w.qacc[l] += alpha * w.sdir[l];
        w.Ma[l] += alpha * w.Ms[l];
      }
      LHW_STRIDED(ed, l, NEDGE) w.ejar[ed] += alpha * w.ejv[ed];
      if (l < NU) {
        w.ljar[l] += alpha * w.ljv[l];
        if constexpr (FLOSS) w.fjar[l] += alpha * w.fjv[l];
      }
      if (l == 31) w.iters_total++;
    }
    LHW_SYNC();
    if (alpha == 0) converged = true;
  }
  LHW_NEWTON_HOOK(2, w, 0);

  // ---------------- P11 what mjData keeps after mj_step (evaluated at the pre-integration state)
  LHW_LANES(l) {
    if (l < NU) {
      w.act_len[l] = w.qpos[7 + l];
      w.act_vel[l] = w.qvel[6 + l];
      w.act_force[l] = w.ctrl[l];
    }
    if (last) {
      if (l >= 12 && l < 15) { w.root_vlin[l - 12] = w.qvel[l - 12]; w.qacc_lag[l - 12] = w.qacc[l - 12]; }
      if (l >= 16 && l < 18) {
        const int f = l - 16, lk = (f + 1) * NJ;
        real t[3];
        cross(w.V[lk], w.xr[lk], t);  // velocity of the link origin: v_o + w x r
        real g = 0;
#pragma unroll
        for (int c = 0; c < 3; c++) w.foot_vel[f][c] = w.V[lk][3 + c] + t[c];
        if constexpr (Cfg<NJ, TK>::STEP) {
          real st[3];
          mv3(w.xmat[lk], m.foot_site[f], st);
#pragma unroll
          for (int c = 0; c < 3; c++) w.site[f][c] = w.o[c] + w.xr[lk][c] + st[c];
        }
        for (int k = 0; k < w.ncon[f]; k++) {
          const real* cf = w.cF[f * CPF + k];
          real nrm = m_sqrt(cf[0] * cf[0] + cf[1] * cf[1] + cf[2] * cf[2]);  // norm of mj_contactForce, friction included
          // SURVEY Appendix C-2: get_*_floor_contacts (robot_interface.py:252-301) skips foot-on-stone contacts (the foot box is
          // geom1 there): only the floor plane's share of a merged corner slot is visible to the task
          if constexpr (Cfg<NJ, TK>::SLABS) nrm *= w.xcd[f * CPF + k];
          g += nrm;
        }
        w.grf[f] = g;
      }
      if (l == 20) {
        real z = 0;
        bool first = true;
        int nfl = 0;
        for (int s = 0; s < NCON; s++)
          if (s - (s / CPF) * CPF < w.ncon[s / CPF]) {
            if constexpr (Cfg<NJ, TK>::SLABS) { if (!(w.xcd[s] > 0)) continue; }
            const real cz = w.o[2] + w.cpos[s][2];
            if (first || cz < z) z = cz;
            first = false;
            nfl++;
          }
        w.cz_min = z;
        w.nfloor = nfl;
      }
    }
    // rhs of the implicit-damping solve: qfrc_smooth + J' f = M a - grad
    if (l < NV) w.vec[l] = w.Ma[l] - w.grad[l];
    if (last) {
      // self-collision capsules: end points relative to o
      // lanes 22..31 take capsules 0..9 (the dof lanes are busy above), lanes 0..5 the rest
      const int c = l >= 22 ? l - 22 : (l < MAXCAP - 10 ? l + 10 : MAXCAP);
      if (c < m.ncap) {
        const int lk = m.cap_link[c];
        real* E = w.capE[c];
        real t[3];
        mv3(w.xmat[lk], m.cap_p0[c], t);
#pragma unroll
        for (int x = 0; x < 3; x++) E[x] = w.xr[lk][x] + t[x];
        mv3(w.xmat[lk], m.cap_p1[c], t);
#pragma unroll
        for (int x = 0; x < 3; x++) E[3 + x] = w.xr[lk][x] + t[x];
      }
      if (l == 31) w.selfcol = 0;
    }
  }
  LHW_SYNC();
  if (last && m.npair > 0) {
    LHW_LANES(l) {
      for (int pi = l; pi < m.npair; pi += 32) {
        const int a = m.pair_a[pi], b = m.pair_b[pi];
        const real* Ea = w.capE[a];
        const real* Eb = w.capE[b];
        const real rr = m.cap_r[a] + m.cap_r[b];
        if (seg_seg_dist2(Ea, Ea + 3, Eb, Eb + 3) < rr * rr) w.selfcol = 1;
      }
    }
    LHW_SYNC();
  }
  // ---------------- P12 mj_Euler: (M + h diag(damping)) a' = qfrc_smooth + qfrc_constraint ; integrate
  if ((PERENV || m.any_damping) && !m.explicit_euler) {
    LHW_LANES(l) {
      constexpr int NW = (int)(sizeof(Arrow<real, NJ, TK>) / sizeof(real));
      const real* src = &w.M.r[0][0];
      real* dst = &w.H.r[0][0];
      for (int it = l; it < NW; it += 32) dst[it] = src[it];
    }
    LHW_SYNC();
    LHW_LANES(l) {
      if (l < 6) w.H.r[l][l] += m.h * LHW_GLD(m, damping[l]);
      else if (l < NV) {
        const int ch = (l - 6) / NJ, k = l - 6 - ch * NJ;
        if constexpr (PERENV) w.H.c[ch][k][k] += m.h * w.p_damping[l - 6];
        else w.H.c[ch][k][k] += m.h * LHW_GLD(m, damping[l]);
      }
    }
    LHW_SYNC();
    arrow_factor_solve<real, NJ, TK>(w, w.vec);
  } else {
    LHW_LANES(l) {
      if (l < NV) w.vec[l] = w.qacc[l];
    }
    LHW_SYNC();
  }
  LHW_LANES(l) {
    if (l < NV) {
      const real a = w.vec[l];
      if (!(m_abs(a) < (real)1e10)) w.status |= 1;
      w.vec[l] = w.qacc_warm[l];   // a_{k-1} for the next substep's warm start (vec is free until P11)
      w.qacc_warm[l] = w.qacc[l];
      w.qvel[l] += m.h * a;
    }
  }
  LHW_SYNC();
  LHW_LANES(l) {
    if (l < 3) w.qpos[l] += m.h * w.qvel[l];
    else if (l == 3) {
      real* q = w.qpos + 3;
      real n = m_rsqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      real q0 = q[0] * n, q1 = q[1] * n, q2 = q[2] * n, q3 = q[3] * n;
      const real* wv = w.qvel + 3;
      const real wn = m_sqrt(wv[0] * wv[0] + wv[1] * wv[1] + wv[2] * wv[2]);
      if (wn > (real)1e-15) {
        real sa, ca;
        m_sincos((real)0.5 * m.h * wn, &sa, &ca);
        sa /= wn;
        const real r0 = ca, r1 = wv[0] * sa, r2 = wv[1] * sa, r3 = wv[2] * sa;
        const real o0 = q0 * r0 - q1 * r1 - q2 * r2 - q3 * r3, o1 = q0 * r1 + q1 * r0 + q2 * r3 - q3 * r2;
        const real o2 = q0 * r2 - q1 * r3 + q2 * r0 + q3 * r1, o3 = q0 * r3 + q1 * r2 - q2 * r1 + q3 * r0;
        n = m_rsqrt(o0 * o0 + o1 * o1 + o2 * o2 + o3 * o3);
        q0 = o0 * n; q1 = o1 * n; q2 = o2 * n; q3 = o3 * n;
      }
      q[0] = q0; q[1] = q1; q[2] = q2; q[3] = q3;
    } else if (l >= 4 && l < 4 + NU) {
      w.qpos[7 + l - 4] += m.h * w.qvel[6 + l - 4];
    }
  }
  LHW_SYNC();
}

// cos / sin of the slab yaws (stepping stones), once per launch and after every task reset
template <class real, int NJ, int TK> LHW_DEV void slab_frames(Work<real, NJ, TK>& w) {
  if constexpr (Cfg<NJ, TK>::SLABS) {
    LHW_LANES(l) {
      if (l < NSLAB) m_sincos(w.seq[l][3], &w.slab_cs[l][1], &w.slab_cs[l][0]);
    }
    LHW_SYNC();
  }
}

// ================================================================= environment level (one control step)
// state record I/O: reals [qpos qvel qacc_warm act_len act_vel prev_pred prev_action prev_torque mode_ref ep_rew],
// ints [phase mode traj_len ep_len rng_ctr have_prev status pad]; env-major, one coalesced stream per warp
template <class real, int NJ, int TK>
LHW_DEV void load_state(Work<real, NJ, TK>& w, const real* sr, const int32_t* si, uint32_t env_id) {
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R;
  real* dst = w.qpos;  // persistent block is contiguous in Work, same order as the record
  LHW_LANES(l) {
    for (int it = l; it < NR; it += 32) dst[it] = sr[it];
    if (l == 0) {
      w.phase = si[0]; w.mode = si[1]; w.traj_len = si[2]; w.ep_len = si[3];
      if constexpr (!Cfg<NJ, TK>::STAND && !Cfg<NJ, TK>::STEP) {
        w.hold = (si[1] & MODE_HELD) != 0;
        w.mode = si[1] & ~MODE_HELD;
      }
      w.rng_ctr = (uint32_t)si[4]; w.have_prev = si[5]; w.status = si[6];
      w.env_id = env_id;
      w.iters_total = 0;
      w.selfcol = 0;
    }
  }
  LHW_SYNC();
  slab_frames<real, NJ, TK>(w);
}
template <class real, int NJ, int TK> LHW_DEV void store_state(const Work<real, NJ, TK>& w, real* sr, int32_t* si) {
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R;
  const real* src = w.qpos;
  LHW_LANES(l) {
    for (int it = l; it < NR; it += 32) sr[it] = src[it];
    if (l == 0) {
      int32_t mode_word = w.mode;
      if constexpr (!Cfg<NJ, TK>::STAND && !Cfg<NJ, TK>::STEP) mode_word |= w.hold ? MODE_HELD : 0;
      si[0] = w.phase; si[1] = mode_word; si[2] = w.traj_len; si[3] = w.ep_len;
      si[4] = (int32_t)w.rng_ctr; si[5] = w.have_prev; si[6] = w.status; si[7] = w.iters_total;
    }
  }
  LHW_SYNC();
}

// WalkModes.sample_ref (tasks/walking_task.py:33-40)
template <class real, int NJ, int TK> LHW_DEV void sample_ref(Work<real, NJ, TK>& w, uint32_t seed, uint32_t stream) {
  uint32_t u[4];
  philox(seed, w.env_id, w.rng_ctr, stream, u);
  if (w.mode == STANDING) {
    for (int x = 0; x < 3; x++) w.mode_ref[x] = (real)-1 + (real)2 * u01<real>(u[x]);
  } else if (w.mode == INPLACE) {
    w.mode_ref[0] = (real)-0.5 + u01<real>(u[0]); w.mode_ref[1] = 0; w.mode_ref[2] = 0;
  } else {
    w.mode_ref[0] = 0; w.mode_ref[1] = (real)0.4 * u01<real>(u[0]); w.mode_ref[2] = 0;
  }
}

// observation (envs/jvrc/jvrc_base.py:133-145 + jvrc_walk.py:65-67): current qpos quat / qvel, LAGGED actuator state
template <class real, int NJ, int TK> LHW_DEV void env_obs(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed) {
  (void)seed;
  constexpr int NU = 2 * NJ, NROBOT = Dims<real, NJ, TK>::NROBOT;
  LHW_LANES(l) {
    if (l == 0) {  // transforms3d quat2euler (sxyz) roll, pitch via quat2mat
      const real qw = w.qpos[3], x = w.qpos[4], y = w.qpos[5], z = w.qpos[6];
      const real s = (real)2 / (qw * qw + x * x + y * y + z * z);
      const real X = x * s, Y = y * s, Z = z * s;
      const real wX = qw * X, wY = qw * Y, wZ = qw * Z, xX = x * X, xY = x * Y, xZ = x * Z, yY = y * Y, yZ = y * Z;
      const real M00 = 1 - (yY + z * Z), M10 = xY + wZ, M20 = xZ - wY, M21 = yZ + wX, M22 = 1 - (xX + yY);
      const real cy = m_sqrt(M00 * M00 + M10 * M10);
      if (cy > (real)(4 * 2.220446049250313e-16)) {
        w.obs[0] = m_atan2(M21, M22);
      } else {
        w.obs[0] = m_atan2(-(yZ - wX), 1 - (xX + z * Z));
      }
      w.obs[1] = m_atan2(-M20, cy);
    } else if (l < 4) {
      w.obs[1 + l] = w.qvel[2 + l];
    } else if (!Cfg<NJ, TK>::STAND && l == 4) {
      real sn, cs;
      m_sincos((real)(2 * M_PI) * w.phase / m.period, &sn, &cs);
      w.obs[NROBOT] = sn; w.obs[NROBOT + 1] = cs;
    } else if (Cfg<NJ, TK>::STEP && l == 5) {
      real* e = w.obs + NROBOT + 2;   // envs/jvrc/jvrc_step.py:67-76: goal steps x[2] y[2] z[2] theta[2]
#pragma unroll
      for (int i = 0; i < 8; i++) e[i] = w.goal[i];
    } else if (!Cfg<NJ, TK>::STAND && !Cfg<NJ, TK>::STEP && l == 5) {
      real* e = w.obs + NROBOT + 2;
      e[0] = w.mode == FORWARD; e[1] = w.mode == INPLACE; e[2] = w.mode == STANDING;
      e[3] = w.mode_ref[0]; e[4] = w.mode_ref[1]; e[5] = w.mode_ref[2];
    } else if (l >= 8 && l < 8 + NU) {
      w.obs[5 + l - 8] = w.act_len[l - 8];
      w.obs[5 + NU + l - 8] = w.act_vel[l - 8];
      if constexpr (Cfg<NJ, TK>::H1OBS) w.obs[5 + 2 * NU + l - 8] = w.act_force[l - 8];   // motor torques (h1_base.py:97)
    }
  }
  LHW_SYNC();
  if constexpr (Cfg<NJ, TK>::H1OBS) {
    // uniform observation noise (base_humanoid_env.py:311-338) on the robot state: value i -> philox stream 40 + i/4, lane i%4.
    // The task's words after it (gait clock, mode, reference) are exact.
    LHW_LANES(l) {
      for (int i = l; i < NROBOT; i += 32) {
        const real sc = i < 2 ? m.obs_noise[0] : i < 5 ? m.obs_noise[1] : i < 5 + NU ? m.obs_noise[2]
                        : i < 5 + 2 * NU ? m.obs_noise[3] : m.obs_noise[4];
        if (sc > 0) {
          uint32_t u[4];
          philox(seed, w.env_id, w.rng_ctr, 40 + (i >> 2), u);
          w.obs[i] += -sc + 2 * sc * u01<real>(u[i & 3]);
        }
      }
    }
    LHW_SYNC();
  }
}

// randomize_dynamics (envs/common/domain_randomization.py:29-56) on counter-based streams: joint j -> stream 16 + j/2,
// lanes 2(j%2) (frictionloss U(0,2)) and 2(j%2)+1 (damping U(0.02,2)); body b (pelvis, then the leg links) -> stream 21+b,
// lane 0 mass scale U(0.95,1.05), lanes 1..3 ipos offset U(-0.01,0.01).  body_inertia is left alone, as in the reference.
template <class real, int NJ, int TK> LHW_DEV void env_randomize(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed) {
  if constexpr (Cfg<NJ, TK>::PERENV) {
    constexpr int NU = 2 * NJ;
    LHW_LANES(l) {
      if (l < NU) {
        uint32_t u[4];
        philox(seed, w.env_id, w.rng_ctr, 16 + (l >> 1), u);
        w.p_floss[l] = (real)2 * u01<real>(u[2 * (l & 1)]);
        w.p_damping[l] = (real)0.02 + (real)1.98 * u01<real>(u[2 * (l & 1) + 1]);
      } else if (l >= 16 && l <= 16 + NU) {
        const int b = l - 16;
        uint32_t u[4];
        philox(seed, w.env_id, w.rng_ctr, 21 + b, u);
        const real sc = (real)0.95 + (real)0.1 * u01<real>(u[0]);
        if (b == 0) {
          // root link = pelvis body (+) welded rest: composite mass, com, inertia about the com
          real cp[3];
#pragma unroll
          for (int x = 0; x < 3; x++) { cp[x] = m.pel_com[x] + ((real)-0.01 + (real)0.02 * u01<real>(u[1 + x])); w.p_pelcom[x] = cp[x]; }
          const real mp = m.pel_mass * sc, M = mp + m.rest_mass;
          real c[3];
#pragma unroll
          for (int x = 0; x < 3; x++) c[x] = (mp * cp[x] + m.rest_mc[x]) / M;
          const real cp2 = dot3(cp, cp), c2 = dot3(c, c);
          const int ra[6] = {0, 1, 2, 0, 0, 1}, rb[6] = {0, 1, 2, 1, 2, 2};
#pragma unroll
          for (int e = 0; e < 6; e++) {
            const int a = ra[e], bb = rb[e];
            const real Io = m.pel_Ic[e] + mp * ((a == bb ? cp2 : (real)0) - cp[a] * cp[bb]) + m.rest_Io[e];
            w.p_inertia0[e] = Io - M * ((a == bb ? c2 : (real)0) - c[a] * c[bb]);
          }
          w.p_mass[0] = M;
#pragma unroll
          for (int x = 0; x < 3; x++) w.p_com[0][x] = c[x];
        } else {
          w.p_mass[b] = m.mass[b] * sc;
#pragma unroll
          for (int x = 0; x < 3; x++) w.p_com[b][x] = m.com[b][x] + ((real)-0.01 + (real)0.02 * u01<real>(u[1 + x]));
        }
      }
    }
    LHW_SYNC();
  }
}

// apply_perturbation (domain_randomization.py:10-26): per body force U(-F,F)^3, torque U(-T,T)^3, then a coin that clears
// the WHOLE xfrc_applied array.  body b -> streams 32+2b (force, lane 3 = coin) and 33+2b (torque)
template <class real, int NJ, int TK> LHW_DEV void env_perturb(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed) {
  if constexpr (Cfg<NJ, TK>::PERENV) {
    LHW_LANES(l) {
      if (l == 0) {
#pragma unroll 1
        for (int b = 0; b < 2; b++) {
          uint32_t uf[4], ut[4];
          philox(seed, w.env_id, w.rng_ctr, 32 + 2 * b, uf);
          philox(seed, w.env_id, w.rng_ctr, 33 + 2 * b, ut);
          for (int x = 0; x < 3; x++) {
            w.xfrc[b][x] = -m.perturb_force + 2 * m.perturb_force * u01<real>(uf[x]);
            w.xfrc[b][3 + x] = -m.perturb_torque + 2 * m.perturb_torque * u01<real>(ut[x]);
          }
          if (randint(uf[3], 2) == 0)
            for (int x = 0; x < 12; x++) (&w.xfrc[0][0])[x] = 0;
        }
      }
    }
    LHW_SYNC();
  }
}

// ---------------- SteppingTask (tasks/stepping_task.py), run by lane 0
// update_target_steps (:207-213)
template <class real, int NJ, int TK> LHW_DEV void step_update_targets(Work<real, NJ, TK>& w) {
  w.tk[1] = w.tk[2];
  w.tk[2] += 1;
  if (w.tk[2] == w.tk[0]) w.tk[2] = w.tk[0] - 1;
}
// update_goal_steps (:188-205): targets t1, t2 in the root frame, R' (p - root_pos) and the yaw of R' Rz(theta)
template <class real, int NJ, int TK> LHW_DEV void step_update_goals(Work<real, NJ, TK>& w) {
#pragma unroll
  for (int i = 0; i < 8; i++) w.goal[i] = 0;
  if (w.mode == ST_STANDING) return;
  const real* R = w.xmat[0];
#pragma unroll 1
  for (int idx = 0; idx < 2; idx++) {
    const int t = (int)w.tk[1 + idx];
    const real* sq = w.seq[t];
    const real d0 = sq[0] - w.o[0], d1 = sq[1] - w.o[1], d2 = sq[2] - w.o[2];
    w.goal[0 + idx] = R[0] * d0 + R[3] * d1 + R[6] * d2;
    w.goal[2 + idx] = R[1] * d0 + R[4] * d1 + R[7] * d2;
    w.goal[4 + idx] = R[2] * d0 + R[5] * d1 + R[8] * d2;
    const real c = w.slab_cs[t][0], sn = w.slab_cs[t][1];
    const real r00 = R[0] * c + R[3] * sn, r10 = R[1] * c + R[4] * sn;
    const real cy = m_sqrt(r00 * r00 + r10 * r10);
    w.goal[6 + idx] = cy > (real)(4 * 2.220446049250313e-16) ? m_atan2(r10, r00) : (real)0;
  }
}
// a chosen footstep plan (lhw_sim_reset_footsteps, DESIGN.md §7.7): mode is an ST_* value and value the FORWARD signed stair
// height (m), the LATERAL side c (+1 = the robot's left), the CURVED plan index (-1: drawn) or 0.  It replaces only the draws that
// pick the plan; every other draw of the reset is the plain reset's
template <class real> struct StepPlan { int mode; real value; };

// the stair curriculum (lhw_sim_step_stairs / lhw_sim_reset_stairs, DESIGN.md §7.8): env i has a level L in [0, n_levels), and its
// FORWARD plans climb or descend stairs of 0.01 L m.  Levels outside the range are clamped on read
enum { STAIR_MAX_LEVELS = 21 };   // 0 .. 0.2 m = 2 slab_half[2], the largest stair a chosen plan may have (lhw_sim_footstep_limits)
LHW_DEV int stair_level_clamp(int level, int n_levels) { return level < 0 ? 0 : level >= n_levels ? n_levels - 1 : level; }
// the magnitude lhw_sim_set_step_height(0.01 L) would store
template <class real> LHW_DEV real stair_level_height(int level) { return (real)(0.01 * level); }
// the level after an ended FORWARD episode that reached target `reached` of a sequence of `seq_len`: up one if it did not fall and
// reached half the sequence, down one if it fell short of half, else unchanged
template <class real> LHW_DEV int stair_level_next(int level, int n_levels, int fell, real reached, real seq_len) {
  const bool far = 2 * reached >= seq_len;
  if (!fell && far) return level + 1 < n_levels ? level + 1 : n_levels - 1;
  if (fell && !far) return level > 0 ? level - 1 : 0;
  return level;
}

// SteppingTask.reset (:243-334); draws: stream 3 lane 0 mode, lane 1 phase, lane 2 first-step offset / plan index / lateral
// sign, lane 3 randint(2,4); stream 4 lane 0 sign of the step height.  PLAN: the plan is `plan`'s, not drawn.  STAIRS: a FORWARD
// plan's stair magnitude is `stair` (the env's curriculum level), not the sim-wide m.step_height; its sign is still drawn
template <class real, int NJ, int TK, bool PLAN = false, bool STAIRS = false>
LHW_DEV void step_task_reset(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed, StepPlan<real> plan = {},
                             real stair = 0) {
  uint32_t u[4], v[4];
  philox(seed, w.env_id, w.rng_ctr, 3, u);
  philox(seed, w.env_id, w.rng_ctr, 4, v);
  w.tk[3] = 0; w.tk[4] = 0; w.tk[1] = 0; w.tk[2] = 0;
  w.phase = randint(u[1], 2) == 0 ? 0 : m.period / 2;
  const real cm = u01<real>(u[0]);
  w.mode = cm < (real)0.15 ? ST_CURVED : cm < (real)(0.15 + 0.05) ? ST_STANDING : cm < (real)(0.15 + 0.05 + 0.2) ? ST_BACKWARD
           : cm < (real)(0.15 + 0.05 + 0.2 + 0.3) ? ST_LATERAL : ST_FORWARD;
  if constexpr (PLAN) w.mode = plan.mode;
  real step_size = (real)0.3, step_height = 0;
  const real step_gap = (real)0.15;
  int num_steps = NSLAB;
  if (w.mode == ST_STANDING) num_steps = 1;
  else if (w.mode == ST_BACKWARD) step_size = (real)-0.1;
  else if (w.mode == ST_LATERAL) step_size = (real)0.4;
  else if (w.mode == ST_FORWARD) {
    if constexpr (PLAN) step_height = plan.value;
    else if constexpr (STAIRS) step_height = randint(v[0], 2) == 0 ? -stair : stair;
    else step_height = randint(v[0], 2) == 0 ? -m.step_height : m.step_height;
  }
  // transform_sequence (:123-136): about the mid-point of the foot bodies, yawed with the root
  const real* R = w.xmat[0];
  const real cyn = m_sqrt(R[0] * R[0] + R[3] * R[3]);
  const real yaw = cyn > (real)(4 * 2.220446049250313e-16) ? m_atan2(R[3], R[0]) : (real)0;
  real sy, cyw;
  m_sincos(yaw, &sy, &cyw);
  const real mid0 = w.o[0] + (w.xr[2 * NJ][0] + w.xr[NJ][0]) / 2, mid1 = w.o[1] + (w.xr[2 * NJ][1] + w.xr[NJ][1]) / 2;
  int n = 0;
  auto put = [&](real x, real y, real z, real th) {
    w.seq[n][0] = mid0 + x * cyw - y * sy;
    w.seq[n][1] = mid1 + x * sy + y * cyw;
    w.seq[n][2] = z;
    w.seq[n][3] = yaw + th;
    n++;
  };
  if (w.mode == ST_CURVED) {
    int k = randint(u[2], m.nplan);
    if constexpr (PLAN) { if (plan.value >= 0 && plan.value < (real)m.nplan) k = (int)plan.value; }   // else the drawn plan
    const real* pl = m.plans + (size_t)k * PLAN_STRIDE;
    const int len = (int)pl[0];
#pragma unroll 1
    for (int i = 0; i < len; i++) put(pl[1 + 3 * i], pl[2 + 3 * i], 0, pl[3 + 3 * i]);
  } else if (w.mode == ST_LATERAL) {
    real y = 0;
    real c = randint(u[2], 2) == 0 ? (real)-1 : (real)1;
    if constexpr (PLAN) c = plan.value;
#pragma unroll 1
    for (int i = 1; i < num_steps; i++) {
      if (i % 2) y += step_size; else y -= (real)(2.0 / 3.0) * step_size;
      put(0, c * y, 0, 0);
    }
  } else {
    const real first = (real)0.095 + (real)(0.105 - 0.095) * u01<real>(u[2]);
    real y;
    if (w.phase == m.period / 2 && 2 * (m.period / 2) == m.period) { put(0, -first, 0, 0); y = -step_gap; }
    else { put(0, first, 0, 0); y = step_gap; }
    real x = 0, z = 0;
    const int c = 2 + randint(u[3], 2);
#pragma unroll 1
    for (int i = 1; i < num_steps - 1; i++) {
      x += step_size;
      y *= -1;
      if (i > c) z += step_height;
      put(x, y, z, 0);
    }
    put(x + step_size, -y, z, 0);
  }
  w.tk[0] = (real)n;
  for (int i = n; i < NSLAB; i++) { w.seq[i][0] = 0; w.seq[i][1] = 0; w.seq[i][2] = -1; w.seq[i][3] = 0; }   // unused boxes (:322)
  step_update_targets<real, NJ, TK>(w);
#pragma unroll
  for (int i = 0; i < 8; i++) w.goal[i] = 0;
}

// terrain extension: re-pose the 20 terraces with the ranges of WalkingTask's manip_hfield hook (tasks/walking_task.py:
// 172-179).  Draws at the current event counter: stream 5 lanes 0..2 = x, y ~ U(-xy, xy), z offset ~ U(zlo, zhi); terrace k's
// bump ~ U(0, bump) = stream 60 + k/4 lane k%4.  Terrace k: centre (px + (k - 4) pitch, py), yaw 0, top at bump_k + zoff.
template <class real, int NJ, int TK>
LHW_DEV void terrain_repose(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed) {
  if constexpr (Cfg<NJ, TK>::TERRAIN) {
    uint32_t u[4], v[4];
    philox(seed, w.env_id, w.rng_ctr, 5, u);
    const real px = -m.terrain_xy + 2 * m.terrain_xy * u01<real>(u[0]), py = -m.terrain_xy + 2 * m.terrain_xy * u01<real>(u[1]);
    const real zo = m.terrain_zlo + (m.terrain_zhi - m.terrain_zlo) * u01<real>(u[2]);
#pragma unroll 1
    for (int k = 0; k < NSLAB; k++) {
      if ((k & 3) == 0) philox(seed, w.env_id, w.rng_ctr, 60 + (k >> 2), v);
      w.seq[k][0] = px + (k - 4) * m.terrain_pitch;
      w.seq[k][1] = py;
      w.seq[k][2] = m.terrain_bump * u01<real>(v[k & 3]) + zo;
      w.seq[k][3] = 0;
    }
    w.tk[0] = (real)NSLAB;
  }
}

// MujocoEnv.reset + BaseHumanoidEnv.reset_model + WalkingTask.reset.  PLAN (SteppingTask only): the footstep plan is `plan`.
// STAIRS (SteppingTask only): a FORWARD plan's stair magnitude is `stair`
template <class real, int NJ, int TK, bool PLAN = false, bool STAIRS = false>
LHW_DEV void env_reset(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, uint32_t seed, StepPlan<real> plan = {}, real stair = 0) {
  static_assert(!PLAN || Cfg<NJ, TK>::STEP, "a footstep plan is a SteppingTask reset");
  static_assert(!STAIRS || Cfg<NJ, TK>::STEP, "a stair curriculum is a SteppingTask reset");
  constexpr int NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ;
  LHW_LANES(l) {
    if (l == 0) w.rng_ctr++;
    if (l < NQ) w.qpos[l] = m.nominal[l];
    if (l < NV) { w.qvel[l] = 0; w.qacc_warm[l] = 0; }
    if (l < NU) { w.ctrl[l] = 0; w.prev_pred[l] = 0; }
    if constexpr (Cfg<NJ, TK>::PERENV) {
      if (l >= 20) (&w.xfrc[0][0])[l - 20] = 0;   // mj_resetData clears xfrc_applied
    }
    if constexpr (Cfg<NJ, TK>::SLABS) {
      // the settling steps below still see the PREVIOUS episode's slabs and floor (the reference edits the model in
      // task.reset, after them); a freshly built env has its boxes below the floor (gen_xml.py:149)
      if (l < NSLAB && w.tk[0] == 0) w.seq[l][2] = -1;
    }
  }
  LHW_SYNC();
  if constexpr (Cfg<NJ, TK>::PERENV) {
    if (m.dynrand_interval > 0) env_randomize<real, NJ, TK>(w, m, seed);   // base_humanoid_env.py:252-253
    else {
      // randomisation disabled: the per-env parameter block is just the nominal model
      LHW_LANES(l) {
        if (l < 1 + NU) {
          w.p_mass[l] = m.mass[l];
          for (int x = 0; x < 3; x++) w.p_com[l][x] = m.com[l][x];
        }
        if (l < NU) { w.p_damping[l] = m.damping[6 + l]; w.p_floss[l] = 0; }
        if (l < 6) w.p_inertia0[l] = m.inertia[0][l];
        if (l < 3) w.p_pelcom[l] = m.pel_com[l];
      }
      LHW_SYNC();
    }
    if (m.init_noise > 0) {
      // _apply_init_noise (base_humanoid_env.py:281-309): stream 50 lanes 0..2 = height, roll, pitch; joint j -> stream
      // 51 + j/4 lane j%4.  euler2quat(r, p, 0) 'sxyz' = (cp cr, cp sr, sp cr, -sp sr)
      const real c = m.init_noise;
      LHW_LANES(l) {
        if (l == 0) {
          uint32_t u[4];
          philox(seed, w.env_id, w.rng_ctr, 50, u);
          w.qpos[2] = m.nominal[2] + (real)0.02 * u01<real>(u[0]);
          const real r = -c + 2 * c * u01<real>(u[1]), p = -c + 2 * c * u01<real>(u[2]);
          real sr, cr, sp, cp;
          m_sincos((real)0.5 * r, &sr, &cr);
          m_sincos((real)0.5 * p, &sp, &cp);
          w.qpos[3] = cp * cr; w.qpos[4] = cp * sr; w.qpos[5] = sp * cr; w.qpos[6] = -sp * sr;
        } else if (l >= 8 && l < 8 + NU) {
          const int j = l - 8;
          uint32_t u[4];
          philox(seed, w.env_id, w.rng_ctr, 51 + (j >> 2), u);
          w.qpos[7 + j] = m.nominal[7 + j] + (-c + 2 * c * u01<real>(u[j & 3]));
        }
      }
      LHW_SYNC();
    }
  }
  for (int i = 0; i < 3; i++) substep<real, NJ, TK>(w, m, false);
  LHW_LANES(l) {
    if (l == 0) {
      if constexpr (Cfg<NJ, TK>::STEP) {
        step_task_reset<real, NJ, TK, PLAN, STAIRS>(w, m, seed, plan, stair);
      } else if constexpr (!Cfg<NJ, TK>::STAND) {
        uint32_t u[4];
        philox(seed, w.env_id, w.rng_ctr, 3, u);
        const real c = u01<real>(u[0]);
        w.mode = c < (real)0.6 ? STANDING : (c < (real)0.8 ? INPLACE : FORWARD);
        w.hold = 0;   // a held command lasts until the env's next reset
        sample_ref<real, NJ, TK>(w, seed, 4);
        w.phase = randint(u[1], m.period);
        if constexpr (Cfg<NJ, TK>::TERRAIN) {
          if (w.tk[0] == 0) terrain_repose<real, NJ, TK>(w, m, seed);   // first reset of a new env: the terrain's initial pose
        }
      }
      w.traj_len = 0; w.ep_len = 0; w.ep_rew = 0; w.status = 0;
    }
  }
  LHW_SYNC();
  slab_frames<real, NJ, TK>(w);
  env_obs<real, NJ, TK>(w, m, seed);
}

struct StepOut {
  void* obs; void* term_obs; void* reward; void* rew_terms;
  int32_t* done; int32_t* ended; int32_t* ep_len; void* ep_rew;
};

// the action delay (lhw_sim_step_delay, DESIGN.md §7.9): an env's delay in physics substeps, clamped to [0, frame_skip] where it
// is read
LHW_DEV int action_delay_clamp(int d, int frame_skip) { return d < 0 ? 0 : d > frame_skip ? frame_skip : d; }

// BaseHumanoidEnv.step + the RolloutWorker's bookkeeping (traj_len truncation, auto-reset, episode stats).  STAIRS (SteppingTask
// only, DESIGN.md §7.8): *level is the env's stair-curriculum level of n_levels; an auto-reset first moves it by the ending episode
// when that was a FORWARD one (stair_level_next), then resets with its stair height.  DELAY (DESIGN.md §7.9): substeps
// 0 .. delay-1 drive the PD loop towards the previous control step's target (prev_action, which holds it until the record update
// below), the rest towards this step's; delay is already clamped to [0, frame_skip].  At delay 0 the step is the plain one.
// PAYLOAD (DESIGN.md §7.10): every substep of the step builds the root link with the payload pay (root_payload); an auto-reset's
// settling substeps do not.  A payload of mass 0 is the plain step.  MOTOR (DESIGN.md §7.11): strength[0 .. NU-1] holds the env's
// per-joint motor strengths; the step's gains become kp_step[l] = s_l kp and kd_step[l] = s_l kd (kp, kd after the pdrand_k draw),
// so the dynamics, act_force, the torque rewards, prev_torque and H1's observed torques all see the scaled torque.  Read once
// per control step, here in the prologue; the substep loop is untouched.  Strength 1 is the plain step (kp 1 is exact)
template <class real, int NJ, int TK, bool STAIRS = false, bool DELAY = false, bool PAYLOAD = false, bool MOTOR = false>
LHW_DEV void env_step(Work<real, NJ, TK>& w, const Model<real, NJ, TK>& m, const real* action, uint32_t seed, int max_traj_len,
                      int autoreset, const int block_sync, const int alive, real* obs_out, real* term_obs_out, real* reward_out, real* rew_terms_out,
                      int32_t* done_out, int32_t* ended_out, int32_t* ep_len_out, real* ep_rew_out, int32_t* level = nullptr,
                      int n_levels = 0, const int delay = 0, const Payload<real> pay = {}, const real* strength = nullptr) {
  constexpr int NU = 2 * NJ, NOBS = Work<real, NJ, TK>::NOBS;
  // action smoothing + nominal offsets (base_humanoid_env.py:209-212, robot_base.py:80-85)
  // one event counter per control step: every draw of this step is keyed by rng_ctr + 1 (stored below)
  LHW_LANES(l) {
    if (l < NU) {
      const real t = m.smoothing * action[l] + (1 - m.smoothing) * w.prev_pred[l] + m.nominal[7 + l];
      w.target[l] = t;
      if (!w.have_prev) { w.prev_action[l] = t; w.prev_torque[l] = 0; }
      real kp = m.kp[l], kd = m.kd[l];
      if (m.pdrand_k > 0) {
        // RobotBase._do_simulation (robots/robot_base.py:41-47): joint u -> stream 8 + u/4 (kp) / 11 + u/4 (kd), lane u%4
        uint32_t u[4];
        philox(seed, w.env_id, w.rng_ctr + 1, 8 + (l >> 2), u);
        real lo = (1 - m.pdrand_k) * kp, hi = (1 + m.pdrand_k) * kp;
        kp = lo + (hi - lo) * u01<real>(u[l & 3]);
        philox(seed, w.env_id, w.rng_ctr + 1, 11 + (l >> 2), u);
        lo = (1 - m.pdrand_k) * kd; hi = (1 + m.pdrand_k) * kd;
        kd = lo + (hi - lo) * u01<real>(u[l & 3]);
      }
      if constexpr (MOTOR) {
        const real s = strength[l];
        kp = s * kp; kd = s * kd;
      }
      w.kp_step[l] = kp; w.kd_step[l] = kd;
    }
  }
  LHW_SYNC();
  for (int sidx = 0; sidx < m.frame_skip; sidx++) {
    LHW_LANES(l) {
      if constexpr (DELAY) {
        if (l < NU) {
          const real tg = sidx < delay ? w.prev_action[l] : w.target[l];
          w.ctrl[l] = w.kp_step[l] * (tg - w.act_len[l]) + w.kd_step[l] * ((real)0 - w.act_vel[l]);
        }
      } else {
        if (l < NU) w.ctrl[l] = w.kp_step[l] * (w.target[l] - w.act_len[l]) + w.kd_step[l] * ((real)0 - w.act_vel[l]);
      }
    }
    LHW_SYNC();
    if constexpr (PAYLOAD) {
      if (alive) substep<real, NJ, TK>(w, m, sidx == m.frame_skip - 1, block_sync, sidx > 0, pay);
      else LHW_BLOCK_SYNC(block_sync & 2);
    } else {
      if (alive) substep<real, NJ, TK>(w, m, sidx == m.frame_skip - 1, block_sync, sidx > 0);
      else LHW_BLOCK_SYNC(block_sync & 2);
    }
    LHW_BLOCK_SYNC((block_sync & 1) && ((sidx + 1) % ((block_sync >> 4) + 1) == 0));   // every (block_sync>>4)+1 substeps
  }
  if (!alive) return;
  // WalkingTask.step (tasks/walking_task.py:149-179)
  LHW_LANES(l) {
    if (l == 0) {
      w.have_prev = 1;
      w.rng_ctr++;
    }
    if (Cfg<NJ, TK>::STEP && l == 0) {
      if constexpr (Cfg<NJ, TK>::STEP) {
        // SteppingTask.step (tasks/stepping_task.py:215-243)
        w.phase += 1;
        if (w.phase >= m.period) w.phase = 0;
        const real* tp = w.seq[(int)w.tk[1]];
        bool in = false;
#pragma unroll
        for (int f = 0; f < 2; f++) {
          const real d0 = w.site[f][0] - tp[0], d1 = w.site[f][1] - tp[1], d2 = w.site[f][2] - tp[2];
          if (m_sqrt(d0 * d0 + d1 * d1 + d2 * d2) < m.target_radius) in = true;
        }
        if (in) { w.tk[3] = 1; w.tk[4] += 1; } else { w.tk[3] = 0; w.tk[4] = 0; }
        if (w.tk[3] != 0 && w.tk[4] >= (real)m.delay_frames) {
          step_update_targets<real, NJ, TK>(w);
          w.tk[3] = 0; w.tk[4] = 0;
        }
        step_update_goals<real, NJ, TK>(w);
      }
    }
    if (!Cfg<NJ, TK>::STAND && !Cfg<NJ, TK>::STEP && l == 0) {
      w.phase += 1;
      if (w.phase >= m.period) w.phase = 0;
      uint32_t u[4];
      philox(seed, w.env_id, w.rng_ctr, 0, u);
      const bool dbl = m.clock[0][w.phase] == (real)1 && m.clock[2][w.phase] == (real)1;
      // a held command (lhw_sim_set_command) skips both mode switches; the draws are counter-based, so nothing else moves
      if (!w.hold) {
        if (randint(u[0], 100) == 0 && dbl) {
          if (w.mode == INPLACE) w.mode = STANDING;
          else if (w.mode == STANDING) w.mode = INPLACE;
          sample_ref<real, NJ, TK>(w, seed, 1);
        }
        if (randint(u[1], 200) == 0 && w.mode != STANDING) {
          if (w.mode == FORWARD) w.mode = INPLACE;
          else if (w.mode == INPLACE) w.mode = FORWARD;
          sample_ref<real, NJ, TK>(w, seed, 2);
        }
      }
      if constexpr (Cfg<NJ, TK>::TERRAIN) {
        if (randint(u[2], m.terrain_interval) == 0 && w.mode != STANDING) terrain_repose<real, NJ, TK>(w, m, seed);
      }
    }
  }
  LHW_SYNC();
  if constexpr (Cfg<NJ, TK>::TERRAIN) slab_frames<real, NJ, TK>(w);
  // WalkingTask.calc_reward (tasks/walking_task.py:85-147, tasks/rewards.py), lane = term
  if constexpr (Cfg<NJ, TK>::STEP) {
    // SteppingTask.calc_reward (tasks/stepping_task.py:66-121), lane = term (6 terms, the rest 0)
    LHW_LANES(l) {
      if (l < NREW) {
        real rfc = m.clock[0][w.phase], rvc = m.clock[1][w.phase], lfc = m.clock[2][w.phase], lvc = m.clock[3][w.phase];
        if (w.mode == ST_STANDING) { rfc = lfc = 1; rvc = lvc = -1; }
        const real PI4 = (real)(M_PI / 4);
        const real* sq = w.seq[(int)w.tk[1]];
        real r = 0;
        if (l == 0) {
          const real nl = m_min(w.grf[1], m.fcap) / m.fcap * 2 - 1, nr = m_min(w.grf[0], m.fcap) / m.fcap * 2 - 1;
          r = (real)0.150 * ((m_tan(PI4 * lfc * nl) + m_tan(PI4 * rfc * nr)) / 2);
        } else if (l == 1) {
          const real lv = m_sqrt(dot3(w.foot_vel[1], w.foot_vel[1])), rv = m_sqrt(dot3(w.foot_vel[0], w.foot_vel[0]));
          const real vl = m_min(lv, (real)0.2) / (real)0.2 * 2 - 1, vr = m_min(rv, (real)0.2) / (real)0.2 * 2 - 1;
          r = (real)0.150 * ((m_tan(PI4 * lvc * vl) + m_tan(PI4 * rvc * vr)) / 2);
        } else if (l == 2) {
          real sh, ch;
          m_sincos((real)0.5 * sq[3], &sh, &ch);   // euler2quat(0, 0, th) = (cos th/2, 0, 0, sin th/2)
          const real inner = ch * w.rquat[0] + sh * w.rquat[3];
          r = (real)0.050 * m_exp(-10 * (1 - inner * inner));
        } else if (l == 3) {
          const real cz = w.nfloor > 0 ? w.cz_min : (real)0;
          real herr = m_abs(w.o[2] - cz - m.goal_height);
          if (herr < (real)0.01) herr = 0;
          r = (real)0.050 * m_exp(-40 * herr * herr);
        } else if (l == 4) {
          real dmin = (real)1e30;
#pragma unroll
          for (int f = 0; f < 2; f++) {
            const real d0 = w.site[f][0] - sq[0], d1 = w.site[f][1] - sq[1], d2 = w.site[f][2] - sq[2];
            dmin = m_min(dmin, m_sqrt(d0 * d0 + d1 * d1 + d2 * d2));
          }
          const real hit = w.tk[3] != 0 ? m_exp(-dmin / (real)0.25) : (real)0;
          const real* s2 = w.seq[(int)w.tk[2]];
          const real mx = (sq[0] + s2[0]) / 2 - w.o[0], my = (sq[1] + s2[1]) / 2 - w.o[1];
          const real progress = m_exp(-m_sqrt(mx * mx + my * my) / 2);
          r = (real)0.450 * ((real)0.8 * hit + (real)0.2 * progress);
        } else if (l == 5) {
          real hp[3];
          mv3(w.xmat[0], m.head, hp);
          r = (real)0.050 * m_exp(-10 * (hp[0] * hp[0] + hp[1] * hp[1]));
        }
        w.rew[l] = r;
      }
    }
  } else if constexpr (Cfg<NJ, TK>::STAND) {
    // StandingTask.calc_reward (tasks/standing_task.py:49-105), lane = term (6 terms, the rest 0)
    LHW_LANES(l) {
      if (l < NREW) {
        real r = 0;
        if (l == 0) {
          const real* R = w.xmat[0];
          const real* v = w.root_vlin;
          const real vx = R[0] * v[0] + R[3] * v[1] + R[6] * v[2], vy = R[1] * v[0] + R[4] * v[1] + R[7] * v[2];
          r = (real)0.3 * m_exp(-4 * (vx * vx + vy * vy));
        } else if (l == 1) {
          r = (real)0.3 * m_exp(-4 * w.qvel[5] * w.qvel[5]);
        } else if (l == 2) {
          const real he = w.o[2] - (real)0.98;
          r = (real)0.1 * m_exp((real)-0.5 * he * he);
        } else if (l == 3) {
          r = (real)0.1 * m_exp(-40 * (m.head[0] * m.head[0] + m.head[1] * m.head[1]));  // torso welded to the pelvis
        } else if (l == 4) {
          real te = 0;
          for (int u = 0; u < NU; u++) te += w.act_force[u] * w.act_force[u];
          r = (real)0.1 * m_exp((real)-5e-5 * te);
        } else if (l == 5) {
          real pe = 0;
          for (int u = 0; u < NU; u++) { const real d = w.act_len[u] - m.nominal[7 + u]; pe += d * d; }
          r = (real)0.1 * m_exp(-pe);
        }
        w.rew[l] = r;
      }
    }
  } else
  LHW_LANES(l) {
    if (l < NREW) {
      real rfc = m.clock[0][w.phase], rvc = m.clock[1][w.phase], lfc = m.clock[2][w.phase], lvc = m.clock[3][w.phase];
      real yaw_ref = w.mode_ref[0], vx = w.mode_ref[1], vy = w.mode_ref[2];
      if (w.mode == STANDING) { rfc = lfc = 1; rvc = lvc = -1; yaw_ref = vx = vy = 0; }
      else if (w.mode == INPLACE) { vx = vy = 0; }
      else { yaw_ref = 0; }
      const real PI4 = (real)(M_PI / 4);
      constexpr int RF = Cfg<NJ, TK>::RFOOT, LF = 1 - RF;
      real r = 0;
      if (l == 0) {
        const real nl = m_min(w.grf[LF], m.fcap) / m.fcap * 2 - 1, nr = m_min(w.grf[RF], m.fcap) / m.fcap * 2 - 1;
        r = (real)0.225 * ((m_tan(PI4 * lfc * nl) + m_tan(PI4 * rfc * nr)) / 2);
      } else if (l == 1) {
        const real lv = m_sqrt(dot3(w.foot_vel[LF], w.foot_vel[LF])), rv = m_sqrt(dot3(w.foot_vel[RF], w.foot_vel[RF]));
        const real vl = m_min(lv, (real)0.2) / (real)0.2 * 2 - 1, vr = m_min(rv, (real)0.2) / (real)0.2 * 2 - 1;
        r = (real)0.225 * ((m_tan(PI4 * lvc * vl) + m_tan(PI4 * rvc * vr)) / 2);
      } else if (l == 2) {
        real err = 0;
        for (int x = 0; x < 3; x++) err += m_abs(w.qvel[3 + x]);
        for (int x = 0; x < 3; x++) err += m_abs(w.qacc_lag[x]);
        r = (real)0.05 * m_exp((real)-0.25 * err);
      } else if (l == 3) {
        const real cz = w.nfloor > 0 ? w.cz_min : (real)0;
        real herr = m_abs(w.o[2] - cz - m.goal_height);
        if (herr < (real)0.01 + (real)0.05 * m_sqrt(vx * vx + vy * vy)) herr = 0;
        r = (real)0.05 * m_exp(-40 * herr * herr);
      } else if (l == 4) {
        const real* R = w.xmat[0];
        const real* v = w.root_vlin;
        const real ex = R[0] * v[0] + R[3] * v[1] + R[6] * v[2] - vx, ey = R[1] * v[0] + R[4] * v[1] + R[7] * v[2] - vy;
        r = (real)0.15 * m_exp(-10 * (ex * ex + ey * ey));
      } else if (l == 5) {
        const real ye = m_abs(w.qvel[5] - yaw_ref);
        r = (real)0.15 * m_exp(-10 * ye * ye * ye);
      } else if (l == 6) {
        real hp[3];
        mv3(w.xmat[0], m.head, hp);
        r = (real)0.05 * m_exp(-10 * m_sqrt(hp[0] * hp[0] + hp[1] * hp[1]));
      } else if (l == 7) {
        real pe = 0;
        for (int u = 0; u < NU; u++) { const real d = m.nominal[7 + u] - w.act_len[u]; pe += d * d; }
        r = (real)0.05 * m_exp(-m_sqrt(pe));
      } else if (l == 8) {
        real te = 0;
        for (int u = 0; u < NU; u++) te += m_abs(w.prev_torque[u] - w.act_force[u]);
        r = (real)0.025 * m_exp((real)-0.25 * (te / NU));
      } else {
        real ae = 0;
        for (int u = 0; u < NU; u++) ae += m_abs(w.prev_action[u] - w.target[u]);
        r = (real)0.025 * m_exp(-5 * ae / NU);
      }
      w.rew[l] = r;
    }
  }
  LHW_SYNC();
  env_obs<real, NJ, TK>(w, m, seed);
  real total = 0;
  for (int i = 0; i < NREW; i++) total += w.rew[i];
  // WalkingTask / StandingTask.done: current root height; SteppingTask.done (stepping_task.py:248-260): lagged root
  // height above the lower foot site
  const int done = Cfg<NJ, TK>::STEP
      ? ((w.o[2] - m_min(w.site[0][2], w.site[1][2]) < m.done_lo) || (w.selfcol != 0) || (w.status != 0))
      : ((w.qpos[2] < m.done_lo) || (w.qpos[2] > m.done_hi) || (w.selfcol != 0) || (w.status != 0));
  const int ended = done || (w.traj_len + 1 >= max_traj_len);
  LHW_SYNC();
  LHW_LANES(l) {
    if (l < NU) {
      w.prev_action[l] = w.target[l];
      w.prev_torque[l] = w.act_force[l];
      w.prev_pred[l] = action[l];
    }
    if (l == 12) { w.traj_len += 1; w.ep_len += 1; w.ep_rew += total; }
    if (l < NREW && rew_terms_out) rew_terms_out[l] = w.rew[l];
    if (l == 13) {
      reward_out[0] = total;
      done_out[0] = done;
      ended_out[0] = ended;
    }
    if (term_obs_out && (ended || !autoreset))
      for (int it = l; it < NOBS; it += 32) term_obs_out[it] = w.obs[it];
  }
  LHW_SYNC();
  if constexpr (Cfg<NJ, TK>::PERENV) {
    // domain randomisation after the observation (base_humanoid_env.py:228-233); decisions on stream 0 lanes 2, 3
    if (m.dynrand_interval > 0 || m.perturb_interval > 0) {
      uint32_t u[4];
      philox(seed, w.env_id, w.rng_ctr, 0, u);
      if (m.dynrand_interval > 0 && randint(u[2], m.dynrand_interval) == 0) env_randomize<real, NJ, TK>(w, m, seed);
      if (m.perturb_interval > 0 && randint(u[3], m.perturb_interval) == 0) env_perturb<real, NJ, TK>(w, m, seed);
    }
  }
  if (ended && autoreset) {
    real stair = 0;   // STAIRS: the next episode's stair magnitude (lane 0's, the lane that builds the plan)
    LHW_LANES(l) {
      if (l == 0) {
        if (ep_len_out) ep_len_out[0] = w.ep_len;
        if (ep_rew_out) ep_rew_out[0] = w.ep_rew;
        if constexpr (STAIRS) {
          int lv = stair_level_clamp(level[0], n_levels);
          if (w.mode == ST_FORWARD) {
            lv = stair_level_next<real>(lv, n_levels, done, w.tk[1], w.tk[0]);
            level[0] = lv;
          }
          stair = stair_level_height<real>(lv);
        }
      }
    }
    LHW_SYNC();
    env_reset<real, NJ, TK, false, STAIRS>(w, m, seed, {}, stair);
  }
  LHW_LANES(l) {
    for (int it = l; it < NOBS; it += 32) obs_out[it] = w.obs[it];
  }
  LHW_SYNC();
}

// ================================================================= evaluation statistics (lhw_sim_eval_accumulate, DESIGN.md §7.4)
// Per env, float64 words: episode length, return, ended-by-done flag, the NREW reward-term sums; per walking mode m
// (STANDING / INPLACE / FORWARD) at EV_TRACK + 4 m: steps in m and the sums of |v_fwd - vx_ref|, |v_lat - vy_ref|,
// |w_z - yaw_ref|; the SteppingTask's target index t1 (= footsteps reached) and sequence length at the last counted step.
// Words a variant has no use for stay 0.
enum { EV_LEN = 0, EV_RET = 1, EV_DONE = 2, EV_TERMS = 3, EV_TRACK = EV_TERMS + NREW, EV_REACHED = EV_TRACK + 12, EV_SEQLEN,
       EV_WORDS };

// The positions eval_accumulate_env reads in the state record: the persistent block of Work, which load_state / store_state
// copy in the order Persist [+ PersistStep] declares it, and the int record's mode word (load_state: w.mode = si[1] without
// MODE_HELD).
template <class real, int NJ, int TK> struct RecordAt {
  static constexpr int NV = 6 + 2 * NJ, NQ = NV + 1, NU = 2 * NJ;
  static constexpr int QPOS = 0, QVEL = NQ, MODE_REF = NQ + 2 * NV + 5 * NU, TK_WORDS = MODE_REF + 4 + 4 * NSLAB;
  static constexpr int I_MODE = 1;
  static_assert(sizeof(Persist<real, NJ, TK>) == sizeof(real) * (MODE_REF + 4) &&
                    sizeof(PersistStep<real, NJ, TK>) == sizeof(real) * (TK_WORDS + 5),
                "RecordAt must follow the persistent block of Work");
};

// The root's linear velocity in its own frame, (R^T v)[0:2] with v = qvel[0:3] (world) and R the rotation of the quaternion
// qpos[3:7] (normalised in the formula): v_fwd and v_lat of DESIGN.md §7.4, in float64 at either precision.
template <class real, int NJ, int TK> LHW_DEV void root_frame_velocity(const real* sr, double& vf, double& vl) {
  using A = RecordAt<real, NJ, TK>;
  const double qw = (double)sr[A::QPOS + 3], x = (double)sr[A::QPOS + 4], y = (double)sr[A::QPOS + 5], z = (double)sr[A::QPOS + 6];
  const double s = 2 / (qw * qw + x * x + y * y + z * z);
  const double X = x * s, Y = y * s, Z = z * s;
  const double wX = qw * X, wY = qw * Y, wZ = qw * Z, xX = x * X, xY = x * Y, xZ = x * Z, yY = y * Y, yZ = y * Z, zZ = z * Z;
  const double v0 = (double)sr[A::QVEL + 0], v1 = (double)sr[A::QVEL + 1], v2 = (double)sr[A::QVEL + 2];
  vf = (1 - (yY + zZ)) * v0 + (xY + wZ) * v1 + (xZ - wY) * v2;   // (R^T v)[0]
  vl = (xY - wZ) * v0 + (1 - (xX + zZ)) * v1 + (yZ + wX) * v2;   // (R^T v)[1]
}

// One control step of one env into its accumulator acc[EV_WORDS], from the step's outputs (reward, rew_terms[NREW], done) and
// the record it left (autoreset off).  An env counts the steps up to and including the first with done set; after that its
// EV_DONE word is 1 and it adds nothing.  The walking-task references are zeroed as the reward zeroes them; v is the
// record's qvel[0:3] in the root frame of qpos[3:7] and w_z is qvel[5] (the reward's root velocity lags these by one substep).
template <class real, int NJ, int TK>
LHW_DEV void eval_accumulate_env(const real* sr, const int32_t* si, real reward, const real* rew_terms, int32_t done, double* acc) {
  using A = RecordAt<real, NJ, TK>;
  if (acc[EV_DONE] != 0) return;
  acc[EV_LEN] += 1;
  acc[EV_RET] += (double)reward;
  for (int k = 0; k < NREW; k++) acc[EV_TERMS + k] += (double)rew_terms[k];
  if constexpr (Cfg<NJ, TK>::STEP) {
    acc[EV_REACHED] = (double)sr[A::TK_WORDS + 1];
    acc[EV_SEQLEN] = (double)sr[A::TK_WORDS + 0];
  } else {
    // the StandingTask holds zero references; a held WalkingTask mode carries MODE_HELD
    const int mode = Cfg<NJ, TK>::STAND ? (int)STANDING : si[A::I_MODE] & ~MODE_HELD;
    double yaw_ref = (double)sr[A::MODE_REF + 0], vx = (double)sr[A::MODE_REF + 1], vy = (double)sr[A::MODE_REF + 2];
    if (mode == STANDING) { yaw_ref = vx = vy = 0; }
    else if (mode == INPLACE) { vx = vy = 0; }
    else { yaw_ref = 0; }
    double vf, vl;
    root_frame_velocity<real, NJ, TK>(sr, vf, vl);
    double* t = acc + EV_TRACK + 4 * mode;
    t[0] += 1;
    t[1] += m_abs(vf - vx);
    t[2] += m_abs(vl - vy);
    t[3] += m_abs((double)sr[A::QVEL + 5] - yaw_ref);
  }
  if (done) acc[EV_DONE] = 1;
}

// ================================================================= root-velocity pushes (lhw_sim_push, DESIGN.md §7.5)
// legged_gym's push_robots: a horizontal velocity impulse on the root, qvel[0:2] (world frame) += Rz(psi) (dx, dy), with psi the
// heading (yaw) of qpos[3:7] and (dx, dy) in the heading frame (x forward, y to the robot's left).  Every link gets the same dv;
// joint velocities are unchanged.  Nothing else of the record is written, and nothing of an env that is not pushed.
// The random pushes draw on their own Philox stream at the env's event counter, which they only read.  The step and reset
// bodies above draw on streams 0-5, 8-13, 16-35, 40-48, 50-54 and 60-64, so with pushes off every trajectory is unchanged.
// The random action delays draw on stream 71 (DELAY_STREAM, delay_draw_env below), the random payloads on stream 72
// (PAYLOAD_STREAM, payload_draw_env below), the random motor strengths on streams 73-75 (MOTOR_STREAM, motor_draw_env below), the
// sensor errors on streams 80-84 (SENSOR_BIAS_STREAM), 96-104 (SENSOR_OBS_STREAM) and 112-120 (SENSOR_TERM_STREAM, sensor_env below).
constexpr uint32_t PUSH_STREAM = 70;

// One env's push; returns 1 when it was pushed.  Explicit mode (d != nullptr): (dx, dy) = (d[0], d[1]), skipped when both are
// exactly 0.  Random mode (d == nullptr): skipped when `ended` (the env was just reset); else pushed with probability 1/interval
// by u = philox(seed, env_id, rng_ctr, PUSH_STREAM): randint(u[0], interval) == 0, then (dx, dy) = vel (2 u01(u[1]) - 1,
// 2 u01(u[2]) - 1).  The arithmetic is float64 at either precision; the sum is rounded once to the record's precision.
template <class real, int NJ, int TK>
LHW_DEV int push_env(real* sr, const int32_t* si, uint32_t seed, uint32_t env_id, int32_t ended, double vel, int interval,
                     const real* d) {
  using A = RecordAt<real, NJ, TK>;
  double dx, dy;
  if (d) {
    if (d[0] == 0 && d[1] == 0) return 0;
    dx = (double)d[0];
    dy = (double)d[1];
  } else {
    if (ended) return 0;
    uint32_t u[4];
    philox(seed, env_id, (uint32_t)si[4], PUSH_STREAM, u);   // si[4]: rng_ctr (load_state)
    if (randint(u[0], interval) != 0) return 0;
    dx = vel * (2 * u01<double>(u[1]) - 1);
    dy = vel * (2 * u01<double>(u[2]) - 1);
  }
  // heading: the first column of the root's rotation matrix (the quaternion normalised as eval_accumulate_env does), projected on
  // the ground plane; (c, s) = (cos psi, sin psi)
  const double qw = (double)sr[A::QPOS + 3], x = (double)sr[A::QPOS + 4], y = (double)sr[A::QPOS + 5], z = (double)sr[A::QPOS + 6];
  const double q2 = 2 / (qw * qw + x * x + y * y + z * z);
  const double r00 = 1 - q2 * (y * y + z * z), r10 = q2 * (x * y + qw * z);
  const double h = m_sqrt(r00 * r00 + r10 * r10);
  const double c = h > 0 ? r00 / h : 1, s = h > 0 ? r10 / h : 0;
  sr[A::QVEL + 0] = (real)((double)sr[A::QVEL + 0] + (c * dx - s * dy));
  sr[A::QVEL + 1] = (real)((double)sr[A::QVEL + 1] + (s * dx + c * dy));
  return 1;
}

// ================================================================= random action delays (lhw_sim_draw_delay, DESIGN.md §7.9)
// An env that was just reset (sel != 0: its ended word or mask word) draws the delay of its new episode, d ~ U{0 .. max_delay}
// substeps: randint(u[0], max_delay + 1) with u = philox(seed, env_id, rng_ctr, DELAY_STREAM), at the event counter the reset left
// (si[4]; every reset increments it).  Only *delay is written.
constexpr uint32_t DELAY_STREAM = 71;

LHW_DEV void delay_draw_env(const int32_t* si, uint32_t seed, uint32_t env_id, int32_t sel, int max_delay, int32_t* delay) {
  if (!sel) return;
  uint32_t u[4];
  philox(seed, env_id, (uint32_t)si[4], DELAY_STREAM, u);
  *delay = randint(u[0], max_delay + 1);
}

// ================================================================= random payloads (lhw_sim_draw_payload, DESIGN.md §7.10)
// An env that was just reset (sel != 0: its ended word or mask word) draws the payload of its new episode: with
// u = philox(seed, env_id, rng_ctr, PAYLOAD_STREAM) at the event counter the reset left (si[4]), mass m = max_mass u01(u[0]) and
// offset r_k = max_offset (2 u01(u[1 + k]) - 1), so m ~ U(0, max_mass) and r ~ U(-max_offset, max_offset)^3.  The arithmetic is
// float64 at either precision, rounded once to the payload's precision.  Only pay[0..3] = (m, rx, ry, rz) is written.
constexpr uint32_t PAYLOAD_STREAM = 72;
constexpr double PAYLOAD_MAX_OFFSET = 0.25;   // m: the largest offset component of a payload

template <class real>
LHW_DEV void payload_draw_env(const int32_t* si, uint32_t seed, uint32_t env_id, int32_t sel, double max_mass, double max_offset,
                              real* pay) {
  if (!sel) return;
  uint32_t u[4];
  philox(seed, env_id, (uint32_t)si[4], PAYLOAD_STREAM, u);
  pay[0] = (real)(max_mass * u01<double>(u[0]));
#pragma unroll
  for (int k = 0; k < 3; k++) pay[1 + k] = (real)(max_offset * (2 * u01<double>(u[1 + k]) - 1));
}

// ================================================================= random motor strengths (lhw_sim_draw_motor, DESIGN.md §7.11)
// An env that was just reset (sel != 0: its ended word or mask word) draws the strengths of its new episode, one per actuated
// joint l < nu: s_l = 1 + max_dev (2 u01(u) - 1) with u = philox(seed, env_id, rng_ctr, MOTOR_STREAM + l/4), lane l % 4, at the
// event counter the reset left (si[4]), so s_l ~ U(1 - max_dev, 1 + max_dev).  The arithmetic is float64 at either precision,
// rounded once to the strength's precision; the product and the sum are rounded separately on the device too (no fused
// multiply-add), so the host body and numpy give the same bits.  Only out[0 .. nu-1] is written.
constexpr uint32_t MOTOR_STREAM = 73;

template <class real>
LHW_DEV void motor_draw_env(const int32_t* si, uint32_t seed, uint32_t env_id, int32_t sel, double max_dev, int nu, real* out) {
  if (!sel) return;
  for (int b = 0; 4 * b < nu; b++) {
    uint32_t u[4];
    philox(seed, env_id, (uint32_t)si[4], MOTOR_STREAM + (uint32_t)b, u);
    for (int k = 0; k < 4 && 4 * b + k < nu; k++) {
      const double dev = max_dev * (2 * u01<double>(u[k]) - 1);
#ifdef __CUDA_ARCH__
      out[4 * b + k] = (real)__dadd_rn(1.0, dev);
#else
      out[4 * b + k] = (real)(1.0 + dev);
#endif
    }
  }
}

// ================================================================= sensor errors (lhw_sim_sense, DESIGN.md §7.12)
// What the policy observes of the robot state, never what the step reads back: a pass over the observation rows after a step or a
// reset.  An env's row [6 + nu] holds its noise multiplier m >= 0, then one offset per calibrated word: roll, pitch (rad), gyro
// x, y, z (rad/s) and the nu motor positions (rad), i.e. obs word i < 5 + nu has offset row[1 + i]; velocity and torque words
// have none.  Word i < nrobot of an observation x becomes
//   x[i] = (real)((double)x[i] + b_i + (m s_g) (2 u01(u[i % 4]) - 1)),   u = philox(seed, env_id, rng_ctr, stream + i/4),
// s_g the noise scale of word i's group (SENSOR_SCALE, the reference's H1 observation_noise.scales), rng_ctr the record's event
// counter (si[4]).  Float64 at either precision, rounded once; the device rounds each product and sum on its own (no fused
// multiply-add), so the host body and numpy give the same bits.  A word with b_i == 0 and m s_g == 0 is not written, so an
// all-zero row leaves every bit of the observation, -0.0 included.  The task words after nrobot are never touched.
constexpr uint32_t SENSOR_BIAS_STREAM = 80, SENSOR_OBS_STREAM = 96, SENSOR_TERM_STREAM = 112;
// the noise scales s_g of the groups root_orient, root_ang_vel, motor_pos, motor_vel, motor_tau, for every robot (model/h1.json
// cfg.observation_noise.scales)
constexpr double SENSOR_SCALE_ORIENT = 0.05, SENSOR_SCALE_GYRO = 0.05, SENSOR_SCALE_POS = 0.02, SENSOR_SCALE_VEL = 0.05,
                 SENSOR_SCALE_TAU = 5.0;
// the largest noise multiplier, and the largest random (and explicit) roll / pitch, gyro and encoder offsets
constexpr double SENSOR_MAX_NOISE = 4, SENSOR_MAX_ORIENT = 0.2, SENSOR_MAX_GYRO = 0.5, SENSOR_MAX_ENCODER = 0.2;

LHW_DEV double sensor_fadd(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dadd_rn(a, b);
#else
  return a + b;
#endif
}

LHW_DEV double sensor_fmul(double a, double b) {
#ifdef __CUDA_ARCH__
  return __dmul_rn(a, b);
#else
  return a * b;
#endif
}

// Words 4g .. 4g+3 (< nrobot) of one observation x with the row, on Philox stream `stream` (+ g); see above.
template <class real>
LHW_DEV void sensor_apply(const real* row, uint32_t seed, uint32_t env_id, uint32_t ctr, uint32_t stream, int g, int nrobot, int nu,
                          real* x) {
  uint32_t u[4];
  philox(seed, env_id, ctr, stream + (uint32_t)g, u);
  const double m = (double)row[0];
#pragma unroll
  for (int k = 0; k < 4; k++) {
    const int i = 4 * g + k;
    const double b = i < 5 + nu ? (double)row[1 + i] : 0.0;
    const double a = sensor_fmul(m, i < 2 ? SENSOR_SCALE_ORIENT : i < 5 ? SENSOR_SCALE_GYRO : i < 5 + nu ? SENSOR_SCALE_POS
                                    : i < 5 + 2 * nu ? SENSOR_SCALE_VEL : SENSOR_SCALE_TAU);
    if (i < nrobot && (b != 0 || a != 0))
      x[i] = (real)sensor_fadd(sensor_fadd((double)x[i], b), sensor_fmul(a, 2 * u01<double>(u[k]) - 1));
  }
}

// One env's group g of four observation words (g < ceil(nrobot / 4)): everything the pass does to those words, so no two calls
// (threads) share a word and none needs another's result.  sel: the env's ended word after a step, its mask word (1 without a
// mask) after a reset.
//   after a step with autoreset, an ended env (sel != 0): term_obs gets the ending episode's row on SENSOR_TERM_STREAM; then, in
//     random mode (draw != 0), the new episode's offsets are drawn; then obs (the new episode's first observation) gets the
//     row on SENSOR_OBS_STREAM.  An env that did not end: obs only.
//   after a step without autoreset: obs, and term_obs (which the step wrote equal to obs) gets the same words, so both stay equal.
//   after a reset: a selected env draws (random mode) and its obs gets the row; an unselected env is not touched.
// The draw (draw != 0, random mode): offset word k (row[1 + k], k < 5 + nu, the ones of this group: k = 4g .. 4g+3) =
// (real)(r_k (2 u01(u[k % 4]) - 1)) with u = philox(seed, env_id, rng_ctr, SENSOR_BIAS_STREAM + k/4) and r_k = r_orient (roll,
// pitch), r_gyro (gyro) or r_enc (motor positions); row[0], the multiplier, is never written.  rng_ctr is si[4] as the step's auto-reset or the reset left it.
template <class real>
LHW_DEV void sensor_env(const int32_t* si, uint32_t seed, uint32_t env_id, int g, int32_t sel, int after_step, int autoreset,
                        int draw, double r_orient, double r_gyro, double r_enc, int nrobot, int nu, real* row, real* obs,
                        real* term_obs) {
  const uint32_t ctr = (uint32_t)si[4];
  if (!after_step && !sel) return;
  const bool new_episode = !after_step || (autoreset && sel);
  if (after_step && new_episode) sensor_apply<real>(row, seed, env_id, ctr, SENSOR_TERM_STREAM, g, nrobot, nu, term_obs);
  if (new_episode && draw) {
    uint32_t u[4];
    philox(seed, env_id, ctr, SENSOR_BIAS_STREAM + (uint32_t)g, u);
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int k = 4 * g + j;
      if (k < 5 + nu) row[1 + k] = (real)sensor_fmul(k < 2 ? r_orient : k < 5 ? r_gyro : r_enc, 2 * u01<double>(u[j]) - 1);
    }
  }
  sensor_apply<real>(row, seed, env_id, ctr, SENSOR_OBS_STREAM, g, nrobot, nu, obs);
  if (after_step && !autoreset)
#pragma unroll
    for (int k = 0; k < 4; k++)
      if (4 * g + k < nrobot) term_obs[4 * g + k] = obs[4 * g + k];
}

// ================================================================= held commands (lhw_sim_set_command, DESIGN.md §7.6)
// legged_gym's `play` command override for the WalkingTask variants.  A command sets the env's mode and reference and holds them:
// the step skips its two random mode switches while MODE_HELD is set, and env_reset clears it.  The body writes the mode word,
// mode_ref and the six task words of the observation (the FORWARD / INPLACE / STANDING one-hot, then mode_ref, as env_obs writes
// them), so the next action already sees the command; nothing else, and nothing of an env whose mode is not 0..2 (-1: untouched).
// ref = (yaw_rate, vx, vy), the record's order.  Returns 1 when the env was given the command.
template <class real, int NJ, int TK>
LHW_DEV int set_command_env(real* sr, int32_t* si, int32_t mode, const real* ref, real* obs) {
  static_assert(!Cfg<NJ, TK>::STAND && !Cfg<NJ, TK>::STEP, "only the WalkingTask variants take a velocity command");
  using A = RecordAt<real, NJ, TK>;
  if (mode < STANDING || mode > FORWARD) return 0;
  si[A::I_MODE] = mode | MODE_HELD;
  real* e = obs + Dims<real, NJ, TK>::NROBOT + 2;
  e[0] = mode == FORWARD; e[1] = mode == INPLACE; e[2] = mode == STANDING;
  for (int x = 0; x < 3; x++) sr[A::MODE_REF + x] = e[3 + x] = ref[x];
  return 1;
}

// The command sweep's signed velocities (lhw_sim_command_accumulate): per env, float64 words [steps, sum v_fwd, sum v_lat,
// sum w_z, ended-by-done], with v_fwd, v_lat and w_z as eval_accumulate_env defines them, over the same steps: up to and including
// the first with done set.
enum { CMD_LEN = 0, CMD_VF = 1, CMD_VL = 2, CMD_WZ = 3, CMD_DONE = 4, CMD_WORDS };

template <class real, int NJ, int TK> LHW_DEV void command_accumulate_env(const real* sr, int32_t done, double* acc) {
  using A = RecordAt<real, NJ, TK>;
  if (acc[CMD_DONE] != 0) return;
  double vf, vl;
  root_frame_velocity<real, NJ, TK>(sr, vf, vl);
  acc[CMD_LEN] += 1;
  acc[CMD_VF] += vf;
  acc[CMD_VL] += vl;
  acc[CMD_WZ] += (double)sr[A::QVEL + 5];
  if (done) acc[CMD_DONE] = 1;
}

}  // namespace lhw
