// sim_kernels.cu — sm_90a kernels + C-ABI for the batched environment (see include/lhw_b200.h).
//
// One environment per warp.  A warp streams its env's state record (env-major, contiguous -> coalesced
// 128 B lines) from HBM into its private slice of shared memory, runs frame_skip physics substeps + reward /
// observation / termination / auto-reset entirely on chip, and streams the record back: one HBM round trip
// per control step (SURVEY.md §8d: 1220 B algorithmic per env-step in fp32).  Inside an environment only __syncwarp()
// is used.  The shipped launch puts 8 (fp64) / 14 (fp32) environments in a block that meets at one __syncthreads() per
// physics substep: the warps then run the same region of a kernel that is far larger than the instruction cache
// (DESIGN.md §4.1, findings 2 and 6); LHW_WARPS_PER_BLOCK=1 gives the original one-warp blocks that never wait.
//
// Every kernel is instantiated for each robot / task variant of sim_core.h's LHW_FOR_EACH_VARIANT at both precisions.  A sim
// is one SimOf<real, NJ, TK>: lhw_sim_create picks it from the model's first word and precision (model_pack.h with_variant),
// and the other entry points call it through lhw_sim's virtual functions.
#include <cuda_runtime.h>
#include <stdio.h>

#include <atomic>
#include <climits>
#include <string>
#include <vector>

#include "../../include/lhw_b200.h"
#define LHW_BLOCK_SYNC(on) do { if (on) __syncthreads(); } while (0)
#include "model_pack.h"
#include "render_core.h"

using namespace lhw;

namespace {

// the constant-bank models, one per variant (sim_core.h LHW_FOR_EACH_VARIANT) and precision.  Named objects in this order:
// their bank offsets are compiled into the kernels' LDC instructions
constexpr int NJ_JVRC = 6;
__constant__ Model<double, 6, 0> c_model_d;
__constant__ Model<float, 6, 0> c_model_f;
__constant__ Model<double, 5, 0> c_model_d5;
__constant__ Model<float, 5, 0> c_model_f5;
__constant__ Model<double, 6, 1> c_model_ds;
__constant__ Model<float, 6, 1> c_model_fs;
__constant__ Model<double, 6, 2> c_model_dt;
__constant__ Model<float, 6, 2> c_model_ft;

// H1 walking (5, 3) has no objects of its own: with them the ten models would need 66 896 of the bank's 65 536 bytes.  Its Model has the
// layout of H1 standing's (5, 0) — the same NJ and foot points — so it borrows that variant's objects, and an h1 and an h1_walk
// sim take turns in them as two sims of one variant do.
template <int NJ, int TK> constexpr int bank_tk() { return NJ == 5 && TK == 3 ? 0 : TK; }
static_assert(sizeof(Model<double, 5, 3>) == sizeof(Model<double, 5, 0>) && sizeof(Model<float, 5, 3>) == sizeof(Model<float, 5, 0>) &&
              Cfg<5, 3>::NPTS == Cfg<5, 0>::NPTS, "h1_walk borrows h1's constant-bank objects: the Model layouts must agree");

// the variant's constant-bank object: the kernels read their model from it, SimOf::bind uploads to it
template <class real, int NJ, int TK> __host__ __device__ __forceinline__ const Model<real, NJ, TK>& cmodel() {
  constexpr bool D = sizeof(real) == 8;
  if constexpr (D && NJ == 6 && TK == 0) return c_model_d;
  if constexpr (!D && NJ == 6 && TK == 0) return c_model_f;
  if constexpr (D && NJ == 5 && TK == 0) return c_model_d5;
  if constexpr (!D && NJ == 5 && TK == 0) return c_model_f5;
  if constexpr (D && NJ == 6 && TK == 1) return c_model_ds;
  if constexpr (!D && NJ == 6 && TK == 1) return c_model_fs;
  if constexpr (D && NJ == 6 && TK == 2) return c_model_dt;
  if constexpr (!D && NJ == 6 && TK == 2) return c_model_ft;
  if constexpr (NJ == 5 && TK == 3) return reinterpret_cast<const Model<real, 5, 3>&>(cmodel<real, 5, 0>());
}

}  // namespace
// tell sim_core.h's out-of-line routines where the model really lives (constant bank -> LDC with immediate offsets)
namespace lhw {
template <int NJ, int TK> struct ModelHome<double, NJ, TK> {
  static __device__ __forceinline__ const Model<double, NJ, TK>& get(const Model<double, NJ, TK>&) { return cmodel<double, NJ, TK>(); }
};
template <int NJ, int TK> struct ModelHome<float, NJ, TK> {
  static __device__ __forceinline__ const Model<float, NJ, TK>& get(const Model<float, NJ, TK>&) { return cmodel<float, NJ, TK>(); }
};
}  // namespace lhw
namespace {

thread_local std::string g_err;
std::atomic<long long> g_launches{0};

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_OK(call)                                                                       \
  do {                                                                                      \
    cudaError_t _e = (call);                                                                \
    if (_e != cudaSuccess) return fail(-10, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// PLAN (jvrc_step only, lhw_sim_reset_footsteps): env i resets with the footstep plan (plan_mode[i], plan_value[i]); rows whose
// mode is not an ST_* value are skipped as masked-out rows are.  STAIRS (jvrc_step only, lhw_sim_reset_stairs): a FORWARD plan of
// env i has the stair magnitude of its curriculum level level[i] of n_levels
template <class real, int NJ, int TK, bool PLAN = false, bool STAIRS = false>
__global__ void __launch_bounds__(32) reset_kernel(real* __restrict__ state_r, int32_t* __restrict__ state_i, int n_envs,
                                                    uint32_t seed, uint32_t first_id, const int32_t* __restrict__ mask,
                                                    int fresh, real* __restrict__ obs_out,
                                                    const int32_t* __restrict__ plan_mode = nullptr,
                                                    const real* __restrict__ plan_value = nullptr,
                                                    const int32_t* __restrict__ level = nullptr, int n_levels = 0) {
  using W = Work<real, NJ, TK>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;
  const int env = blockIdx.x;
  if (env >= n_envs) return;
  if (mask && !mask[env]) return;
  StepPlan<real> plan = {};
  if constexpr (PLAN) {
    plan = {plan_mode[env], plan_value[env]};
    if (plan.mode < ST_CURVED || plan.mode > ST_FORWARD) return;
  }
  W& w = *reinterpret_cast<W*>(smem_raw);
  const Model<real, NJ, TK>& m = cmodel<real, NJ, TK>();
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R;
  real* sr = state_r + (size_t)env * NR;
  int32_t* si = state_i + (size_t)env * NSTATE_I;
  if (fresh) {
    for (int it = lane; it < NR; it += 32) sr[it] = 0;
    if (lane < NSTATE_I) si[lane] = 0;
    __syncwarp();
  }
  load_state<real, NJ, TK>(w, sr, si, first_id + env);
  real stair = 0;
  if constexpr (STAIRS) stair = stair_level_height<real>(stair_level_clamp(level[env], n_levels));
  env_reset<real, NJ, TK, PLAN, STAIRS>(w, m, seed, plan, stair);
  store_state<real, NJ, TK>(w, sr, si);
  if (obs_out)
    for (int it = lane; it < W::NOBS; it += 32) obs_out[(size_t)env * W::NOBS + it] = w.obs[it];
}

// ONE warp per block: the warp's Work struct then sits at a link-time-constant shared-memory address, so every
// access is [index + immediate] and no base register has to be kept (or rematerialised).  fp32: 28 blocks/SM (register
// bound: 28 x 132 = 3696 environments at once on an H100, so a 4096-env batch is two waves); fp64: 16 blocks/SM (shared-memory bound).
// STAIRS (jvrc_step only, lhw_sim_step_stairs): level [n_envs] holds the envs' stair-curriculum levels of n_levels, moved and used
// by the auto-resets (sim_core.h env_step).  DELAY (lhw_sim_step_delay): delay [n_envs] holds each env's action delay in substeps,
// read once into a register and clamped to [0, frame_skip].  PAYLOAD (lhw_sim_step_payload, instantiated with DELAY): payload
// [n_envs][4] holds each env's (m, rx, ry, rz), read once per control step; delay may then be null, which is delay 0.  MOTOR
// (lhw_sim_step_motor, instantiated with DELAY and PAYLOAD): strength [n_envs][NU] holds each env's per-joint motor strengths,
// read once per control step; delay and payload may then be null, which is delay 0 and mass 0
template <class real, int NJ, int TK, bool STAIRS = false, bool DELAY = false, bool PAYLOAD = false, bool MOTOR = false>
__global__ void __launch_bounds__(32, sizeof(real) == 4 ? (Cfg<NJ, TK>::SLABS ? 24 : 28) : (Cfg<NJ, TK>::SLABS ? 12 : (NJ == NJ_JVRC ? 16 : 15)))
    step_kernel(real* __restrict__ state_r, int32_t* __restrict__ state_i, int n_envs, uint32_t seed, uint32_t first_id,
                const real* __restrict__ actions, int max_traj_len, int autoreset, real* __restrict__ obs,
                real* __restrict__ term_obs, real* __restrict__ reward, real* __restrict__ rew_terms,
                int32_t* __restrict__ done, int32_t* __restrict__ ended, int32_t* __restrict__ ep_len,
                real* __restrict__ ep_rew, int32_t* __restrict__ level = nullptr, int n_levels = 0,
                const int32_t* __restrict__ delay = nullptr, const real* __restrict__ payload = nullptr,
                const real* __restrict__ strength = nullptr) {
  using W = Work<real, NJ, TK>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int env = blockIdx.x;
  if (env >= n_envs) return;
  W& w = *reinterpret_cast<W*>(smem_raw);
  const Model<real, NJ, TK>& m = cmodel<real, NJ, TK>();
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NU = 2 * NJ;
  real* sr = state_r + (size_t)env * NR;
  int32_t* si = state_i + (size_t)env * NSTATE_I;
  load_state<real, NJ, TK>(w, sr, si, first_id + env);
  const int d = DELAY && (!PAYLOAD || delay) ? action_delay_clamp(delay[env], m.frame_skip) : 0;
  Payload<real> pl = {};
  if constexpr (PAYLOAD) {
    if (!MOTOR || payload) pl = {payload[4 * (size_t)env], {payload[4 * (size_t)env + 1], payload[4 * (size_t)env + 2], payload[4 * (size_t)env + 3]}};
  }
  env_step<real, NJ, TK, STAIRS, DELAY, PAYLOAD, MOTOR>(w, m, actions + (size_t)env * NU, seed, max_traj_len, autoreset, 0, 1, obs + (size_t)env * W::NOBS,
                     term_obs ? term_obs + (size_t)env * W::NOBS : nullptr, reward + env,
                     rew_terms ? rew_terms + (size_t)env * NREW : nullptr, done + env, ended + env,
                     ep_len ? ep_len + env : nullptr, ep_rew ? ep_rew + env : nullptr, STAIRS ? level + env : nullptr, n_levels, d, pl,
                     MOTOR ? strength + (size_t)env * NU : nullptr);
  store_state<real, NJ, TK>(w, sr, si);
}

// the shipped carving: W warps per block (one env each), a __syncthreads() per substep so the warps of an SM share
// instruction-cache fills (far fewer no-instruction stalls); W from LHW_WARPS_PER_BLOCK or the defaults below.  STAIRS, DELAY,
// PAYLOAD, MOTOR: as step_kernel
template <class real, int NJ, int TK, bool STAIRS = false, bool DELAY = false, bool PAYLOAD = false, bool MOTOR = false>
// LHW_X_REGCAP (candidate, tools/ab_variants.py): the register budget of the fp64 lock-step kernel as "threads per SM" — 512 = 127
// registers (16 warps per SM, the shipped kernel), 576 = 112 (18 warps), 640 = 96 (20 warps)
#ifndef LHW_X_REGCAP
#define LHW_X_REGCAP 512
#endif
__global__ void __launch_bounds__(sizeof(real) == 8 ? LHW_X_REGCAP : 896, 1)
    step_kernel_mw(real* __restrict__ state_r, int32_t* __restrict__ state_i, int n_envs, uint32_t seed, uint32_t first_id,
                   const real* __restrict__ actions, int max_traj_len, int autoreset, real* __restrict__ obs,
                   real* __restrict__ term_obs, real* __restrict__ reward, real* __restrict__ rew_terms,
                   int32_t* __restrict__ done, int32_t* __restrict__ ended, int32_t* __restrict__ ep_len,
                   real* __restrict__ ep_rew, int sync_mode, int32_t* __restrict__ level = nullptr, int n_levels = 0,
                   const int32_t* __restrict__ delay = nullptr, const real* __restrict__ payload = nullptr,
                   const real* __restrict__ strength = nullptr) {
  using W = Work<real, NJ, TK>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5;
  const int env = blockIdx.x * (blockDim.x >> 5) + warp;
  const int alive = env < n_envs;
  const int e = alive ? env : n_envs - 1;
  W& w = reinterpret_cast<W*>(smem_raw)[warp];
  const Model<real, NJ, TK>& m = cmodel<real, NJ, TK>();
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NU = 2 * NJ;
  real* sr = state_r + (size_t)e * NR;
  int32_t* si = state_i + (size_t)e * NSTATE_I;
  if (alive) load_state<real, NJ, TK>(w, sr, si, first_id + e);
  const int d = DELAY && (!PAYLOAD || delay) ? action_delay_clamp(delay[e], m.frame_skip) : 0;
  Payload<real> pl = {};
  if constexpr (PAYLOAD) {
    if (!MOTOR || payload) pl = {payload[4 * (size_t)e], {payload[4 * (size_t)e + 1], payload[4 * (size_t)e + 2], payload[4 * (size_t)e + 3]}};
  }
  env_step<real, NJ, TK, STAIRS, DELAY, PAYLOAD, MOTOR>(w, m, actions + (size_t)e * NU, seed, max_traj_len, autoreset, sync_mode, alive, obs + (size_t)e * W::NOBS,
                     term_obs ? term_obs + (size_t)e * W::NOBS : nullptr, reward + e,
                     rew_terms ? rew_terms + (size_t)e * NREW : nullptr, done + e, ended + e,
                     ep_len ? ep_len + e : nullptr, ep_rew ? ep_rew + e : nullptr, STAIRS ? level + e : nullptr, n_levels, d, pl,
                     MOTOR ? strength + (size_t)e * NU : nullptr);
  if (alive) store_state<real, NJ, TK>(w, sr, si);
}

// evaluation statistics: one thread per env (a few dozen words read and written per env, no cross-env work; the record is read
// in place, nothing of it is written)
template <class real, int NJ, int TK>
__global__ void __launch_bounds__(256) eval_accumulate_kernel(const real* __restrict__ state_r, const int32_t* __restrict__ state_i,
                                                             int n_envs, const real* __restrict__ reward,
                                                             const real* __restrict__ rew_terms, const int32_t* __restrict__ done,
                                                             double* __restrict__ acc) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  eval_accumulate_env<real, NJ, TK>(state_r + (size_t)env * Dims<real, NJ, TK>::NSTATE_R, state_i + (size_t)env * NSTATE_I, reward[env],
                                    rew_terms + (size_t)env * NREW, done[env], acc + (size_t)env * EV_WORDS);
}

// root-velocity pushes: one thread per env, qvel[0:2] of the pushed envs written in place, nothing else (sim_core.h push_env)
template <class real, int NJ, int TK>
__global__ void __launch_bounds__(256) push_kernel(real* __restrict__ state_r, const int32_t* __restrict__ state_i, int n_envs,
                                                  uint32_t seed, uint32_t first_id, const int32_t* __restrict__ ended, double vel,
                                                  int interval, const real* __restrict__ d) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  push_env<real, NJ, TK>(state_r + (size_t)env * Dims<real, NJ, TK>::NSTATE_R, state_i + (size_t)env * NSTATE_I, seed, first_id + env,
                         ended ? ended[env] : 0, vel, interval, d ? d + 2 * (size_t)env : nullptr);
}

// random action delays: one thread per env, delay[i] of the selected envs (mask[i] != 0, or every env without a mask) redrawn,
// nothing else written (sim_core.h delay_draw_env); no model constants, so one kernel serves every variant
__global__ void __launch_bounds__(256) delay_draw_kernel(const int32_t* __restrict__ state_i, int n_envs, uint32_t seed,
                                                        uint32_t first_id, const int32_t* __restrict__ mask, int max_delay,
                                                        int32_t* __restrict__ delay) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  delay_draw_env(state_i + (size_t)env * NSTATE_I, seed, first_id + env, mask ? mask[env] : 1, max_delay, delay + env);
}

// random payloads: one thread per env, payload[i][0..3] of the selected envs (mask[i] != 0, or every env without a mask) redrawn,
// nothing else written (sim_core.h payload_draw_env); no model constants, so one kernel per precision serves every variant
template <class real>
__global__ void __launch_bounds__(256) payload_draw_kernel(const int32_t* __restrict__ state_i, int n_envs, uint32_t seed,
                                                          uint32_t first_id, const int32_t* __restrict__ mask, double max_mass,
                                                          double max_offset, real* __restrict__ payload) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  payload_draw_env<real>(state_i + (size_t)env * NSTATE_I, seed, first_id + env, mask ? mask[env] : 1, max_mass, max_offset,
                         payload + 4 * (size_t)env);
}

// random motor strengths: one thread per env, strength[i][0 .. nu-1] of the selected envs (mask[i] != 0, or every env without a
// mask) redrawn, nothing else written (sim_core.h motor_draw_env); nu is an argument and no other model constant is read, so one
// kernel per precision serves every variant
template <class real>
__global__ void __launch_bounds__(256) motor_draw_kernel(const int32_t* __restrict__ state_i, int n_envs, uint32_t seed,
                                                        uint32_t first_id, const int32_t* __restrict__ mask, double max_dev, int nu,
                                                        real* __restrict__ strength) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  motor_draw_env<real>(state_i + (size_t)env * NSTATE_I, seed, first_id + env, mask ? mask[env] : 1, max_dev, nu,
                       strength + (size_t)nu * env);
}

// sensor errors: one thread per (env, group of four observation words), ngroup = ceil(nrobot / 4) threads per env (sim_core.h
// sensor_env); nrobot, nu and obs_dim are arguments and no model constant is read, so one kernel per precision serves every variant
template <class real>
__global__ void __launch_bounds__(256) sensor_kernel(const int32_t* __restrict__ state_i, int n_envs, uint32_t seed, uint32_t first_id,
                                                    const int32_t* __restrict__ sel, int after_step, int autoreset, double3 draw,
                                                    int has_draw, int nrobot, int nu, int obs_dim, real* __restrict__ sensor,
                                                    real* __restrict__ obs, real* __restrict__ term_obs) {
  const int ngroup = (nrobot + 3) / 4;
  const int t = blockIdx.x * blockDim.x + threadIdx.x;   // the host keeps n_envs * ngroup within int
  if (t >= n_envs * ngroup) return;
  const int env = t / ngroup, g = t - env * ngroup;
  sensor_env<real>(state_i + (size_t)env * NSTATE_I, seed, first_id + env, g, sel ? sel[env] : 1, after_step, autoreset, has_draw,
                   draw.x, draw.y, draw.z, nrobot, nu, sensor + (size_t)(6 + nu) * env, obs + (size_t)obs_dim * env,
                   term_obs ? term_obs + (size_t)obs_dim * env : nullptr);
}

// held commands (WalkingTask variants only): one thread per env, the mode word, mode_ref and the obs task words of the envs given
// one (sim_core.h set_command_env)
template <class real, int NJ, int TK>
__global__ void __launch_bounds__(256) set_command_kernel(real* __restrict__ state_r, int32_t* __restrict__ state_i, int n_envs,
                                                         const int32_t* __restrict__ mode, const real* __restrict__ ref,
                                                         real* __restrict__ obs) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  set_command_env<real, NJ, TK>(state_r + (size_t)env * Dims<real, NJ, TK>::NSTATE_R, state_i + (size_t)env * NSTATE_I, mode[env],
                                ref + 3 * (size_t)env, obs + (size_t)env * Dims<real, NJ, TK>::NOBS);
}

// the command sweep's signed velocities: one thread per env, the record only read (sim_core.h command_accumulate_env)
template <class real, int NJ, int TK>
__global__ void __launch_bounds__(256) command_accumulate_kernel(const real* __restrict__ state_r, int n_envs,
                                                                const int32_t* __restrict__ done, double* __restrict__ acc) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  command_accumulate_env<real, NJ, TK>(state_r + (size_t)env * Dims<real, NJ, TK>::NSTATE_R, done[env], acc + (size_t)env * CMD_WORDS);
}

}  // namespace

// what every sim has, whichever its variant; SimOf<real, NJ, TK> holds its model and launches its kernels
struct lhw_sim {
  int precision, device, warps_per_block, sync_mode;
  size_t work_bytes;
  int state_reals, obs_dim, act_dim, nrobot;   // nrobot: the robot-state words that lead an observation
  virtual ~lhw_sim() = default;
  virtual int bind(cudaStream_t st) = 0;
  virtual void reset(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                     int fresh, void* obs, cudaStream_t st) = 0;
  virtual void step(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                    int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                    int32_t* ended, int32_t* ep_len, void* ep_rew, cudaStream_t st) = 0;
  virtual void render(const void* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids, int n_ids, int width,
                      int height, const render::Camera& cam, uint8_t* rgb, cudaStream_t st) = 0;
  virtual void eval_accumulate(const void* state_r, const int32_t* state_i, int n_envs, const void* reward, const void* rew_terms,
                               const int32_t* done, double* acc, cudaStream_t st) = 0;
  virtual void push(void* state_r, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* ended,
                    double vel, int interval, const void* d, cudaStream_t st) = 0;
  virtual int set_command(void* state_r, int32_t* state_i, int n_envs, const int32_t* mode, const void* ref, void* obs,
                          cudaStream_t st) = 0;
  virtual void command_accumulate(const void* state_r, int n_envs, const int32_t* done, double* acc, cudaStream_t st) = 0;
  virtual int footstep_limits(int* nplan, double* max_height) const = 0;
  virtual void reset_footsteps(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mode,
                               const void* value, int fresh, void* obs, cudaStream_t st) = 0;
  virtual int stairs_refusal() const = 0;
  virtual void reset_stairs(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                            int fresh, void* obs, const int32_t* level, int n_levels, cudaStream_t st) = 0;
  virtual void step_stairs(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                           int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                           int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels, cudaStream_t st) = 0;
  virtual void step_delay(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                          int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                          int32_t* ended, int32_t* ep_len, void* ep_rew, const int32_t* delay, int32_t* level, int n_levels,
                          cudaStream_t st) = 0;
  virtual void step_payload(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                            int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                            int32_t* ended, int32_t* ep_len, void* ep_rew, const void* payload, const int32_t* delay, int32_t* level,
                            int n_levels, cudaStream_t st) = 0;
  virtual void step_motor(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                          int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                          int32_t* ended, int32_t* ep_len, void* ep_rew, const void* strength, const void* payload,
                          const int32_t* delay, int32_t* level, int n_levels, cudaStream_t st) = 0;
  virtual int frame_skip() const = 0;
  virtual void set_step_height(double h) = 0;
};

namespace {

template <class K> int prepare_kernel(K kernel, size_t smem) {
  CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return 0;
}

template <class real, int NJ, int TK> int prepare_variant(lhw_sim* s) {
  s->work_bytes = sizeof(Work<real, NJ, TK>);
  s->state_reals = Dims<real, NJ, TK>::NSTATE_R;
  s->obs_dim = Dims<real, NJ, TK>::NOBS;
  s->nrobot = Dims<real, NJ, TK>::NROBOT;
  int maxsmem = 0;
  CUDA_OK(cudaDeviceGetAttribute(&maxsmem, cudaDevAttrMaxSharedMemoryPerBlockOptin, s->device));
  // lock-step blocks: as many warps as the launch bound and the shared memory of one SM allow, two blocks per SM
  const int cap_threads = (sizeof(real) == 8 ? LHW_X_REGCAP : 896) / 32;
  if (s->warps_per_block > cap_threads) s->warps_per_block = cap_threads;
  while (s->warps_per_block > 1 && s->work_bytes * s->warps_per_block > (size_t)maxsmem) s->warps_per_block--;
  if (s->warps_per_block < 1) s->warps_per_block = 1;
  if ((int)s->work_bytes > maxsmem) return fail(-5, "working set does not fit in shared memory");
  if (prepare_kernel(step_kernel<real, NJ, TK>, s->work_bytes) || prepare_kernel(reset_kernel<real, NJ, TK>, s->work_bytes)) return -10;
  if constexpr (Cfg<NJ, TK>::STEP) {
    if (prepare_kernel(reset_kernel<real, NJ, TK, true>, s->work_bytes)) return -10;
    if (prepare_kernel(reset_kernel<real, NJ, TK, false, true>, s->work_bytes) || prepare_kernel(step_kernel<real, NJ, TK, true>, s->work_bytes))
      return -10;
  }
  if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK>, s->work_bytes * s->warps_per_block)) return -10;
  if constexpr (Cfg<NJ, TK>::STEP) {
    if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, true>, s->work_bytes * s->warps_per_block)) return -10;
  }
  if (prepare_kernel(step_kernel<real, NJ, TK, false, true>, s->work_bytes)) return -10;
  if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, false, true>, s->work_bytes * s->warps_per_block)) return -10;
  if constexpr (Cfg<NJ, TK>::STEP) {
    if (prepare_kernel(step_kernel<real, NJ, TK, true, true>, s->work_bytes)) return -10;
    if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, true, true>, s->work_bytes * s->warps_per_block)) return -10;
  }
  if (prepare_kernel(step_kernel<real, NJ, TK, false, true, true>, s->work_bytes)) return -10;
  if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, false, true, true>, s->work_bytes * s->warps_per_block))
    return -10;
  if constexpr (Cfg<NJ, TK>::STEP) {
    if (prepare_kernel(step_kernel<real, NJ, TK, true, true, true>, s->work_bytes)) return -10;
    if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, true, true, true>, s->work_bytes * s->warps_per_block))
      return -10;
  }
  if (prepare_kernel(step_kernel<real, NJ, TK, false, true, true, true>, s->work_bytes)) return -10;
  if (s->warps_per_block > 1 && prepare_kernel(step_kernel_mw<real, NJ, TK, false, true, true, true>, s->work_bytes * s->warps_per_block))
    return -10;
  if constexpr (Cfg<NJ, TK>::STEP) {
    if (prepare_kernel(step_kernel<real, NJ, TK, true, true, true, true>, s->work_bytes)) return -10;
    if (s->warps_per_block > 1 &&
        prepare_kernel(step_kernel_mw<real, NJ, TK, true, true, true, true>, s->work_bytes * s->warps_per_block))
      return -10;
  }
  return 0;
}

// the sim whose model sits in a constant-bank object now, one record per object
template <class real, int NJ, int BANK_TK> struct BankOwner { static inline const lhw_sim* sim = nullptr; };

template <class real, int NJ, int TK> struct SimOf final : lhw_sim {
  using M = Model<real, NJ, TK>;
  // the sim whose model sits in cmodel<real, NJ, TK>() now
  static const lhw_sim*& owner() { return BankOwner<real, NJ, bank_tk<NJ, TK>()>::sim; }
  M model;
  M* d_twin = nullptr;       // the model once more, in global memory (lane-indexed tables are read from there)
  real* d_plans = nullptr;   // SteppingTask footstep plans in HBM ([MAXPLAN][PLAN_STRIDE])

  ~SimOf() override {
    if (owner() == this) owner() = nullptr;
    if (d_plans) cudaFree(d_plans);
    if (d_twin) cudaFree(d_twin);
  }

  int init(const double* flat, int n_flat, int dev) {
    precision = sizeof(real) == 8 ? 64 : 32;
    device = dev;
    act_dim = 2 * NJ;
    std::vector<real> plans(Cfg<NJ, TK>::STEP ? (size_t)MAXPLAN * PLAN_STRIDE : 0);
    const int rc = fill_model(model, flat, n_flat, plans.data());
    if (rc != 0) return fail(-4, "malformed model array (fill_model rc " + std::to_string(rc) + ")");
    if constexpr (Cfg<NJ, TK>::STEP) {
      // SteppingTask: the footstep plans go to HBM in the sim's precision; the model constants hold the device pointer
      cudaError_t e = cudaMalloc(&d_plans, plans.size() * sizeof(real));
      if (e == cudaSuccess) e = cudaMemcpy(d_plans, plans.data(), plans.size() * sizeof(real), cudaMemcpyHostToDevice);
      if (e != cudaSuccess) return fail(-10, std::string("footstep plan upload: ") + cudaGetErrorString(e));
      model.plans = d_plans;
    }
    const char* env_wpb = getenv("LHW_WARPS_PER_BLOCK");
    // lock-step blocks of 8 (fp64) / 14 (fp32) warps, 2 blocks per SM: what the 64 K registers and 228 KB of shared memory of
    // an H100 SM hold at the kernels' launch bounds (prepare_variant shrinks the block when the device has less)
    warps_per_block = env_wpb ? atoi(env_wpb) : (sizeof(real) == 8 ? (NJ == NJ_JVRC && !TK ? 8 : 7) : 14);
    const char* env_sync = getenv("LHW_BLOCK_SYNC_MODE");
    sync_mode = env_sync ? atoi(env_sync) : 1;
    if (warps_per_block < 1) warps_per_block = 1;
    return prepare_variant<real, NJ, TK>(this);
  }

  // make this sim's model the one in the constant bank, and copy it to the twin as well
  int bind(cudaStream_t st) override {
    if (owner() == this) return 0;
    if (!d_twin) CUDA_OK(cudaMalloc(&d_twin, sizeof(M)));
    model.gm = d_twin;
    CUDA_OK(cudaMemcpyAsync(d_twin, &model, sizeof(M), cudaMemcpyHostToDevice, st));
    CUDA_OK(cudaMemcpyToSymbolAsync(cmodel<real, NJ, TK>(), &model, sizeof(M), 0, cudaMemcpyHostToDevice, st));
    owner() = this;
    return 0;
  }

  void reset(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask, int fresh,
             void* obs, cudaStream_t st) override {
    reset_kernel<real, NJ, TK><<<n_envs, 32, work_bytes, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id, mask, fresh,
                                                             (real*)obs);
  }

  void step(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
            int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
            int32_t* ended, int32_t* ep_len, void* ep_rew, cudaStream_t st) override {
    const int wpb = warps_per_block, grid = (n_envs + wpb - 1) / wpb;
    const size_t smem = work_bytes * wpb;
    if (wpb > 1)
      step_kernel_mw<real, NJ, TK><<<grid, wpb * 32, smem, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id,
                                                            (const real*)actions, max_traj_len, autoreset, (real*)obs,
                                                            (real*)term_obs, (real*)reward, (real*)rew_terms, done, ended,
                                                            ep_len, (real*)ep_rew, sync_mode);
    else
      step_kernel<real, NJ, TK><<<grid, 32, smem, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id,
                                                   (const real*)actions, max_traj_len, autoreset, (real*)obs, (real*)term_obs,
                                                   (real*)reward, (real*)rew_terms, done, ended, ep_len, (real*)ep_rew);
  }

  // the renderer reads the sim's own global-memory model twin, whichever sim owns the constant bank
  void render(const void* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids, int n_ids, int width, int height,
              const render::Camera& cam, uint8_t* rgb, cudaStream_t st) override {
    render_launch<real, NJ, TK>(d_twin, (const real*)state_r, state_i, n_envs, env_ids, n_ids, width, height, cam, rgb, st);
  }

  void eval_accumulate(const void* state_r, const int32_t* state_i, int n_envs, const void* reward, const void* rew_terms,
                       const int32_t* done, double* acc, cudaStream_t st) override {
    eval_accumulate_kernel<real, NJ, TK><<<(n_envs + 255) / 256, 256, 0, st>>>((const real*)state_r, state_i, n_envs, (const real*)reward,
                                                                               (const real*)rew_terms, done, acc);
  }

  void push(void* state_r, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* ended, double vel,
            int interval, const void* d, cudaStream_t st) override {
    push_kernel<real, NJ, TK><<<(n_envs + 255) / 256, 256, 0, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id, ended, vel,
                                                                    interval, (const real*)d);
  }

  int set_command(void* state_r, int32_t* state_i, int n_envs, const int32_t* mode, const void* ref, void* obs,
                  cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STAND || Cfg<NJ, TK>::STEP) {
      return fail(-2, std::string(Cfg<NJ, TK>::STEP ? "jvrc_step (SteppingTask)" : "h1 (StandingTask)") +
                          " has no velocity command: only the WalkingTask variants jvrc_walk, jvrc_walk_terrain and h1_walk take one");
    } else {
      set_command_kernel<real, NJ, TK><<<(n_envs + 255) / 256, 256, 0, st>>>((real*)state_r, state_i, n_envs, mode, (const real*)ref,
                                                                             (real*)obs);
      return 0;
    }
  }

  void command_accumulate(const void* state_r, int n_envs, const int32_t* done, double* acc, cudaStream_t st) override {
    command_accumulate_kernel<real, NJ, TK><<<(n_envs + 255) / 256, 256, 0, st>>>((const real*)state_r, n_envs, done, acc);
  }

  int footstep_limits(int* nplan, double* max_height) const override {
    if constexpr (Cfg<NJ, TK>::STEP) {
      *nplan = model.nplan;
      *max_height = 2 * (double)model.slab_half[2];   // above it a slab's side face no longer covers the riser below the next slab
      return 0;
    } else {
      return fail(-2, std::string(NJ == 5 ? (TK == 3 ? "h1_walk" : "h1") : TK == 2 ? "jvrc_walk_terrain" : "jvrc_walk") +
                          " has no footstep plan: only jvrc_step (SteppingTask) takes one");
    }
  }

  void reset_footsteps(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mode,
                       const void* value, int fresh, void* obs, cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP)
      reset_kernel<real, NJ, TK, true><<<n_envs, 32, work_bytes, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id, nullptr,
                                                                       fresh, (real*)obs, mode, (const real*)value);
  }

  int stairs_refusal() const override {
    if constexpr (Cfg<NJ, TK>::STEP) return 0;
    else
      return fail(-2, std::string(NJ == 5 ? (TK == 3 ? "h1_walk" : "h1") : TK == 2 ? "jvrc_walk_terrain" : "jvrc_walk") +
                          " has no stair curriculum: only jvrc_step (SteppingTask) takes one");
  }

  void reset_stairs(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask, int fresh,
                    void* obs, const int32_t* level, int n_levels, cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP)
      reset_kernel<real, NJ, TK, false, true><<<n_envs, 32, work_bytes, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id, mask,
                                                                              fresh, (real*)obs, nullptr, nullptr, level, n_levels);
  }

  void step_stairs(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                   int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                   int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels, cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP) {
      const int wpb = warps_per_block, grid = (n_envs + wpb - 1) / wpb;
      const size_t smem = work_bytes * wpb;
      if (wpb > 1)
        step_kernel_mw<real, NJ, TK, true><<<grid, wpb * 32, smem, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id,
                                                                         (const real*)actions, max_traj_len, autoreset, (real*)obs,
                                                                         (real*)term_obs, (real*)reward, (real*)rew_terms, done, ended,
                                                                         ep_len, (real*)ep_rew, sync_mode, level, n_levels);
      else
        step_kernel<real, NJ, TK, true><<<grid, 32, smem, st>>>((real*)state_r, state_i, n_envs, seed, first_env_id,
                                                                (const real*)actions, max_traj_len, autoreset, (real*)obs, (real*)term_obs,
                                                                (real*)reward, (real*)rew_terms, done, ended, ep_len, (real*)ep_rew,
                                                                level, n_levels);
    }
  }

  // DELAY, and with a level array (jvrc_step only) STAIRS as well
  void step_delay(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                  int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                  int32_t* ended, int32_t* ep_len, void* ep_rew, const int32_t* delay, int32_t* level, int n_levels,
                  cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP) {
      if (level) {
        launch_step<true, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward,
                                rew_terms, done, ended, ep_len, ep_rew, level, n_levels, delay, st);
        return;
      }
    }
    launch_step<false, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward,
                             rew_terms, done, ended, ep_len, ep_rew, nullptr, 0, delay, st);
  }

  // PAYLOAD (with DELAY: a null delay array is delay 0), and with a level array (jvrc_step only) STAIRS as well
  void step_payload(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                    int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                    int32_t* ended, int32_t* ep_len, void* ep_rew, const void* payload, const int32_t* delay, int32_t* level,
                    int n_levels, cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP) {
      if (level) {
        launch_step<true, true, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs,
                                      reward, rew_terms, done, ended, ep_len, ep_rew, level, n_levels, delay, st, payload);
        return;
      }
    }
    launch_step<false, true, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs,
                                   reward, rew_terms, done, ended, ep_len, ep_rew, nullptr, 0, delay, st, payload);
  }

  // MOTOR (with DELAY and PAYLOAD: a null delay array is delay 0, a null payload array mass 0), and with a level array (jvrc_step
  // only) STAIRS as well
  void step_motor(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                  int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                  int32_t* ended, int32_t* ep_len, void* ep_rew, const void* strength, const void* payload, const int32_t* delay,
                  int32_t* level, int n_levels, cudaStream_t st) override {
    if constexpr (Cfg<NJ, TK>::STEP) {
      if (level) {
        launch_step<true, true, true, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs,
                                            term_obs, reward, rew_terms, done, ended, ep_len, ep_rew, level, n_levels, delay, st,
                                            payload, strength);
        return;
      }
    }
    launch_step<false, true, true, true>(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs,
                                         reward, rew_terms, done, ended, ep_len, ep_rew, nullptr, 0, delay, st, payload, strength);
  }

  template <bool STAIRS, bool DELAY, bool PAYLOAD = false, bool MOTOR = false>
  void launch_step(void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const void* actions,
                   int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                   int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels, const int32_t* delay, cudaStream_t st,
                   const void* payload = nullptr, const void* strength = nullptr) {
    const int wpb = warps_per_block, grid = (n_envs + wpb - 1) / wpb;
    const size_t smem = work_bytes * wpb;
    if (wpb > 1)
      step_kernel_mw<real, NJ, TK, STAIRS, DELAY, PAYLOAD, MOTOR><<<grid, wpb * 32, smem, st>>>(
          (real*)state_r, state_i, n_envs, seed, first_env_id, (const real*)actions, max_traj_len, autoreset, (real*)obs, (real*)term_obs,
          (real*)reward, (real*)rew_terms, done, ended, ep_len, (real*)ep_rew, sync_mode, level, n_levels, delay, (const real*)payload,
          (const real*)strength);
    else
      step_kernel<real, NJ, TK, STAIRS, DELAY, PAYLOAD, MOTOR><<<grid, 32, smem, st>>>(
          (real*)state_r, state_i, n_envs, seed, first_env_id, (const real*)actions, max_traj_len, autoreset, (real*)obs, (real*)term_obs,
          (real*)reward, (real*)rew_terms, done, ended, ep_len, (real*)ep_rew, level, n_levels, delay, (const real*)payload,
          (const real*)strength);
  }

  int frame_skip() const override { return model.frame_skip; }

  void set_step_height(double h) override {
    if constexpr (Cfg<NJ, TK>::STEP) {   // only the SteppingTask has a curriculum
      model.step_height = (real)h;
      if (owner() == this) owner() = nullptr;   // re-upload the constants at the next launch / lhw_sim_bind
    }
  }
};

}  // namespace

extern "C" {

int lhw_version(void) { return 3; }
const char* lhw_last_error(void) { return g_err.c_str(); }
long long lhw_launch_count(void) { return g_launches.load(); }
void lhw_count_launch(void) { g_launches++; }

int lhw_sim_create(lhw_sim** out, const double* flat, int n_flat, int precision, int device) {
  if (!out || !flat || n_flat < 1) return fail(-1, "null argument");
  if (precision != 64 && precision != 32) return fail(-2, "precision must be 32 or 64");
  int ndev = 0;
  CUDA_OK(cudaGetDeviceCount(&ndev));
  if (device < 0 || device >= ndev) return fail(-3, "no such CUDA device");
  CUDA_OK(cudaSetDevice(device));
  const int var = (int)flat[0];
  lhw_sim* s = nullptr;
  int rc = 0;
  const int unknown = with_variant(var, precision, [&](auto v) {
    using V = decltype(v);
    auto* sv = new SimOf<typename V::real, V::NJ, V::TK>();
    s = sv;
    rc = sv->init(flat, n_flat, device);
  });
  if (unknown) return fail(-4, "unsupported robot / task variant " + std::to_string(var));
  if (rc != 0) { delete s; return rc; }
  *out = s;
  return 0;
}

int lhw_sim_destroy(lhw_sim* s) {
  delete s;
  return 0;
}

int lhw_sim_set_step_height(lhw_sim* s, double h) {
  if (!s) return fail(-1, "null argument");
  s->set_step_height(h);   // no-op but for the SteppingTask
  return 0;
}

int lhw_sim_state_reals(const lhw_sim* s) { return s ? s->state_reals : Dims<double, NJ_JVRC, 0>::NSTATE_R; }
int lhw_sim_state_ints(const lhw_sim*) { return NSTATE_I; }
int lhw_sim_obs_dim(const lhw_sim* s) { return s ? s->obs_dim : Dims<double, NJ_JVRC, 0>::NOBS; }
int lhw_sim_act_dim(const lhw_sim* s) { return s ? s->act_dim : 2 * NJ_JVRC; }
int lhw_sim_smem_bytes_per_env(const lhw_sim* s) { return (int)s->work_bytes; }
int lhw_sim_precision(const lhw_sim* s) { return s ? s->precision : 0; }
int lhw_sim_device(const lhw_sim* s) { return s ? s->device : -1; }

int lhw_sim_bind(lhw_sim* s, void* stream) {
  if (!s) return fail(-1, "null argument");
  return s->bind((cudaStream_t)stream);
}

int lhw_sim_reset(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                  const int32_t* mask, int fresh, void* obs, void* stream) {
  if (!s || !state_r || !state_i) return fail(-1, "null argument");
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->reset(state_r, state_i, n_envs, seed, first_env_id, mask, fresh, obs, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_step(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                 const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                 void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, void* stream) {
  if (!s || !state_r || !state_i || !actions || !obs || !reward || !done || !ended) return fail(-1, "null argument");
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->step(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward, rew_terms, done,
          ended, ep_len, ep_rew, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_render(lhw_sim* s, const void* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids, int n_ids, int width,
                   int height, double dx, double dy, double z, double distance, double azimuth, double elevation, double fovy,
                   uint8_t* rgb, void* stream) {
  if (!s || !state_r || !state_i || !env_ids || !rgb) return fail(-1, "null argument");
  if (n_envs <= 0 || n_ids <= 0 || n_ids > 65535) return fail(-2, "n_envs must be positive and n_ids in 1..65535");
  if (width < 16 || width > 4096 || height < 16 || height > 4096) return fail(-2, "width and height must lie in 16..4096");
  if (!(distance > 0) || !(fovy > 0 && fovy < 180)) return fail(-2, "distance must be positive and fovy in (0, 180) degrees");
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;   // leaves the sim's current model in its twin
  const render::Camera cam = render::make_camera(dx, dy, z, distance, azimuth, elevation, fovy, width, height);
  s->render(state_r, state_i, n_envs, env_ids, n_ids, width, height, cam, rgb, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_eval_words(void) { return EV_WORDS; }

int lhw_sim_eval_accumulate(lhw_sim* s, const void* state_r, const int32_t* state_i, int n_envs, const void* reward,
                            const void* rew_terms, const int32_t* done, double* acc, void* stream) {
  if (!s || !state_r || !state_i || !reward || !rew_terms || !done || !acc) return fail(-1, "null argument");
  if (n_envs <= 0) return 0;
  s->eval_accumulate(state_r, state_i, n_envs, reward, rew_terms, done, acc, (cudaStream_t)stream);   // reads no model constants
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_push(lhw_sim* s, void* state_r, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                 const int32_t* ended, double vel, int interval_steps, const void* d, void* stream) {
  if (!s || !state_r || !state_i || (!d && !ended)) return fail(-1, "null argument");
  if (!d && !(vel >= 0 && vel <= 1e30)) return fail(-2, "push velocity must be finite and non-negative");
  if (!d && interval_steps < 1) return fail(-2, "push interval must be at least one control step");
  if (n_envs <= 0) return 0;
  s->push(state_r, state_i, n_envs, seed, first_env_id, ended, vel, interval_steps, d, (cudaStream_t)stream);   // no model constants
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_set_command(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, const int32_t* mode, const void* ref, void* obs,
                        void* stream) {
  if (!s || !state_r || !state_i || !mode || !ref || !obs) return fail(-1, "null argument");
  if (n_envs <= 0) return 0;
  const int rc = s->set_command(state_r, state_i, n_envs, mode, ref, obs, (cudaStream_t)stream);   // no model constants
  if (rc) return rc;
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_footstep_limits(const lhw_sim* s, int* nplan, double* max_height) {
  if (!s || !nplan || !max_height) return fail(-1, "null argument");
  return s->footstep_limits(nplan, max_height);
}

int lhw_sim_reset_footsteps(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                            const int32_t* mode, const void* value, int fresh, void* obs, void* stream) {
  if (!s || !state_r || !state_i || !mode || !value) return fail(-1, "null argument");
  int nplan = 0;
  double max_height = 0;
  if (const int rc = s->footstep_limits(&nplan, &max_height)) return rc;
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->reset_footsteps(state_r, state_i, n_envs, seed, first_env_id, mode, value, fresh, obs, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

static int check_stairs(const lhw_sim* s, int n_levels, const char* what) {
  if (const int rc = s->stairs_refusal()) return fail(rc, std::string(what) + ": " + g_err);
  if (n_levels < 2 || n_levels > STAIR_MAX_LEVELS)
    return fail(-2, std::string(what) + ": n_levels must lie in 2.." + std::to_string(STAIR_MAX_LEVELS) + ", got " + std::to_string(n_levels));
  return 0;
}

int lhw_sim_reset_stairs(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                         const int32_t* mask, int fresh, void* obs, const int32_t* level, int n_levels, void* stream) {
  if (!s || !state_r || !state_i || !level) return fail(-1, "null argument");
  if (const int rc = check_stairs(s, n_levels, "lhw_sim_reset_stairs")) return rc;
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->reset_stairs(state_r, state_i, n_envs, seed, first_env_id, mask, fresh, obs, level, n_levels, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_step_stairs(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                        const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                        void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels,
                        void* stream) {
  if (!s || !state_r || !state_i || !actions || !obs || !reward || !done || !ended || !level) return fail(-1, "null argument");
  if (const int rc = check_stairs(s, n_levels, "lhw_sim_step_stairs")) return rc;
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->step_stairs(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward, rew_terms,
                 done, ended, ep_len, ep_rew, level, n_levels, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_step_delay(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                       const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                       void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const int32_t* delay,
                       int32_t* level, int n_levels, void* stream) {
  if (!s || !state_r || !state_i || !actions || !obs || !reward || !done || !ended || !delay) return fail(-1, "null argument");
  if (level) {
    if (const int rc = check_stairs(s, n_levels, "lhw_sim_step_delay")) return rc;
  }
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->step_delay(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward, rew_terms,
                done, ended, ep_len, ep_rew, delay, level, n_levels, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_draw_delay(lhw_sim* s, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                       int max_delay, int32_t* delay, void* stream) {
  if (!s || !state_i || !delay) return fail(-1, "null argument");
  if (max_delay < 0 || max_delay > s->frame_skip())
    return fail(-2, "lhw_sim_draw_delay: the largest delay must lie in 0.." + std::to_string(s->frame_skip()) +
                        " substeps (frame_skip), got " + std::to_string(max_delay));
  if (n_envs <= 0) return 0;
  delay_draw_kernel<<<(n_envs + 255) / 256, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, mask, max_delay,
                                                                            delay);   // no model constants
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_step_payload(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                         const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                         void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const void* payload,
                         const int32_t* delay, int32_t* level, int n_levels, void* stream) {
  if (!s || !state_r || !state_i || !actions || !obs || !reward || !done || !ended || !payload) return fail(-1, "null argument");
  if (level) {
    if (const int rc = check_stairs(s, n_levels, "lhw_sim_step_payload")) return rc;
  }
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->step_payload(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward, rew_terms,
                  done, ended, ep_len, ep_rew, payload, delay, level, n_levels, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_draw_payload(lhw_sim* s, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                         double max_mass, double max_offset, void* payload, void* stream) {
  if (!s || !state_i || !payload) return fail(-1, "null argument");
  if (!(max_mass >= 0 && max_mass < INFINITY))
    return fail(-2, "lhw_sim_draw_payload: the largest payload mass must be finite and >= 0 kg, got " + std::to_string(max_mass));
  if (!(max_offset >= 0 && max_offset <= PAYLOAD_MAX_OFFSET))
    return fail(-2, "lhw_sim_draw_payload: the largest payload offset must lie in [0, 0.25] m, got " + std::to_string(max_offset));
  if (n_envs <= 0) return 0;
  const int grid = (n_envs + 255) / 256;   // no model constants
  if (s->precision == 64)
    payload_draw_kernel<double><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, mask, max_mass, max_offset,
                                                                        (double*)payload);
  else
    payload_draw_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, mask, max_mass, max_offset,
                                                                       (float*)payload);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_step_motor(lhw_sim* s, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                       const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                       void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const void* strength,
                       const void* payload, const int32_t* delay, int32_t* level, int n_levels, void* stream) {
  if (!s || !state_r || !state_i || !actions || !obs || !reward || !done || !ended || !strength) return fail(-1, "null argument");
  if (level) {
    if (const int rc = check_stairs(s, n_levels, "lhw_sim_step_motor")) return rc;
  }
  if (n_envs <= 0) return 0;
  cudaStream_t st = (cudaStream_t)stream;
  if (s->bind(st)) return -10;
  s->step_motor(state_r, state_i, n_envs, seed, first_env_id, actions, max_traj_len, autoreset, obs, term_obs, reward, rew_terms,
                done, ended, ep_len, ep_rew, strength, payload, delay, level, n_levels, st);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_draw_motor(lhw_sim* s, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                       double max_dev, void* strength, void* stream) {
  if (!s || !state_i || !strength) return fail(-1, "null argument");
  if (!(max_dev >= 0 && max_dev <= 1))
    return fail(-2, "lhw_sim_draw_motor: the largest strength deviation must lie in [0, 1], got " + std::to_string(max_dev));
  if (n_envs <= 0) return 0;
  const int grid = (n_envs + 255) / 256;   // no model constants but the joint count
  if (s->precision == 64)
    motor_draw_kernel<double><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, mask, max_dev, s->act_dim,
                                                                      (double*)strength);
  else
    motor_draw_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, mask, max_dev, s->act_dim,
                                                                     (float*)strength);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_sense(lhw_sim* s, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* sel,
                  int after_step, int autoreset, const double* draw, void* sensor, void* obs, void* term_obs, void* stream) {
  if (!s || !state_i || !sensor || !obs) return fail(-1, "null argument");
  if (after_step && !term_obs) return fail(-2, "lhw_sim_sense: after a step the pass needs the step's term_obs");
  if (draw) {
    static const char* what[3] = {"roll / pitch offset", "gyro offset", "encoder offset"};
    const double hi[3] = {SENSOR_MAX_ORIENT, SENSOR_MAX_GYRO, SENSOR_MAX_ENCODER};
    for (int k = 0; k < 3; k++)
      if (!(draw[k] >= 0 && draw[k] <= hi[k]))
        return fail(-2, std::string("lhw_sim_sense: the largest ") + what[k] + " must lie in [0, " + std::to_string(hi[k]) + "], got " +
                            std::to_string(draw[k]));
  }
  if (n_envs <= 0) return 0;
  const long long threads = (long long)n_envs * ((s->nrobot + 3) / 4);
  if (threads > INT_MAX) return fail(-2, "lhw_sim_sense: too many environments for one launch");
  const int grid = (int)((threads + 255) / 256);   // no model constants but the three sizes
  const double3 r = draw ? make_double3(draw[0], draw[1], draw[2]) : make_double3(0, 0, 0);
  if (s->precision == 64)
    sensor_kernel<double><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, sel, after_step, autoreset, r,
                                                                  draw != nullptr, s->nrobot, s->act_dim, s->obs_dim, (double*)sensor,
                                                                  (double*)obs, (double*)term_obs);
  else
    sensor_kernel<float><<<grid, 256, 0, (cudaStream_t)stream>>>(state_i, n_envs, seed, first_env_id, sel, after_step, autoreset, r,
                                                                 draw != nullptr, s->nrobot, s->act_dim, s->obs_dim, (float*)sensor,
                                                                 (float*)obs, (float*)term_obs);
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

int lhw_sim_command_words(void) { return CMD_WORDS; }

int lhw_sim_command_accumulate(lhw_sim* s, const void* state_r, int n_envs, const int32_t* done, double* acc, void* stream) {
  if (!s || !state_r || !done || !acc) return fail(-1, "null argument");
  if (n_envs <= 0) return 0;
  s->command_accumulate(state_r, n_envs, done, acc, (cudaStream_t)stream);   // reads no model constants
  g_launches++;
  CUDA_OK(cudaGetLastError());
  return 0;
}

}  // extern "C"
