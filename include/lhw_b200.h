/*
 * lhw_b200.h — C-ABI of the H100-native (sm_90a) rollout / PPO data path (liblhw_b200.so).
 *
 * The reference (rohanpsingh/LearningHumanoidWalking) has no FFI of its own: its seams are Python
 * duck-typed protocols and the arithmetic sits behind the `mujoco` pybind module.  Each entry point
 * below names the reference interface it replaces (paths relative to the reference repo root).
 * Plain pointers and sizes only; all buffers are caller-owned DEVICE memory (the Python host uses
 * torch tensors) unless a parameter says "host".  `stream` is a cudaStream_t passed as void*.
 * Every function returns 0 on success, a negative code on error (lhw_last_error() has the text).
 *
 * `precision` is 64 (float64 state and arithmetic, the reference's numeric type) or 32 (float32).
 * Typed `void*` buffers hold doubles or floats accordingly.
 */
#ifndef LHW_B200_H
#define LHW_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lhw_sim lhw_sim;

int lhw_version(void);
const char* lhw_last_error(void);

/* ---- environment batch --------------------------------------------------------------------------
 * lhw_sim_create: replaces MujocoEnv.__init__ (envs/common/mujoco_env.py:16-36: MjSpec.compile +
 * MjData) and JvrcBaseEnv._setup_robot (envs/jvrc/jvrc_base.py:38-67): takes the compiled model
 * constants as a flat HOST float64 array (layout: learninghumanoidwalking_b200/model/loader.py).
 * The first word selects the robot/task variant: 106 = JVRC-1 + SteppingTask (envs/jvrc/jvrc_step.py,
 * tasks/stepping_task.py: footstep sequences, 20 per-env stepping-stone slabs, floor dropped in FORWARD mode),
 * 206 = JVRC-1 + WalkingTask on uneven / compliant terrain (an EXTENSION: the reference only has the unused
 * WalkingTask(manip_hfield) hook, tasks/walking_task.py:57,172-179; 20 terraces re-posed with that hook's ranges),
 * 6 = JVRC-1 + WalkingTask (envs/jvrc/jvrc_walk.py),
 * 5 = Unitree H1 + StandingTask (envs/h1/h1_env.py, envs/h1/h1_base.py:31-63: mass overrides, PD gains,
 * StandingTask), whose step also runs the observation noise, dynamics randomisation, random pushes and
 * initial-pose noise of envs/common/base_humanoid_env.py:228-338 + envs/common/domain_randomization.py inside
 * the kernel (per-env randomised parameters live at the tail of the state record). */
int lhw_sim_create(lhw_sim** out, const double* model_flat_host, int n_flat, int precision, int device);
int lhw_sim_destroy(lhw_sim* sim);
int lhw_sim_state_reals(const lhw_sim* sim); /* real words per env in the state record */
int lhw_sim_state_ints(const lhw_sim* sim);  /* int32 words per env in the state record */
int lhw_sim_obs_dim(const lhw_sim* sim);     /* env.observation_space.shape[0] (37 jvrc_walk, 39 jvrc_step, 35 h1) */
int lhw_sim_act_dim(const lhw_sim* sim);     /* env.action_space.shape[0] (12 jvrc_walk, 10 h1) */
int lhw_sim_smem_bytes_per_env(const lhw_sim* sim);
int lhw_sim_precision(const lhw_sim* sim);   /* 64 or 32 */
int lhw_sim_device(const lhw_sim* sim);      /* CUDA device ordinal the sim was created on */

/* lhw_sim_reset: MujocoEnv.reset + BaseHumanoidEnv.reset_model + WalkingTask.reset
 * (envs/common/mujoco_env.py:113-116, envs/common/base_humanoid_env.py:247-309,
 * tasks/walking_task.py:194-205 / tasks/standing_task.py:33) for every env whose mask[i] != 0 (mask == NULL: all).
 * `fresh` != 0 zero-initialises the record first (a newly constructed env).
 * state_r: [n_envs, state_reals] reals; state_i: [n_envs, state_ints] int32; obs: [n_envs, obs_dim]. */
int lhw_sim_reset(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                  const int32_t* mask, int fresh, void* obs, void* stream);

/* lhw_sim_step: BaseHumanoidEnv.step (envs/common/base_humanoid_env.py:199-227) ->
 * RobotBase.step/_do_simulation (robots/robot_base.py:41-98) -> frame_skip x {RobotInterface.step_pd,
 * set_motor_torque, mujoco.mj_step} (envs/common/robot_interface.py:493-546) -> WalkingTask.step /
 * calc_reward / done (tasks/walking_task.py:85-192; tasks/standing_task.py:49-131 for h1) -> get_obs (base_humanoid_env.py:177-197), for
 * n_envs environments in one launch.  With autoreset != 0 it also does the RolloutWorker's episode
 * bookkeeping (rl/workers/rollout_worker.py:146-176): ended = done || traj_len >= max_traj_len; an ended env
 * is reset inside the same launch and `obs` is the post-reset observation while `term_obs` keeps the
 * pre-reset one (for the truncation bootstrap critic(next_state)).
 * actions [n,act_dim]; obs, term_obs [n,obs_dim]; reward [n]; rew_terms [n,10] (may be NULL);
 * done, ended, ep_len [n] int32; ep_rew [n]  (ep_len/ep_rew written only where ended). */
int lhw_sim_step(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                 const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                 void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, void* stream);

/* lhw_sim_bind: make `sim`'s model constants the resident ones (they live in one __constant__ object per (robot, precision),
 * shared by all sims of the process; lhw_sim_step/reset do this implicitly, a replayed CUDA graph cannot). */
int lhw_sim_bind(lhw_sim* sim, void* stream);

/* lhw_sim_set_step_height: SteppingTask curriculum (tasks/stepping_task.py:312): the host computes
 * h = clip((iteration_count - 3000) / 8000, 0, 1) * 0.1 from `env.robot.iteration_count` (rl/workers/rollout_worker.py:95)
 * and passes it here; it takes effect at the next task reset.  No-op for the other variants. */
int lhw_sim_set_step_height(lhw_sim* sim, double h);

/* lhw_sim_render: replaces EvaluateEnv.run's frames (rl/utils/eval.py:37-86: mujoco.Renderer offscreen rendering of the
 * roll-out into an mp4).  Ray-casts n_ids images of the environments env_ids[k] (device int32, each in [0, n_envs)) into
 * rgb [n_ids, height, width, 3] uint8, row 0 at the top, in one launch; state_r / state_i are only read.  Drawn: every link
 * as its equivalent-inertia box, the contact geometry of the feet, the slabs of jvrc_step / terrain, a checkerboard floor,
 * one directional light with hard shadows (csrc/render_core.h has the scene and shading formulas).  Pinhole camera looking
 * at (root_x + dx, root_y + dy, z) of each environment from `distance` metres, at `azimuth` / `elevation` (degrees,
 * elevation > 0 looks down), vertical field of view `fovy` degrees.  width, height in 16..4096; distance > 0; fovy in (0, 180). */
int lhw_sim_render(lhw_sim* sim, const void* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids, int n_ids,
                   int width, int height, double dx, double dy, double z, double distance, double azimuth, double elevation,
                   double fovy, uint8_t* rgb, void* stream);

/* lhw_sim_eval_accumulate: evaluation statistics of one control step, on the device (DESIGN.md §7.4; the reference only has
 * EvaluateEnv's single roll-out, rl/utils/eval.py).  After an lhw_sim_step with autoreset == 0 it reads the step's reward [n],
 * rew_terms [n,10] and done [n] and the records state_r / state_i (only read) and updates acc [n, lhw_sim_eval_words()]
 * float64 (zero it before the first step).  Per env, while its ended-by-done word is 0: episode length, return, ended-by-done
 * (set by the step whose done is set, which is counted), the 10 reward-term sums; walking tasks (and h1 against zero
 * references), per mode STANDING / INPLACE / FORWARD: steps and the sums of |v_fwd - vx_ref|, |v_lat - vy_ref|, |w_z - yaw_ref|
 * with the references zeroed as the reward zeroes them; jvrc_step: footstep targets reached and sequence length.  The word
 * layout is sim_core.h's EV_* enum. */
int lhw_sim_eval_words(void);
int lhw_sim_eval_accumulate(lhw_sim* sim, const void* state_r, const int32_t* state_i, int n_envs, const void* reward,
                            const void* rew_terms, const int32_t* done, double* acc, void* stream);

/* lhw_sim_push: root-velocity pushes (DESIGN.md §7.5; legged_gym's push_robots, the reference has none).  One launch over n envs
 * that adds Rz(psi) (dx, dy) to qvel[0:2] of the records state_r it pushes (world frame; psi = heading of qpos[3:7], (dx, dy) in
 * the heading frame: x forward, y to the robot's left) and writes nothing else.  state_i is only read.
 * Explicit mode, d != NULL: d [n, 2] in the sim's precision; rows that are exactly 0 are skipped (ended, vel, interval unused).
 * Random mode, d == NULL: after an lhw_sim_step over the same envs; an env whose ended [n] flag is 0 is pushed when
 * randint(u0, interval_steps) == 0 for u = philox(seed, first_env_id + i, rng_ctr, 70), by vel (2 u01(u1) - 1, 2 u01(u2) - 1).
 * vel must be finite and >= 0, interval_steps >= 1.  Reads no model constants. */
int lhw_sim_push(lhw_sim* sim, void* state_r, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                 const int32_t* ended, double vel, int interval_steps, const void* d, void* stream);

/* lhw_sim_set_command: hold a velocity command (DESIGN.md §7.6; legged_gym's `play` command override, the reference has none).
 * WalkingTask variants only (jvrc_walk, jvrc_walk_terrain, h1_walk); the others are refused with -2 and a message that names them.
 * One launch over n envs: an env whose mode [n] (int32) is STANDING = 0, INPLACE = 1 or FORWARD = 2 gets that mode, the held flag
 * (bit 30 of state_i's mode word, state_i[1]) and mode_ref = ref[i] (ref [n, 3] in the sim's precision, the record's order
 * (yaw_rate, vx, vy)), and its six task words of obs [n, obs_dim] (from obs_dim - 6: the FORWARD / INPLACE / STANDING one-hot, then
 * mode_ref) are rewritten as the step would write them.  Any other mode value (-1) leaves the env untouched; nothing else is written.
 * A held env's step skips the WalkingTask's random mode switches; its next reset (autoreset or lhw_sim_reset) clears the flag.
 * Reads no model constants. */
int lhw_sim_set_command(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, const int32_t* mode, const void* ref, void* obs,
                        void* stream);

/* lhw_sim_command_accumulate: the command sweep's signed velocities of one control step.  After an lhw_sim_step with autoreset == 0
 * it reads done [n] and the records state_r (only read) and updates acc [n, lhw_sim_command_words()] float64 (zero it before the
 * first step): while its ended-by-done word is 0, steps, the sums of v_fwd, v_lat and w_z as lhw_sim_eval_accumulate defines
 * them, and ended-by-done, over exactly the steps that lhw_sim_eval_accumulate counts.  The word layout is sim_core.h's CMD_* enum. */
int lhw_sim_command_words(void);
int lhw_sim_command_accumulate(lhw_sim* sim, const void* state_r, int n_envs, const int32_t* done, double* acc, void* stream);

/* lhw_sim_reset_footsteps: lhw_sim_reset with a chosen stepping-stone plan (DESIGN.md §7.7).  jvrc_step only; the other variants
 * are refused with -2 and a message that names them.  An env whose mode [n] (int32) is an ST_* value (CURVED = 0, STANDING = 1,
 * BACKWARD = 2, LATERAL = 3, FORWARD = 4) is reset as lhw_sim_reset resets it, with that plan type and value [n] (the sim's
 * precision): FORWARD the signed stair height in m (for the sign draw and the curriculum height), LATERAL the side +1 (the robot's
 * left) or -1, CURVED a plan index in [0, nplan) (any other value: the reset's own draw), STANDING and BACKWARD 0.  Every other
 * draw is the plain reset's.  Any other mode (-1) leaves the env untouched.  `fresh` and obs as for lhw_sim_reset.  The plan
 * lasts for the episode: the next reset draws one again.
 * lhw_sim_footstep_limits: the values the plan may take, nplan and the largest stair height |h| (2 slab_half[2]); -2 as above. */
int lhw_sim_footstep_limits(const lhw_sim* sim, int* nplan, double* max_height);
int lhw_sim_reset_footsteps(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                            const int32_t* mode, const void* value, int fresh, void* obs, void* stream);

/* lhw_sim_step_stairs / lhw_sim_reset_stairs: lhw_sim_step / lhw_sim_reset with a stair curriculum per env (DESIGN.md §7.8;
 * legged_gym's terrain levels).  jvrc_step only; the other variants are refused with -2 and a message that names them, as is
 * n_levels outside 2..21.  level [n] (device int32) holds each env's level L, clamped to [0, n_levels) where it is read.  Every reset
 * these launches do builds a FORWARD plan with the stair magnitude (real)(0.01 L) in place of the sim-wide step height; its sign
 * and every other draw are the plain reset's.  lhw_sim_step_stairs with autoreset != 0 moves the level of an env whose ended
 * episode was a FORWARD one, just before its reset: r = footstep targets reached, n = sequence length, fell = done; L + 1 (at most
 * n_levels - 1) if !fell and 2 r >= n, L - 1 (at least 0) if fell and 2 r < n, else unchanged.  Nothing else writes level;
 * lhw_sim_reset_stairs only reads it. */
int lhw_sim_reset_stairs(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                         const int32_t* mask, int fresh, void* obs, const int32_t* level, int n_levels, void* stream);
int lhw_sim_step_stairs(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                        const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                        void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels,
                        void* stream);

/* lhw_sim_step_delay: lhw_sim_step with an action delay per env (DESIGN.md §7.9), every variant.  delay [n] (device int32) holds
 * each env's delay d in physics substeps, clamped to [0, frame_skip] where it is read, once per control step.  In the control
 * step, substeps 0 .. d-1 drive the PD loop towards the previous control step's target, substeps d .. frame_skip-1 towards this
 * step's; nothing else changes (smoothing, gains, rewards, observations, termination, auto-reset).  The first step of an episode
 * has no previous target and so is never delayed.  d = 0 is lhw_sim_step bit for bit; d = frame_skip delays the action by one
 * whole control step.  level != NULL (jvrc_step only) adds the stair curriculum of lhw_sim_step_stairs, with its refusals.
 * Nothing writes delay.
 * lhw_sim_draw_delay: the random delays.  Every env whose mask [n] word is non-zero (every env when mask is NULL; pass the step's
 * `ended`, or a reset's mask) gets delay[i] = randint(u[0], max_delay + 1) with u = philox(seed, first_env_id + i, rng_ctr,
 * 71), rng_ctr the record's event counter (state_i[i][4]) as the reset left it.  Only delay is written; max_delay outside
 * 0..frame_skip is refused with -2.  Reads no model constants. */
int lhw_sim_step_delay(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                       const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                       void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const int32_t* delay,
                       int32_t* level, int n_levels, void* stream);
int lhw_sim_draw_delay(lhw_sim* sim, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                       int max_delay, int32_t* delay, void* stream);

/* lhw_sim_step_payload: lhw_sim_step with a payload carried by each env's root link (DESIGN.md §7.10), every variant.  payload
 * [n][4] (device, the sim's precision) holds each env's (m, rx, ry, rz): a point mass m >= 0 kg rigidly attached to the root link
 * at r (m), given in the root link's frame relative to the compiled model's root-link centre of mass.  It is read once per control
 * step.  Every physics substep of the control step builds the root link's mass, centre of mass and inertia as the composite of
 * the link and the point mass (H1: on top of the env's randomised link); an auto-reset's settling substeps run without it.
 * Observations, rewards, termination and the contact regularisation constants are unchanged.  An env whose mass is exactly 0 is
 * lhw_sim_step bit for bit, whatever its offset.  delay [n] (device int32, or NULL for none) adds the action delays of
 * lhw_sim_step_delay; level != NULL (jvrc_step only) adds the stair curriculum of lhw_sim_step_stairs, with its refusals.
 * Nothing writes payload or delay.
 * lhw_sim_draw_payload: the random payloads.  Every env whose mask [n] word is non-zero (every env when mask is NULL; pass the
 * step's `ended`, or a reset's mask) gets payload[i] = (max_mass u01(u[0]), max_offset (2 u01(u[1..3]) - 1)) with
 * u = philox(seed, first_env_id + i, rng_ctr, 72), rng_ctr the record's event counter (state_i[i][4]) as the reset left it.
 * Only payload is written.  max_mass not finite or negative, or max_offset outside [0, 0.25], is refused with -2; the host
 * bounds max_mass by half the robot's mass.  Reads no model constants. */
int lhw_sim_step_payload(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                         const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                         void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const void* payload,
                         const int32_t* delay, int32_t* level, int n_levels, void* stream);
int lhw_sim_draw_payload(lhw_sim* sim, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                         double max_mass, double max_offset, void* payload, void* stream);

/* lhw_sim_step_motor: lhw_sim_step with a motor strength per env and actuated joint (DESIGN.md §7.11), every variant.  strength
 * [n][NU] (device, the sim's precision; NU = act_dim, in get_motor_names() order) holds each env's factors s_l >= 0, read once
 * per control step: the step's PD gains become kp_step[l] = s_l kp, kd_step[l] = s_l kd (kp, kd after the pdrand_k draw when that
 * is on), so the dynamics, act_force, the torque reward terms, prev_torque and H1's observed motor torques all see the scaled
 * torque.  The substep loop and an auto-reset's settling (ctrl = 0) are unchanged.  An env whose factors are all exactly 1 is
 * lhw_sim_step bit for bit; s_l = 0 leaves joint l limp.  payload [n][4] (or NULL for none) adds the payloads of
 * lhw_sim_step_payload, delay [n] (device int32, or NULL for none) the action delays of lhw_sim_step_delay; level != NULL
 * (jvrc_step only) adds the stair curriculum of lhw_sim_step_stairs, with its refusals.  Nothing writes strength, payload or delay.
 * lhw_sim_draw_motor: the random strengths.  Every env whose mask [n] word is non-zero (every env when mask is NULL; pass the
 * step's `ended`, or a reset's mask) gets strength[i][l] = 1 + max_dev (2 u01(u[l % 4]) - 1) with
 * u = philox(seed, first_env_id + i, rng_ctr, 73 + l / 4), rng_ctr the record's event counter (state_i[i][4]) as the reset left
 * it.  Only strength is written.  max_dev not finite or outside [0, 1] is refused with -2.  Reads no model constant but NU. */
int lhw_sim_step_motor(lhw_sim* sim, void* state_r, int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id,
                       const void* actions, int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward,
                       void* rew_terms, int32_t* done, int32_t* ended, int32_t* ep_len, void* ep_rew, const void* strength,
                       const void* payload, const int32_t* delay, int32_t* level, int n_levels, void* stream);
int lhw_sim_draw_motor(lhw_sim* sim, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* mask,
                       double max_dev, void* strength, void* stream);

/* lhw_sim_sense: sensor errors on the observations (DESIGN.md §7.12), every variant; a pass over obs (and term_obs) [n][obs_dim]
 * after a step or a reset, on the same stream.  sensor [n][6 + NU] (device, the sim's precision) holds per env the noise
 * multiplier m >= 0, then one offset per calibrated observation word: roll, pitch (rad), gyro x, y, z (rad/s) and the NU motor
 * positions (rad, get_motor_names() order).  Word i < NROBOT (the robot-state words: 29 on JVRC-1, 35 on H1) of a treated
 * observation x becomes (real)(x[i] + b_i + (m s_g) (2 u01(u[i % 4]) - 1)) in float64, b_i its offset (0 for velocities and
 * torques), s_g its group's noise scale (orient 0.05, gyro 0.05, motor_pos 0.02, motor_vel 0.05, motor_tau 5) and
 * u = philox(seed, first_env_id + i_env, rng_ctr, stream + i / 4) at the record's event counter (state_i[i_env][4]); a word with
 * b_i == 0 and m s_g == 0 is not written.  The task words after NROBOT, the records and everything a step reads are never written.
 * after_step != 0 (sel: the step's `ended`, term_obs required, else -2): with autoreset, an env that ended has its term_obs treated
 * with its old row (stream 112), then draws (below), then its obs treated (stream 96); an env that did not end has its obs
 * treated.  Without autoreset every obs is treated and term_obs gets the same words.  after_step == 0 (a reset; sel: its mask, or
 * NULL for every env): a selected env draws, then its obs is treated; the others are not touched.  draw (host, {O, G, E}, or NULL
 * for none): a drawing env's offsets become U(-O, O) for roll and pitch, U(-G, G) for the gyro, U(-E, E) for each motor position,
 * offset k = (real)(r_k (2 u01(u[k % 4]) - 1)) with u = philox(seed, env id, rng_ctr, 80 + k / 4); the multiplier is never
 * written.  O outside [0, 0.2], G outside [0, 0.5], E outside [0, 0.2] or not finite is refused with -2.  Reads no model constant
 * but NROBOT, NU and obs_dim. */
int lhw_sim_sense(lhw_sim* sim, const int32_t* state_i, int n_envs, uint32_t seed, uint32_t first_env_id, const int32_t* sel,
                  int after_step, int autoreset, const double* draw, void* sensor, void* obs, void* term_obs, void* stream);

/* number of kernels this library has launched since load (the bench's gpu_launches claim) */
long long lhw_launch_count(void);

/* ---- PPO data path (float32, as rl/algos/ppo.py:474-477 casts the batch) ---------------------------
 * lhw_gae: PPOBuffer.finish_path (rl/storage/rollout_storage.py:53-85) for a [T, N] rollout stored time-major:
 * per env a reverse scan with the path broken wherever ended[t] != 0, bootstrapping with boot[t] there
 * ((not done) * critic(next_state), rl/workers/rollout_worker.py:166) and with last_val[n] after t = T-1
 * when the final transition did not end an episode (rollout_worker.py:183-186).
 * rewards, values, boot [T,N] f32; ended [T,N] int32; last_val [N]; returns [T,N] out.
 * adv_partials (may be NULL): lhw_gae_partial_words(N) doubles; the launch then also leaves per-block (sum, sumsq) of
 * returns - values there, which lhw_adv_stats_from_gae folds into stats[0:2] — the advantage normalisation
 * (rl/algos/ppo.py:484-485) then costs one 12 B/sample pass (lhw_adv_apply) instead of a statistics pass plus that. */
int lhw_gae(const float* rewards, const float* values, const int32_t* ended, const float* boot, const float* last_val,
            float* returns, int T, int N, float gamma, float lam, double* adv_partials_or_null, void* stream);
int lhw_gae_partial_words(int N);
int lhw_adv_stats_from_gae(const double* adv_partials, int N, double* stats, void* stream);

/* lhw_adv_norm: rl/algos/ppo.py:484-485 — adv = returns - values; (adv - mean) / (std_unbiased + eps).
 * stats: device scratch of lhw_adv_stats_words() doubles, {sum, sumsq, mean, std, per-block partials...}
 * (partials are combined in a fixed order, so the result is run-to-run deterministic). With world > 1 the
 * caller all-reduces stats[0:2] between lhw_adv_stats and lhw_adv_apply (count_total = global sample count). */
int lhw_adv_stats_words(void);
int lhw_adv_stats(const float* returns, const float* values, double* stats, long long count, void* stream);
int lhw_adv_apply(const float* returns, const float* values, float* adv, double* stats, long long count,
                  long long count_total, float eps, void* stream);

/* lhw_ppo_loss: the loss tail of PPO.update_actor_critic (rl/algos/ppo.py:302-386), forward and backward in one launch, for a
 * Gaussian policy with fixed per-action std: from the policy means mu / old_mu [B,A], the taken actions, advantages, returns,
 * values and (optional) mirrored actions it writes out8 = {actor_loss, entropy_penalty, critic_loss, approx_kl_div, mirror_loss,
 * imitation_loss (0), clip_fraction, total} and the gradients of total = actor + mirror_coeff * mirror + ent_coeff * entropy_penalty
 * + critic w.r.t. mu (g_mu), the mirrored actions (g_mirr) and the values (g_val).  partials: lhw_ppo_loss_partial_words(B)
 * doubles; ticket: one zero-initialised uint32.  Deterministic (block-ordered reduction). */
int lhw_ppo_loss_partial_words(int B);
int lhw_ppo_loss(const float* mu, const float* old_mu, const float* act, const float* adv, const float* ret, const float* val,
                 const float* mirr_or_null, const float* stds, int B, int A, float clip, float mirror_coeff, float ent_coeff,
                 float* g_mu, float* g_mirr_or_null, float* g_val, double* partials, unsigned int* ticket, float* out8, void* stream);
/* lhw_ppo_loss_imitation: lhw_ppo_loss plus the imitation term of a teacher policy (rl/algos/ppo.py:361-368): from the teacher's
 * actions teacher_mu [B,A] and an optional per-sample mask [B] (NULL = all ones), out8[5] = imitation_loss = mean over B*A of
 * mask_b (mu_bk - teacher_bk)^2, total (out8[7]) gains imitate_coeff * imitation_loss and g_mu its gradient.  Same partials,
 * ticket and determinism as lhw_ppo_loss. */
int lhw_ppo_loss_imitation(const float* mu, const float* old_mu, const float* act, const float* adv, const float* ret, const float* val,
                           const float* mirr_or_null, const float* stds, const float* teacher_mu, const float* mask_or_null, int B,
                           int A, float clip, float mirror_coeff, float ent_coeff, float imitate_coeff, float* g_mu,
                           float* g_mirr_or_null, float* g_val, double* partials, unsigned int* ticket, float* out8, void* stream);

/* lhw_linear_wgrad: what `loss.backward()` (rl/algos/ppo.py:389-392) does per Linear layer of the actor / critic MLPs
 * (rl/policies/actor.py:122-189, critic.py) for its parameters: gW [N,K] = gy [M,N]^T x [M,K] and gb [N] = column sums of gy
 * (gb_or_null = NULL: weights only), M = minibatch rows, row-major contiguous operands.  One streaming launch over (gy, x) plus
 * an ordered reduction of the batch slices (deterministic).  workspace: lhw_linear_wgrad_workspace_floats(M, N, K) floats of
 * device scratch, free to reuse once the call's work has run on `stream`.  M = 0 zero-fills the outputs. */
long long lhw_linear_wgrad_workspace_floats(int M, int N, int K);
int lhw_linear_wgrad(const float* gy, const float* x, int M, int N, int K, float* gW, float* gb_or_null, float* workspace,
                     void* stream);

/* lhw_gather_minibatch: the fancy-index gathers of rl/algos/ppo.py:535-538 in one launch.
 * idx [B] int64 sample indices into the flattened batch. */
int lhw_gather_minibatch(const float* obs, const float* act, const float* ret, const float* adv, const int64_t* idx,
                         float* obs_b, float* act_b, float* ret_b, float* adv_b, int B, int obs_dim, int act_dim,
                         void* stream);

/* lhw_clip_adam: torch.nn.utils.clip_grad_norm_(params, max_norm) followed by optim.Adam.step
 * (rl/algos/ppo.py:393-396, Adam(lr, eps) created at :429-430) over ONE flat parameter buffer:
 * lhw_grad_sumsq accumulates sum(g^2) into norm_scratch[0] (zeroed by the call), lhw_clip_adam applies
 * clip_coef = min(1, max_norm / (sqrt(sumsq) + 1e-6)) and the Adam update (beta1 .9, beta2 .999, no weight
 * decay, no amsgrad). grad_scale multiplies g first (1/world after a sum all-reduce). */
int lhw_grad_sumsq(const float* grad, float* norm_scratch, long long n, float grad_scale, void* stream);
int lhw_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* norm_scratch,
                  long long n, int step, float lr, float beta1, float beta2, float eps, float max_norm,
                  float grad_scale, void* stream);
/* same update, Adam step number kept in DEVICE memory (step_dev[0] = completed steps, incremented by the call): the whole
 * optimiser step of rl/algos/ppo.py:389-396 can then be replayed from a CUDA graph */
int lhw_clip_adam_dev(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* norm_scratch,
                      long long n, int* step_dev, float lr, float beta1, float beta2, float eps, float max_norm,
                      float grad_scale, void* stream);

/* ---- multi-GPU exchange step, fused (csrc/comm_kernels.cu) ------------------------------------------
 * Replaces, on N >= 1 GPUs, the sequence of rl/algos/ppo.py:389-396: (gradient all-reduce) -> clip_grad_norm_(actor),
 * clip_grad_norm_(critic) -> actor Adam.step, critic Adam.step, by three ordinary (CUDA-graph capturable) launches that
 * read the peers' flat gradients over NVLink peer memory (CUDA IPC, 16-byte loads), sum them in fixed rank order, and
 * apply clip + Adam; the Adam step number and the peer-barrier epoch live in device memory.
 * lhw_comm owns a cudaMalloc'ed IPC-exported gradient buffer of n_floats floats (lhw_comm_grad_ptr) — the host
 * makes the modules' .grad tensors views of it. Handles are exchanged by the host (torch.distributed
 * all_gather of lhw_comm_handle_size() bytes per rank) and mapped with lhw_comm_import.
 * n_actor: the first n_actor floats belong to the actor (own norm / clip), the rest to the critic.
 * lhw_comm_status: error word of the peer barrier (non-zero: a peer did not arrive within the spin limit; returns -20),
 * completed Adam steps, the two gradient norms of the last step; synchronises `stream`.
 * lhw_comm_set_step: set the device-side Adam step number (resume). */
typedef struct lhw_comm lhw_comm;
const char* lhw_comm_last_error(void);
int lhw_comm_handle_size(void);
int lhw_comm_create(lhw_comm** out, long long n_floats, int rank, int world, int device);
void* lhw_comm_grad_ptr(lhw_comm* comm);
long long lhw_comm_size(const lhw_comm* comm);   /* n_floats */
int lhw_comm_device(const lhw_comm* comm);
int lhw_comm_export(lhw_comm* comm, void* handle_blob_host);
int lhw_comm_import(lhw_comm* comm, const void* all_handle_blobs_host);
int lhw_comm_destroy(lhw_comm* comm);
int lhw_fused_allreduce_clip_adam(lhw_comm* comm, float* param, float* exp_avg, float* exp_avg_sq, long long n_actor,
                                  long long n_total, float lr, float beta1, float beta2, float eps, float max_norm,
                                  void* stream);
int lhw_comm_status(lhw_comm* comm, int* error_word, int* adam_steps, float* norms2, void* stream);
int lhw_comm_set_step(lhw_comm* comm, int adam_steps, void* stream);
/* KL-adaptive learning rate (rsl_rl's schedule, DESIGN.md §7.3), the same three launches otherwise.  Each rank publishes its
 * minibatch KL (kl: one device float, e.g. the loss's approx_kl_div) in its comm block after the flag words; once every peer
 * is ready, K1 takes the rank-order float64 mean of the W KL words and updates the float64 rate lr_dev[0] (device memory):
 * mean > 2 desired_kl -> lr = max(1e-5, lr / 1.5); 0 < mean < desired_kl / 2 -> lr = min(1e-2, lr * 1.5); otherwise (NaN
 * included) unchanged.  Adam then uses (float)lr_dev[0] in the same step.  Every rank computes the same bits, and the
 * launches stay graph-capturable: the rate is never a by-value argument.  desired_kl > 0.
 * lhw_comm_lr_ptr: the comm's own float64 rate word (the host passes it as lr_dev); lhw_comm_get_lr / lhw_comm_set_lr read
 * and write it (logging, resume) and synchronise `stream`; set_lr needs lr > 0. */
int lhw_fused_allreduce_clip_adam_adaptive(lhw_comm* comm, float* param, float* exp_avg, float* exp_avg_sq, long long n_actor,
                                           long long n_total, const float* kl, double* lr_dev, double desired_kl, float beta1,
                                           float beta2, float eps, float max_norm, void* stream);
double* lhw_comm_lr_ptr(lhw_comm* comm);
int lhw_comm_get_lr(lhw_comm* comm, double* lr_host, void* stream);
int lhw_comm_set_lr(lhw_comm* comm, double lr, void* stream);

#ifdef __cplusplus
}
#endif
#endif
