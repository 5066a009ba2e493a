// torch_ops.cpp — the entry points of include/lhw_b200.h registered with PyTorch's C++ extension ABI (TORCH_LIBRARY):
// torch.ops.lhw.sim_step(...), .sim_reset, .sim_render, .sim_eval_accumulate, .sim_push, .sim_set_command, .sim_command_accumulate, .sim_reset_footsteps, .sim_step_stairs, .sim_reset_stairs, .sim_step_delay, .sim_draw_delay, .sim_step_payload, .sim_draw_payload, .sim_step_motor, .sim_draw_motor, .sim_sense, .gae, .adv_stats, .adv_apply, .gather_minibatch, .grad_sumsq, .clip_adam_dev,
// .fused_exchange, .fused_exchange_adaptive.  Thin: every op validates its tensors (device, dtype, contiguity, shape against the sim / comm
// handle) with TORCH_CHECK, takes the CURRENT CUDA stream of the tensors' device and calls the C-ABI of liblhw_b200.so
// underneath — a wrong-length or wrong-dtype tensor is an exception here instead of an out-of-bounds write in a kernel.
// Handles (lhw_sim*, lhw_comm*) travel as int64, as the Python host already holds them.  All ops mutate their output
// arguments in place and return nothing, so they can be captured into CUDA graphs like the plain launches they are.
//
// Reference seams these ops stand behind (SURVEY.md §8b): env.step / env.reset (envs/common/base_humanoid_env.py:199-276),
// PPOBuffer.finish_path (rl/storage/rollout_storage.py:53-85), rl/algos/ppo.py:484-485, :535-538, :389-396.
#include <ATen/ATen.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <cmath>

#include "../../include/lhw_b200.h"

namespace {

using at::Tensor;
using OptTensor = std::optional<at::Tensor>;

void* stream_of(const Tensor& t) { return (void*)c10::cuda::getCurrentCUDAStream(t.get_device()).stream(); }

void check_cuda(const Tensor& t, const char* name, at::ScalarType dt, int device) {
  TORCH_CHECK(t.is_cuda(), "lhw: ", name, " must be a CUDA tensor (no CPU fallback on this path)");
  TORCH_CHECK(t.get_device() == device, "lhw: ", name, " is on cuda:", t.get_device(), ", expected cuda:", device);
  TORCH_CHECK(t.scalar_type() == dt, "lhw: ", name, " has dtype ", t.scalar_type(), ", expected ", dt);
  TORCH_CHECK(t.is_contiguous(), "lhw: ", name, " must be contiguous");
}
void check_shape(const Tensor& t, const char* name, std::initializer_list<int64_t> shape) {
  TORCH_CHECK(t.sizes() == at::IntArrayRef(shape), "lhw: ", name, " has shape ", t.sizes(), ", expected ", at::IntArrayRef(shape));
}
void ok(int rc, const char* what) { TORCH_CHECK(rc == 0, "lhw: ", what, " failed (rc=", rc, "): ", lhw_last_error()); }

struct SimInfo {
  lhw_sim* s;
  at::ScalarType real;
  int device, nr, ni, nobs, nact;
};
SimInfo sim_info(int64_t handle) {
  TORCH_CHECK(handle != 0, "lhw: null sim handle");
  lhw_sim* s = reinterpret_cast<lhw_sim*>(handle);
  return {s, lhw_sim_precision(s) == 64 ? at::kDouble : at::kFloat, lhw_sim_device(s), lhw_sim_state_reals(s), lhw_sim_state_ints(s),
          lhw_sim_obs_dim(s), lhw_sim_act_dim(s)};
}

void check_reset(const SimInfo& I, const Tensor& state_r, const Tensor& state_i, const OptTensor& mask, const Tensor& obs) {
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(obs, "obs", I.real, I.device); check_shape(obs, "obs", {n, I.nobs});
  if (mask) { check_cuda(*mask, "mask", at::kInt, I.device); check_shape(*mask, "mask", {n}); }
}

void sim_reset(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const OptTensor& mask, bool fresh,
               Tensor obs) {
  const SimInfo I = sim_info(sim);
  const int64_t n = state_r.size(0);
  check_reset(I, state_r, state_i, mask, obs);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_reset(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                   mask ? mask->data_ptr<int32_t>() : nullptr, fresh ? 1 : 0, obs.data_ptr(), stream_of(state_r)), "lhw_sim_reset");
}

void check_step(const SimInfo& I, const Tensor& state_r, const Tensor& state_i, const Tensor& actions, int64_t max_traj_len, const Tensor& obs,
                const OptTensor& term_obs, const Tensor& reward, const OptTensor& rew_terms, const Tensor& done, const Tensor& ended,
                const OptTensor& ep_len, const OptTensor& ep_rew) {
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(actions, "actions", I.real, I.device); check_shape(actions, "actions", {n, I.nact});
  check_cuda(obs, "obs", I.real, I.device); check_shape(obs, "obs", {n, I.nobs});
  check_cuda(reward, "reward", I.real, I.device); check_shape(reward, "reward", {n});
  check_cuda(done, "done", at::kInt, I.device); check_shape(done, "done", {n});
  check_cuda(ended, "ended", at::kInt, I.device); check_shape(ended, "ended", {n});
  if (term_obs) { check_cuda(*term_obs, "term_obs", I.real, I.device); check_shape(*term_obs, "term_obs", {n, I.nobs}); }
  if (rew_terms) { check_cuda(*rew_terms, "rew_terms", I.real, I.device); check_shape(*rew_terms, "rew_terms", {n, 10}); }
  if (ep_len) { check_cuda(*ep_len, "ep_len", at::kInt, I.device); check_shape(*ep_len, "ep_len", {n}); }
  if (ep_rew) { check_cuda(*ep_rew, "ep_rew", I.real, I.device); check_shape(*ep_rew, "ep_rew", {n}); }
  TORCH_CHECK(max_traj_len > 0, "lhw: max_traj_len must be positive");
}

void sim_step(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& actions,
              int64_t max_traj_len, bool autoreset, Tensor obs, const OptTensor& term_obs, Tensor reward, const OptTensor& rew_terms,
              Tensor done, Tensor ended, const OptTensor& ep_len, const OptTensor& ep_rew) {
  const SimInfo I = sim_info(sim);
  const int64_t n = state_r.size(0);
  check_step(I, state_r, state_i, actions, max_traj_len, obs, term_obs, reward, rew_terms, done, ended, ep_len, ep_rew);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_step(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                  actions.data_ptr(), (int)max_traj_len, autoreset ? 1 : 0, obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr,
                  reward.data_ptr(), rew_terms ? rew_terms->data_ptr() : nullptr, done.data_ptr<int32_t>(), ended.data_ptr<int32_t>(),
                  ep_len ? ep_len->data_ptr<int32_t>() : nullptr, ep_rew ? ep_rew->data_ptr() : nullptr, stream_of(state_r)), "lhw_sim_step");
}

void sim_render(int64_t sim, const Tensor& state_r, const Tensor& state_i, const Tensor& env_ids, int64_t width, int64_t height, double dx,
                double dy, double z, double distance, double azimuth, double elevation, double fovy, Tensor rgb) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(width >= 16 && width <= 4096 && height >= 16 && height <= 4096, "lhw: width and height must lie in 16..4096, got ", width,
              " x ", height);
  TORCH_CHECK(distance > 0, "lhw: camera distance must be positive, got ", distance);
  TORCH_CHECK(fovy > 0 && fovy < 180, "lhw: fovy must lie in (0, 180) degrees, got ", fovy);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(env_ids, "env_ids", at::kInt, I.device);
  TORCH_CHECK(env_ids.dim() == 1 && env_ids.numel() >= 1 && env_ids.numel() <= 65535, "lhw: env_ids must be a 1-D tensor of 1..65535 ids");
  const int64_t k = env_ids.numel();
  check_cuda(rgb, "rgb", at::kByte, I.device); check_shape(rgb, "rgb", {k, height, width, 3});
  TORCH_CHECK(n >= 1, "lhw: no environments");
  TORCH_CHECK(env_ids.min().item<int32_t>() >= 0 && env_ids.max().item<int32_t>() < n, "lhw: env_ids must lie in [0, ", n, ")");
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_render(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, env_ids.data_ptr<int32_t>(), (int)k, (int)width, (int)height,
                    dx, dy, z, distance, azimuth, elevation, fovy, rgb.data_ptr<uint8_t>(), stream_of(state_r)), "lhw_sim_render");
}

void sim_eval_accumulate(int64_t sim, const Tensor& state_r, const Tensor& state_i, const Tensor& reward, const Tensor& rew_terms,
                         const Tensor& done, Tensor acc) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(reward, "reward", I.real, I.device); check_shape(reward, "reward", {n});
  check_cuda(rew_terms, "rew_terms", I.real, I.device); check_shape(rew_terms, "rew_terms", {n, 10});
  check_cuda(done, "done", at::kInt, I.device); check_shape(done, "done", {n});
  check_cuda(acc, "acc", at::kDouble, I.device); check_shape(acc, "acc", {n, lhw_sim_eval_words()});
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_eval_accumulate(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, reward.data_ptr(), rew_terms.data_ptr(),
                             done.data_ptr<int32_t>(), acc.data_ptr<double>(), stream_of(state_r)), "lhw_sim_eval_accumulate");
}

void sim_push(int64_t sim, Tensor state_r, const Tensor& state_i, int64_t seed, int64_t first_env_id, const OptTensor& ended, double vel,
              int64_t interval_steps, const OptTensor& d) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  TORCH_CHECK(d.has_value() != ended.has_value(), "lhw: sim_push takes either d (explicit pushes) or ended (random pushes)");
  if (d) { check_cuda(*d, "d", I.real, I.device); check_shape(*d, "d", {n, 2}); }
  if (ended) {
    check_cuda(*ended, "ended", at::kInt, I.device); check_shape(*ended, "ended", {n});
    TORCH_CHECK(std::isfinite(vel) && vel >= 0, "lhw: push velocity must be finite and non-negative, got ", vel);
    TORCH_CHECK(interval_steps >= 1 && interval_steps <= INT32_MAX, "lhw: push interval must be at least one control step, got ",
                interval_steps);
  }
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_push(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                  ended ? ended->data_ptr<int32_t>() : nullptr, vel, (int)interval_steps, d ? d->data_ptr() : nullptr, stream_of(state_r)),
     "lhw_sim_push");
}

void sim_set_command(int64_t sim, Tensor state_r, Tensor state_i, const Tensor& mode, const Tensor& ref, Tensor obs) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(mode, "mode", at::kInt, I.device); check_shape(mode, "mode", {n});
  check_cuda(ref, "ref", I.real, I.device); check_shape(ref, "ref", {n, 3});
  check_cuda(obs, "obs", I.real, I.device); check_shape(obs, "obs", {n, I.nobs});
  c10::cuda::CUDAGuard guard(I.device);
  // called once per episode, outside graphs: the host syncs on the values are affordable
  TORCH_CHECK(!((mode < -1) | (mode > 2)).any().item<bool>(), "lhw: mode must be -1 (untouched), 0 (STANDING), 1 (INPLACE) or 2 (FORWARD)");
  TORCH_CHECK(ref.isfinite().all().item<bool>(), "lhw: ref must be finite");
  ok(lhw_sim_set_command(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, mode.data_ptr<int32_t>(), ref.data_ptr(),
                         obs.data_ptr(), stream_of(state_r)), "lhw_sim_set_command");
}

void sim_command_accumulate(int64_t sim, const Tensor& state_r, const Tensor& done, Tensor acc) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(done, "done", at::kInt, I.device); check_shape(done, "done", {n});
  check_cuda(acc, "acc", at::kDouble, I.device); check_shape(acc, "acc", {n, lhw_sim_command_words()});
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_command_accumulate(I.s, state_r.data_ptr(), (int)n, done.data_ptr<int32_t>(), acc.data_ptr<double>(), stream_of(state_r)),
     "lhw_sim_command_accumulate");
}

void sim_reset_footsteps(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& mode,
                         const Tensor& value, bool fresh, Tensor obs) {
  const SimInfo I = sim_info(sim);
  int nplan = 0;
  double max_height = 0;
  ok(lhw_sim_footstep_limits(I.s, &nplan, &max_height), "lhw_sim_reset_footsteps");   // names a variant without plans
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_cuda(state_r, "state_r", I.real, I.device); check_shape(state_r, "state_r", {n, I.nr});
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(mode, "mode", at::kInt, I.device); check_shape(mode, "mode", {n});
  check_cuda(value, "value", I.real, I.device); check_shape(value, "value", {n});
  check_cuda(obs, "obs", I.real, I.device); check_shape(obs, "obs", {n, I.nobs});
  c10::cuda::CUDAGuard guard(I.device);
  // called once per evaluation, outside graphs: the host syncs on the values are affordable
  TORCH_CHECK(!((mode < -1) | (mode > 4)).any().item<bool>(),
              "lhw: mode must be -1 (untouched), 0 (CURVED), 1 (STANDING), 2 (BACKWARD), 3 (LATERAL) or 4 (FORWARD)");
  TORCH_CHECK(value.isfinite().all().item<bool>(), "lhw: value must be finite");
  const Tensor v = value.to(at::kDouble);
  TORCH_CHECK(!((mode == 4) & (v.abs() > max_height)).any().item<bool>(), "lhw: a FORWARD stair height must lie in [-", max_height,
              ", ", max_height, "] m (2 slab_half[2]: above it a slab's side face no longer covers the riser below the next slab)");
  TORCH_CHECK(!((mode == 3) & (v != 1) & (v != -1)).any().item<bool>(), "lhw: a LATERAL value must be +1 (left) or -1 (right)");
  TORCH_CHECK(!((mode == 0) & (v != -1) & ((v < 0) | (v >= nplan) | (v != v.floor()))).any().item<bool>(),
              "lhw: a CURVED value must be -1 (drawn) or a plan index in [0, ", nplan, ")");
  TORCH_CHECK(!(((mode == 1) | (mode == 2)) & (v != 0)).any().item<bool>(), "lhw: a STANDING or BACKWARD value must be 0");
  ok(lhw_sim_reset_footsteps(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                             mode.data_ptr<int32_t>(), value.data_ptr(), fresh ? 1 : 0, obs.data_ptr(), stream_of(state_r)),
     "lhw_sim_reset_footsteps");
}

// the stair curriculum's level tensor [n] int32 and its level count (lhw_sim_step_stairs / lhw_sim_reset_stairs, DESIGN.md §7.8);
// a variant without the curriculum is named by the C-ABI's refusal
void check_stairs(const SimInfo& I, const Tensor& level, int64_t n, int64_t n_levels) {
  check_cuda(level, "level", at::kInt, I.device); check_shape(level, "level", {n});
  TORCH_CHECK(n_levels >= 2 && n_levels <= 21, "lhw: n_levels must lie in 2..21, got ", n_levels);
}

void sim_step_stairs(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& actions,
                     int64_t max_traj_len, bool autoreset, Tensor obs, const OptTensor& term_obs, Tensor reward, const OptTensor& rew_terms,
                     Tensor done, Tensor ended, const OptTensor& ep_len, const OptTensor& ep_rew, Tensor level, int64_t n_levels) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_step(I, state_r, state_i, actions, max_traj_len, obs, term_obs, reward, rew_terms, done, ended, ep_len, ep_rew);
  check_stairs(I, level, n, n_levels);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_step_stairs(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                         actions.data_ptr(), (int)max_traj_len, autoreset ? 1 : 0, obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr,
                         reward.data_ptr(), rew_terms ? rew_terms->data_ptr() : nullptr, done.data_ptr<int32_t>(), ended.data_ptr<int32_t>(),
                         ep_len ? ep_len->data_ptr<int32_t>() : nullptr, ep_rew ? ep_rew->data_ptr() : nullptr, level.data_ptr<int32_t>(),
                         (int)n_levels, stream_of(state_r)),
     "lhw_sim_step_stairs");
}

void sim_reset_stairs(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const OptTensor& mask, bool fresh,
                      Tensor obs, const Tensor& level, int64_t n_levels) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_reset(I, state_r, state_i, mask, obs);
  check_stairs(I, level, n, n_levels);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_reset_stairs(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                          mask ? mask->data_ptr<int32_t>() : nullptr, fresh ? 1 : 0, obs.data_ptr(), level.data_ptr<int32_t>(),
                          (int)n_levels, stream_of(state_r)),
     "lhw_sim_reset_stairs");
}

// the action delays (lhw_sim_step_delay / lhw_sim_draw_delay, DESIGN.md §7.9): delay [n] int32 substeps
void sim_step_delay(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& actions,
                    int64_t max_traj_len, bool autoreset, Tensor obs, const OptTensor& term_obs, Tensor reward, const OptTensor& rew_terms,
                    Tensor done, Tensor ended, const OptTensor& ep_len, const OptTensor& ep_rew, const Tensor& delay, const OptTensor& level,
                    int64_t n_levels) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_step(I, state_r, state_i, actions, max_traj_len, obs, term_obs, reward, rew_terms, done, ended, ep_len, ep_rew);
  check_cuda(delay, "delay", at::kInt, I.device); check_shape(delay, "delay", {n});
  if (level) check_stairs(I, *level, n, n_levels);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_step_delay(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                        actions.data_ptr(), (int)max_traj_len, autoreset ? 1 : 0, obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr,
                        reward.data_ptr(), rew_terms ? rew_terms->data_ptr() : nullptr, done.data_ptr<int32_t>(), ended.data_ptr<int32_t>(),
                        ep_len ? ep_len->data_ptr<int32_t>() : nullptr, ep_rew ? ep_rew->data_ptr() : nullptr, delay.data_ptr<int32_t>(),
                        level ? level->data_ptr<int32_t>() : nullptr, (int)n_levels, stream_of(state_r)),
     "lhw_sim_step_delay");
}

// the largest delay is checked against the sim's frame_skip by the C-ABI, before its launch
void sim_draw_delay(int64_t sim, const Tensor& state_i, int64_t seed, int64_t first_env_id, const OptTensor& mask, int64_t max_delay,
                    Tensor delay) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_i.dim() == 2, "lhw: state_i must be [n_envs, state_ints]");
  const int64_t n = state_i.size(0);
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(delay, "delay", at::kInt, I.device); check_shape(delay, "delay", {n});
  if (mask) { check_cuda(*mask, "mask", at::kInt, I.device); check_shape(*mask, "mask", {n}); }
  TORCH_CHECK(max_delay >= 0 && max_delay <= INT32_MAX, "lhw: the largest delay must be a non-negative number of substeps, got ", max_delay);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_draw_delay(I.s, state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                        mask ? mask->data_ptr<int32_t>() : nullptr, (int)max_delay, delay.data_ptr<int32_t>(), stream_of(state_i)),
     "lhw_sim_draw_delay");
}

// the carried payloads (lhw_sim_step_payload / lhw_sim_draw_payload, DESIGN.md §7.10): payload [n, 4] of the sim's precision,
// (m, rx, ry, rz) per env; the optional delay [n] int32 and level [n] int32 as sim_step_delay takes them
void sim_step_payload(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& actions,
                      int64_t max_traj_len, bool autoreset, Tensor obs, const OptTensor& term_obs, Tensor reward, const OptTensor& rew_terms,
                      Tensor done, Tensor ended, const OptTensor& ep_len, const OptTensor& ep_rew, const Tensor& payload,
                      const OptTensor& delay, const OptTensor& level, int64_t n_levels) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_step(I, state_r, state_i, actions, max_traj_len, obs, term_obs, reward, rew_terms, done, ended, ep_len, ep_rew);
  check_cuda(payload, "payload", I.real, I.device); check_shape(payload, "payload", {n, 4});
  if (delay) { check_cuda(*delay, "delay", at::kInt, I.device); check_shape(*delay, "delay", {n}); }
  if (level) check_stairs(I, *level, n, n_levels);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_step_payload(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                          actions.data_ptr(), (int)max_traj_len, autoreset ? 1 : 0, obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr,
                          reward.data_ptr(), rew_terms ? rew_terms->data_ptr() : nullptr, done.data_ptr<int32_t>(), ended.data_ptr<int32_t>(),
                          ep_len ? ep_len->data_ptr<int32_t>() : nullptr, ep_rew ? ep_rew->data_ptr() : nullptr, payload.data_ptr(),
                          delay ? delay->data_ptr<int32_t>() : nullptr, level ? level->data_ptr<int32_t>() : nullptr, (int)n_levels,
                          stream_of(state_r)),
     "lhw_sim_step_payload");
}

// the largest mass and offset are checked by the C-ABI before its launch (the mass's bound of half the robot is the host's)
void sim_draw_payload(int64_t sim, const Tensor& state_i, int64_t seed, int64_t first_env_id, const OptTensor& mask, double max_mass,
                      double max_offset, Tensor payload) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_i.dim() == 2, "lhw: state_i must be [n_envs, state_ints]");
  const int64_t n = state_i.size(0);
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(payload, "payload", I.real, I.device); check_shape(payload, "payload", {n, 4});
  if (mask) { check_cuda(*mask, "mask", at::kInt, I.device); check_shape(*mask, "mask", {n}); }
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_draw_payload(I.s, state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                          mask ? mask->data_ptr<int32_t>() : nullptr, max_mass, max_offset, payload.data_ptr(), stream_of(state_i)),
     "lhw_sim_draw_payload");
}

// the motor strengths (lhw_sim_step_motor / lhw_sim_draw_motor, DESIGN.md §7.11): strength [n, NU] of the sim's precision, the
// factors of each env's actuated joints; the optional payload [n, 4], delay [n] int32 and level [n] int32 as sim_step_payload takes them
void sim_step_motor(int64_t sim, Tensor state_r, Tensor state_i, int64_t seed, int64_t first_env_id, const Tensor& actions,
                    int64_t max_traj_len, bool autoreset, Tensor obs, const OptTensor& term_obs, Tensor reward, const OptTensor& rew_terms,
                    Tensor done, Tensor ended, const OptTensor& ep_len, const OptTensor& ep_rew, const Tensor& strength,
                    const OptTensor& payload, const OptTensor& delay, const OptTensor& level, int64_t n_levels) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_r.dim() == 2, "lhw: state_r must be [n_envs, state_reals]");
  const int64_t n = state_r.size(0);
  check_step(I, state_r, state_i, actions, max_traj_len, obs, term_obs, reward, rew_terms, done, ended, ep_len, ep_rew);
  check_cuda(strength, "strength", I.real, I.device); check_shape(strength, "strength", {n, I.nact});
  if (payload) { check_cuda(*payload, "payload", I.real, I.device); check_shape(*payload, "payload", {n, 4}); }
  if (delay) { check_cuda(*delay, "delay", at::kInt, I.device); check_shape(*delay, "delay", {n}); }
  if (level) check_stairs(I, *level, n, n_levels);
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_step_motor(I.s, state_r.data_ptr(), state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                        actions.data_ptr(), (int)max_traj_len, autoreset ? 1 : 0, obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr,
                        reward.data_ptr(), rew_terms ? rew_terms->data_ptr() : nullptr, done.data_ptr<int32_t>(), ended.data_ptr<int32_t>(),
                        ep_len ? ep_len->data_ptr<int32_t>() : nullptr, ep_rew ? ep_rew->data_ptr() : nullptr, strength.data_ptr(),
                        payload ? payload->data_ptr() : nullptr, delay ? delay->data_ptr<int32_t>() : nullptr,
                        level ? level->data_ptr<int32_t>() : nullptr, (int)n_levels, stream_of(state_r)),
     "lhw_sim_step_motor");
}

// the largest deviation is checked by the C-ABI before its launch
void sim_draw_motor(int64_t sim, const Tensor& state_i, int64_t seed, int64_t first_env_id, const OptTensor& mask, double max_dev,
                    Tensor strength) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_i.dim() == 2, "lhw: state_i must be [n_envs, state_ints]");
  const int64_t n = state_i.size(0);
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(strength, "strength", I.real, I.device); check_shape(strength, "strength", {n, I.nact});
  if (mask) { check_cuda(*mask, "mask", at::kInt, I.device); check_shape(*mask, "mask", {n}); }
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_draw_motor(I.s, state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                        mask ? mask->data_ptr<int32_t>() : nullptr, max_dev, strength.data_ptr(), stream_of(state_i)),
     "lhw_sim_draw_motor");
}

// the sensor errors (lhw_sim_sense, DESIGN.md §7.12): sensor [n, 6 + NU] of the sim's precision; sel [n] int32 (the step's ended,
// a reset's mask, or None for every env); term_obs is needed after a step; draw = [O, G, E] (random mode) or None, checked by the
// C-ABI before its launch
void sim_sense(int64_t sim, const Tensor& state_i, int64_t seed, int64_t first_env_id, const OptTensor& sel, bool after_step,
               bool autoreset, std::optional<at::ArrayRef<double>> draw, Tensor sensor, Tensor obs, const OptTensor& term_obs) {
  const SimInfo I = sim_info(sim);
  TORCH_CHECK(state_i.dim() == 2, "lhw: state_i must be [n_envs, state_ints]");
  const int64_t n = state_i.size(0);
  check_cuda(state_i, "state_i", at::kInt, I.device); check_shape(state_i, "state_i", {n, I.ni});
  check_cuda(sensor, "sensor", I.real, I.device); check_shape(sensor, "sensor", {n, 6 + I.nact});
  check_cuda(obs, "obs", I.real, I.device); check_shape(obs, "obs", {n, I.nobs});
  if (term_obs) { check_cuda(*term_obs, "term_obs", I.real, I.device); check_shape(*term_obs, "term_obs", {n, I.nobs}); }
  TORCH_CHECK(!after_step || term_obs.has_value(), "lhw: sim_sense after a step needs the step's term_obs");
  if (sel) { check_cuda(*sel, "sel", at::kInt, I.device); check_shape(*sel, "sel", {n}); }
  TORCH_CHECK(!draw.has_value() || draw->size() == 3, "lhw: draw must be [O, G, E] (the largest orient, gyro and encoder offsets)");
  c10::cuda::CUDAGuard guard(I.device);
  ok(lhw_sim_sense(I.s, state_i.data_ptr<int32_t>(), (int)n, (uint32_t)seed, (uint32_t)first_env_id,
                   sel ? sel->data_ptr<int32_t>() : nullptr, after_step ? 1 : 0, autoreset ? 1 : 0, draw.has_value() ? draw->data() : nullptr,
                   sensor.data_ptr(), obs.data_ptr(), term_obs ? term_obs->data_ptr() : nullptr, stream_of(state_i)),
     "lhw_sim_sense");
}

void gae(const Tensor& rewards, const Tensor& values, const Tensor& ended, const Tensor& boot, const Tensor& last_val, Tensor returns,
         double gamma, double lam, const OptTensor& adv_partials) {
  TORCH_CHECK(rewards.dim() == 2, "lhw: rewards must be [T, N]");
  const int64_t T = rewards.size(0), N = rewards.size(1);
  const int dev = rewards.is_cuda() ? rewards.get_device() : -1;
  check_cuda(rewards, "rewards", at::kFloat, dev); check_cuda(values, "values", at::kFloat, dev); check_shape(values, "values", {T, N});
  check_cuda(ended, "ended", at::kInt, dev); check_shape(ended, "ended", {T, N});
  check_cuda(boot, "boot", at::kFloat, dev); check_shape(boot, "boot", {T, N});
  check_cuda(last_val, "last_val", at::kFloat, dev); check_shape(last_val, "last_val", {N});
  check_cuda(returns, "returns", at::kFloat, dev); check_shape(returns, "returns", {T, N});
  if (adv_partials) { check_cuda(*adv_partials, "adv_partials", at::kDouble, dev); check_shape(*adv_partials, "adv_partials", {lhw_gae_partial_words((int)N)}); }
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_gae(rewards.data_ptr<float>(), values.data_ptr<float>(), ended.data_ptr<int32_t>(), boot.data_ptr<float>(),
             last_val.data_ptr<float>(), returns.data_ptr<float>(), (int)T, (int)N, (float)gamma, (float)lam,
             adv_partials ? adv_partials->data_ptr<double>() : nullptr, stream_of(rewards)), "lhw_gae");
}

void adv_stats_from_gae(const Tensor& adv_partials, int64_t n_envs, Tensor stats) {
  const int dev = adv_partials.is_cuda() ? adv_partials.get_device() : -1;
  check_cuda(adv_partials, "adv_partials", at::kDouble, dev); check_shape(adv_partials, "adv_partials", {lhw_gae_partial_words((int)n_envs)});
  check_cuda(stats, "stats", at::kDouble, dev); check_shape(stats, "stats", {lhw_adv_stats_words()});
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_adv_stats_from_gae(adv_partials.data_ptr<double>(), (int)n_envs, stats.data_ptr<double>(), stream_of(adv_partials)), "lhw_adv_stats_from_gae");
}

void adv_stats(const Tensor& returns, const Tensor& values, Tensor stats) {
  const int dev = returns.is_cuda() ? returns.get_device() : -1;
  check_cuda(returns, "returns", at::kFloat, dev); check_cuda(values, "values", at::kFloat, dev);
  TORCH_CHECK(values.numel() == returns.numel(), "lhw: returns / values differ in size");
  check_cuda(stats, "stats", at::kDouble, dev); check_shape(stats, "stats", {lhw_adv_stats_words()});
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_adv_stats(returns.data_ptr<float>(), values.data_ptr<float>(), stats.data_ptr<double>(), returns.numel(), stream_of(returns)),
     "lhw_adv_stats");
}

void adv_apply(const Tensor& returns, const Tensor& values, Tensor adv, Tensor stats, int64_t count_total, double eps) {
  const int dev = returns.is_cuda() ? returns.get_device() : -1;
  check_cuda(returns, "returns", at::kFloat, dev); check_cuda(values, "values", at::kFloat, dev); check_cuda(adv, "adv", at::kFloat, dev);
  TORCH_CHECK(values.numel() == returns.numel() && adv.numel() == returns.numel(), "lhw: returns / values / adv differ in size");
  check_cuda(stats, "stats", at::kDouble, dev); check_shape(stats, "stats", {lhw_adv_stats_words()});
  TORCH_CHECK(count_total >= returns.numel() && count_total > 1, "lhw: count_total must be the global sample count");
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_adv_apply(returns.data_ptr<float>(), values.data_ptr<float>(), adv.data_ptr<float>(), stats.data_ptr<double>(), returns.numel(),
                   count_total, (float)eps, stream_of(returns)), "lhw_adv_apply");
}

void gather_minibatch(const Tensor& obs, const Tensor& act, const Tensor& ret, const Tensor& adv, const Tensor& idx, Tensor obs_b,
                      Tensor act_b, Tensor ret_b, Tensor adv_b) {
  TORCH_CHECK(obs.dim() == 2 && act.dim() == 2, "lhw: obs / act must be [S, dim]");
  const int64_t S = obs.size(0), od = obs.size(1), ad = act.size(1), B = idx.numel();
  const int dev = obs.is_cuda() ? obs.get_device() : -1;
  check_cuda(obs, "obs", at::kFloat, dev); check_cuda(act, "act", at::kFloat, dev); check_shape(act, "act", {S, ad});
  check_cuda(ret, "ret", at::kFloat, dev); check_cuda(adv, "adv", at::kFloat, dev);
  TORCH_CHECK(ret.numel() == S && adv.numel() == S, "lhw: ret / adv must hold one value per sample");
  check_cuda(idx, "idx", at::kLong, dev);
  check_cuda(obs_b, "obs_b", at::kFloat, dev); check_shape(obs_b, "obs_b", {B, od});
  check_cuda(act_b, "act_b", at::kFloat, dev); check_shape(act_b, "act_b", {B, ad});
  check_cuda(ret_b, "ret_b", at::kFloat, dev); check_cuda(adv_b, "adv_b", at::kFloat, dev);
  TORCH_CHECK(ret_b.numel() == B && adv_b.numel() == B, "lhw: ret_b / adv_b must hold one value per minibatch sample");
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_gather_minibatch(obs.data_ptr<float>(), act.data_ptr<float>(), ret.data_ptr<float>(), adv.data_ptr<float>(),
                          idx.data_ptr<int64_t>(), obs_b.data_ptr<float>(), act_b.data_ptr<float>(), ret_b.data_ptr<float>(),
                          adv_b.data_ptr<float>(), (int)B, (int)od, (int)ad, stream_of(obs)), "lhw_gather_minibatch");
}

// the checks of ppo_loss's tensors, shared with ppo_loss_imitation; returns the device
int check_ppo_loss(const Tensor& mu, const Tensor& old_mu, const Tensor& act, const Tensor& adv, const Tensor& ret, const Tensor& val,
                   const OptTensor& mirr, const Tensor& stds, const Tensor& g_mu, const OptTensor& g_mirr, const Tensor& g_val,
                   const Tensor& partials, const Tensor& ticket, const Tensor& out8) {
  TORCH_CHECK(mu.dim() == 2, "lhw: mu must be [B, A]");
  const int64_t B = mu.size(0), A = mu.size(1);
  const int dev = mu.is_cuda() ? mu.get_device() : -1;
  check_cuda(mu, "mu", at::kFloat, dev); check_cuda(old_mu, "old_mu", at::kFloat, dev); check_shape(old_mu, "old_mu", {B, A});
  check_cuda(act, "act", at::kFloat, dev); check_shape(act, "act", {B, A});
  check_cuda(adv, "adv", at::kFloat, dev); check_cuda(ret, "ret", at::kFloat, dev); check_cuda(val, "val", at::kFloat, dev);
  TORCH_CHECK(adv.numel() == B && ret.numel() == B && val.numel() == B, "lhw: adv / ret / val must hold one value per sample");
  check_cuda(stds, "stds", at::kFloat, dev); check_shape(stds, "stds", {A});
  check_cuda(g_mu, "g_mu", at::kFloat, dev); check_shape(g_mu, "g_mu", {B, A});
  check_cuda(g_val, "g_val", at::kFloat, dev); TORCH_CHECK(g_val.numel() == B, "lhw: g_val must hold one value per sample");
  TORCH_CHECK(mirr.has_value() == g_mirr.has_value(), "lhw: mirr and g_mirr go together");
  if (mirr) { check_cuda(*mirr, "mirr", at::kFloat, dev); check_shape(*mirr, "mirr", {B, A}); check_cuda(*g_mirr, "g_mirr", at::kFloat, dev); check_shape(*g_mirr, "g_mirr", {B, A}); }
  check_cuda(partials, "partials", at::kDouble, dev); check_shape(partials, "partials", {lhw_ppo_loss_partial_words((int)B)});
  check_cuda(ticket, "ticket", at::kInt, dev); TORCH_CHECK(ticket.numel() >= 1, "lhw: ticket is empty");
  check_cuda(out8, "out8", at::kFloat, dev); check_shape(out8, "out8", {8});
  return dev;
}

void ppo_loss(const Tensor& mu, const Tensor& old_mu, const Tensor& act, const Tensor& adv, const Tensor& ret, const Tensor& val,
              const OptTensor& mirr, const Tensor& stds, double clip, double mirror_coeff, double ent_coeff, Tensor g_mu,
              const OptTensor& g_mirr, Tensor g_val, Tensor partials, Tensor ticket, Tensor out8) {
  const int dev = check_ppo_loss(mu, old_mu, act, adv, ret, val, mirr, stds, g_mu, g_mirr, g_val, partials, ticket, out8);
  const int64_t B = mu.size(0), A = mu.size(1);
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_ppo_loss(mu.data_ptr<float>(), old_mu.data_ptr<float>(), act.data_ptr<float>(), adv.data_ptr<float>(), ret.data_ptr<float>(),
                  val.data_ptr<float>(), mirr ? mirr->data_ptr<float>() : nullptr, stds.data_ptr<float>(), (int)B, (int)A, (float)clip,
                  (float)mirror_coeff, (float)ent_coeff, g_mu.data_ptr<float>(), g_mirr ? g_mirr->data_ptr<float>() : nullptr,
                  g_val.data_ptr<float>(), partials.data_ptr<double>(), (unsigned int*)ticket.data_ptr<int>(), out8.data_ptr<float>(),
                  stream_of(mu)), "lhw_ppo_loss");
}

void ppo_loss_imitation(const Tensor& mu, const Tensor& old_mu, const Tensor& act, const Tensor& adv, const Tensor& ret, const Tensor& val,
                        const OptTensor& mirr, const Tensor& stds, const Tensor& teacher_mu, const OptTensor& mask, double clip,
                        double mirror_coeff, double ent_coeff, double imitate_coeff, Tensor g_mu, const OptTensor& g_mirr, Tensor g_val,
                        Tensor partials, Tensor ticket, Tensor out8) {
  const int dev = check_ppo_loss(mu, old_mu, act, adv, ret, val, mirr, stds, g_mu, g_mirr, g_val, partials, ticket, out8);
  const int64_t B = mu.size(0), A = mu.size(1);
  check_cuda(teacher_mu, "teacher_mu", at::kFloat, dev); check_shape(teacher_mu, "teacher_mu", {B, A});
  if (mask) { check_cuda(*mask, "mask", at::kFloat, dev); TORCH_CHECK(mask->numel() == B, "lhw: mask must hold one value per sample"); }
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_ppo_loss_imitation(mu.data_ptr<float>(), old_mu.data_ptr<float>(), act.data_ptr<float>(), adv.data_ptr<float>(),
                            ret.data_ptr<float>(), val.data_ptr<float>(), mirr ? mirr->data_ptr<float>() : nullptr, stds.data_ptr<float>(),
                            teacher_mu.data_ptr<float>(), mask ? mask->data_ptr<float>() : nullptr, (int)B, (int)A, (float)clip,
                            (float)mirror_coeff, (float)ent_coeff, (float)imitate_coeff, g_mu.data_ptr<float>(),
                            g_mirr ? g_mirr->data_ptr<float>() : nullptr, g_val.data_ptr<float>(), partials.data_ptr<double>(),
                            (unsigned int*)ticket.data_ptr<int>(), out8.data_ptr<float>(), stream_of(mu)), "lhw_ppo_loss_imitation");
}

void linear_wgrad(const Tensor& gy, const Tensor& x, Tensor gw, const OptTensor& gb, Tensor workspace) {
  TORCH_CHECK(gy.dim() == 2 && x.dim() == 2 && gy.size(0) == x.size(0), "lhw: gy [M, N] and x [M, K] must share their rows");
  const int64_t M = gy.size(0), N = gy.size(1), K = x.size(1);
  const int dev = gy.is_cuda() ? gy.get_device() : -1;
  check_cuda(gy, "gy", at::kFloat, dev); check_cuda(x, "x", at::kFloat, dev);
  check_cuda(gw, "gw", at::kFloat, dev); check_shape(gw, "gw", {N, K});
  if (gb) { check_cuda(*gb, "gb", at::kFloat, dev); check_shape(*gb, "gb", {N}); }
  check_cuda(workspace, "workspace", at::kFloat, dev);
  TORCH_CHECK(M < (1LL << 31) && N * K < (1LL << 31), "lhw: linear_wgrad operands too large");
  TORCH_CHECK(workspace.numel() >= lhw_linear_wgrad_workspace_floats((int)M, (int)N, (int)K), "lhw: linear_wgrad workspace too small");
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_linear_wgrad(gy.data_ptr<float>(), x.data_ptr<float>(), (int)M, (int)N, (int)K, gw.data_ptr<float>(),
                      gb ? gb->data_ptr<float>() : nullptr, workspace.data_ptr<float>(), stream_of(gy)), "lhw_linear_wgrad");
}

void grad_sumsq(const Tensor& grad, Tensor norm, double grad_scale) {
  const int dev = grad.is_cuda() ? grad.get_device() : -1;
  check_cuda(grad, "grad", at::kFloat, dev); check_cuda(norm, "norm", at::kFloat, dev);
  TORCH_CHECK(norm.numel() >= 1, "lhw: norm scratch is empty");
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_grad_sumsq(grad.data_ptr<float>(), norm.data_ptr<float>(), grad.numel(), (float)grad_scale, stream_of(grad)), "lhw_grad_sumsq");
}

void clip_adam_dev(Tensor param, const Tensor& grad, Tensor exp_avg, Tensor exp_avg_sq, const Tensor& norm, Tensor step_dev, double lr,
                   double beta1, double beta2, double eps, double max_norm, double grad_scale) {
  const int dev = param.is_cuda() ? param.get_device() : -1;
  const int64_t n = param.numel();
  check_cuda(param, "param", at::kFloat, dev); check_cuda(grad, "grad", at::kFloat, dev); check_cuda(exp_avg, "exp_avg", at::kFloat, dev);
  check_cuda(exp_avg_sq, "exp_avg_sq", at::kFloat, dev); check_cuda(norm, "norm", at::kFloat, dev); check_cuda(step_dev, "step_dev", at::kInt, dev);
  TORCH_CHECK(grad.numel() == n && exp_avg.numel() == n && exp_avg_sq.numel() == n, "lhw: param / grad / moments differ in size");
  TORCH_CHECK(norm.numel() >= 1 && step_dev.numel() >= 1, "lhw: norm / step scratch is empty");
  c10::cuda::CUDAGuard guard(dev);
  ok(lhw_clip_adam_dev(param.data_ptr<float>(), grad.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(),
                       norm.data_ptr<float>(), n, step_dev.data_ptr<int>(), (float)lr, (float)beta1, (float)beta2, (float)eps,
                       (float)max_norm, (float)grad_scale, stream_of(param)), "lhw_clip_adam_dev");
}

void fused_exchange(int64_t comm, Tensor param, Tensor exp_avg, Tensor exp_avg_sq, int64_t n_actor, double lr, double beta1, double beta2,
                    double eps, double max_norm) {
  TORCH_CHECK(comm != 0, "lhw: null comm handle");
  lhw_comm* c = reinterpret_cast<lhw_comm*>(comm);
  const int64_t n = lhw_comm_size(c);
  const int dev = lhw_comm_device(c);
  check_cuda(param, "param", at::kFloat, dev); check_shape(param, "param", {n});
  check_cuda(exp_avg, "exp_avg", at::kFloat, dev); check_shape(exp_avg, "exp_avg", {n});
  check_cuda(exp_avg_sq, "exp_avg_sq", at::kFloat, dev); check_shape(exp_avg_sq, "exp_avg_sq", {n});
  TORCH_CHECK(n_actor >= 0 && n_actor <= n, "lhw: n_actor out of range");
  c10::cuda::CUDAGuard guard(dev);
  const int rc = lhw_fused_allreduce_clip_adam(c, param.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(), n_actor, n,
                                               (float)lr, (float)beta1, (float)beta2, (float)eps, (float)max_norm, stream_of(param));
  TORCH_CHECK(rc == 0, "lhw: lhw_fused_allreduce_clip_adam failed (rc=", rc, "): ", lhw_comm_last_error());
}

void fused_exchange_adaptive(int64_t comm, Tensor param, Tensor exp_avg, Tensor exp_avg_sq, int64_t n_actor, const Tensor& kl, Tensor lr,
                             double desired_kl, double beta1, double beta2, double eps, double max_norm) {
  TORCH_CHECK(comm != 0, "lhw: null comm handle");
  lhw_comm* c = reinterpret_cast<lhw_comm*>(comm);
  const int64_t n = lhw_comm_size(c);
  const int dev = lhw_comm_device(c);
  check_cuda(param, "param", at::kFloat, dev); check_shape(param, "param", {n});
  check_cuda(exp_avg, "exp_avg", at::kFloat, dev); check_shape(exp_avg, "exp_avg", {n});
  check_cuda(exp_avg_sq, "exp_avg_sq", at::kFloat, dev); check_shape(exp_avg_sq, "exp_avg_sq", {n});
  check_cuda(kl, "kl", at::kFloat, dev);
  TORCH_CHECK(kl.numel() == 1 && kl.dim() <= 1, "lhw: kl has shape ", kl.sizes(), ", expected one float ([] or [1])");
  check_cuda(lr, "lr", at::kDouble, dev); check_shape(lr, "lr", {1});
  TORCH_CHECK(n_actor >= 0 && n_actor <= n, "lhw: n_actor out of range");
  TORCH_CHECK(desired_kl > 0.0, "lhw: desired_kl must be > 0, got ", desired_kl);
  c10::cuda::CUDAGuard guard(dev);
  const int rc = lhw_fused_allreduce_clip_adam_adaptive(c, param.data_ptr<float>(), exp_avg.data_ptr<float>(), exp_avg_sq.data_ptr<float>(),
                                                        n_actor, n, kl.data_ptr<float>(), lr.data_ptr<double>(), desired_kl, (float)beta1,
                                                        (float)beta2, (float)eps, (float)max_norm, stream_of(param));
  TORCH_CHECK(rc == 0, "lhw: lhw_fused_allreduce_clip_adam_adaptive failed (rc=", rc, "): ", lhw_comm_last_error());
}

}  // namespace

TORCH_LIBRARY(lhw, m) {
  m.def("sim_reset(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor? mask, bool fresh, Tensor(c!) obs) -> ()");
  m.def("sim_step(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor actions, int max_traj_len, "
        "bool autoreset, Tensor(c!) obs, Tensor(d!)? term_obs, Tensor(e!) reward, Tensor(f!)? rew_terms, Tensor(g!) done, Tensor(h!) ended, "
        "Tensor(i!)? ep_len, Tensor(j!)? ep_rew) -> ()");
  m.def("sim_render(int sim, Tensor state_r, Tensor state_i, Tensor env_ids, int width, int height, float dx, float dy, float z, "
        "float distance, float azimuth, float elevation, float fovy, Tensor(a!) rgb) -> ()");
  m.def("sim_eval_accumulate(int sim, Tensor state_r, Tensor state_i, Tensor reward, Tensor rew_terms, Tensor done, Tensor(a!) acc) -> ()");
  m.def("sim_push(int sim, Tensor(a!) state_r, Tensor state_i, int seed, int first_env_id, Tensor? ended, float vel, int interval_steps, "
        "Tensor? d) -> ()");
  m.def("sim_set_command(int sim, Tensor(a!) state_r, Tensor(b!) state_i, Tensor mode, Tensor ref, Tensor(c!) obs) -> ()");
  m.def("sim_command_accumulate(int sim, Tensor state_r, Tensor done, Tensor(a!) acc) -> ()");
  m.def("sim_reset_footsteps(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor mode, Tensor value, "
        "bool fresh, Tensor(c!) obs) -> ()");
  m.def("sim_step_stairs(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor actions, int max_traj_len, "
        "bool autoreset, Tensor(c!) obs, Tensor(d!)? term_obs, Tensor(e!) reward, Tensor(f!)? rew_terms, Tensor(g!) done, Tensor(h!) ended, "
        "Tensor(i!)? ep_len, Tensor(j!)? ep_rew, Tensor(k!) level, int n_levels) -> ()");
  m.def("sim_reset_stairs(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor? mask, bool fresh, "
        "Tensor(c!) obs, Tensor level, int n_levels) -> ()");
  m.def("sim_step_delay(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor actions, int max_traj_len, "
        "bool autoreset, Tensor(c!) obs, Tensor(d!)? term_obs, Tensor(e!) reward, Tensor(f!)? rew_terms, Tensor(g!) done, Tensor(h!) ended, "
        "Tensor(i!)? ep_len, Tensor(j!)? ep_rew, Tensor delay, Tensor(k!)? level=None, int n_levels=0) -> ()");
  m.def("sim_draw_delay(int sim, Tensor state_i, int seed, int first_env_id, Tensor? mask, int max_delay, Tensor(a!) delay) -> ()");
  m.def("sim_step_payload(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor actions, int max_traj_len, "
        "bool autoreset, Tensor(c!) obs, Tensor(d!)? term_obs, Tensor(e!) reward, Tensor(f!)? rew_terms, Tensor(g!) done, Tensor(h!) ended, "
        "Tensor(i!)? ep_len, Tensor(j!)? ep_rew, Tensor payload, Tensor? delay=None, Tensor(k!)? level=None, int n_levels=0) -> ()");
  m.def("sim_draw_payload(int sim, Tensor state_i, int seed, int first_env_id, Tensor? mask, float max_mass, float max_offset, "
        "Tensor(a!) payload) -> ()");
  m.def("sim_step_motor(int sim, Tensor(a!) state_r, Tensor(b!) state_i, int seed, int first_env_id, Tensor actions, int max_traj_len, "
        "bool autoreset, Tensor(c!) obs, Tensor(d!)? term_obs, Tensor(e!) reward, Tensor(f!)? rew_terms, Tensor(g!) done, Tensor(h!) ended, "
        "Tensor(i!)? ep_len, Tensor(j!)? ep_rew, Tensor strength, Tensor? payload=None, Tensor? delay=None, Tensor(k!)? level=None, "
        "int n_levels=0) -> ()");
  m.def("sim_draw_motor(int sim, Tensor state_i, int seed, int first_env_id, Tensor? mask, float max_dev, Tensor(a!) strength) -> ()");
  m.def("sim_sense(int sim, Tensor state_i, int seed, int first_env_id, Tensor? sel, bool after_step, bool autoreset, float[]? draw, "
        "Tensor(a!) sensor, Tensor(b!) obs, Tensor(c!)? term_obs) -> ()");
  m.def("gae(Tensor rewards, Tensor values, Tensor ended, Tensor boot, Tensor last_val, Tensor(a!) returns, float gamma, float lam, "
        "Tensor(b!)? adv_partials) -> ()");
  m.def("adv_stats_from_gae(Tensor adv_partials, int n_envs, Tensor(a!) stats) -> ()");
  m.def("adv_stats(Tensor returns, Tensor values, Tensor(a!) stats) -> ()");
  m.def("adv_apply(Tensor returns, Tensor values, Tensor(a!) adv, Tensor(b!) stats, int count_total, float eps) -> ()");
  m.def("gather_minibatch(Tensor obs, Tensor act, Tensor ret, Tensor adv, Tensor idx, Tensor(a!) obs_b, Tensor(b!) act_b, Tensor(c!) ret_b, "
        "Tensor(d!) adv_b) -> ()");
  m.def("ppo_loss(Tensor mu, Tensor old_mu, Tensor act, Tensor adv, Tensor ret, Tensor val, Tensor? mirr, Tensor stds, float clip, "
        "float mirror_coeff, float ent_coeff, Tensor(a!) g_mu, Tensor(b!)? g_mirr, Tensor(c!) g_val, Tensor(d!) partials, Tensor(e!) ticket, "
        "Tensor(f!) out8) -> ()");
  m.def("ppo_loss_imitation(Tensor mu, Tensor old_mu, Tensor act, Tensor adv, Tensor ret, Tensor val, Tensor? mirr, Tensor stds, "
        "Tensor teacher_mu, Tensor? mask, float clip, float mirror_coeff, float ent_coeff, float imitate_coeff, Tensor(a!) g_mu, "
        "Tensor(b!)? g_mirr, Tensor(c!) g_val, Tensor(d!) partials, Tensor(e!) ticket, Tensor(f!) out8) -> ()");
  m.def("linear_wgrad(Tensor gy, Tensor x, Tensor(a!) gw, Tensor(b!)? gb, Tensor(c!) workspace) -> ()");
  m.def("grad_sumsq(Tensor grad, Tensor(a!) norm, float grad_scale) -> ()");
  m.def("clip_adam_dev(Tensor(a!) param, Tensor grad, Tensor(b!) exp_avg, Tensor(c!) exp_avg_sq, Tensor norm, Tensor(d!) step_dev, float lr, "
        "float beta1, float beta2, float eps, float max_norm, float grad_scale) -> ()");
  m.def("fused_exchange(int comm, Tensor(a!) param, Tensor(b!) exp_avg, Tensor(c!) exp_avg_sq, int n_actor, float lr, float beta1, float beta2, "
        "float eps, float max_norm) -> ()");
  m.def("fused_exchange_adaptive(int comm, Tensor(a!) param, Tensor(b!) exp_avg, Tensor(c!) exp_avg_sq, int n_actor, Tensor kl, "
        "Tensor(d!) lr, float desired_kl, float beta1, float beta2, float eps, float max_norm) -> ()");
}

// CompositeExplicitAutograd: the checks must also reject CPU tensors with OUR message (a CUDA-only registration would answer
// "no kernel for the CPU backend"); there is no CPU implementation behind them.
TORCH_LIBRARY_IMPL(lhw, CompositeExplicitAutograd, m) {
  m.impl("sim_reset", &sim_reset);
  m.impl("sim_step", &sim_step);
  m.impl("sim_render", &sim_render);
  m.impl("sim_eval_accumulate", &sim_eval_accumulate);
  m.impl("sim_push", &sim_push);
  m.impl("sim_set_command", &sim_set_command);
  m.impl("sim_command_accumulate", &sim_command_accumulate);
  m.impl("sim_reset_footsteps", &sim_reset_footsteps);
  m.impl("sim_step_stairs", &sim_step_stairs);
  m.impl("sim_reset_stairs", &sim_reset_stairs);
  m.impl("sim_step_delay", &sim_step_delay);
  m.impl("sim_draw_delay", &sim_draw_delay);
  m.impl("sim_step_payload", &sim_step_payload);
  m.impl("sim_draw_payload", &sim_draw_payload);
  m.impl("sim_step_motor", &sim_step_motor);
  m.impl("sim_draw_motor", &sim_draw_motor);
  m.impl("sim_sense", &sim_sense);
  m.impl("gae", &gae);
  m.impl("adv_stats_from_gae", &adv_stats_from_gae);
  m.impl("adv_stats", &adv_stats);
  m.impl("adv_apply", &adv_apply);
  m.impl("gather_minibatch", &gather_minibatch);
  m.impl("ppo_loss", &ppo_loss);
  m.impl("ppo_loss_imitation", &ppo_loss_imitation);
  m.impl("linear_wgrad", &linear_wgrad);
  m.impl("grad_sumsq", &grad_sumsq);
  m.impl("clip_adam_dev", &clip_adam_dev);
  m.impl("fused_exchange", &fused_exchange);
  m.impl("fused_exchange_adaptive", &fused_exchange_adaptive);
}
