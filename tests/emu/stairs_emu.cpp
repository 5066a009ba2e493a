// tests/emu/stairs_emu.cpp — TEST HARNESS ONLY.  The stair curriculum's step and reset (the bodies of lhw_sim_step_stairs's and
// lhw_sim_reset_stairs's kernels, step_kernel<real, 6, 1, true> and reset_kernel<real, 6, 1, false, true>: sim_core.h
// env_step<..., STAIRS = true> and env_reset<..., STAIRS = true>) compiled for the host, next to sim_emu.cpp's entry points, whose
// handles they take; one call = one launch over n envs.  tests/test_stair_curriculum.py drives it.
#include "sim_emu.cpp"

template <class real>
static void reset_stairs_all(void* p, real* sr, int32_t* si, int n_envs, uint32_t seed, uint32_t first_id, const int32_t* mask,
                             const int32_t* level, int n_levels, real* obs, int fresh) {
  auto* e = (Emu<real, 6, 1>*)p;
  constexpr int NR = Dims<real, 6, 1>::NSTATE_R, NOBS = Work<real, 6, 1>::NOBS;
  for (int i = 0; i < n_envs; i++) {
    if (mask && !mask[i]) continue;
    if (fresh) {
      for (int k = 0; k < NR; k++) sr[(size_t)i * NR + k] = 0;
      for (int k = 0; k < NSTATE_I; k++) si[(size_t)i * NSTATE_I + k] = 0;
    }
    load_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, first_id + i);
    const real stair = stair_level_height<real>(stair_level_clamp(level[i], n_levels));   // as reset_kernel<..., STAIRS> reads it
    env_reset<real, 6, 1, false, true>(e->work, e->model, seed, StepPlan<real>{}, stair);
    store_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I);
    for (int k = 0; k < NOBS; k++) obs[(size_t)i * NOBS + k] = e->work.obs[k];
  }
}

template <class real>
static void step_stairs_all(void* p, real* sr, int32_t* si, int n_envs, uint32_t seed, uint32_t first_id, const real* actions,
                            int max_traj_len, int autoreset, real* obs, real* term_obs, real* reward, real* rew_terms, int32_t* done,
                            int32_t* ended, int32_t* ep_len, real* ep_rew, int32_t* level, int n_levels) {
  auto* e = (Emu<real, 6, 1>*)p;
  constexpr int NR = Dims<real, 6, 1>::NSTATE_R, NOBS = Work<real, 6, 1>::NOBS, NU = 12;
  for (int i = 0; i < n_envs; i++) {
    load_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, first_id + i);
    env_step<real, 6, 1, true>(e->work, e->model, actions + (size_t)i * NU, seed, max_traj_len, autoreset, 0, 1, obs + (size_t)i * NOBS,
                               term_obs + (size_t)i * NOBS, reward + i, rew_terms + (size_t)i * NREW, done + i, ended + i, ep_len + i,
                               ep_rew + i, level + i, n_levels);
    store_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I);
  }
}

extern "C" {
// 0, or -2 for a handle that is not jvrc_step
int stairs_emu_reset(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* mask,
                     const int32_t* level, int n_levels, void* obs, int fresh) {
  Handle* h = (Handle*)hv;
  if (h->var != 106) return -2;
  if (precision == 64) reset_stairs_all<double>(h->p, (double*)sr, si, n, seed, first_id, mask, level, n_levels, (double*)obs, fresh);
  else reset_stairs_all<float>(h->p, (float*)sr, si, n, seed, first_id, mask, level, n_levels, (float*)obs, fresh);
  return 0;
}

int stairs_emu_step(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const void* actions,
                    int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                    int32_t* ended, int32_t* ep_len, void* ep_rew, int32_t* level, int n_levels) {
  Handle* h = (Handle*)hv;
  if (h->var != 106) return -2;
#define CALL(R)                                                                                                                    \
  step_stairs_all<R>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs, (R*)term_obs,       \
                     (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew, level, n_levels)
  if (precision == 64) CALL(double);
  else CALL(float);
#undef CALL
  return 0;
}
}
