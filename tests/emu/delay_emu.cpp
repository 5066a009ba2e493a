// tests/emu/delay_emu.cpp — TEST HARNESS ONLY.  The action delay's step (the body of lhw_sim_step_delay's kernels,
// step_kernel<real, NJ, TK, STAIRS, true>: sim_core.h env_step<..., DELAY = true>) and the random draw (sim_core.h delay_draw_env,
// the body of lhw_sim_draw_delay's kernel) compiled for the host, for every variant of LHW_FOR_EACH_VARIANT, next to
// sim_emu_variants.cpp's entry points, whose handles they take; one call = one launch over n envs.  tests/test_action_delay.py
// drives it.
#include "sim_emu_variants.cpp"

template <class real, int NJ, int TK, bool STAIRS>
static void step_delay_all(void* p, real* sr, int32_t* si, int n_envs, uint32_t seed, uint32_t first_id, const real* actions,
                           int max_traj_len, int autoreset, real* obs, real* term_obs, real* reward, real* rew_terms, int32_t* done,
                           int32_t* ended, int32_t* ep_len, real* ep_rew, const int32_t* delay, int32_t* level, int n_levels) {
  auto* e = (Emu<real, NJ, TK>*)p;
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NOBS = Work<real, NJ, TK>::NOBS, NU = 2 * NJ;
  for (int i = 0; i < n_envs; i++) {
    load_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, first_id + i);
    const int d = action_delay_clamp(delay[i], e->model.frame_skip);   // as step_kernel<..., DELAY> reads it
    env_step<real, NJ, TK, STAIRS, true>(e->work, e->model, actions + (size_t)i * NU, seed, max_traj_len, autoreset, 0, 1,
                                         obs + (size_t)i * NOBS, term_obs + (size_t)i * NOBS, reward + i, rew_terms + (size_t)i * NREW,
                                         done + i, ended + i, ep_len + i, ep_rew + i, STAIRS ? level + i : nullptr, n_levels, d);
    store_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I);
  }
}

extern "C" {
// level != NULL: the stair curriculum as well (jvrc_step only; -2 for another variant)
int delay_emu_step(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const void* actions,
                   int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                   int32_t* ended, int32_t* ep_len, void* ep_rew, const int32_t* delay, int32_t* level, int n_levels) {
  Handle* h = (Handle*)hv;
  if (level) {
    if (h->var != 106) return -2;
#define CALL(R)                                                                                                                    \
  step_delay_all<R, 6, 1, true>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs,          \
                                (R*)term_obs, (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew, delay, level, n_levels)
    if (precision == 64) CALL(double);
    else CALL(float);
#undef CALL
    return 0;
  }
#define CALL(R, J, T)                                                                                                              \
  step_delay_all<R, J, T, false>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs,         \
                                 (R*)term_obs, (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew, delay, nullptr, 0)
  VDISPATCH(h, precision, CALL);
#undef CALL
  return 0;
}

void delay_emu_draw(const int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* mask, int max_delay, int32_t* delay) {
  for (int i = 0; i < n; i++) delay_draw_env(si + (size_t)i * NSTATE_I, seed, first_id + i, mask ? mask[i] : 1, max_delay, delay + i);
}
}
