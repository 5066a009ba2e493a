// tests/emu/motor_emu.cpp — TEST HARNESS ONLY.  The motor step (the body of lhw_sim_step_motor's kernels,
// step_kernel<real, NJ, TK, STAIRS, true, true, true>: sim_core.h env_step<..., DELAY = true, PAYLOAD = true, MOTOR = true>) and the
// random draw (sim_core.h motor_draw_env, the body of lhw_sim_draw_motor's kernel) compiled for the host, for every variant of
// LHW_FOR_EACH_VARIANT, next to sim_emu_variants.cpp's entry points, whose handles they take; one call = one launch over n envs.
// tests/test_motor_strength.py drives it.
#include "sim_emu_variants.cpp"

template <class real, int NJ, int TK, bool STAIRS>
static void step_motor_all(void* p, real* sr, int32_t* si, int n_envs, uint32_t seed, uint32_t first_id, const real* actions,
                           int max_traj_len, int autoreset, real* obs, real* term_obs, real* reward, real* rew_terms, int32_t* done,
                           int32_t* ended, int32_t* ep_len, real* ep_rew, const real* strength, const real* payload,
                           const int32_t* delay, int32_t* level, int n_levels) {
  auto* e = (Emu<real, NJ, TK>*)p;
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NOBS = Work<real, NJ, TK>::NOBS, NU = 2 * NJ;
  for (int i = 0; i < n_envs; i++) {
    load_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, first_id + i);
    // as step_kernel<..., DELAY, PAYLOAD, MOTOR> reads them
    const int d = delay ? action_delay_clamp(delay[i], e->model.frame_skip) : 0;
    Payload<real> pl = {};
    if (payload) {
      const real* q = payload + 4 * (size_t)i;
      pl = {q[0], {q[1], q[2], q[3]}};
    }
    env_step<real, NJ, TK, STAIRS, true, true, true>(e->work, e->model, actions + (size_t)i * NU, seed, max_traj_len, autoreset, 0, 1,
                                                     obs + (size_t)i * NOBS, term_obs + (size_t)i * NOBS, reward + i,
                                                     rew_terms + (size_t)i * NREW, done + i, ended + i, ep_len + i, ep_rew + i,
                                                     STAIRS ? level + i : nullptr, n_levels, d, pl, strength + (size_t)i * NU);
    store_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I);
  }
}

extern "C" {
// payload and delay may be NULL (mass 0, delay 0); level != NULL: the stair curriculum as well (jvrc_step only; -2 for another
// variant)
int motor_emu_step(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const void* actions,
                   int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
                   int32_t* ended, int32_t* ep_len, void* ep_rew, const void* strength, const void* payload, const int32_t* delay,
                   int32_t* level, int n_levels) {
  Handle* h = (Handle*)hv;
  if (level) {
    if (h->var != 106) return -2;
#define CALL(R)                                                                                                                    \
  step_motor_all<R, 6, 1, true>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs,          \
                                (R*)term_obs, (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew, (const R*)strength,       \
                                (const R*)payload, delay, level, n_levels)
    if (precision == 64) CALL(double);
    else CALL(float);
#undef CALL
    return 0;
  }
#define CALL(R, J, T)                                                                                                              \
  step_motor_all<R, J, T, false>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs,         \
                                 (R*)term_obs, (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew, (const R*)strength,      \
                                 (const R*)payload, delay, nullptr, 0)
  VDISPATCH(h, precision, CALL);
#undef CALL
  return 0;
}

void motor_emu_draw(int precision, const int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* mask, double max_dev,
                    int nu, void* strength) {
  for (int i = 0; i < n; i++) {
    if (precision == 64)
      motor_draw_env<double>(si + (size_t)i * NSTATE_I, seed, first_id + i, mask ? mask[i] : 1, max_dev, nu,
                             (double*)strength + (size_t)nu * i);
    else
      motor_draw_env<float>(si + (size_t)i * NSTATE_I, seed, first_id + i, mask ? mask[i] : 1, max_dev, nu,
                            (float*)strength + (size_t)nu * i);
  }
}
}
