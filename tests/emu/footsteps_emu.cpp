// tests/emu/footsteps_emu.cpp — TEST HARNESS ONLY.  The reset with a chosen footstep plan (the body of lhw_sim_reset_footsteps's
// kernel, reset_kernel<real, 6, 1, true>: sim_core.h env_reset<..., PLAN = true>) compiled for the host, next to sim_emu.cpp's
// entry points, whose handles it takes; one call = one launch over n envs.  tests/test_footsteps.py drives it.
#include "sim_emu.cpp"

template <class real>
static void reset_footsteps_all(void* p, real* sr, int32_t* si, int n_envs, uint32_t seed, uint32_t first_id, const int32_t* mode,
                                const real* value, real* obs, int fresh) {
  auto* e = (Emu<real, 6, 1>*)p;
  constexpr int NR = Dims<real, 6, 1>::NSTATE_R, NOBS = Work<real, 6, 1>::NOBS;
  for (int i = 0; i < n_envs; i++) {
    if (mode[i] < ST_CURVED || mode[i] > ST_FORWARD) continue;   // the kernel's skipped rows
    if (fresh) {
      for (int k = 0; k < NR; k++) sr[(size_t)i * NR + k] = 0;
      for (int k = 0; k < NSTATE_I; k++) si[(size_t)i * NSTATE_I + k] = 0;
    }
    load_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, first_id + i);
    env_reset<real, 6, 1, true>(e->work, e->model, seed, StepPlan<real>{mode[i], value[i]});
    store_state(e->work, sr + (size_t)i * NR, si + (size_t)i * NSTATE_I);
    for (int k = 0; k < NOBS; k++) obs[(size_t)i * NOBS + k] = e->work.obs[k];
  }
}

extern "C" {
// 0, or -2 for a handle that is not jvrc_step
int footsteps_emu_reset(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* mode,
                        const void* value, void* obs, int fresh) {
  Handle* h = (Handle*)hv;
  if (h->var != 106) return -2;
  if (precision == 64) reset_footsteps_all<double>(h->p, (double*)sr, si, n, seed, first_id, mode, (const double*)value, (double*)obs, fresh);
  else reset_footsteps_all<float>(h->p, (float*)sr, si, n, seed, first_id, mode, (const float*)value, (float*)obs, fresh);
  return 0;
}
}
