// tests/emu/sensor_emu.cpp — TEST HARNESS ONLY.  The sensor pass (sim_core.h sensor_env, the body of lhw_sim_sense's kernel)
// compiled for the host, next to sim_emu_variants.cpp's entry points (whose step and reset the closed-loop tests run before it);
// one call = one launch over n envs, every (env, group) in turn.  tests/test_sensor_errors.py drives it.
#include "sim_emu_variants.cpp"

template <class real>
static void sense_all(const int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* sel, int after_step, int autoreset,
                      const double* draw, int nrobot, int nu, int obs_dim, real* sensor, real* obs, real* term_obs) {
  const int ngroup = (nrobot + 3) / 4;
  for (int i = 0; i < n; i++)
    for (int g = 0; g < ngroup; g++)
      sensor_env<real>(si + (size_t)i * NSTATE_I, seed, first_id + i, g, sel ? sel[i] : 1, after_step, autoreset, draw != nullptr,
                       draw ? draw[0] : 0.0, draw ? draw[1] : 0.0, draw ? draw[2] : 0.0, nrobot, nu,
                       sensor + (size_t)(6 + nu) * i, obs + (size_t)obs_dim * i, term_obs ? term_obs + (size_t)obs_dim * i : nullptr);
}

extern "C" {
void sensor_emu_sense(int precision, const int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* sel, int after_step,
                      int autoreset, const double* draw, int nrobot, int nu, int obs_dim, void* sensor, void* obs, void* term_obs) {
  if (precision == 64)
    sense_all<double>(si, n, seed, first_id, sel, after_step, autoreset, draw, nrobot, nu, obs_dim, (double*)sensor, (double*)obs,
                      (double*)term_obs);
  else
    sense_all<float>(si, n, seed, first_id, sel, after_step, autoreset, draw, nrobot, nu, obs_dim, (float*)sensor, (float*)obs,
                     (float*)term_obs);
}
}
