// tests/emu/sim_emu_variants.cpp — TEST HARNESS ONLY.  The CPU emulation of sim_emu.cpp, entered through model_pack.h's
// with_variant, so that every variant of sim_core.h's LHW_FOR_EACH_VARIANT runs on the host (sim_emu.cpp's own entry points
// know the first four).  The entry points are sim_emu.cpp's, named emuv_* (tests/emu/emu_variants.py).
#include "sim_emu.cpp"

#define VDISPATCH(h, prec, CALL)                                             \
  with_variant((h)->var, (prec), [&](auto v_) {                              \
    using V_ = decltype(v_);                                                 \
    CALL(typename V_::real, V_::NJ, V_::TK);                                 \
  })

extern "C" {
void* emuv_create(const double* flat, int n, int precision) {
  Handle tmp{(int)flat[0], nullptr};
  void* p = nullptr;
#define CALL(R, J, T) p = create<R, J, T>(flat, n)
  if (VDISPATCH(&tmp, precision, CALL) != 0 || !p) return nullptr;
#undef CALL
  return new Handle{tmp.var, p};
}
int emuv_state_words(void* hv) {
  int out = 0;
#define CALL(R, J, T) out = Dims<double, J, T>::NSTATE_R
  VDISPATCH((Handle*)hv, 64, CALL);
#undef CALL
  return out;
}
int emuv_obs_dim(void* hv) {
  int out = 0;
#define CALL(R, J, T) out = Dims<double, J, T>::NOBS
  VDISPATCH((Handle*)hv, 64, CALL);
#undef CALL
  return out;
}
int emuv_work_bytes(void* hv, int precision) {
  int out = 0;
#define CALL(R, J, T) out = (int)sizeof(Work<R, J, T>)
  VDISPATCH((Handle*)hv, precision, CALL);
#undef CALL
  return out;
}
void emuv_reset(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, void* obs, int fresh) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) reset_all<R, J, T>(h->p, (R*)sr, si, n, seed, first_id, (R*)obs, fresh)
  VDISPATCH(h, precision, CALL);
#undef CALL
}
void emuv_step(void* hv, int precision, void* sr, int32_t* si, int n, uint32_t seed, uint32_t first_id, const void* actions,
               int max_traj_len, int autoreset, void* obs, void* term_obs, void* reward, void* rew_terms, int32_t* done,
               int32_t* ended, int32_t* ep_len, void* ep_rew) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T)                                                                                          \
  step_all<R, J, T>(h->p, (R*)sr, si, n, seed, first_id, (const R*)actions, max_traj_len, autoreset, (R*)obs,    \
                    (R*)term_obs, (R*)reward, (R*)rew_terms, done, ended, ep_len, (R*)ep_rew)
  VDISPATCH(h, precision, CALL);
#undef CALL
}
void emuv_substep64(void* hv, double* sr, int32_t* si, const double* ctrl, int nsteps) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) substeps64<J, T>(h->p, sr, si, ctrl, nsteps)
  VDISPATCH(h, 64, CALL);
#undef CALL
}
void emuv_set_step_height(void* hv, int precision, double h_) { emu_set_step_height(hv, precision, h_); }
}
