// tests/dev/substep_emu.cpp — TEST HARNESS ONLY.  The host twin of tests/dev/substep_dev.cu: load_state -> substep x nsub ->
// store_state of the step kernel source compiled for the host with LHW_CPU_EMU (the 32 lanes of a warp run one after another),
// substep s with last = (s == nsub - 1) and chained = (s > 0) as env_step runs them, for every variant at both precisions.
// The same entry points as the device harness, with emu_ in front and no warps per block; tests/test_substep_harness.py holds
// it to the oracle without a GPU.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/model_pack.h"
#include "substep_record.h"

#include <vector>

using namespace lhw;

namespace {

struct Harness {
  int code, precision;
  std::vector<double> flat;
};

template <class real, int NJ, int TK>
int run(const Harness* h, int n, int nsub, void* sr_v, int32_t* si, const void* ctrl_v, void* work_v) {
  using W = Work<real, NJ, TK>;
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NU = 2 * NJ;
  if (n < 1 || nsub < 1) return -2;
  std::vector<Model<real, NJ, TK>> m(1);
  std::vector<real> plans((size_t)MAXPLAN * PLAN_STRIDE);
  if (fill_model(m[0], h->flat.data(), (int)h->flat.size(), plans.data())) return -4;
  m[0].plans = plans.data();
  real* sr = (real*)sr_v;
  const real* ctrl = (const real*)ctrl_v;
  W* wout = (W*)work_v;
  std::vector<W> wv(1);
  W& w = wv[0];
  for (int p = 0; p < n; p++) {
    memset(&w, 0, sizeof(W));
    load_state<real, NJ, TK>(w, sr + (size_t)p * NR, si + (size_t)p * NSTATE_I, (uint32_t)p);
    for (int l = 0; l < NU; l++) w.ctrl[l] = ctrl[(size_t)p * NU + l];
    for (int s = 0; s < nsub; s++) substep<real, NJ, TK>(w, m[0], s == nsub - 1, 0, s > 0);
    store_state<real, NJ, TK>(w, sr + (size_t)p * NR, si + (size_t)p * NSTATE_I);
    memcpy(&wout[p], &w, sizeof(W));
  }
  return 0;
}

}  // namespace

extern "C" {
void* emu_substep_create(const double* flat, int n_flat, int precision) {
  long long probe[substep_record::NFIELDS];
  if (n_flat < 1 || substep_record::layout_any((int)flat[0], precision, probe)) return nullptr;
  return new Harness{(int)flat[0], precision, std::vector<double>(flat, flat + n_flat)};
}

void emu_substep_destroy(void* hv) { delete (Harness*)hv; }

int emu_substeps(void* hv, int n, int nsub, void* sr, int32_t* si, const void* ctrl, void* work) {
  const Harness* h = (const Harness*)hv;
  int rc = -1;
  substep_record::dispatch(h->code, h->precision, [&](auto v) {
    using V = decltype(v);
    rc = run<typename V::real, V::NJ, V::TK>(h, n, nsub, sr, si, ctrl, work);
  });
  return rc;
}

int emu_substep_layout(int code, int precision, long long* out) { return substep_record::layout_any(code, precision, out); }
}
