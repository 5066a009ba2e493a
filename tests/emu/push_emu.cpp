// tests/emu/push_emu.cpp — TEST HARNESS ONLY.  The root-velocity push of the product (sim_core.h push_env, the body of lhw_sim_push's
// kernel) compiled for the host, for every variant of LHW_FOR_EACH_VARIANT through model_pack.h's with_variant; one call = one
// launch over n envs.  tests/test_push.py feeds it records of sim_emu_variants.cpp.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/model_pack.h"

using namespace lhw;

extern "C" {
// 0, or -1 for an unknown variant code; pushed[i] = 1 where env i was pushed
int push_emu(int variant, int precision, void* sr, const int32_t* si, int n, uint32_t seed, uint32_t first_id, const int32_t* ended,
             double vel, int interval, const void* d, int32_t* pushed) {
  return with_variant(variant, precision, [&](auto v) {
    using V = decltype(v);
    using R = typename V::real;
    constexpr int NR = Dims<R, V::NJ, V::TK>::NSTATE_R;
    for (int i = 0; i < n; i++)
      pushed[i] = push_env<R, V::NJ, V::TK>((R*)sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, seed, first_id + i, ended ? ended[i] : 0,
                                            vel, interval, d ? (const R*)d + 2 * (size_t)i : nullptr);
  });
}
}
