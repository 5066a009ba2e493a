// tests/emu/eval_emu.cpp — TEST HARNESS ONLY.  The evaluation accumulator of the product (sim_core.h eval_accumulate_env, the
// body of lhw_sim_eval_accumulate's kernel) compiled for the host, for every variant of LHW_FOR_EACH_VARIANT through model_pack.h's
// with_variant; one call = one launch over n envs.  tests/test_eval_stats.py feeds it roll-outs of sim_emu_variants.cpp.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/model_pack.h"

using namespace lhw;

extern "C" {
int eval_emu_words(void) { return EV_WORDS; }

// 0, or -1 for an unknown variant code
int eval_emu_accumulate(int variant, int precision, const void* sr, const int32_t* si, int n, const void* reward,
                        const void* rew_terms, const int32_t* done, double* acc) {
  return with_variant(variant, precision, [&](auto v) {
    using V = decltype(v);
    using R = typename V::real;
    constexpr int NR = Dims<R, V::NJ, V::TK>::NSTATE_R;
    for (int i = 0; i < n; i++)
      eval_accumulate_env<R, V::NJ, V::TK>((const R*)sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, ((const R*)reward)[i],
                                           (const R*)rew_terms + (size_t)i * NREW, done[i], acc + (size_t)i * EV_WORDS);
  });
}
}
