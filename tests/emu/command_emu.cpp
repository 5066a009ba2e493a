// tests/emu/command_emu.cpp — TEST HARNESS ONLY.  The held-command bodies of the product (sim_core.h set_command_env and
// command_accumulate_env, the bodies of lhw_sim_set_command's and lhw_sim_command_accumulate's kernels) compiled for the host, for
// every variant of LHW_FOR_EACH_VARIANT through model_pack.h's with_variant; one call = one launch over n envs.
// tests/test_command.py feeds them records of sim_emu_variants.cpp.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/model_pack.h"

using namespace lhw;

extern "C" {
int command_emu_words(void) { return CMD_WORDS; }

// 0; -1 for an unknown variant code, -2 for a variant without a velocity command (the kernel's refusal); given[i] = 1 where env i
// took the command
int command_emu_set(int variant, int precision, void* sr, int32_t* si, int n, const int32_t* mode, const void* ref, void* obs,
                    int32_t* given) {
  int rc = 0;
  const int unknown = with_variant(variant, precision, [&](auto v) {
    using V = decltype(v);
    using R = typename V::real;
    if constexpr (Cfg<V::NJ, V::TK>::STAND || Cfg<V::NJ, V::TK>::STEP) {
      rc = -2;
    } else {
      constexpr int NR = Dims<R, V::NJ, V::TK>::NSTATE_R, NOBS = Dims<R, V::NJ, V::TK>::NOBS;
      for (int i = 0; i < n; i++)
        given[i] = set_command_env<R, V::NJ, V::TK>((R*)sr + (size_t)i * NR, si + (size_t)i * NSTATE_I, mode[i],
                                                    (const R*)ref + 3 * (size_t)i, (R*)obs + (size_t)i * NOBS);
    }
  });
  return unknown ? -1 : rc;
}

// 0, or -1 for an unknown variant code
int command_emu_accumulate(int variant, int precision, const void* sr, int n, const int32_t* done, double* acc) {
  return with_variant(variant, precision, [&](auto v) {
    using V = decltype(v);
    using R = typename V::real;
    constexpr int NR = Dims<R, V::NJ, V::TK>::NSTATE_R;
    for (int i = 0; i < n; i++)
      command_accumulate_env<R, V::NJ, V::TK>((const R*)sr + (size_t)i * NR, done[i], acc + (size_t)i * CMD_WORDS);
  });
}
}
