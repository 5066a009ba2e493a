// tests/dev/solver_emu.cpp — TEST HARNESS ONLY.  The host twin of tests/dev/solver_dev.cu: newton_hessian_f64 and
// arrow_factor_solve of the step kernel source compiled for the host with LHW_CPU_EMU (as tests/emu/dmma_emu.cpp compiles the
// Hessian), run on the same Work records through the same entry points (emu_ in front, no warps per block);
// tests/test_solver_harness.py holds it to numpy without a GPU, and tests/test_gpu_solver_pieces.py holds the device to it.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/sim_core.h"
#include "solver_record.h"

using namespace lhw;

extern "C" {
// newton_hessian_f64 of a variant (variant_code: 6, 5, 106, 206, 305) on n problems; rec_in / rec_out (n records, or null)
// receive the records before and after
int emu_hessian(int variant, int n, const double* S, const double* Af, const int* ncon, const double* M, const int* lside,
                const double* ljar, const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T,
                unsigned char* rec_in, unsigned char* rec_out) {
  return solver_record::hessian_any(variant, n, S, Af, ncon, M, lside, ljar, lD, fjar, flim, fD, H, T, rec_in, rec_out, [](auto& w) {
    for (auto& r : w) newton_hessian_f64(r);
    return 0;
  });
}

// arrow_factor_solve(w, w.sdir) of a variant at precision 64 or 32 on n problems
int arrow_emu_solve(int variant, int precision, int n, const double* H, const double* b, const int* status, double* F, double* hdinv,
                    double* x, int* status_out, unsigned char* rec_in, unsigned char* rec_out) {
  return solver_record::arrow_any(variant, precision, n, H, b, status, F, hdinv, x, status_out, rec_in, rec_out, [](auto& w) {
    for (auto& r : w) arrow_factor_solve(r, r.sdir);
    return 0;
  });
}

int emu_layout(int variant, int precision, long long* out) { return solver_record::layout_any(variant, precision, out); }
}
