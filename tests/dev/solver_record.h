// tests/dev/solver_record.h — TEST HARNESS ONLY.  The host side shared by the two builds of the Newton solver pieces of
// sim_core.h: tests/dev/solver_dev.cu (device) and tests/dev/solver_emu.cpp (host emulation).  Include it after sim_core.h.
// It fills one Work record per problem from flat host arrays, hands the records to `run` (a launch, or a host loop), and
// reads the results back.  Each record is first filled with fixed pseudo-random bytes, so a test can tell every byte the
// piece wrote from one it left alone (the records before and after are returned whole).
#pragma once
#include <stdint.h>
#include <string.h>

#include <vector>

namespace solver_record {
using namespace lhw;

template <int NJ> constexpr int arrow_words() { return 36 + 12 * NJ + 2 * NJ * NJ; }   // Arrow r, x, c without tail padding

template <class W> void scramble(W& w, int p) {
  unsigned char* b = reinterpret_cast<unsigned char*>(&w);
  uint32_t s = 0x9E3779B9u * (uint32_t)(p + 1);
  for (size_t i = 0; i < sizeof(W); i++) {
    s = s * 1664525u + 1013904223u;
    b[i] = (unsigned char)(s >> 24);
  }
}

// byte offsets and sizes of what the pieces read and write:
// [sizeof(Work), H, H bytes, hdinv, hdinv bytes, sdir, sdir bytes, status, T, T bytes]
template <class real, int NJ, int TK> void layout(long long* out) {
  using W = Work<real, NJ, TK>;
  std::vector<W> v(1);
  W& w = v[0];
  const char* b = reinterpret_cast<const char*>(&w);
  const long long o[] = {(long long)sizeof(W), reinterpret_cast<const char*>(&w.H) - b, (long long)(arrow_words<NJ>() * sizeof(real)),
                         reinterpret_cast<const char*>(w.hdinv) - b, (long long)sizeof(w.hdinv),
                         reinterpret_cast<const char*>(w.sdir) - b, (long long)sizeof(w.sdir),
                         reinterpret_cast<const char*>(&w.status) - b, reinterpret_cast<const char*>(w.T) - b, (long long)sizeof(w.T)};
  memcpy(out, o, sizeof(o));
}

template <class W> void records_out(const std::vector<W>& w, unsigned char* rec) {
  if (rec) memcpy(rec, w.data(), w.size() * sizeof(W));
}

// newton_hessian_f64 on n problems; inputs as tests/emu/dmma_emu.cpp dmma_emu_hessian's, problem-major.  Every word of H starts
// as 1e300, so an entry the build does not write (the upper triangles of H.r and H.c) shows
template <int NJ, int TK, class Run>
int hessian_problems(int n, const double* S, const double* Af, const int* ncon, const double* M, const int* lside, const double* ljar,
                     const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T,
                     unsigned char* rec_in, unsigned char* rec_out, Run run) {
  using W = Work<double, NJ, TK>;
  constexpr int NV = 6 + 2 * NJ, NU = 2 * NJ, NA = 6 + NJ, NW = arrow_words<NJ>();
  std::vector<W> w(n);
  for (int p = 0; p < n; p++) {
    W& r = w[p];
    scramble(r, p);
    memcpy(r.S, S + (size_t)p * NV * 6, sizeof(r.S));
    memcpy(r.Af, Af + (size_t)p * 72, sizeof(r.Af));
    memcpy(&r.M, M + (size_t)p * NW, NW * sizeof(double));
    for (int f = 0; f < 2; f++) r.ncon[f] = ncon[2 * p + f];
    for (int j = 0; j < NU; j++) {
      r.lside[j] = lside[p * NU + j];
      r.ljar[j] = ljar[p * NU + j];
      r.lD[j] = lD[p * NU + j];
    }
    if constexpr (Cfg<NJ, TK>::FLOSS)
      for (int j = 0; j < NU; j++) {
        r.fjar[j] = fjar[p * NU + j];
        r.flim[j] = flim[p * NU + j];
        r.fD[j] = fD[p * NU + j];
      }
    for (int i = 0; i < NW; i++) (&r.H.r[0][0])[i] = 1e300;
  }
  records_out(w, rec_in);
  if (const int e = run(w)) return e;
  for (int p = 0; p < n; p++) {
    memcpy(H + (size_t)p * NW, &w[p].H, NW * sizeof(double));
    memcpy(T + (size_t)p * 2 * NA * 6, w[p].T, sizeof(w[p].T));
  }
  records_out(w, rec_out);
  return 0;
}

// arrow_factor_solve(w, w.sdir) on n problems: H (Arrow words, lower triangles read) and b in double, rounded to `real`; status is
// the record's status word before the solve.  Out: the factor in H's words, hdinv, x, status
template <class real, int NJ, int TK, class Run>
int arrow_problems(int n, const double* H, const double* b, const int* status, double* F, double* hdinv, double* x, int* status_out,
                   unsigned char* rec_in, unsigned char* rec_out, Run run) {
  using W = Work<real, NJ, TK>;
  constexpr int NV = 6 + 2 * NJ, NW = arrow_words<NJ>();
  std::vector<W> w(n);
  for (int p = 0; p < n; p++) {
    W& r = w[p];
    scramble(r, p);
    for (int i = 0; i < NW; i++) (&r.H.r[0][0])[i] = (real)H[(size_t)p * NW + i];
    for (int i = 0; i < NV; i++) r.sdir[i] = (real)b[p * NV + i];
    r.status = status[p];
  }
  records_out(w, rec_in);
  if (const int e = run(w)) return e;
  for (int p = 0; p < n; p++) {
    for (int i = 0; i < NW; i++) F[(size_t)p * NW + i] = (&w[p].H.r[0][0])[i];
    for (int i = 0; i < NV; i++) {
      hdinv[p * NV + i] = w[p].hdinv[i];
      x[p * NV + i] = w[p].sdir[i];
    }
    status_out[p] = w[p].status;
  }
  records_out(w, rec_out);
  return 0;
}

// variant = variant_code(nj, tk) (6, 5, 106, 206, 305), precision 64 or 32; -1 for anything else
template <class Run>
int hessian_any(int variant, int n, const double* S, const double* Af, const int* ncon, const double* M, const int* lside,
                const double* ljar, const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T,
                unsigned char* rec_in, unsigned char* rec_out, Run run) {
#define SOLVER_RECORD_X(nj, tk)                                                                                                  \
  if (variant == variant_code(nj, tk))                                                                                          \
    return hessian_problems<nj, tk>(n, S, Af, ncon, M, lside, ljar, lD, fjar, flim, fD, H, T, rec_in, rec_out, run);
  LHW_FOR_EACH_VARIANT(SOLVER_RECORD_X)
#undef SOLVER_RECORD_X
  return -1;
}

template <class Run>
int arrow_any(int variant, int precision, int n, const double* H, const double* b, const int* status, double* F, double* hdinv, double* x,
              int* status_out, unsigned char* rec_in, unsigned char* rec_out, Run run) {
#define SOLVER_RECORD_X(nj, tk)                                                                                                  \
  if (variant == variant_code(nj, tk) && precision == 64)                                                                       \
    return arrow_problems<double, nj, tk>(n, H, b, status, F, hdinv, x, status_out, rec_in, rec_out, run);                       \
  if (variant == variant_code(nj, tk) && precision == 32)                                                                       \
    return arrow_problems<float, nj, tk>(n, H, b, status, F, hdinv, x, status_out, rec_in, rec_out, run);
  LHW_FOR_EACH_VARIANT(SOLVER_RECORD_X)
#undef SOLVER_RECORD_X
  return -1;
}

inline int layout_any(int variant, int precision, long long* out) {
#define SOLVER_RECORD_X(nj, tk)                                                                                                  \
  if (variant == variant_code(nj, tk) && precision == 64) return layout<double, nj, tk>(out), 0;                                \
  if (variant == variant_code(nj, tk) && precision == 32) return layout<float, nj, tk>(out), 0;
  LHW_FOR_EACH_VARIANT(SOLVER_RECORD_X)
#undef SOLVER_RECORD_X
  return -1;
}

}  // namespace solver_record
