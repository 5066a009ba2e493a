// tests/emu/dmma_emu.cpp — TEST HARNESS ONLY.  The fp64 tensor-core pieces of the step kernel source (sim_core.h warp_mma_f64 and
// newton_hessian_f64) compiled for the host with LHW_CPU_EMU;
// tests/test_dmma_hessian.py holds them to numpy.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/sim_core.h"

#include <string.h>

using namespace lhw;

template <int KS> static void lanes(const double* a, const double* b, const double* c, double* d) {
  warp_mma_f64<KS>([&](int l, int k) { return a[l * KS + k]; }, [&](int l, int k) { return b[l * KS + k]; },
                   [&](int l, int i) { return c[l * 2 + i]; }, [&](int l, int i, double v) { d[l * 2 + i] = v; });
}

template <int NJ, int TK>
static void hessian(const double* S, const double* Af, const int* ncon, const double* M, const int* lside, const double* ljar,
                    const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T) {
  using W = Work<double, NJ, TK>;
  constexpr int NU = 2 * NJ;
  W* w = new W();
  memcpy(w->S, S, sizeof(w->S));
  memcpy(w->Af, Af, sizeof(w->Af));
  memcpy(&w->M, M, sizeof(w->M));
  for (int f = 0; f < 2; f++) w->ncon[f] = ncon[f];
  for (int j = 0; j < NU; j++) {
    w->lside[j] = lside[j];
    w->ljar[j] = ljar[j];
    w->lD[j] = lD[j];
  }
  if constexpr (Cfg<NJ, TK>::FLOSS)
    for (int j = 0; j < NU; j++) {
      w->fjar[j] = fjar[j];
      w->flim[j] = flim[j];
      w->fD[j] = fD[j];
    }
  // garbage in what must come out of the build, so that an entry it does not write shows
  double* h = &w->H.r[0][0];
  for (size_t i = 0; i < sizeof(w->H) / sizeof(double); i++) h[i] = 1e300;
  newton_hessian_f64<double, NJ, TK>(*w);
  memcpy(H, &w->H, sizeof(w->H));
  memcpy(T, w->T, sizeof(w->T));
  delete w;
}

extern "C" {
// one tile from raw per-lane fragments: a, b [32][ks], c, d [32][2]; 0, or -1 for an unsupported ks
int dmma_emu_lanes(int ks, const double* a, const double* b, const double* c, double* d) {
  switch (ks) {
    case 1: lanes<1>(a, b, c, d); return 0;
    case 2: lanes<2>(a, b, c, d); return 0;
    case 3: lanes<3>(a, b, c, d); return 0;
    case 4: lanes<4>(a, b, c, d); return 0;
  }
  return -1;
}

// the Newton Hessian of the JVRC-1 (nj = 6, no friction loss) or H1 (nj = 5, friction-loss rows) walking variants
int dmma_emu_hessian(int nj, const double* S, const double* Af, const int* ncon, const double* M, const int* lside, const double* ljar,
                     const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T) {
  if (nj == 6) hessian<6, 0>(S, Af, ncon, M, lside, ljar, lD, fjar, flim, fD, H, T);
  else if (nj == 5) hessian<5, 3>(S, Af, ncon, M, lside, ljar, lD, fjar, flim, fD, H, T);
  else return -1;
  return 0;
}
}
