// tests/emu/render_emu.cpp — TEST HARNESS ONLY.  Compiles the product's renderer source (csrc/render_core.h) for the host,
// so that the `-m "not gpu"` tier can check its forward kinematics and images against oracle/render_oracle.py and the GPU
// tier can hold the device images to this build.  Never linked into or reachable from the product.
#define LHW_CPU_EMU 1
#include "../../learninghumanoidwalking_b200/csrc/model_pack.h"
#include "../../learninghumanoidwalking_b200/csrc/render_core.h"

using namespace lhw;

template <class real, int NJ, int TK> struct RModel {
  Model<real, NJ, TK> model;
  real plans[MAXPLAN * PLAN_STRIDE];
};

template <class real, int NJ, int TK> static void* create(const double* flat, int n) {
  auto* e = new RModel<real, NJ, TK>();
  if (fill_model(e->model, flat, n, e->plans) != 0) { delete e; return nullptr; }
  return e;
}

template <class real, int NJ, int TK> static void fk(void* h, const real* qpos, float* xpos, float* xmat) {
  constexpr int NL = 1 + 2 * NJ;
  float p[NL][3], R[NL][9];
  render::scene_fk(((RModel<real, NJ, TK>*)h)->model, qpos, p, R);
  for (int i = 0; i < NL; i++) {
    for (int k = 0; k < 3; k++) xpos[3 * i + k] = p[i][k];
    for (int k = 0; k < 9; k++) xmat[9 * i + k] = R[i][k];
  }
}

// `only_box` >= 0: keep that robot box (link or foot box) and move every other robot primitive 1e6 m up, out of the picture
template <class real, int NJ, int TK>
static void image(void* h, const real* sr, const int32_t* si, int W, int H, const double* c7, int only_box, uint8_t* rgb, float* boxes) {
  using S = render::Scene<NJ, TK>;
  const render::Camera cam = render::make_camera(c7[0], c7[1], c7[2], c7[3], c7[4], c7[5], c7[6], W, H);
  S* s = new S();
  render::build_scene(((RModel<real, NJ, TK>*)h)->model, sr, si, cam, *s);
  if (only_box >= 0) {
    for (int b = 0; b < S::NL + S::NFOOT; b++)
      if (b != only_box) s->bc[b][2] += 1e6f;
    for (int k = 0; k < S::NSPH; k++) s->sc[k][2] += 1e6f;
  }
  for (int b = 0; boxes && b < S::NBOX; b++) {
    for (int k = 0; k < 3; k++) boxes[15 * b + k] = s->bc[b][k];
    for (int k = 0; k < 9; k++) boxes[15 * b + 3 + k] = s->br[b][k];
    for (int k = 0; k < 3; k++) boxes[15 * b + 12 + k] = s->bh[b][k];
  }
  for (int py = 0; py < H; py++)
    for (int px = 0; px < W; px++) render::shade_pixel(*s, cam, px, py, W, H, rgb + 3 * ((size_t)py * W + px));
  delete s;
}

struct Handle { int var; void* p; };
#define DISPATCH(h, prec, CALL)                                                                       \
  do {                                                                                                \
    if ((h)->var == 6) { if ((prec) == 64) { CALL(double, 6, 0); } else { CALL(float, 6, 0); } }      \
    else if ((h)->var == 106) { if ((prec) == 64) { CALL(double, 6, 1); } else { CALL(float, 6, 1); } } \
    else if ((h)->var == 206) { if ((prec) == 64) { CALL(double, 6, 2); } else { CALL(float, 6, 2); } } \
    else { if ((prec) == 64) { CALL(double, 5, 0); } else { CALL(float, 5, 0); } }                    \
  } while (0)

extern "C" {
void* render_emu_create(const double* flat, int n, int precision) {
  const int var = (int)flat[0];
  if (var != 6 && var != 5 && var != 106 && var != 206) return nullptr;
  Handle tmp{var, nullptr};
  void* p = nullptr;
#define CALL(R, J, T) p = create<R, J, T>(flat, n)
  DISPATCH(&tmp, precision, CALL);
#undef CALL
  return p ? new Handle{var, p} : nullptr;
}
void render_emu_fk(void* hv, int precision, const void* qpos, float* xpos, float* xmat) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) fk<R, J, T>(h->p, (const R*)qpos, xpos, xmat)
  DISPATCH(h, precision, CALL);
#undef CALL
}
// one environment's record -> rgb [H, W, 3]; c7 = (dx, dy, z, distance, azimuth, elevation, fovy); boxes (may be NULL):
// [NBOX][centre 3, rotation 9, half sizes 3] of the scene as built
void render_emu_image(void* hv, int precision, const void* sr, const int32_t* si, int W, int H, const double* c7, int only_box,
                      uint8_t* rgb, float* boxes) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) image<R, J, T>(h->p, (const R*)sr, si, W, H, c7, only_box, rgb, boxes)
  DISPATCH(h, precision, CALL);
#undef CALL
}
}
