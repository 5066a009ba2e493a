// tests/emu/render_emu_variants.cpp — TEST HARNESS ONLY.  The host build of the renderer (render_emu.cpp), entered through
// model_pack.h's with_variant, so that every variant of sim_core.h's LHW_FOR_EACH_VARIANT renders on the host (render_emu.cpp's
// own entry points know the first four).  The entry points are render_emu.cpp's, named render_emuv_* (tests/emu/emu_variants.py).
#include "render_emu.cpp"

#define VDISPATCH(h, prec, CALL)                                             \
  with_variant((h)->var, (prec), [&](auto v_) {                              \
    using V_ = decltype(v_);                                                 \
    CALL(typename V_::real, V_::NJ, V_::TK);                                 \
  })

extern "C" {
void* render_emuv_create(const double* flat, int n, int precision) {
  Handle tmp{(int)flat[0], nullptr};
  void* p = nullptr;
#define CALL(R, J, T) p = create<R, J, T>(flat, n)
  if (VDISPATCH(&tmp, precision, CALL) != 0 || !p) return nullptr;
#undef CALL
  return new Handle{tmp.var, p};
}
void render_emuv_fk(void* hv, int precision, const void* qpos, float* xpos, float* xmat) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) fk<R, J, T>(h->p, (const R*)qpos, xpos, xmat)
  VDISPATCH(h, precision, CALL);
#undef CALL
}
void render_emuv_image(void* hv, int precision, const void* sr, const int32_t* si, int W, int H, const double* c7, int only_box,
                       uint8_t* rgb, float* boxes) {
  Handle* h = (Handle*)hv;
#define CALL(R, J, T) image<R, J, T>(h->p, (const R*)sr, si, W, H, c7, only_box, rgb, boxes)
  VDISPATCH(h, precision, CALL);
#undef CALL
}
}
