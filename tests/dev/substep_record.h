// tests/dev/substep_record.h — TEST HARNESS ONLY.  The host side shared by the two builds of one physics substep of sim_core.h:
// tests/dev/substep_dev.cu (device) and tests/dev/substep_emu.cpp (host emulation).  Include it after sim_core.h.
// It names the Work fields the tests read after the last substep (their byte offsets, through layout()) and dispatches on
// (variant code, precision).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace substep_record {
using namespace lhw;

constexpr int NFIELDS = 25;

// byte offsets of the Work fields the tests read, in this order (tests/dev/substep_cases.py FIELDS); the first word is sizeof(Work)
template <class real, int NJ, int TK> void layout(long long* out) {
  using W = Work<real, NJ, TK>;
  static W w;   // Work is not standard-layout (its persistent block is a base class): offsets from an object, not offsetof
  const char* b = reinterpret_cast<const char*>(&w);
  auto at = [&](const void* f) { return (long long)(reinterpret_cast<const char*>(f) - b); };
  const long long o[] = {(long long)sizeof(W), at(w.qpos), at(w.qvel), at(w.qacc_warm), at(w.qacc), at(w.qfs), at(w.act_force),
                         at(&w.M), at(w.ncon), at(w.ncorner), at(w.nside), at(w.cmul), at(w.cn), at(w.cpos), at(w.xcd), at(w.lside),
                         at(w.grf), at(&w.cz_min), at(w.foot_vel), at(w.root_vlin), at(&w.status), at(&w.nfloor), at(&w.iters_total),
                         at(w.flim), at(w.fjar)};
  static_assert(sizeof(o) / sizeof(o[0]) == NFIELDS, "FIELDS of tests/dev/substep_cases.py");
  memcpy(out, o, sizeof(o));
}

// calls f(Variant<real, NJ, TK>{}) for (code, precision); -1 for an unknown pair (model_pack.h with_variant)
template <class F> int dispatch(int code, int precision, F&& f) {
  if (precision != 64 && precision != 32) return -1;
  return with_variant(code, precision, f);
}

template <class real, int NJ, int TK> int layout_of(long long* out) {
  layout<real, NJ, TK>(out);
  return 0;
}

inline int layout_any(int code, int precision, long long* out) {
  int rc = -1;
  dispatch(code, precision, [&](auto v) {
    using V = decltype(v);
    rc = layout_of<typename V::real, V::NJ, V::TK>(out);
  });
  return rc;
}
}  // namespace substep_record
