// tools/newton_census.cpp — DEVELOPMENT TOOL ONLY (tools/newton_census.py).  The CPU emulation of the kernel source
// (tests/emu/sim_emu.cpp, included unchanged) with sim_core.h's Newton-step hook defined: one (env id, Newton steps,
// line-search evaluations after the one at alpha = 0) record per contact solve, in the order the solves run.
#include <stdint.h>

#include <vector>

static std::vector<int32_t> g_census;
static int g_census_it0, g_census_ls;
static void census_hook(int event, uint32_t env, int iters, int n) {
  if (event == 0) { g_census_it0 = iters; g_census_ls = 0; }
  else if (event == 1) g_census_ls += n > 0;
  else { g_census.push_back((int32_t)env); g_census.push_back(iters - g_census_it0); g_census.push_back(g_census_ls); }
}
#define LHW_NEWTON_HOOK(event, w, n) census_hook(event, (w).env_id, (w).iters_total, n)

#include "../tests/emu/sim_emu.cpp"

// moves the records gathered since the last call to out (3 int32 each); returns the number of records
extern "C" int emu_census_take(int32_t* out, int cap_records) {
  const int n = (int)(g_census.size() / 3) < cap_records ? (int)(g_census.size() / 3) : cap_records;
  for (int i = 0; i < 3 * n; i++) out[i] = g_census[i];
  g_census.erase(g_census.begin(), g_census.begin() + 3 * n);
  return n;
}
