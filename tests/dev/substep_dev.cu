// tests/dev/substep_dev.cu — TEST HARNESS ONLY.  Physics substeps of the step kernel source on the device, one problem per warp:
// load_state -> substep x nsub -> store_state of sim_core.h, run as env_step runs them (substep s has last = (s == nsub - 1) and
// chained = (s > 0); in a block of several warps every warp meets the block at one barrier per substep, as step_kernel_mw's
// warps do, and a warp past the last problem only keeps those barriers).  tests/test_gpu_substep_edges.py holds the results to
// the float64 oracle at crafted states; its host twin is tests/dev/substep_emu.cpp (the same entry points, emu_ in front).
//
// The product's sim_kernels.cu is compiled here unchanged, so substep reads its model from the variant's __constant__ object
// through the ModelHome specialisation exactly as the shipped kernels do (a model read through a generic pointer compiles to
// different code), and the model is bound through lhw_sim_create / lhw_sim_bind.  Built with -fvisibility=hidden: the harness's
// own copies of the C-ABI functions (and render_kernels.cu, linked in beside it) bind inside this library and neither see nor shadow those of liblhw_b200.so in the same
// process; only the dev_* entry points below are exported.
#include "../../learninghumanoidwalking_b200/csrc/sim_kernels.cu"
#include "substep_record.h"

#define DEV_EXPORT extern "C" __attribute__((visibility("default")))

namespace {

// nsub substeps of n problems; sr / si / ctrl: problem-major records and controls; wout: the Work record of each problem after
// the last substep.  The launch bound is step_kernel_mw's, so this kernel asks no more of substep's registers than it does
template <class real, int NJ, int TK>
__global__ void __launch_bounds__(sizeof(real) == 8 ? LHW_X_REGCAP : 896, 1)
    substep_kernel(real* __restrict__ state_r, int32_t* __restrict__ state_i, const real* __restrict__ ctrl, int n, int nsub,
                   Work<real, NJ, TK>* __restrict__ wout) {
  using W = Work<real, NJ, TK>;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = threadIdx.x >> 5;
  const int p = blockIdx.x * (blockDim.x >> 5) + warp;
  const int alive = p < n;
  const int sync = blockDim.x > 32 ? 1 : 0;   // step_kernel_mw's default sync_mode; step_kernel passes 0
  W& w = reinterpret_cast<W*>(smem_raw)[warp];
  const Model<real, NJ, TK>& m = cmodel<real, NJ, TK>();
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NU = 2 * NJ;
  real* sr = state_r + (size_t)(alive ? p : 0) * NR;
  int32_t* si = state_i + (size_t)(alive ? p : 0) * NSTATE_I;
  if (alive) {
    load_state<real, NJ, TK>(w, sr, si, (uint32_t)p);
    LHW_LANES(l) {
      if (l < NU) w.ctrl[l] = ctrl[(size_t)p * NU + l];
    }
    LHW_SYNC();
  }
  for (int s = 0; s < nsub; s++) {
    if (alive) substep<real, NJ, TK>(w, m, s == nsub - 1, sync, s > 0);
    else LHW_BLOCK_SYNC(sync & 2);
    LHW_BLOCK_SYNC(sync & 1);
  }
  if (!alive) return;
  store_state<real, NJ, TK>(w, sr, si);
  const int4* src = reinterpret_cast<const int4*>(&w);
  int4* dst = reinterpret_cast<int4*>(wout + p);
  for (int i = (int)(threadIdx.x & 31); i < (int)(sizeof(W) / 16); i += 32) dst[i] = src[i];
}

struct Harness {
  lhw_sim* sim;
  int code, precision;
};

#define DEV_OK(x)                         \
  do {                                    \
    if ((x) != cudaSuccess) return -100;  \
  } while (0)

template <class real, int NJ, int TK>
int run(Harness* h, int n, int n_warps, int nsub, void* sr_h, int32_t* si_h, const void* ctrl_h, void* work_h) {
  using W = Work<real, NJ, TK>;
  constexpr int NR = Dims<real, NJ, TK>::NSTATE_R, NU = 2 * NJ;
  if (n < 1 || nsub < 1 || n_warps < 1) return -2;
  if (lhw_sim_bind(h->sim, nullptr)) return -3;
  const size_t smem = sizeof(W) * n_warps;
  DEV_OK(cudaFuncSetAttribute(substep_kernel<real, NJ, TK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const size_t b_sr = (size_t)n * NR * sizeof(real), b_si = (size_t)n * NSTATE_I * sizeof(int32_t);
  const size_t b_ctrl = (size_t)n * NU * sizeof(real), b_w = (size_t)n * sizeof(W);
  char* d = nullptr;
  DEV_OK(cudaMalloc(&d, b_sr + b_si + b_ctrl + b_w + 64));
  real* d_sr = reinterpret_cast<real*>(d);
  int32_t* d_si = reinterpret_cast<int32_t*>(d + b_sr);
  real* d_ctrl = reinterpret_cast<real*>(d + b_sr + b_si);
  W* d_w = reinterpret_cast<W*>(d + ((b_sr + b_si + b_ctrl + 15) / 16) * 16);
  int rc = 0;
  if (cudaMemcpy(d_sr, sr_h, b_sr, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_si, si_h, b_si, cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(d_ctrl, ctrl_h, b_ctrl, cudaMemcpyHostToDevice) != cudaSuccess || cudaMemset(d_w, 0, b_w) != cudaSuccess)
    rc = -101;
  if (!rc) {
    substep_kernel<real, NJ, TK><<<(n + n_warps - 1) / n_warps, 32 * n_warps, smem>>>(d_sr, d_si, d_ctrl, n, nsub, d_w);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = -102;
  }
  if (!rc && (cudaMemcpy(sr_h, d_sr, b_sr, cudaMemcpyDeviceToHost) != cudaSuccess ||
              cudaMemcpy(si_h, d_si, b_si, cudaMemcpyDeviceToHost) != cudaSuccess ||
              cudaMemcpy(work_h, d_w, b_w, cudaMemcpyDeviceToHost) != cudaSuccess))
    rc = -103;
  cudaFree(d);
  return rc;
}

}  // namespace

// a harness for the model `flat` (model/loader.py pack_model) at precision 64 or 32 on the current device; null on failure
DEV_EXPORT void* dev_substep_create(const double* flat, int n_flat, int precision) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  lhw_sim* s = nullptr;
  if (lhw_sim_create(&s, flat, n_flat, precision, dev)) return nullptr;
  return new Harness{s, (int)flat[0], precision};
}

DEV_EXPORT void dev_substep_destroy(void* hv) {
  Harness* h = (Harness*)hv;
  lhw_sim_destroy(h->sim);
  delete h;
}

// nsub substeps of n problems, n_warps of them per block (the last block ragged when n_warps does not divide n).  sr [n][NSTATE_R]
// and si [n][NSTATE_I] (the sim's precision) are stepped in place, ctrl [n][2 NJ] is held over the substeps, work [n] receives the
// Work records.  0, or < 0 on a bad argument or a CUDA error
DEV_EXPORT int dev_substeps(void* hv, int n, int n_warps, int nsub, void* sr, int32_t* si, const void* ctrl, void* work) {
  Harness* h = (Harness*)hv;
  int rc = -1;
  substep_record::dispatch(h->code, h->precision, [&](auto v) {
    using V = decltype(v);
    rc = run<typename V::real, V::NJ, V::TK>(h, n, n_warps, nsub, sr, si, ctrl, work);
  });
  return rc;
}

DEV_EXPORT int dev_substep_layout(int code, int precision, long long* out) { return substep_record::layout_any(code, precision, out); }

DEV_EXPORT const char* dev_substep_error(void) { return lhw_last_error(); }
