// tests/dev/solver_dev.cu — TEST HARNESS ONLY.  The Newton solver pieces of the step kernel source (sim_core.h warp_mma_f64,
// newton_hessian_f64 and arrow_factor_solve) compiled for the device as they are, each launched on its own;
// tests/test_gpu_solver_pieces.py holds them to numpy float64.  Its host twin is tests/dev/solver_emu.cpp: the same entry points and
// argument order, with dev_ in front and the number of warps per block after the number of problems.  dev_mma_lanes takes the
// arguments of tests/emu/dmma_emu.cpp dmma_emu_lanes.
// One warp per problem: the warp copies its Work record into dynamic shared memory (arrow_factor_solve and newton_hessian_f64
// assume their record is there), calls the piece and copies the whole record back.  A block carries n_warps problems, the
// record of warp i at smem[i], as step_kernel_mw lays them out.
#include "../../learninghumanoidwalking_b200/csrc/sim_core.h"
#include "solver_record.h"

#include <cuda_runtime.h>

using namespace lhw;

template <class W> __device__ __forceinline__ void copy_record(W* dst, const W* src) {
  static_assert(sizeof(W) % 16 == 0, "Work is 16-byte aligned");
  const int4* s = reinterpret_cast<const int4*>(src);
  int4* d = reinterpret_cast<int4*>(dst);
  for (int i = (int)(threadIdx.x & 31); i < (int)(sizeof(W) / 16); i += 32) d[i] = s[i];
}

// the warp's record in shared memory, loaded; nullptr for a warp past the last problem
template <class W> __device__ __forceinline__ W* load_record(W* g, int n) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int warp = (int)(threadIdx.x >> 5), p = (int)blockIdx.x * (int)(blockDim.x >> 5) + warp;
  if (p >= n) return nullptr;
  W* w = reinterpret_cast<W*>(smem_raw) + warp;
  copy_record(w, g + p);
  __syncwarp();
  return w;
}

template <class W> __device__ __forceinline__ void store_record(W* g, const W* w) {
  __syncwarp();
  copy_record(g + (int)blockIdx.x * (int)(blockDim.x >> 5) + (int)(threadIdx.x >> 5), w);
}

template <int NJ, int TK> __global__ void k_hessian(Work<double, NJ, TK>* g, int n) {
  Work<double, NJ, TK>* w = load_record(g, n);
  if (!w) return;
  newton_hessian_f64<double, NJ, TK>(*w);
  store_record(g, w);
}

template <class real, int NJ, int TK> __global__ void k_arrow(Work<real, NJ, TK>* g, int n) {
  Work<real, NJ, TK>* w = load_record(g, n);
  if (!w) return;
  arrow_factor_solve<real, NJ, TK>(*w, w->sdir);
  store_record(g, w);
}

template <int KS> __global__ void k_lanes(const double* a, const double* b, const double* c, double* d) {
  warp_mma_f64<KS>([&](int l, int k) { return a[l * KS + k]; }, [&](int l, int k) { return b[l * KS + k]; },
                   [&](int l, int i) { return c[l * 2 + i]; }, [&](int l, int i, double v) { d[l * 2 + i] = v; });
}

#define DEV_OK(x)                          \
  do {                                     \
    if ((x) != cudaSuccess) return -100;   \
  } while (0)

// the records through kernel(records, n), n_warps of them per block; the records come back whole
template <class W> static int launch(void (*kernel)(W*, int), std::vector<W>& w, int n_warps) {
  const int n = (int)w.size();
  if (n_warps < 1) return -2;
  const size_t bytes = w.size() * sizeof(W), smem = sizeof(W) * n_warps;
  W* d = nullptr;
  DEV_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  DEV_OK(cudaMalloc(&d, bytes));
  int rc = 0;
  if (cudaMemcpy(d, w.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) rc = -101;
  if (!rc) {
    kernel<<<(n + n_warps - 1) / n_warps, 32 * n_warps, smem>>>(d, n);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = -102;
  }
  if (!rc && cudaMemcpy(w.data(), d, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) rc = -103;
  cudaFree(d);
  return rc;
}

template <int NJ, int TK> static int launch_hessian(std::vector<Work<double, NJ, TK>>& w, int n_warps) {
  return launch(k_hessian<NJ, TK>, w, n_warps);
}
template <class real, int NJ, int TK> static int launch_arrow(std::vector<Work<real, NJ, TK>>& w, int n_warps) {
  return launch(k_arrow<real, NJ, TK>, w, n_warps);
}

template <int KS> static int lanes(const double* a, const double* b, const double* c, double* d) {
  double* m = nullptr;   // a, b [32][KS], c, d [32][2]
  DEV_OK(cudaMalloc(&m, (64 * KS + 128) * sizeof(double)));
  int rc = 0;
  if (cudaMemcpy(m, a, 32 * KS * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(m + 32 * KS, b, 32 * KS * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess ||
      cudaMemcpy(m + 64 * KS, c, 64 * sizeof(double), cudaMemcpyHostToDevice) != cudaSuccess)
    rc = -101;
  if (!rc) {
    k_lanes<KS><<<1, 32>>>(m, m + 32 * KS, m + 64 * KS, m + 64 * KS + 64);
    if (cudaGetLastError() != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess) rc = -102;
  }
  if (!rc && cudaMemcpy(d, m + 64 * KS + 64, 64 * sizeof(double), cudaMemcpyDeviceToHost) != cudaSuccess) rc = -103;
  cudaFree(m);
  return rc;
}

extern "C" {
// one tile from raw per-lane fragments: a, b [32][ks], c, d [32][2]; 0, -1 for an unsupported ks, < -1 for a CUDA error
int dev_mma_lanes(int ks, const double* a, const double* b, const double* c, double* d) {
  switch (ks) {
    case 1: return lanes<1>(a, b, c, d);
    case 2: return lanes<2>(a, b, c, d);
    case 3: return lanes<3>(a, b, c, d);
    case 4: return lanes<4>(a, b, c, d);
  }
  return -1;
}

// newton_hessian_f64 of a variant (variant_code: 6, 5, 106, 206, 305) on n problems; rec_in / rec_out (n records, or null)
// receive the records before and after
int dev_hessian(int variant, int n, int n_warps, const double* S, const double* Af, const int* ncon, const double* M, const int* lside,
                const double* ljar, const double* lD, const double* fjar, const double* flim, const double* fD, double* H, double* T,
                unsigned char* rec_in, unsigned char* rec_out) {
  return solver_record::hessian_any(variant, n, S, Af, ncon, M, lside, ljar, lD, fjar, flim, fD, H, T, rec_in, rec_out,
                                    [&](auto& w) { return launch_hessian(w, n_warps); });
}

// arrow_factor_solve(w, w.sdir) of a variant at precision 64 or 32 on n problems
int dev_arrow_solve(int variant, int precision, int n, int n_warps, const double* H, const double* b, const int* status, double* F,
                    double* hdinv, double* x, int* status_out, unsigned char* rec_in, unsigned char* rec_out) {
  return solver_record::arrow_any(variant, precision, n, H, b, status, F, hdinv, x, status_out, rec_in, rec_out,
                                  [&](auto& w) { return launch_arrow(w, n_warps); });
}

int dev_layout(int variant, int precision, long long* out) { return solver_record::layout_any(variant, precision, out); }
}
