// render_kernels.cu — sm_90a ray-caster of the environments' scenes (csrc/render_core.h), behind lhw_sim_render.
//
// One thread per pixel, blockIdx.y selects the image.  Each block builds its image's scene once in shared memory (forward
// kinematics in one thread while another warp runs the per-link Jacobi solves), then shades a tile of 256 consecutive pixels
// and writes its 768 output bytes through shared memory, so that every store instruction of a warp covers 32 consecutive
// bytes.  Kept out of sim_kernels.cu: that object's SASS is the step kernel's fingerprint (build_record.json).
// Built with -fmad=false (build.py): without contraction the device arithmetic is the host build's (tests/emu/render_emu.cpp).
#include <cuda_runtime.h>

#include "render_core.h"

namespace lhw {
namespace {

constexpr int RENDER_THREADS = 256;

template <class real, int NJ, int TK>
__global__ void __launch_bounds__(RENDER_THREADS) render_kernel(const Model<real, NJ, TK>* __restrict__ mg, const real* __restrict__ state_r,
                                                                const int32_t* __restrict__ state_i, int n_envs,
                                                                const int32_t* __restrict__ env_ids, int W, int H, render::Camera cam,
                                                                uint8_t* __restrict__ rgb) {
  using S = render::Scene<NJ, TK>;
  constexpr int NL = S::NL, NR = Dims<real, NJ, TK>::NSTATE_R;
  __shared__ S s;
  __shared__ uint8_t tile[3 * RENDER_THREADS];
  const int img = blockIdx.y, tid = threadIdx.x;
  const int env = env_ids[img];
  if (env < 0 || env >= n_envs) return;   // torch.ops.lhw.sim_render rejects such ids before the launch
  const Model<real, NJ, TK>& m = *mg;
  const real* sr = state_r + (size_t)env * NR;
  const int32_t* si = state_i + (size_t)env * NSTATE_I;
  if (tid == 0) {
    render::scene_fk(m, sr, s.xpos, s.xmat);
    render::scene_view(sr, si, cam, s);
  } else if (tid >= 32 && tid < 32 + NL) {
    render::scene_inertia_box(m, tid - 32, s.lv[tid - 32], s.lh[tid - 32]);
  } else if (tid >= 64 && tid < 64 + S::NSL) {
    render::scene_slab(m, sr, tid - 64, s);
  }
  __syncthreads();
  if (tid < NL) render::scene_link(m, tid, s);
  else if (tid < NL + 2) render::scene_foot(m, tid - NL, s);
  __syncthreads();
  const long long npix = (long long)W * H, p0 = (long long)blockIdx.x * RENDER_THREADS, p = p0 + tid;
  if (p < npix) {
    uint8_t c[3];
    render::shade_pixel(s, cam, (int)(p % W), (int)(p / W), W, H, c);
    tile[3 * tid] = c[0]; tile[3 * tid + 1] = c[1]; tile[3 * tid + 2] = c[2];
  }
  __syncthreads();
  const long long nbytes = 3 * (npix - p0 < RENDER_THREADS ? npix - p0 : RENDER_THREADS);
  uint8_t* out = rgb + ((size_t)img * npix + p0) * 3;
  for (int k = tid; k < nbytes; k += RENDER_THREADS) out[k] = tile[k];
}

}  // namespace

template <class real, int NJ, int TK>
int render_launch(const Model<real, NJ, TK>* d_model, const real* state_r, const int32_t* state_i, int n_envs, const int32_t* env_ids,
                  int n_ids, int width, int height, const render::Camera& cam, uint8_t* rgb, cudaStream_t stream) {
  const long long npix = (long long)width * height;
  const dim3 grid((unsigned)((npix + RENDER_THREADS - 1) / RENDER_THREADS), (unsigned)n_ids);
  render_kernel<real, NJ, TK><<<grid, RENDER_THREADS, 0, stream>>>(d_model, state_r, state_i, n_envs, env_ids, width, height, cam, rgb);
  return 0;
}

#define LHW_RENDER_INSTANCE(R, J, T)                                                                                              \
  template int render_launch<R, J, T>(const Model<R, J, T>*, const R*, const int32_t*, int, const int32_t*, int, int, int,        \
                                      const render::Camera&, uint8_t*, cudaStream_t);
#define LHW_RENDER_VARIANT(J, T) LHW_RENDER_INSTANCE(double, J, T) LHW_RENDER_INSTANCE(float, J, T)
LHW_FOR_EACH_VARIANT(LHW_RENDER_VARIANT)
#undef LHW_RENDER_VARIANT
#undef LHW_RENDER_INSTANCE

}  // namespace lhw
