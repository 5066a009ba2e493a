// comm_kernels.cu — the one exchange step of the path, fused and graph-capturable: gradient all-reduce over NVLink peer
// memory + clip_grad_norm_ (actor and critic separately) + Adam, as three ordinary launches per optimiser step.
//
// Replaces rl/algos/ppo.py:389-396 on N >= 1 GPUs: (NCCL all-reduce) -> clip_grad_norm_ x2 -> Adam.step x2.
// Every rank owns a cudaMalloc'ed, CUDA-IPC exported block {flat gradient | flags}; peers map it once
// (cudaIpcOpenMemHandle).  One optimiser step is
//   K1 exchange_reduce_kernel   block 0 tells every peer "my gradient is complete" (st.release.sys of the epoch into the
//        peer's flag word for this rank); EVERY block then waits until all peers said so (ld.acquire.sys on its own,
//        local, flag words), pulls its slice of all W gradients with 16-byte P2P loads (one-shot all-reduce: each GPU
//        reads W x 617 KB over NVLink), sums them in fixed rank order (bit-identical on every rank -> replicas never
//        drift), stores the averaged gradient locally and leaves per-block partial sums of squares per network.  The
//        last block to finish (ticket counter) adds the partials in index order (deterministic), writes both clip
//        coefficients, and tells every peer "I have finished reading your gradient" (epoch + 1).
//   K2 clip_adam_pair_kernel    clip + Adam for actor and critic over the flat parameter buffer (Adam step number and
//        the clip coefficients come from device memory).
//   K3 exchange_finish_kernel   one warp: waits until every peer has finished reading THIS rank's gradient (so the next
//        backward pass may overwrite it), then advances the epoch and the Adam step number in device memory.
// No cooperative launch, no grid-wide barrier, no by-value step / epoch arguments: the three launches can be captured
// into the CUDA graph of the optimiser step and replayed (every rank replays the same number of steps).  A peer that
// never arrives does not hang the GPU: the spins are bounded and leave an error word that the host reads with
// lhw_comm_status once per iteration.  At W = 1 the flag traffic vanishes and this is simply the fused clip + Adam.
//
// The adaptive instantiation (<true>, lhw_fused_allreduce_clip_adam_adaptive) adds rsl_rl's KL-adaptive learning rate
// (DESIGN.md §7.3).  Block 0 of K1 copies this rank's minibatch KL into the KL word of its comm block (after the flag
// words) before it says "ready"; the last block of K1, after every peer said so and before it says "done reading", sums
// the W KL words in rank order in float64, divides by W and updates the float64 rate in device memory (same bits on every
// rank); K2 then takes (float)rate for this very step.  The <false> instantiations are the fixed-rate kernels unchanged.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/lhw_b200.h"

extern "C" void lhw_count_launch(void);

namespace {

constexpr int MAX_WORLD = 16;
constexpr int COMM_BLOCK = 256;
constexpr int VEC_PER_THREAD = 1;          // float4 per thread in K1: 154 381 floats -> 151 blocks, one per SM
constexpr int KL_WORDS = 4;                // after the MAX_WORLD flag words of a comm block: [0] = this rank's KL (float)
// rsl_rl's adaptive schedule (DESIGN.md §7.3); rl/schedule.py holds the same constants and rule for the host
constexpr double LR_MIN = 1e-5, LR_MAX = 1e-2, LR_FACTOR = 1.5;
thread_local std::string g_cerr;

struct Peers {
  const float* grad[MAX_WORLD];    // peer r's flat gradient (device pointer valid on this GPU)
  unsigned int* flags[MAX_WORLD];  // peer r's flag array: flags[r][me] is written by me
};

// device-side state words
enum { ST_EPOCH = 0, ST_ERROR = 1, ST_TICKET = 2, ST_STEP = 3, ST_WORDS = 4 };
enum { ERR_READY_TIMEOUT = 1, ERR_DONE_TIMEOUT = 2 };

__device__ __forceinline__ void st_release_sys(unsigned int* p, unsigned int v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned int ld_acquire_sys(const unsigned int* p) {
  unsigned int v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// peer memory is rewritten every step: never serve it from a stale L1 line
__device__ __forceinline__ float4 ld_peer4(const float* p) { return __ldcv(reinterpret_cast<const float4*>(p)); }
__device__ __forceinline__ float ld_peer1(const float* p) { return __ldcv(p); }

// wait until every peer has written at least `epoch` into my flag word for it; false on time-out
__device__ __forceinline__ bool wait_peers(const unsigned int* my_flags, int world, unsigned int epoch, long long spin_limit) {
  bool ok = true;
  if ((int)threadIdx.x < world) {
    long long spins = 0;
    while ((int)(ld_acquire_sys(my_flags + threadIdx.x) - epoch) < 0)
      if (++spins > spin_limit) { ok = false; break; }
  }
  return ok;
}

// the peer's KL word sits right after its MAX_WORLD flag words
__device__ __forceinline__ float* kl_word(unsigned int* flags) { return reinterpret_cast<float*>(flags + MAX_WORLD); }

// the rule of DESIGN.md §7.3 in IEEE float64; a NaN KL fails every comparison and leaves the rate alone
__device__ __forceinline__ double adapt_lr(double lr, double kl, double desired_kl) {
  if (kl > 2.0 * desired_kl) return fmax(LR_MIN, lr / LR_FACTOR);
  if (kl > 0.0 && kl < desired_kl / 2.0) return fmin(LR_MAX, lr * LR_FACTOR);
  return lr;
}

template <bool ADAPTIVE>
__global__ void __launch_bounds__(COMM_BLOCK)
    exchange_reduce_kernel(Peers P, unsigned int* __restrict__ my_flags, unsigned int* __restrict__ state,
                           float* __restrict__ reduced, double* __restrict__ partials, float* __restrict__ coef,
                           long long n_actor, long long n_total, int rank, int world, float max_norm, long long spin_limit,
                           const float* __restrict__ kl, double* __restrict__ lr, double desired_kl) {
  __shared__ double sh[2][COMM_BLOCK / 32];
  __shared__ int sh_last;
  const unsigned int epoch = state[ST_EPOCH];
  if constexpr (ADAPTIVE) {
    // this rank's KL into its comm block before any "ready": peers read it once they have seen the flag
    if (blockIdx.x == 0) {
      if (threadIdx.x == 0) {
        *kl_word(my_flags) = *kl;
        __threadfence_system();
      }
      __syncthreads();
    }
  }
  if (world > 1) {
    // my backward pass precedes this kernel in stream order: the gradient is complete -> tell the peers
    if (blockIdx.x == 0 && (int)threadIdx.x < world) st_release_sys(P.flags[threadIdx.x] + rank, epoch);
    if (!wait_peers(my_flags, world, epoch, spin_limit)) atomicOr(state + ST_ERROR, (unsigned)ERR_READY_TIMEOUT);
    __syncthreads();
  }
  // ---- one-shot all-reduce of this block's slice (fixed rank order) + per-network sum of squares of the AVERAGE
  const float inv_w = 1.0f / (float)world;
  const long long n4 = n_total >> 2;
  double sa = 0, sc = 0;
  for (long long q = (long long)blockIdx.x * blockDim.x * VEC_PER_THREAD + threadIdx.x; q < n4;
       q += (long long)gridDim.x * blockDim.x * VEC_PER_THREAD) {
    float4 g = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int r = 0; r < world; r++) {
      const float4 v = ld_peer4(P.grad[r] + 4 * q);
      g.x += v.x; g.y += v.y; g.z += v.z; g.w += v.w;
    }
    g.x *= inv_w; g.y *= inv_w; g.z *= inv_w; g.w *= inv_w;
    reinterpret_cast<float4*>(reduced)[q] = g;
    const float e[4] = {g.x, g.y, g.z, g.w};
#pragma unroll
    for (int k = 0; k < 4; k++) {
      const double gg = (double)e[k] * (double)e[k];
      if (4 * q + k < n_actor) sa += gg; else sc += gg;
    }
  }
  if (blockIdx.x == gridDim.x - 1) {   // the 0..3 floats after the last full float4
    const long long i = 4 * n4 + threadIdx.x;
    if (i < n_total) {
      float g = 0;
      for (int r = 0; r < world; r++) g += ld_peer1(P.grad[r] + i);
      g *= inv_w;
      reduced[i] = g;
      const double gg = (double)g * (double)g;
      if (i < n_actor) sa += gg; else sc += gg;
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) { sa += __shfl_xor_sync(0xffffffffu, sa, o); sc += __shfl_xor_sync(0xffffffffu, sc, o); }
  if ((threadIdx.x & 31) == 0) { sh[0][threadIdx.x >> 5] = sa; sh[1][threadIdx.x >> 5] = sc; }
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0, c = 0;
#pragma unroll
    for (int k = 0; k < COMM_BLOCK / 32; k++) { a += sh[0][k]; c += sh[1][k]; }
    partials[2 * blockIdx.x] = a;
    partials[2 * blockIdx.x + 1] = c;
    __threadfence();                                       // partials (and this block's peer reads) before the ticket
    sh_last = atomicAdd(state + ST_TICKET, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!sh_last) return;
  // ---- last block: norms in block-index order (the same order on every rank and in every run), clip coefficients
  __threadfence();
  if (threadIdx.x < 32) {
    double na = 0, nc = 0;
    for (int b = threadIdx.x; b < (int)gridDim.x; b += 32) { na += __ldcg(partials + 2 * b); nc += __ldcg(partials + 2 * b + 1); }
#pragma unroll
    for (int o = 16; o; o >>= 1) { na += __shfl_xor_sync(0xffffffffu, na, o); nc += __shfl_xor_sync(0xffffffffu, nc, o); }
    if (threadIdx.x == 0) {
      const float ta = (float)sqrt(na), tc = (float)sqrt(nc);
      float ca = max_norm / (ta + 1e-6f), cc = max_norm / (tc + 1e-6f);   // torch.nn.utils.clip_grad_norm_
      coef[0] = ca > 1.0f ? 1.0f : ca;
      coef[1] = cc > 1.0f ? 1.0f : cc;
      coef[2] = ta;
      coef[3] = tc;
      state[ST_TICKET] = 0;
    }
  }
  if constexpr (ADAPTIVE) {
    // every peer's KL word was written before its "ready", which this block's thread r acquired for peer r
    __shared__ float sh_kl[MAX_WORLD];
    if ((int)threadIdx.x < world) sh_kl[threadIdx.x] = __ldcv(kl_word(P.flags[threadIdx.x]));
    __syncthreads();
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int r = 0; r < world; r++) s += (double)sh_kl[r];     // rank order: the same bits on every rank
      *lr = adapt_lr(*lr, s / (double)world, desired_kl);
    }
  }
  // every block of this rank has consumed the peers' gradients: they may be overwritten
  if (world > 1 && (int)threadIdx.x < world) st_release_sys(P.flags[threadIdx.x] + rank, epoch + 1);
}

// clip + Adam (rl/algos/ppo.py:393-396) for both networks; coef[0/1] from K1, the Adam step number from device memory;
// ADAPTIVE: the rate is (float) of the float64 rate K1 has just updated, the conversion the host applies to a fixed `lr`
template <bool ADAPTIVE>
__global__ void __launch_bounds__(COMM_BLOCK)
    clip_adam_pair_kernel(const float* __restrict__ reduced, const float* __restrict__ coef, const unsigned int* __restrict__ state,
                          float* __restrict__ param, float* __restrict__ m, float* __restrict__ v, long long n_actor,
                          long long n_total, float lr, float b1, float b2, float eps, const double* __restrict__ lr_dev) {
  if constexpr (ADAPTIVE) lr = (float)*lr_dev;
  const float t = (float)(state[ST_STEP] + 1u);
  const float bc1 = 1.0f - powf(b1, t), bc2_sqrt = sqrtf(1.0f - powf(b2, t));
  const float step_size = lr / bc1, coef_a = coef[0], coef_c = coef[1];
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n_total; i += (long long)gridDim.x * blockDim.x) {
    const float gi = reduced[i] * (i < n_actor ? coef_a : coef_c);
    const float mi = m[i] + (1.0f - b1) * (gi - m[i]);
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    param[i] -= step_size * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

// nobody zeroes / rewrites a gradient a peer is still reading; then the device-side counters advance
__global__ void __launch_bounds__(32)
    exchange_finish_kernel(const unsigned int* __restrict__ my_flags, unsigned int* __restrict__ state, int world,
                           long long spin_limit) {
  const unsigned int epoch = state[ST_EPOCH];
  if (world > 1 && !wait_peers(my_flags, world, epoch + 1, spin_limit)) atomicOr(state + ST_ERROR, (unsigned)ERR_DONE_TIMEOUT);
  __syncwarp();
  if (threadIdx.x == 0) {
    state[ST_EPOCH] = epoch + 2;
    state[ST_STEP] += 1u;
  }
}

}  // namespace

struct lhw_comm {
  int rank, world, device, grid;
  long long n, spin_limit;   // spin_limit: polls of a flag word before a wait gives up (about a microsecond each)
  unsigned char* block;  // [n floats grad | MAX_WORLD flags]
  float* grad;
  unsigned int* flags;
  float* reduced;
  double* partials;
  float* coef;           // clip coefficients (actor, critic), then the two gradient norms
  unsigned int* state;   // ST_* words
  double* lr;            // the adaptive schedule's learning rate (lhw_comm_lr_ptr)
  Peers peers;
  void* opened[MAX_WORLD];
};

namespace {
int cfail(int code, const std::string& s) { g_cerr = s; return code; }
#define COK(call)                                                                              \
  do {                                                                                         \
    cudaError_t _e = (call);                                                                   \
    if (_e != cudaSuccess) return cfail(-10, std::string(#call) + ": " + cudaGetErrorString(_e)); \
  } while (0)
size_t grad_bytes(long long n) { return ((size_t)n * 4 + 255) / 256 * 256; }
}  // namespace

extern "C" {

const char* lhw_comm_last_error(void) { return g_cerr.c_str(); }
int lhw_comm_handle_size(void) { return (int)sizeof(cudaIpcMemHandle_t); }

int lhw_comm_create(lhw_comm** out, long long n_floats, int rank, int world, int device) {
  if (!out || n_floats <= 0 || world < 1 || world > MAX_WORLD || rank < 0 || rank >= world) return cfail(-1, "bad argument");
  COK(cudaSetDevice(device));
  lhw_comm* c = new lhw_comm();
  memset(c, 0, sizeof(*c));
  c->rank = rank; c->world = world; c->device = device; c->n = n_floats;
  // a healthy peer answers within microseconds, but ranks may be seconds apart on the host (graph capture, a checkpoint
  // written by rank 0): the default waits about a minute before it reports; LHW_COMM_SPIN_LOG2 overrides it
  const char* sl = getenv("LHW_COMM_SPIN_LOG2");
  c->spin_limit = 1ll << (sl && atoi(sl) > 0 && atoi(sl) < 40 ? atoi(sl) : 26);
  const size_t gb = grad_bytes(n_floats);
  COK(cudaMalloc(&c->block, gb + (MAX_WORLD + KL_WORDS) * sizeof(unsigned int)));
  COK(cudaMemset(c->block, 0, gb + (MAX_WORLD + KL_WORDS) * sizeof(unsigned int)));
  c->grad = (float*)c->block;
  c->flags = (unsigned int*)(c->block + gb);
  COK(cudaMalloc(&c->reduced, gb));
  const long long per_block = (long long)COMM_BLOCK * VEC_PER_THREAD * 4;
  long long need = (n_floats + per_block - 1) / per_block;
  int nsm = 0;
  COK(cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, device));
  // every block of K1 spins until the peers arrive: all of them must be resident at once (8 x 256 threads fit on an SM)
  const long long cap = (long long)nsm * 8;
  c->grid = (int)(need < 1 ? 1 : (need > cap ? cap : need));
  COK(cudaMalloc(&c->partials, 2 * (size_t)c->grid * sizeof(double)));
  COK(cudaMalloc(&c->coef, 4 * sizeof(float)));
  COK(cudaMemset(c->coef, 0, 4 * sizeof(float)));
  COK(cudaMalloc(&c->state, ST_WORDS * sizeof(unsigned int)));
  const unsigned int init[ST_WORDS] = {1u, 0u, 0u, 0u};
  COK(cudaMemcpy(c->state, init, sizeof(init), cudaMemcpyHostToDevice));
  COK(cudaMalloc(&c->lr, sizeof(double)));
  COK(cudaMemset(c->lr, 0, sizeof(double)));
  c->peers.grad[rank] = c->grad;
  c->peers.flags[rank] = c->flags;
  *out = c;
  return 0;
}

void* lhw_comm_grad_ptr(lhw_comm* c) { return c ? c->grad : nullptr; }
double* lhw_comm_lr_ptr(lhw_comm* c) { return c ? c->lr : nullptr; }
long long lhw_comm_size(const lhw_comm* c) { return c ? c->n : 0; }
int lhw_comm_device(const lhw_comm* c) { return c ? c->device : -1; }

int lhw_comm_export(lhw_comm* c, void* blob_host) {
  if (!c || !blob_host) return cfail(-1, "null argument");
  cudaIpcMemHandle_t h;
  COK(cudaIpcGetMemHandle(&h, c->block));
  memcpy(blob_host, &h, sizeof(h));
  return 0;
}

int lhw_comm_import(lhw_comm* c, const void* all_blobs_host) {
  if (!c || !all_blobs_host) return cfail(-1, "null argument");
  COK(cudaSetDevice(c->device));
  const size_t gb = grad_bytes(c->n);
  for (int r = 0; r < c->world; r++) {
    if (r == c->rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, (const unsigned char*)all_blobs_host + (size_t)r * sizeof(h), sizeof(h));
    void* p = nullptr;
    COK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess));
    c->opened[r] = p;
    c->peers.grad[r] = (const float*)p;
    c->peers.flags[r] = (unsigned int*)((unsigned char*)p + gb);
  }
  return 0;
}

int lhw_comm_destroy(lhw_comm* c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  for (int r = 0; r < c->world; r++)
    if (c->opened[r]) cudaIpcCloseMemHandle(c->opened[r]);
  cudaFree(c->block);
  cudaFree(c->reduced);
  cudaFree(c->partials);
  cudaFree(c->coef);
  cudaFree(c->state);
  cudaFree(c->lr);
  delete c;
  return 0;
}

}  // extern "C"

namespace {
// the three launches of one optimiser step; ADAPTIVE: kl / lr_dev / desired_kl drive the rate (kl, lr_dev unused otherwise)
template <bool ADAPTIVE>
int fused_step(lhw_comm* c, float* param, float* exp_avg, float* exp_avg_sq, long long n_actor, long long n_total, float lr,
               float beta1, float beta2, float eps, float max_norm, const float* kl, double* lr_dev, double desired_kl,
               void* stream) {
  if (!c || !param || !exp_avg || !exp_avg_sq) return cfail(-1, "null argument");
  if (n_total != c->n || n_actor < 0 || n_actor > n_total) return cfail(-2, "size mismatch");
  cudaStream_t st = (cudaStream_t)stream;
  exchange_reduce_kernel<ADAPTIVE><<<c->grid, COMM_BLOCK, 0, st>>>(c->peers, c->flags, c->state, c->reduced, c->partials, c->coef,
                                                                   n_actor, n_total, c->rank, c->world, max_norm, c->spin_limit, kl,
                                                                   lr_dev, desired_kl);
  lhw_count_launch();
  COK(cudaGetLastError());
  int grid2 = (int)((n_total + COMM_BLOCK - 1) / COMM_BLOCK);
  if (grid2 > 132 * 4) grid2 = 132 * 4;   // 4 blocks per SM of an H100 SXM (132 SMs)
  clip_adam_pair_kernel<ADAPTIVE><<<grid2, COMM_BLOCK, 0, st>>>(c->reduced, c->coef, c->state, param, exp_avg, exp_avg_sq, n_actor,
                                                                n_total, lr, beta1, beta2, eps, lr_dev);
  lhw_count_launch();
  COK(cudaGetLastError());
  exchange_finish_kernel<<<1, 32, 0, st>>>(c->flags, c->state, c->world, c->spin_limit);
  lhw_count_launch();
  COK(cudaGetLastError());
  return 0;
}
}  // namespace

extern "C" {

int lhw_fused_allreduce_clip_adam(lhw_comm* c, float* param, float* exp_avg, float* exp_avg_sq, long long n_actor,
                                  long long n_total, float lr, float beta1, float beta2, float eps, float max_norm,
                                  void* stream) {
  return fused_step<false>(c, param, exp_avg, exp_avg_sq, n_actor, n_total, lr, beta1, beta2, eps, max_norm, nullptr, nullptr, 0.0,
                           stream);
}

int lhw_fused_allreduce_clip_adam_adaptive(lhw_comm* c, float* param, float* exp_avg, float* exp_avg_sq, long long n_actor,
                                           long long n_total, const float* kl, double* lr_dev, double desired_kl, float beta1,
                                           float beta2, float eps, float max_norm, void* stream) {
  if (!kl || !lr_dev) return cfail(-1, "null argument");
  if (!(desired_kl > 0.0)) return cfail(-1, "desired_kl must be > 0");
  return fused_step<true>(c, param, exp_avg, exp_avg_sq, n_actor, n_total, 0.0f, beta1, beta2, eps, max_norm, kl, lr_dev, desired_kl,
                          stream);
}

int lhw_comm_status(lhw_comm* c, int* error_word, int* adam_steps, float* norms2, void* stream) {
  if (!c) return cfail(-1, "null argument");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int h[ST_WORDS];
  float hc[4];
  COK(cudaMemcpyAsync(h, c->state, sizeof(h), cudaMemcpyDeviceToHost, st));
  COK(cudaMemcpyAsync(hc, c->coef, sizeof(hc), cudaMemcpyDeviceToHost, st));
  COK(cudaStreamSynchronize(st));
  if (error_word) *error_word = (int)h[ST_ERROR];
  if (adam_steps) *adam_steps = (int)h[ST_STEP];
  if (norms2) { norms2[0] = hc[2]; norms2[1] = hc[3]; }
  if (h[ST_ERROR]) return cfail(-20, std::string("peer exchange timed out (error word ") + std::to_string(h[ST_ERROR]) +
                                     "): a rank did not reach the gradient exchange");
  return 0;
}

int lhw_comm_set_step(lhw_comm* c, int adam_steps, void* stream) {
  if (!c || adam_steps < 0) return cfail(-1, "bad argument");
  const unsigned int v = (unsigned int)adam_steps;
  COK(cudaMemcpyAsync(c->state + ST_STEP, &v, sizeof(v), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  COK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

int lhw_comm_get_lr(lhw_comm* c, double* lr_host, void* stream) {
  if (!c || !lr_host) return cfail(-1, "null argument");
  COK(cudaMemcpyAsync(lr_host, c->lr, sizeof(double), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
  COK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

int lhw_comm_set_lr(lhw_comm* c, double lr, void* stream) {
  if (!c || !(lr > 0.0)) return cfail(-1, "bad argument");
  COK(cudaMemcpyAsync(c->lr, &lr, sizeof(double), cudaMemcpyHostToDevice, (cudaStream_t)stream));
  COK(cudaStreamSynchronize((cudaStream_t)stream));
  return 0;
}

}  // extern "C"
