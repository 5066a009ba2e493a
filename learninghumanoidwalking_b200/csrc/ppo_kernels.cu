// ppo_kernels.cu — sm_90a kernels for the PPO data path (include/lhw_b200.h, "PPO data path").
// All of these are HBM-streaming ops; the rollout is stored time-major [T, N, .] so that every access below is
// coalesced across the env index.  Replaces rl/storage/rollout_storage.py:53-85 (GAE), rl/algos/ppo.py:484-485
// (advantage normalisation), :535-538 (minibatch gathers) and :393-396 (clip_grad_norm_ + Adam.step).
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

#include "../../include/lhw_b200.h"

extern "C" void lhw_count_launch(void);

namespace {

thread_local std::string g_perr;

// GAE(lambda) as a two-level reverse scan.  A_t = delta_t + c_t A_{t+1} with c_t = gamma*lambda (0 where an episode
// ended) is an affine recurrence, and V(s_{t+1}) is data (the next row of `val`, or the bootstrap where the path ends),
// so only the scalar A crosses a segment boundary.  Block = 32 envs x GAE_SEG time segments: (1) every thread scans its
// segment with A_in = 0 and keeps (A_out, C = prod c_t); (2) the carry into each segment is the fixed-order composition
// of the later segments' (A, C) through shared memory; (3) the segment is rescanned with the right A_in and written.
// 2 x 16 B reads + 4 B write per sample, coalesced across the env index, T*N/GAE_LEN threads instead of N.
// float64 accumulation like the reference's buffers (rl/storage/rollout_storage.py:26-31).
constexpr int GAE_SEG = 16;
__global__ void __launch_bounds__(32 * GAE_SEG) gae_kernel(const float* __restrict__ rew, const float* __restrict__ val,
                                                           const int32_t* __restrict__ ended, const float* __restrict__ boot,
                                                           const float* __restrict__ last_val, float* __restrict__ ret, int T,
                                                           int N, double gamma, double lam, double* __restrict__ adv_part) {
  __shared__ double shA[GAE_SEG][32], shC[GAE_SEG][32];
  const int lane = threadIdx.x & 31, seg = threadIdx.x >> 5;
  const int n = blockIdx.x * 32 + lane;
  const int len = (T + GAE_SEG - 1) / GAE_SEG;
  const int t_lo = seg * len, t_hi = min(T, t_lo + len) - 1;   // this thread owns t_lo..t_hi (may be empty)
  const bool live = n < N && t_lo <= t_hi;
  const double gl = gamma * lam;
  double A = 0.0, C = 1.0;
  if (live) {
    double next_val = t_hi == T - 1 ? (double)last_val[n] : (double)val[(size_t)(t_hi + 1) * N + n];
    // branch-free body, unrolled: the four loads of a time step do not depend on the previous step's arithmetic, so the
    // unrolled iterations' loads are in flight together (one DRAM latency per group instead of one per step)
#pragma unroll 5
    for (int t = t_hi; t >= t_lo; t--) {
      const size_t i = (size_t)t * N + n;
      const int e = ended[i];
      const double v = (double)val[i], r = (double)rew[i], b = (double)boot[i];
      const double nv = e ? b : next_val, Ap = e ? 0.0 : A;
      A = (r + gamma * nv - v) + gl * Ap;
      C = (e ? 0.0 : C) * gl;
      next_val = v;
    }
  }
  shA[seg][lane] = A;
  shC[seg][lane] = live ? C : 1.0;
  __syncthreads();
  double s1 = 0.0, s2sum = 0.0;   // sum / sum of squares of the advantage (returns - values) of this thread's samples
  if (live) {
    // carry into this segment = A of everything later, composed from the last segment backwards (fixed order)
    double carry = 0.0;
    for (int s2 = GAE_SEG - 1; s2 > seg; s2--) carry = shA[s2][lane] + shC[s2][lane] * carry;
    double gae = carry;
    double next_val = t_hi == T - 1 ? (double)last_val[n] : (double)val[(size_t)(t_hi + 1) * N + n];
#pragma unroll 5
    for (int t = t_hi; t >= t_lo; t--) {
      const size_t i = (size_t)t * N + n;
      const int e = ended[i];
      const double v = (double)val[i], rw = (double)rew[i], b = (double)boot[i];
      gae = (rw + gamma * (e ? b : next_val) - v) + gl * (e ? 0.0 : gae);
      const float r = (float)(gae + v);
      ret[i] = r;
      const double a = (double)r - v;     // the advantage as the learner forms it: float32 returns - float32 values
      s1 += a;
      s2sum += a * a;
      next_val = v;
    }
  }
  if (adv_part) {
    // the statistics of rl/algos/ppo.py:484-485 as a by-product of the pass that produces the returns: fixed-order block
    // reduction, one (sum, sumsq) pair per block -> the normalisation needs no statistics pass of its own
    __syncthreads();
#pragma unroll
    for (int o = 16; o; o >>= 1) { s1 += __shfl_xor_sync(0xffffffffu, s1, o); s2sum += __shfl_xor_sync(0xffffffffu, s2sum, o); }
    if (lane == 0) { shA[seg][0] = s1; shC[seg][0] = s2sum; }
    __syncthreads();
    if (threadIdx.x == 0) {
      double a = 0.0, b = 0.0;
#pragma unroll
      for (int k = 0; k < GAE_SEG; k++) { a += shA[k][0]; b += shC[k][0]; }
      adv_part[blockIdx.x] = a;
      adv_part[gridDim.x + blockIdx.x] = b;
    }
  }
}

// stats[0:2] = (sum, sumsq) from the per-block pairs lhw_gae left behind; one warp, index order -> deterministic
__global__ void adv_from_gae_kernel(const double* __restrict__ part, int nblk, double* __restrict__ stats) {
  double a = 0.0, b = 0.0;
  for (int k = threadIdx.x; k < nblk; k += 32) { a += part[k]; b += part[nblk + k]; }
#pragma unroll
  for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(0xffffffffu, a, o); b += __shfl_xor_sync(0xffffffffu, b, o); }
  if (threadIdx.x == 0) { stats[0] = a; stats[1] = b; }
}

// deterministic block reduction helper (fixed tree)
template <int BLOCK> __device__ __forceinline__ double block_sum(double v, double* sh) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  v = threadIdx.x < BLOCK / 32 ? sh[threadIdx.x] : 0.0;
  if (warp == 0)
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  __syncthreads();
  return v;  // valid in warp 0
}

constexpr int NUM_SMS = 132;      // H100 SXM
constexpr int STAT_BLOCKS = NUM_SMS;  // one partial per SM; partials are combined in a fixed order -> deterministic
// stats layout (double[4 + 2*STAT_BLOCKS]): {sum, sumsq, mean, std, partial sums..., partial sumsq...}
__global__ void __launch_bounds__(1024) adv_partial_kernel(const float* __restrict__ ret, const float* __restrict__ val,
                                                           double* __restrict__ stats, long long n) {
  __shared__ double sh[32];
  double s = 0, ss = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double a = (double)ret[i] - (double)val[i];
    s += a;
    ss += a * a;
  }
  s = block_sum<1024>(s, sh);
  ss = block_sum<1024>(ss, sh);
  if (threadIdx.x == 0) {
    stats[4 + blockIdx.x] = s;
    stats[4 + STAT_BLOCKS + blockIdx.x] = ss;
  }
}
__global__ void adv_final_kernel(double* __restrict__ stats) {
  if (threadIdx.x == 0) {
    double s = 0, ss = 0;
    for (int b = 0; b < STAT_BLOCKS; b++) { s += stats[4 + b]; ss += stats[4 + STAT_BLOCKS + b]; }
    stats[0] = s;
    stats[1] = ss;
  }
}
__global__ void adv_apply_kernel(const float* __restrict__ ret, const float* __restrict__ val, float* __restrict__ adv,
                                 double* __restrict__ stats, long long n, long long n_total, double eps) {
  const double mean = stats[0] / (double)n_total;
  double var = (stats[1] - (double)n_total * mean * mean) / (double)(n_total - 1);  // unbiased, torch.std default
  if (var < 0) var = 0;
  const double sd = sqrt(var);
  if (blockIdx.x == 0 && threadIdx.x == 0) { stats[2] = mean; stats[3] = sd; }
  const float fm = (float)mean, inv = (float)(1.0 / (sd + eps));
  const long long tid = (long long)blockIdx.x * blockDim.x + threadIdx.x, stride = (long long)gridDim.x * blockDim.x;
  if ((((uintptr_t)ret | (uintptr_t)val | (uintptr_t)adv) & 15) == 0) {   // 16-byte accesses: 12 B/sample as three vector streams
    const long long n4 = n >> 2;
    const float4* r4 = reinterpret_cast<const float4*>(ret);
    const float4* v4 = reinterpret_cast<const float4*>(val);
    float4* a4 = reinterpret_cast<float4*>(adv);
    for (long long q = tid; q < n4; q += stride) {
      const float4 r = r4[q], v = v4[q];
      a4[q] = make_float4(((r.x - v.x) - fm) * inv, ((r.y - v.y) - fm) * inv, ((r.z - v.z) - fm) * inv, ((r.w - v.w) - fm) * inv);
    }
    for (long long i = 4 * n4 + tid; i < n; i += stride) adv[i] = ((ret[i] - val[i]) - fm) * inv;
  } else {
    for (long long i = tid; i < n; i += stride) adv[i] = ((ret[i] - val[i]) - fm) * inv;
  }
}

__global__ void gather_kernel(const float* __restrict__ obs, const float* __restrict__ act, const float* __restrict__ ret,
                              const float* __restrict__ adv, const int64_t* __restrict__ idx, float* __restrict__ obs_b,
                              float* __restrict__ act_b, float* __restrict__ ret_b, float* __restrict__ adv_b, int B,
                              int obs_dim, int act_dim) {
  const int cols = obs_dim + act_dim + 2;
  const long long total = (long long)B * cols;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const int b = (int)(i / cols), c = (int)(i - (long long)b * cols);
    const long long src = idx[b];
    if (c < obs_dim) obs_b[(size_t)b * obs_dim + c] = obs[src * obs_dim + c];
    else if (c < obs_dim + act_dim) act_b[(size_t)b * act_dim + (c - obs_dim)] = act[src * act_dim + (c - obs_dim)];
    else if (c == obs_dim + act_dim) ret_b[b] = ret[src];
    else adv_b[b] = adv[src];
  }
}

// ||g||^2 with a single block: fixed summation order -> run-to-run deterministic (the reference's determinism
// tests demand bit-identical weights for identical seeds, tests/test_determinism.py:79-146)
__global__ void __launch_bounds__(1024) sumsq_kernel(const float* __restrict__ g, float* __restrict__ out, long long n,
                                                     float scale) {
  __shared__ double sh[32];
  double s = 0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const double v = (double)(g[i] * scale);
    s += v * v;
  }
  s = block_sum<1024>(s, sh);
  if (threadIdx.x == 0) out[0] = (float)s;
}

__global__ void clip_adam_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                 float* __restrict__ v, const float* __restrict__ sumsq, long long n, float lr, float b1,
                                 float b2, float eps, float max_norm, float scale, float bc1, float bc2_sqrt) {
  const float total_norm = sqrtf(sumsq[0]);
  float coef = max_norm / (total_norm + 1e-6f);
  coef = coef > 1.0f ? 1.0f : coef;
  const float gs = scale * coef, step_size = lr / bc1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * gs;
    const float mi = m[i] + (1.0f - b1) * (gi - m[i]);
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= step_size * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}

// the same update with the Adam step number read from device memory: lets the whole optimiser step live inside a CUDA graph
// (a by-value step would be frozen at capture time); step_dev[0] holds the number of completed steps
__global__ void clip_adam_dev_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                     float* __restrict__ v, const float* __restrict__ sumsq, long long n,
                                     const int* __restrict__ step_dev, float lr, float b1, float b2, float eps, float max_norm,
                                     float scale) {
  const float t = (float)(step_dev[0] + 1);
  const float bc1 = 1.0f - powf(b1, t), bc2_sqrt = sqrtf(1.0f - powf(b2, t));
  const float total_norm = sqrtf(sumsq[0]);
  float coef = max_norm / (total_norm + 1e-6f);
  coef = coef > 1.0f ? 1.0f : coef;
  const float gs = scale * coef, step_size = lr / bc1;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const float gi = g[i] * gs;
    const float mi = m[i] + (1.0f - b1) * (gi - m[i]);
    const float vi = b2 * v[i] + (1.0f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    p[i] -= step_size * (mi / (sqrtf(vi) / bc2_sqrt + eps));
  }
}
__global__ void step_inc_kernel(int* step_dev) { step_dev[0] += 1; }

int perr(int code, const char* what, cudaError_t e) {
  g_perr = std::string(what) + ": " + cudaGetErrorString(e);
  return code;
}
#define KCHECK(what)                                   \
  do {                                                 \
    lhw_count_launch();                                \
    cudaError_t _e = cudaGetLastError();               \
    if (_e != cudaSuccess) return perr(-10, what, _e); \
  } while (0)

}  // namespace

extern "C" {

int lhw_gae(const float* rewards, const float* values, const int32_t* ended, const float* boot, const float* last_val,
            float* returns, int T, int N, float gamma, float lam, double* adv_partials_or_null, void* stream) {
  if (T <= 0 || N <= 0) return 0;
  gae_kernel<<<(N + 31) / 32, 32 * GAE_SEG, 0, (cudaStream_t)stream>>>(rewards, values, ended, boot, last_val, returns, T, N,
                                                                (double)gamma, (double)lam, adv_partials_or_null);
  KCHECK("gae_kernel");
  return 0;
}

int lhw_gae_partial_words(int N) { return 2 * ((N + 31) / 32); }

int lhw_adv_stats_from_gae(const double* adv_partials, int N, double* stats, void* stream) {
  if (!adv_partials || !stats || N <= 0) return 0;
  adv_from_gae_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(adv_partials, (N + 31) / 32, stats);
  KCHECK("adv_from_gae_kernel");
  return 0;
}

int lhw_adv_stats_words(void) { return 4 + 2 * STAT_BLOCKS; }

int lhw_adv_stats(const float* returns, const float* values, double* stats, long long count, void* stream) {
  adv_partial_kernel<<<STAT_BLOCKS, 1024, 0, (cudaStream_t)stream>>>(returns, values, stats, count);
  KCHECK("adv_partial_kernel");
  adv_final_kernel<<<1, 32, 0, (cudaStream_t)stream>>>(stats);
  KCHECK("adv_final_kernel");
  return 0;
}

int lhw_adv_apply(const float* returns, const float* values, float* adv, double* stats, long long count,
                  long long count_total, float eps, void* stream) {
  int grid = (int)((count / 4 + 255) / 256);      // one float4 per thread where the batch allows it
  if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
  if (grid < 1) grid = 1;
  adv_apply_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(returns, values, adv, stats, count, count_total, (double)eps);
  KCHECK("adv_apply_kernel");
  return 0;
}

int lhw_gather_minibatch(const float* obs, const float* act, const float* ret, const float* adv, const int64_t* idx,
                         float* obs_b, float* act_b, float* ret_b, float* adv_b, int B, int obs_dim, int act_dim,
                         void* stream) {
  if (B <= 0) return 0;
  const long long total = (long long)B * (obs_dim + act_dim + 2);
  int grid = (int)((total + 255) / 256);
  if (grid > NUM_SMS * 8) grid = NUM_SMS * 8;
  gather_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(obs, act, ret, adv, idx, obs_b, act_b, ret_b, adv_b, B, obs_dim,
                                                        act_dim);
  KCHECK("gather_kernel");
  return 0;
}

int lhw_grad_sumsq(const float* grad, float* norm_scratch, long long n, float grad_scale, void* stream) {
  sumsq_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(grad, norm_scratch, n, grad_scale);
  KCHECK("sumsq_kernel");
  return 0;
}

int lhw_clip_adam(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* norm_scratch,
                  long long n, int step, float lr, float beta1, float beta2, float eps, float max_norm,
                  float grad_scale, void* stream) {
  if (n <= 0) return 0;
  const float bc1 = 1.0f - powf(beta1, (float)step);
  const float bc2_sqrt = sqrtf(1.0f - powf(beta2, (float)step));
  int grid = (int)((n + 255) / 256);
  if (grid > NUM_SMS * 4) grid = NUM_SMS * 4;
  clip_adam_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, norm_scratch, n, lr, beta1,
                                                           beta2, eps, max_norm, grad_scale, bc1, bc2_sqrt);
  KCHECK("clip_adam_kernel");
  return 0;
}

int lhw_clip_adam_dev(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, const float* norm_scratch,
                      long long n, int* step_dev, float lr, float beta1, float beta2, float eps, float max_norm,
                      float grad_scale, void* stream) {
  if (n <= 0 || !step_dev) return 0;
  int grid = (int)((n + 255) / 256);
  if (grid > NUM_SMS * 4) grid = NUM_SMS * 4;
  clip_adam_dev_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(param, grad, exp_avg, exp_avg_sq, norm_scratch, n, step_dev, lr,
                                                               beta1, beta2, eps, max_norm, grad_scale);
  KCHECK("clip_adam_dev_kernel");
  step_inc_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(step_dev);
  KCHECK("step_inc_kernel");
  return 0;
}

}  // extern "C"

// ================================================================= fused PPO loss tail (rl/algos/ppo.py:302-386)
// Everything between the network outputs and the scalar loss, forward AND backward, in one pass over the minibatch:
//   log-probabilities of the taken actions under the new and the old policy (fixed per-action std), ratio, clipped surrogate,
//   value MSE, entropy, mirror MSE, approximate KL, clip fraction -> 7 scalars; and the gradients of
//   total = actor + mirror_coeff * mirror + ent_coeff * entropy_penalty + critic  w.r.t. the policy mean, the mirrored
//   mean and the values.  torch autograd then only runs the three MLP backward passes (cuBLAS).  One thread per sample,
//   per-block partial sums combined in block order by the last block (ticket) -> run-to-run deterministic.
// IMIT = true adds the imitation term (DESIGN §7.2): imitation = mean over B*A of m_b (mu_bk - teacher_bk)^2 with the mask
//   m_b (1 where `imask` is null), in the spare partial slot 5, and imitate_coeff * imitation in the total.  IMIT = false is the
//   kernel without it, instruction for instruction (the imitation arguments come last, so the others keep their offsets).
namespace {
constexpr int LOSS_BLOCK = 256, LOSS_NS = 6;   // partial sums: surrogate, clipfrac, critic, kl, mirror, imitation
template <bool IMIT>
__global__ void __launch_bounds__(LOSS_BLOCK)
    ppo_loss_kernel(const float* __restrict__ mu, const float* __restrict__ old_mu, const float* __restrict__ act,
                    const float* __restrict__ adv, const float* __restrict__ ret, const float* __restrict__ val,
                    const float* __restrict__ mirr /* [B,A] mirrored actions or null */, const float* __restrict__ stds, int B, int A,
                    float clip, float mirror_coeff, float ent_coeff, float* __restrict__ g_mu, float* __restrict__ g_mirr,
                    float* __restrict__ g_val, double* __restrict__ partials, unsigned int* __restrict__ ticket,
                    float* __restrict__ out7, const float* __restrict__ teacher /* [B,A] teacher actions (IMIT) */,
                    const float* __restrict__ imask /* [B] mask or null (IMIT) */, float imitate_coeff) {
  __shared__ double sh[LOSS_NS][LOSS_BLOCK / 32];
  __shared__ int last;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  double s[LOSS_NS] = {0, 0, 0, 0, 0, 0};
  const float invB = 1.0f / (float)B, invBA = 1.0f / ((float)B * (float)A);
  if (b < B) {
    const float* m = mu + (size_t)b * A;
    const float* om = old_mu + (size_t)b * A;
    const float* a = act + (size_t)b * A;
    float lp = 0.f, olp = 0.f;
    for (int k = 0; k < A; k++) {      // Normal(mu, sd).log_prob(a) summed over the action dims (the constant terms cancel in lp - olp)
      const float sd = stds[k], z = (a[k] - m[k]) / sd, zo = (a[k] - om[k]) / sd;
      lp += -0.5f * z * z;
      olp += -0.5f * zo * zo;
    }
    const float dlp = lp - olp, ratio = expf(dlp), ad = adv[b];
    const float cpi = ratio * ad, rc = fminf(fmaxf(ratio, 1.0f - clip), 1.0f + clip), cl = rc * ad;
    s[0] = (double)fminf(cpi, cl);
    s[1] = fabsf(ratio - 1.0f) > clip ? 1.0 : 0.0;
    const float dv = val[b] - ret[b];
    s[2] = (double)dv * dv;
    s[3] = (double)((ratio - 1.0f) - dlp);
    // d(-mean min(cpi, clip)) / d lp : the clamp passes the gradient inside [1-c, 1+c]; outside, only the unclipped branch
    // has one, and torch.min hands it the gradient when it is the smaller of the two
    const bool inside = ratio >= 1.0f - clip && ratio <= 1.0f + clip;
    const float glp = (inside || cpi < cl) ? -invB * ratio * ad : 0.0f;
    g_val[b] = 2.0f * dv * invB;
    float ci = 0.f, mb = 1.f;     // d imitate_coeff * imitation / d (mu - teacher) = ci * (mu - teacher)
    if constexpr (IMIT) {
      mb = imask ? imask[b] : 1.0f;
      ci = imitate_coeff * 2.0f * mb * invBA;
    }
    for (int k = 0; k < A; k++) {
      const float sd = stds[k];
      float g = glp * (a[k] - m[k]) / (sd * sd);
      if (mirr) {
        const float d = m[k] - mirr[(size_t)b * A + k];
        s[4] += (double)d * d;
        const float gm = mirror_coeff * 2.0f * d * invBA;
        g += gm;
        g_mirr[(size_t)b * A + k] = -gm;
      }
      if constexpr (IMIT) {
        const float d = m[k] - teacher[(size_t)b * A + k];
        s[5] += (double)mb * ((double)d * d);
        if (ci != 0.f) g += ci * d;     // a zero mask or coefficient leaves g exactly as the kernel without the term has it
      }
      g_mu[(size_t)b * A + k] = g;
    }
  }
#pragma unroll
  for (int q = 0; q < LOSS_NS; q++) {
    double v = s[q];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if ((threadIdx.x & 31) == 0) sh[q][threadIdx.x >> 5] = v;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int q = 0; q < LOSS_NS; q++) {
      double v = 0;
      for (int w = 0; w < LOSS_BLOCK / 32; w++) v += sh[q][w];
      partials[(size_t)blockIdx.x * LOSS_NS + q] = v;
    }
    __threadfence();
    last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!last || threadIdx.x >= 32) return;
  __threadfence();
  double t[LOSS_NS];
#pragma unroll
  for (int q = 0; q < LOSS_NS; q++) {
    double v = 0;
    for (int k = threadIdx.x; k < (int)gridDim.x; k += 32) v += __ldcg(partials + (size_t)k * LOSS_NS + q);
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    t[q] = v;
  }
  if (threadIdx.x == 0) {
    float ent = 0.f;     // Normal.entropy() = 0.5 + 0.5 log(2 pi) + log sd per action dim, the same for every sample
    for (int k = 0; k < A; k++) ent += 0.5f + 0.9189385332046727f + logf(stds[k]);
    ent /= (float)A;
    const float actor = (float)(-t[0] / B), critic = (float)(t[2] / B), mirror = mirr ? (float)(t[4] / ((double)B * A)) : 0.f;
    out7[0] = actor;                    // actor_loss
    out7[1] = -ent;                     // entropy_penalty
    out7[2] = critic;                   // critic_loss
    out7[3] = (float)(t[3] / B);        // approx_kl_div
    out7[4] = mirror;                   // mirror_loss
    const float imitation = IMIT ? (float)(t[5] / ((double)B * A)) : 0.f;
    out7[5] = imitation;                // imitation_loss (0 without a teacher)
    out7[6] = (float)(t[1] / B);        // clip_fraction
    if constexpr (IMIT)
      out7[7] = actor + mirror_coeff * mirror + imitate_coeff * imitation + ent_coeff * (-ent) + critic;   // total
    else
      out7[7] = actor + mirror_coeff * mirror + ent_coeff * (-ent) + critic;   // total
    *ticket = 0;
  }
}

template <bool IMIT>
int launch_ppo_loss(const float* mu, const float* old_mu, const float* act, const float* adv, const float* ret, const float* val,
                    const float* mirr, const float* stds, int B, int A, float clip, float mirror_coeff, float ent_coeff, float* g_mu,
                    float* g_mirr, float* g_val, double* partials, unsigned int* ticket, float* out8, const float* teacher,
                    const float* imask, float imitate_coeff, void* stream) {
  ppo_loss_kernel<IMIT><<<(B + LOSS_BLOCK - 1) / LOSS_BLOCK, LOSS_BLOCK, 0, (cudaStream_t)stream>>>(
      mu, old_mu, act, adv, ret, val, mirr, stds, B, A, clip, mirror_coeff, ent_coeff, g_mu, g_mirr, g_val, partials, ticket, out8,
      teacher, imask, imitate_coeff);
  KCHECK("ppo_loss_kernel");
  return 0;
}
}  // namespace

extern "C" int lhw_ppo_loss_partial_words(int B) { return LOSS_NS * ((B + LOSS_BLOCK - 1) / LOSS_BLOCK); }

extern "C" int lhw_ppo_loss(const float* mu, const float* old_mu, const float* act, const float* adv, const float* ret, const float* val,
                            const float* mirr_or_null, const float* stds, int B, int A, float clip, float mirror_coeff, float ent_coeff,
                            float* g_mu, float* g_mirr_or_null, float* g_val, double* partials, unsigned int* ticket, float* out8,
                            void* stream) {
  if (B <= 0 || A <= 0) return 0;
  if (mirr_or_null && !g_mirr_or_null) { g_perr = "lhw_ppo_loss: mirrored actions without a gradient buffer"; return -1; }
  return launch_ppo_loss<false>(mu, old_mu, act, adv, ret, val, mirr_or_null, stds, B, A, clip, mirror_coeff, ent_coeff, g_mu,
                                g_mirr_or_null, g_val, partials, ticket, out8, nullptr, nullptr, 0.f, stream);
}

extern "C" int lhw_ppo_loss_imitation(const float* mu, const float* old_mu, const float* act, const float* adv, const float* ret,
                                      const float* val, const float* mirr_or_null, const float* stds, const float* teacher_mu,
                                      const float* mask_or_null, int B, int A, float clip, float mirror_coeff, float ent_coeff,
                                      float imitate_coeff, float* g_mu, float* g_mirr_or_null, float* g_val, double* partials,
                                      unsigned int* ticket, float* out8, void* stream) {
  if (B <= 0 || A <= 0) return 0;
  if (mirr_or_null && !g_mirr_or_null) { g_perr = "lhw_ppo_loss_imitation: mirrored actions without a gradient buffer"; return -1; }
  if (!teacher_mu) { g_perr = "lhw_ppo_loss_imitation: no teacher actions"; return -1; }
  return launch_ppo_loss<true>(mu, old_mu, act, adv, ret, val, mirr_or_null, stds, B, A, clip, mirror_coeff, ent_coeff, g_mu,
                               g_mirr_or_null, g_val, partials, ticket, out8, teacher_mu, mask_or_null, imitate_coeff, stream);
}
