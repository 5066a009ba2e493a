// Device harness of the fused gradient exchange (learninghumanoidwalking_b200/csrc/comm_kernels.cu) for
// tests/test_gpu_exchange_ranks.py: W comm records on ONE device stand in for W ranks.  Record r's peer table points straight
// at the other records' gradients and flag words (no CUDA IPC), and the ranks step one after another on one stream.  Before
// rank q's step the flag words of the ranks that step after it are set ahead of any epoch (bytes 0x3F: 0x3F3F3F3F), and the
// ranks before it have already written epoch + 1 there themselves, so no wait of the kernels spins: each rank does exactly the
// loads, rank-order sums, flag writes and coefficient work it does on its own GPU.
//
// The product source is compiled unchanged.  Built with -fvisibility=hidden: the harness's own copies of lhw_comm_create and
// the other C-ABI functions bind inside this library and neither see nor shadow those of liblhw_b200.so in the same process;
// only the cx_* entry points below are exported.
#include "../../learninghumanoidwalking_b200/csrc/comm_kernels.cu"

extern "C" void lhw_count_launch(void) {}

#define CX_EXPORT extern "C" __attribute__((visibility("default")))

// W records of n floats on `device`, each wired to all the others
CX_EXPORT int cx_create(lhw_comm** cs, long long n, int world, int device) {
  for (int r = 0; r < world; r++) {
    const int rc = lhw_comm_create(&cs[r], n, r, world, device);
    if (rc) {
      while (r-- > 0) lhw_comm_destroy(cs[r]);
      return rc;
    }
  }
  for (int r = 0; r < world; r++)
    for (int q = 0; q < world; q++) {
      cs[r]->peers.grad[q] = cs[q]->grad;
      cs[r]->peers.flags[q] = cs[q]->flags;
    }
  return 0;
}

CX_EXPORT void cx_destroy(lhw_comm** cs, int world) {
  for (int r = 0; r < world; r++) lhw_comm_destroy(cs[r]);
}

// device addresses: grad, flags (MAX_WORLD flag words, then the KL words), reduced, coef, state, lr; then the float count
// the gradient and `reduced` allocations hold (n rounded up to 256 bytes) and the words of `flags`
CX_EXPORT void cx_pointers(const lhw_comm* c, unsigned long long* out) {
  out[0] = (unsigned long long)c->grad;
  out[1] = (unsigned long long)c->flags;
  out[2] = (unsigned long long)c->reduced;
  out[3] = (unsigned long long)c->coef;
  out[4] = (unsigned long long)c->state;
  out[5] = (unsigned long long)c->lr;
  out[6] = grad_bytes(c->n) / sizeof(float);
  out[7] = MAX_WORLD + KL_WORDS;
}

CX_EXPORT void cx_set_spin_limit(lhw_comm* c, long long polls) { c->spin_limit = polls; }

// the flag words of the ranks after c->rank in the stepping order, set ahead of any epoch; a memset node when captured
CX_EXPORT int cx_preset_later_peers(lhw_comm* c, void* stream) {
  if (c->rank + 1 >= c->world) return 0;
  COK(cudaMemsetAsync(c->flags + c->rank + 1, 0x3F, (size_t)(c->world - c->rank - 1) * sizeof(unsigned int), (cudaStream_t)stream));
  return 0;
}

CX_EXPORT int cx_step(lhw_comm* c, float* param, float* m, float* v, long long n_actor, long long n_total, float lr, float beta1,
                      float beta2, float eps, float max_norm, void* stream) {
  return lhw_fused_allreduce_clip_adam(c, param, m, v, n_actor, n_total, lr, beta1, beta2, eps, max_norm, stream);
}

CX_EXPORT int cx_step_adaptive(lhw_comm* c, float* param, float* m, float* v, long long n_actor, long long n_total, const float* kl,
                               double* lr_dev, double desired_kl, float beta1, float beta2, float eps, float max_norm, void* stream) {
  return lhw_fused_allreduce_clip_adam_adaptive(c, param, m, v, n_actor, n_total, kl, lr_dev, desired_kl, beta1, beta2, eps, max_norm,
                                                stream);
}

CX_EXPORT int cx_status(lhw_comm* c, int* error_word, int* adam_steps, float* norms2, void* stream) {
  return lhw_comm_status(c, error_word, adam_steps, norms2, stream);
}

CX_EXPORT const char* cx_last_error(void) { return lhw_comm_last_error(); }
