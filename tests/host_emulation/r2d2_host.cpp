// TEST HARNESS (never part of libseedrl_b200.so): compiles the per-thread bodies of the R2D2
// kernels -- the same source text the GPU kernels execute, seed_rl_b200/csrc/r2d2_thread.inl --
// as plain host C++ and runs them thread by thread, so that the CPU test suite can check the
// algorithm and its indexing against oracle/r2d2_oracle.py without a GPU.
//   g++ -O2 -shared -fPIC -o _r2d2_host.so r2d2_host.cpp
#define SEEDRL_HD inline
#include "../../seed_rl_b200/csrc/r2d2_thread.inl"

#include <math.h>

extern "C" int emu_stack_frames(int T, int B, int P, int S, const uint8_t* frames, const int32_t* state_in,
                                const uint8_t* done, uint8_t* stacked, int32_t* state_out) {
  for (int b = 0; b < B; ++b)
    for (int p = 0; p < P; ++p) {
      if (S == 4) seedrl::r2d2_stack_frames_thread<4>(T, B, P, b, p, frames, state_in, done, stacked, state_out);
      else if (S == 3) seedrl::r2d2_stack_frames_thread<3>(T, B, P, b, p, frames, state_in, done, stacked, state_out);
      else if (S == 2) seedrl::r2d2_stack_frames_thread<2>(T, B, P, b, p, frames, state_in, done, stacked, state_out);
      else return 1;
    }
  return 0;
}

extern "C" int emu_r2d2_loss(int T, int B, int A, const float* q_train, const float* q_target,
                             const int64_t* replay_action, const float* reward, const uint8_t* done,
                             const float* is_weights, float gamma, int n_steps, float eta, float eps, float* loss,
                             float* priorities, float* dq, float* scratch) {
  seedrl::R2d2LossParams p;
  p.T = T; p.B = B; p.A = A; p.n_steps = n_steps;
  p.q_train = q_train; p.q_target = q_target; p.replay_action = replay_action; p.reward = reward; p.done = done;
  p.is_weights = is_weights; p.gamma = gamma; p.eta = eta; p.eps = eps;
  for (int k = 0; k < 8; ++k) p.gamma_pow[k] = (float)pow((double)gamma, (double)k);   // as seedrl_r2d2_loss_fwd_bwd
  p.loss = loss; p.priorities = priorities; p.dq = dq; p.scratch = scratch;
  for (int b = 0; b < B; ++b) seedrl::r2d2_loss_thread(p, b);
  return 0;
}

// the value rescaling h (inverse = 0) or h^-1 (inverse = 1) of the loss bodies, elementwise
extern "C" int emu_vf_rescale(int n, const float* x, float eps, int inverse, float* out) {
  for (int i = 0; i < n; ++i) out[i] = inverse ? seedrl::vf_rescale_inv(x[i], eps) : seedrl::vf_rescale(x[i], eps);
  return 0;
}

// replay_sample_kernel's phases in the order the kernel runs them (one CTA); prefix_only draws with
// the overload that takes the probability from cdf[i] - cdf[i-1] instead of the item's mass
static void replay_sample(bool prefix_only, int limit, const float* priorities, float priority_exp, float is_exp,
                          int num_samples, const float* uniforms, int64_t* indices, float* weights,
                          float* probs_out) {
  float* cdf = new float[limit];
  for (int i = 0; i < limit; ++i) seedrl::replay_pow_thread(i, priorities, priority_exp, cdf);
  const float total = seedrl::replay_prefix_serial(limit, cdf);
  if (probs_out)
    for (int i = 0; i < limit; ++i) probs_out[i] = seedrl::replay_mass(i, priorities, priority_exp) / total;
  float wmax = 0.f;
  for (int j = 0; j < num_samples; ++j)
    wmax = fmaxf(wmax, prefix_only
                           ? seedrl::replay_sample_thread(j, limit, cdf, total, is_exp, uniforms, indices, weights)
                           : seedrl::replay_sample_thread(j, limit, cdf, total, priorities, priority_exp, is_exp,
                                                          uniforms, indices, weights));
  for (int j = 0; j < num_samples; ++j) weights[j] /= wmax;
  delete[] cdf;
}

extern "C" int emu_replay_sample(int limit, const float* priorities, float priority_exp, float is_exp,
                                 int num_samples, const float* uniforms, int64_t* indices, float* weights,
                                 float* probs_out) {
  replay_sample(false, limit, priorities, priority_exp, is_exp, num_samples, uniforms, indices, weights, probs_out);
  return 0;
}

extern "C" int emu_replay_sample_prefix_only(int limit, const float* priorities, float priority_exp, float is_exp,
                                             int num_samples, const float* uniforms, int64_t* indices,
                                             float* weights) {
  replay_sample(true, limit, priorities, priority_exp, is_exp, num_samples, uniforms, indices, weights, nullptr);
  return 0;
}
