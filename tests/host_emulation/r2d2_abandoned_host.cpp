// TEST HARNESS (never part of libseedrl_b200.so): r2d2_loss_thread and r2d2_retrace_loss_thread -- the bodies
// the GPU kernels execute, from seed_rl_b200/csrc/r2d2_thread.inl -- compiled as plain host C++ with an
// abandoned mask (NULL = none), so that the CPU test suite can check them against
// tests/abandoned_float64_reference.py and against the same bodies without the mask.
//   g++ -O2 -shared -fPIC -o _r2d2_abandoned_host.so r2d2_abandoned_host.cpp
#include <math.h>
#define SEEDRL_HD inline
#include "../../seed_rl_b200/csrc/r2d2_thread.inl"

extern "C" int emu_r2d2_loss_abandoned(int T, int B, int A, const float* q_train, const float* q_target,
                                       const int64_t* replay_action, const float* reward, const uint8_t* done,
                                       const uint8_t* abandoned, const float* is_weights, float gamma, int n_steps,
                                       float eta, float eps, float* loss, float* priorities, float* dq,
                                       float* scratch) {
  seedrl::R2d2LossParams p;
  p.T = T; p.B = B; p.A = A; p.n_steps = n_steps;
  p.q_train = q_train; p.q_target = q_target; p.replay_action = replay_action; p.reward = reward; p.done = done;
  p.is_weights = is_weights; p.gamma = gamma; p.eta = eta; p.eps = eps;
  for (int k = 0; k < 8; ++k) p.gamma_pow[k] = (float)pow((double)gamma, (double)k);   // as the C entry point
  p.loss = loss; p.priorities = priorities; p.dq = dq; p.scratch = scratch;
  p.abandoned = abandoned;
  for (int b = 0; b < B; ++b) seedrl::r2d2_loss_thread(p, b);
  return 0;
}

extern "C" int emu_r2d2_retrace_loss_abandoned(int T, int B, int A, const float* q_train, const float* q_target,
                                               const int64_t* replay_action, const float* reward,
                                               const uint8_t* done, const uint8_t* abandoned,
                                               const float* is_weights, float gamma, float lambda_, float eta,
                                               float eps, float* loss, float* priorities, float* dq,
                                               float* scratch) {
  seedrl::R2d2RetraceParams p;
  p.T = T; p.B = B; p.A = A;
  p.q_train = q_train; p.q_target = q_target; p.replay_action = replay_action; p.reward = reward; p.done = done;
  p.is_weights = is_weights; p.gamma = gamma; p.lambda = lambda_; p.eta = eta; p.eps = eps;
  p.loss = loss; p.priorities = priorities; p.dq = dq; p.scratch = scratch;
  p.abandoned = abandoned;
  for (int b = 0; b < B; ++b) seedrl::r2d2_retrace_loss_thread(p, b);
  return 0;
}
