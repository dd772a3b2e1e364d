// R2D2 (SURVEY 8(a) row a11) post-network kernels for sm_90a:
//
//   r2d2_stack_frames_kernel   atari/networks.py:57-173   bit-packed frame stacking (uint8/int32)
//   r2d2_loss_kernel           agents/r2d2/learner.py:180-330  h / h^-1, n-step double-DQN
//                              targets, per-sequence loss, priorities and d loss / d q
//   r2d2_retrace_loss_kernel   the same loss with Retrace(lambda) targets (Munos et al. 2016), greedy
//                              target policy; not in the reference (opt-in)
//   replay_sample_kernel       common/utils.py:327-352    p_i ~ prio_i^alpha, inverse-CDF draw,
//                              importance weights normalised by their max
//   global-norm clip           tf.clip_by_global_norm, learner.py:608 (clip_norm = 40)
//   r2d2_epsilon_greedy_kernel agents/r2d2/learner.py:155-177  epsilon-greedy on the device, Philox
//                              offset from a device counter (CUDA-graph replays)
//
// Parity: tests/test_gpu_r2d2.py against oracle/r2d2_oracle.py / oracle/r2d2_learner_oracle.py (frame
// stacking and replay indices bit-exact, loss / priorities / dq within fp32 rounding), on an H100.
// The network itself (DuelingLSTMDQNNet forward / backward) is csrc/r2d2_net.cu.  Nothing on the
// V-trace path calls these kernels.
//
// All of it is HBM-/latency-bound byte and elementwise work: coalesced accesses across the
// pixel or batch axis, sequential walks along time in registers.
#include <math.h>

#include "common.cuh"
#include "r2d2_thread.inl"

namespace seedrl {

// ---------------------------------------------------------------------------------------
// The per-thread bodies live in r2d2_thread.inl (shared with the host emulation harness).
template <int S>
__global__ void r2d2_stack_frames_kernel(int T, int B, int P, const uint8_t* __restrict__ frames,
                                         const int32_t* __restrict__ state_in,
                                         const uint8_t* __restrict__ done,
                                         uint8_t* __restrict__ stacked, int32_t* __restrict__ state_out) {
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= P) return;
  r2d2_stack_frames_thread<S>(T, B, P, blockIdx.y, p, frames, state_in, done, stacked, state_out);
}

__global__ void r2d2_loss_kernel(const R2d2LossParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  r2d2_loss_thread(p, b);
}

__global__ void r2d2_retrace_loss_kernel(const R2d2RetraceParams p) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.B) return;
  r2d2_retrace_loss_thread(p, b);
}

// ---------------------------------------------------------------------------------------
// Single CTA (the replay holds ~100 unrolls): inclusive CDF of prio^alpha in shared memory; sample
// j = first i with cdf[i] > u_j * total; prob_i = prio_i^alpha / total from the item's own mass
// (for the weights and probs_out alike); weights = ((1/limit)/prob_i)^beta / max.
constexpr int kReplayMax = 8192;
__global__ void __launch_bounds__(1024)
replay_sample_kernel(int limit, const float* __restrict__ priorities, float priority_exp, float is_exp,
                     int num_samples, const float* __restrict__ uniforms, int64_t* __restrict__ indices,
                     float* __restrict__ weights, float* __restrict__ probs_out) {
  __shared__ float s_cdf[kReplayMax];
  __shared__ float s_red[32];
  const int tid = threadIdx.x;
  for (int i = tid; i < limit; i += blockDim.x) replay_pow_thread(i, priorities, priority_exp, s_cdf);
  __syncthreads();
  // serial prefix by one thread in index order: deterministic, and 100..8192 adds are nothing
  if (tid == 0) s_red[0] = replay_prefix_serial(limit, s_cdf);
  __syncthreads();
  const float total = s_red[0];
  if (probs_out)
    for (int i = tid; i < limit; i += blockDim.x) probs_out[i] = replay_mass(i, priorities, priority_exp) / total;
  float wmax = 0.f;
  for (int j = tid; j < num_samples; j += blockDim.x)
    wmax = fmaxf(wmax, replay_sample_thread(j, limit, s_cdf, total, priorities, priority_exp, is_exp, uniforms,
                                            indices, weights));
  // max over the CTA, then normalise
  for (int o = 16; o; o >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xffffffffu, wmax, o));
  __syncthreads();
  if ((tid & 31) == 0) s_red[tid >> 5] = wmax;
  __syncthreads();
  float m = 0.f;
  for (int k = 0; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, s_red[k]);
  for (int j = tid; j < num_samples; j += blockDim.x) weights[j] /= m;
}

// ---------------------------------------------------------------------------------------
// tf.clip_by_global_norm: g *= clip * min(1/norm, 1/clip) + (norm - norm), norm = ||g||_2.  The
// (norm - norm) term is TF's: an infinite or NaN norm turns every element into NaN, so a broken
// gradient is visible instead of being zeroed (inf) or passed unclipped (NaN).  Deterministic
// two-stage reduction.
__global__ void sumsq_partial_kernel(size_t n, const float* __restrict__ g, float* __restrict__ partial) {
  __shared__ float red[32];
  float s = 0.f;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    s = fmaf(g[i], g[i], s);
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < (int)(blockDim.x >> 5); ++k) t += red[k];
    partial[blockIdx.x] = t;
  }
}
__global__ void clip_scale_kernel(size_t n, float* __restrict__ g, const float* __restrict__ partial, int nparts,
                                  float clip_norm, float* __restrict__ norm_out) {
  __shared__ float s_scale;
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int k = 0; k < nparts; ++k) t += partial[k];        // fixed order
    const float norm = sqrtf(t);
    // fminf drops a NaN operand: the NaN of a non-finite norm comes in through (norm - norm) only
    s_scale = clip_norm * fminf(1.f / norm, 1.f / clip_norm) + (norm - norm);
    if (norm_out && blockIdx.x == 0) *norm_out = norm;
  }
  __syncthreads();
  const float sc = s_scale;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    g[i] *= sc;
}

// ---------------------------------------------------------------------------------------
// Epsilon-greedy: row n draws r = philox4x32_10((counter lo, counter hi, n, 0), seed); it explores
// iff (r.x >> 8) * 2^-24 < epsilon(env), with the uniform action (r.y * A) >> 32.  The formulas are
// part of the interface: tests restate them in numpy bit for bit.
__global__ void r2d2_epsilon_greedy_kernel(int N, int A, const int32_t* __restrict__ env_ids,
                                           const float* __restrict__ envs_epsilon, uint64_t seed,
                                           const uint64_t* __restrict__ counter, int32_t* __restrict__ actions) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  const uint64_t c = *counter;
  const uint4 r = philox4x32_10(make_uint4((uint32_t)c, (uint32_t)(c >> 32), (uint32_t)n, 0u),
                                make_uint2((uint32_t)seed, (uint32_t)(seed >> 32)));
  if ((float)(r.x >> 8) * 5.9604644775390625e-8f < envs_epsilon[env_ids[n]])
    actions[n] = (int32_t)(((uint64_t)r.y * (uint64_t)A) >> 32);
}

// a separate one-thread launch, so that no block of the draw can see the incremented counter
__global__ void r2d2_bump_counter_kernel(uint64_t* counter) { *counter += 1; }

}  // namespace seedrl

using namespace seedrl;

extern "C" int seedrl_r2d2_stack_frames(int T, int B, int P, int stack_size, const uint8_t* frames,
                                        const int32_t* state_in, const uint8_t* done, uint8_t* stacked,
                                        int32_t* state_out, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T >= 0 && B >= 1 && P >= 1, "bad T/B/P");
  SEEDRL_CHECK_ARG(stack_size >= 2 && stack_size <= 4,
                   "Only up to stack size 4 is supported due to bit-packing.");   // networks.py:98-99
  SEEDRL_CHECK_ARG(frames && state_in && done && stacked && state_out, "null pointer");
  const dim3 grid(ceil_div(P, 256), B);
  cudaStream_t st = (cudaStream_t)stream;
  if (stack_size == 4) r2d2_stack_frames_kernel<4><<<grid, 256, 0, st>>>(T, B, P, frames, state_in, done, stacked, state_out);
  else if (stack_size == 3) r2d2_stack_frames_kernel<3><<<grid, 256, 0, st>>>(T, B, P, frames, state_in, done, stacked, state_out);
  else r2d2_stack_frames_kernel<2><<<grid, 256, 0, st>>>(T, B, P, frames, state_in, done, stacked, state_out);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" size_t seedrl_r2d2_loss_scratch_bytes(int T, int B, int n_steps) {
  return (size_t)B * (size_t)(T + n_steps) * sizeof(float);
}

extern "C" int seedrl_r2d2_loss_fwd_bwd(int T, int B, int A, const float* q_train, const float* q_target,
                                        const int64_t* replay_action, const float* reward, const uint8_t* done,
                                        const float* importance_weights, float gamma, int n_steps, float eta,
                                        float value_rescaling_eps, float* loss, float* priorities, float* dq,
                                        void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T >= 2 && B >= 1 && A >= 1, "need T>=2, B>=1, A>=1");
  SEEDRL_CHECK_ARG(n_steps >= 1 && n_steps <= 8, "n_steps must be in [1, 8]");
  SEEDRL_CHECK_ARG(q_train && q_target && replay_action && reward && done && loss && priorities && dq && scratch,
                   "null pointer");
  R2d2LossParams p;
  p.T = T; p.B = B; p.A = A; p.n_steps = n_steps;
  p.q_train = q_train; p.q_target = q_target; p.replay_action = replay_action; p.reward = reward;
  p.done = done; p.is_weights = importance_weights; p.gamma = gamma; p.eta = eta; p.eps = value_rescaling_eps;
  for (int k = 0; k < 8; ++k) p.gamma_pow[k] = (float)pow((double)gamma, (double)k);   // fp32(gamma ** k)
  p.loss = loss; p.priorities = priorities; p.dq = dq; p.scratch = reinterpret_cast<float*>(scratch);
  r2d2_loss_kernel<<<ceil_div(B, 64), 64, 0, (cudaStream_t)stream>>>(p);
  count_launch(PC_LOSS, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" size_t seedrl_r2d2_retrace_loss_scratch_bytes(int T, int B) {
  return (size_t)B * (size_t)T * sizeof(float);
}

extern "C" int seedrl_r2d2_retrace_loss_fwd_bwd(int T, int B, int A, const float* q_train, const float* q_target,
                                                const int64_t* replay_action, const float* reward,
                                                const uint8_t* done, const float* importance_weights, float gamma,
                                                float lambda_, float eta, float value_rescaling_eps, float* loss,
                                                float* priorities, float* dq, void* scratch,
                                                seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T >= 2 && B >= 1 && A >= 1, "need T>=2, B>=1, A>=1");
  SEEDRL_CHECK_ARG(lambda_ >= 0.f && lambda_ <= 1.f, "lambda must be in [0, 1]");   // false for NaN
  SEEDRL_CHECK_ARG(q_train && q_target && replay_action && reward && done && loss && priorities && dq && scratch,
                   "null pointer");
  R2d2RetraceParams p;
  p.T = T; p.B = B; p.A = A;
  p.q_train = q_train; p.q_target = q_target; p.replay_action = replay_action; p.reward = reward;
  p.done = done; p.is_weights = importance_weights;
  p.gamma = gamma; p.lambda = lambda_; p.eta = eta; p.eps = value_rescaling_eps;
  p.loss = loss; p.priorities = priorities; p.dq = dq; p.scratch = reinterpret_cast<float*>(scratch);
  r2d2_retrace_loss_kernel<<<ceil_div(B, 64), 64, 0, (cudaStream_t)stream>>>(p);
  count_launch(PC_LOSS, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_replay_sample(int limit, const float* priorities, float priority_exp,
                                    float importance_sampling_exp, int num_samples, const float* uniforms,
                                    int64_t* indices, float* weights, float* probs_out,
                                    seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(limit >= 1 && limit <= kReplayMax, "replay limit must be in [1, 8192]");
  SEEDRL_CHECK_ARG(num_samples >= 1 && priorities && uniforms && indices && weights, "bad arguments");
  replay_sample_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(limit, priorities, priority_exp,
                                                            importance_sampling_exp, num_samples, uniforms,
                                                            indices, weights, probs_out);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_r2d2_epsilon_greedy(int N, int A, const int32_t* env_ids, const float* envs_epsilon,
                                          uint64_t seed, uint64_t* counter_dev, int32_t* actions,
                                          seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 0 && A >= 1, "need N >= 0, A >= 1");
  SEEDRL_CHECK_ARG(env_ids && envs_epsilon && counter_dev && actions, "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (N > 0) {
    r2d2_epsilon_greedy_kernel<<<ceil_div(N, 128), 128, 0, st>>>(N, A, env_ids, envs_epsilon, seed, counter_dev,
                                                                  actions);
    count_launch(PC_MISC, st);
    SEEDRL_CHECK_LAUNCH();
  }
  r2d2_bump_counter_kernel<<<1, 1, 0, st>>>(counter_dev);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" size_t seedrl_clip_scratch_bytes(void) { return 1024 * sizeof(float); }

extern "C" int seedrl_clip_by_global_norm(size_t n, float* grads, float clip_norm, float* norm_out,
                                          void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG((grads || n == 0) && scratch && clip_norm > 0.f, "bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {                                              // the norm of an empty arena is 0
    if (norm_out) SEEDRL_CUDA(cudaMemsetAsync(norm_out, 0, sizeof(float), st));
    return SEEDRL_OK;
  }
  const int parts = 4 * kNumSMs;
  float* partial = reinterpret_cast<float*>(scratch);
  sumsq_partial_kernel<<<parts, 256, 0, st>>>(n, grads, partial);
  count_launch(PC_ADAM, st);
  SEEDRL_CHECK_LAUNCH();
  clip_scale_kernel<<<parts, 256, 0, st>>>(n, grads, partial, parts, clip_norm, norm_out);
  count_launch(PC_ADAM, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}
