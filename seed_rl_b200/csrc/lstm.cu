// The LSTM recurrence of one network call, in each lstm_mode: the one place that dispatches on the mode
// (net.cu and r2d2_net.cu call it), and its C-ABI test hook, which makes the same calls.
#include "schedule.h"

namespace seedrl {

int lstm_recurrence_forward(int mode, int H, int T1, int B, const float* U, const uint8_t* done, float* z,
                            const float* h0, const float* c0, float* hs, float* cs, float* hp, unsigned int* counter,
                            int* err, cudaStream_t st) {
  // one kernel for the whole recurrence, CTA = (batch tile, 16 units) (lstm_tiled.cu)
  if (mode == 2) return lstm_forward_tiled(H, T1, B, U, done, z, h0, c0, hs, cs, hp, counter, err, st);
  // the same recurrence with the recurrent products on the tensor cores (lstm_tc.cu)
  if (mode == 3) return lstm_forward_tc(H, T1, B, U, done, z, h0, c0, hs, cs, hp, counter, err, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm mode must be 2 (tiled) or 3 (tc3)");
}

int lstm_recurrence_backward(int mode, int H, int T1, int B, const float* U, const uint8_t* done, const float* gates,
                             const float* cs, const float* c0, const float* dhs, float* dz, unsigned int* counter,
                             int* err, cudaStream_t st) {
  if (mode == 2) return lstm_backward_tiled(H, T1, B, U, done, gates, cs, c0, dhs, dz, counter, err, st);
  if (mode == 3) return lstm_backward_tc(H, T1, B, U, done, gates, cs, c0, dhs, dz, counter, err, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm mode must be 2 (tiled) or 3 (tc3)");
}

// ---- the recurrent core of both nets ---------------------------------------------------------
Core core_create(ParamTable& t, const std::string& dense, int H, int flat, int A, bool clip_reward, bool flat_relu) {
  Core k;
  k.H = H; k.flat = flat; k.A = A; k.core_in = H + 1 + A;
  k.clip_reward = clip_reward; k.flat_relu = flat_relu;
  k.dense_w = t.add(dense + "/kernel", {flat, H});
  k.dense_b = t.add(dense + "/bias", {H});
  k.w = t.add("core/kernel", {k.core_in, 4 * H});
  k.u = t.add("core/recurrent_kernel", {H, 4 * H});
  k.b = t.add("core/bias", {4 * H});
  return k;
}

CorePlan core_plan(const Core& k, Bump& b, int T1, int B) {
  CorePlan p;
  p.T1 = T1; p.B = B; p.N = T1 * B;
  const size_t N = (size_t)p.N, H = (size_t)k.H;
  p.xc = b.take(N * k.core_in * 4);
  p.z = b.take(N * 4 * H * 4);
  p.hp = b.take(N * H * 4);
  p.cs = b.take(N * H * 4);
  p.hs = b.take(N * H * 4);
  p.c0buf = b.take((size_t)B * H * 4);
  p.dhs = b.take(N * H * 4);
  p.dz = b.take(N * 4 * H * 4);
  p.dd = b.take(N * H * 4);
  p.counter = b.take(256);
  return p;
}

// core_in[n] = concat(dense_out[n] (D columns, already written), reward[n] (clipped to [-1, 1] if `clip`),
// one_hot(prev_action[n], A))
__global__ void core_input_tail_kernel(int Nrows, int D, int A, bool clip, const float* __restrict__ reward,
                                       const int64_t* __restrict__ prev_action, float* __restrict__ core_in) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int Wd = 1 + A;
  if (i >= Nrows * Wd) return;
  const int n = i / Wd, j = i - n * Wd;
  float v;
  if (j == 0) v = clip ? fminf(fmaxf(reward[n], -1.f), 1.f) : reward[n];
  else v = prev_action[n] == (int64_t)(j - 1) ? 1.f : 0.f;
  core_in[(size_t)n * (D + Wd) + D + j] = v;
}

int core_forward(const Core& k, const ParamTable& t, const CorePlan& p, const GemmExec& ex, void* ws, const float* prm,
                 const float* flat, const float* reward, const int64_t* prev_actions, const uint8_t* done,
                 const float* h0, const float* c0) {
  cudaStream_t st = ex.st;
  const int N = p.N, H = k.H, CI = k.core_in;
  float* xc = W<float>(ws, p.xc);
  float* z = W<float>(ws, p.z);
  float* c0buf = W<float>(ws, p.c0buf);
  // Dense + ReLU written straight into the first H columns of the core input
  GemmEpi e = epi_none();
  e.bias = prm + t.offset(k.dense_b); e.relu = 1; e.a_relu = k.flat_relu;
  SEEDRL_TRY(ex.gemm(false, false, N, H, k.flat, flat, k.flat, prm + t.offset(k.dense_w), H, xc, CI, e));
  core_input_tail_kernel<<<ceil_div(N * (1 + k.A), 256), 256, 0, st>>>(N, H, k.A, k.clip_reward, reward,
                                                                       prev_actions, xc);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  // input projection for all T at once: z = xc W + b
  e = epi_none();
  e.bias = prm + t.offset(k.b);
  SEEDRL_TRY(ex.gemm(false, false, N, 4 * H, CI, xc, CI, prm + t.offset(k.w), 4 * H, z, 4 * H, e));
  SEEDRL_CUDA(cudaMemcpyAsync(c0buf, c0, (size_t)p.B * H * 4, cudaMemcpyDeviceToDevice, st));
  return lstm_recurrence_forward(k.lstm_mode, H, p.T1, p.B, prm + t.offset(k.u), done, z, h0, c0buf,
                                 W<float>(ws, p.hs), W<float>(ws, p.cs), W<float>(ws, p.hp),
                                 W<unsigned int>(ws, p.counter), ex.err, st);
}

int core_final_state(const Core& k, const CorePlan& p, cudaStream_t st, void* ws, float* h_out, float* c_out) {
  const size_t last = (size_t)(p.T1 - 1) * p.B * k.H, bytes = (size_t)p.B * k.H * 4;
  if (h_out)
    SEEDRL_CUDA(cudaMemcpyAsync(h_out, W<float>(ws, p.hs) + last, bytes, cudaMemcpyDeviceToDevice, st));
  if (c_out)
    SEEDRL_CUDA(cudaMemcpyAsync(c_out, W<float>(ws, p.cs) + last, bytes, cudaMemcpyDeviceToDevice, st));
  return SEEDRL_OK;
}

int core_backward(const Core& k, const ParamTable& t, const CorePlan& p, const GemmExec& ex, void* ws,
                  const float* prm, float* grd, const uint8_t* done, const float* flat, float* dflat,
                  cudaEvent_t head_ready) {
  const int N = p.N, H = k.H, CI = k.core_in;
  const float* xc = W<float>(ws, p.xc);
  float* dz = W<float>(ws, p.dz);
  float* dd = W<float>(ws, p.dd);
  const GemmEpi e = epi_none();
  // BPTT
  SEEDRL_TRY(lstm_recurrence_backward(k.lstm_mode, H, p.T1, p.B, prm + t.offset(k.u), done, W<float>(ws, p.z),
                                      W<float>(ws, p.cs), W<float>(ws, p.c0buf), W<float>(ws, p.dhs), dz,
                                      W<unsigned int>(ws, p.counter), ex.err, ex.st));
  SEEDRL_TRY(ex.gemm(true, false, H, 4 * H, N, W<float>(ws, p.hp), H, dz, 4 * H, grd + t.offset(k.u), 4 * H, e));
  SEEDRL_TRY(ex.gemm(true, false, CI, 4 * H, N, xc, CI, dz, 4 * H, grd + t.offset(k.w), 4 * H, e));
  SEEDRL_TRY(ex.colsum(N, 4 * H, dz, 4 * H, grd + t.offset(k.b)));
  // d dense_out = (dz W[:H,:]^T) * (dense_out > 0)
  GemmEpi em = epi_none();
  em.mask = xc; em.ldm = CI;
  SEEDRL_TRY(ex.gemm(false, true, N, H, 4 * H, dz, 4 * H, prm + t.offset(k.w), 4 * H, dd, H, em));
  // Dense
  GemmEpi ea = epi_none();
  ea.a_relu = k.flat_relu;
  SEEDRL_TRY(ex.gemm(true, false, k.flat, H, N, flat, k.flat, dd, H, grd + t.offset(k.dense_w), H, ea));
  SEEDRL_TRY(ex.colsum(N, H, dd, H, grd + t.offset(k.dense_b)));
  if (head_ready) SEEDRL_CUDA(cudaEventRecord(head_ready, ex.st));
  em.mask = flat; em.ldm = k.flat;
  return ex.gemm(false, true, N, k.flat, H, dd, H, prm + t.offset(k.dense_w), H, dflat, k.flat, em);
}

}  // namespace seedrl

using namespace seedrl;

// The test hook's workspace: the 64 barrier counters.
extern "C" size_t seedrl_debug_lstm_workspace_bytes(int mode, int H, int T1, int B) {
  if (mode < 2 || mode > 3 || H < 1 || T1 < 1 || B < 1) return 0;
  return 256;
}

// A batch a mode cannot take is refused by its launcher, before anything is launched.
static int debug_lstm_check(int mode, int H, int T1, int B, size_t ws_bytes) {
  SEEDRL_CHECK_ARG(mode == 2 || mode == 3, "lstm mode must be 2 (tiled) or 3 (tc3)");
  SEEDRL_CHECK_ARG(H == 256 || H == 512, "lstm: hidden size must be 256 or 512");
  SEEDRL_CHECK_ARG(T1 >= 1 && B >= 1 && (size_t)T1 * B * 4 * H < ((size_t)1 << 31), "bad T1 / B");
  SEEDRL_CHECK_ARG(ws_bytes >= 256, "workspace too small");
  return SEEDRL_OK;
}

extern "C" int seedrl_debug_lstm_forward(int mode, int H, int T1, int B, const float* U, const uint8_t* done, float* z,
                                         const float* h0, const float* c0, float* hs, float* cs, float* hp, void* ws,
                                         size_t ws_bytes, int* error_flag, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(U && done && z && h0 && c0 && hs && cs && hp && ws && error_flag, "null pointer");
  SEEDRL_TRY(debug_lstm_check(mode, H, T1, B, ws_bytes));
  return lstm_recurrence_forward(mode, H, T1, B, U, done, z, h0, c0, hs, cs, hp, (unsigned int*)ws, error_flag,
                                 (cudaStream_t)stream);
}

extern "C" int seedrl_debug_lstm_backward(int mode, int H, int T1, int B, const float* U, const uint8_t* done,
                                          const float* gates, const float* cs, const float* c0, const float* dhs,
                                          float* dz, void* ws, size_t ws_bytes, int* error_flag,
                                          seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(U && done && gates && cs && c0 && dhs && dz && ws && error_flag, "null pointer");
  SEEDRL_TRY(debug_lstm_check(mode, H, T1, B, ws_bytes));
  return lstm_recurrence_backward(mode, H, T1, B, U, done, gates, cs, c0, dhs, dz, (unsigned int*)ws, error_flag,
                                  (cudaStream_t)stream);
}
