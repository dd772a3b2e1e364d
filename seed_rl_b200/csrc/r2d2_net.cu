// (a11) R2D2 agent network: atari/networks.py:221-340 DuelingLSTMDQNNet as a fixed schedule of
// this library's kernels -- forward unroll (_torso folded over T*B by batch_apply; LSTMCell(512)
// over T with done-resets, _unroll_cell :176-218; dueling _head :275-288) and the matching
// backward (what tf.GradientTape computes at agents/r2d2/learner.py:596-609).
//
// The three 'valid' strided convolutions (8x8/4 -> 32, 4x4/2 -> 64, 3x3/1 -> 64) run as
// im2col + tensor-core GEMM (strided_conv.cu; gemm_tc_kernel, bf16x3 = fp32-faithful; fp32 SIMT sgemm
// in mode 0).  The im2col matrices of the training unroll are kept for the backward (HBM is plentiful:
// 4.5 GB at T=101, B=64).  Frames arrive already stacked ([T,B,H,W,C] uint8, C = stack_size; the
// bit-packed frame stacking is r2d2_kernels.cu::stack_frames) and are scaled by 1/255 inside im2col.
//
// Parameters: one flat fp32 arena in tf.Module.trainable_variables order (attribute-name order:
// _advantage, _body, _core, _value), Keras layouts, tensor starts aligned to 64 floats.
#include "schedule.h"

namespace seedrl {

constexpr int kRH = 512;                 // LSTMCell(512), Dense(512) (networks.py:240-252)

}  // namespace seedrl

struct seedrl_r2d2_net {
  int A, H, W, C;
  int mode;                               // 0 = fp32 SIMT GEMMs, 2 = wgmma bf16x3
  seedrl::ParamTable params;
  size_t logical_params;
  seedrl::StridedConv conv[3];
  int conv_w[3], conv_b[3];               // param indices
  seedrl::Core core;                      // Dense(512) + LSTM(512); lstm_mode 2 or 3 (schedule.h)
  int p_ah_w, p_ah_b, p_a_w, p_vh_w, p_vh_b, p_v_w, p_v_b;
};

namespace seedrl {

struct RPlan {
  size_t N;
  size_t col[3], act[3];                  // im2col matrices, post-ReLU conv outputs (NHWC)
  CorePlan core;
  size_t vh, ah, v, adv;
  size_t dv, dadv, dvh, dah, g[3];
  size_t gemm_ws, tcerr;
  size_t total;
};

static RPlan r_plan(const seedrl_r2d2_net* n, int T, int B) {
  RPlan p;
  Bump b;
  const size_t N = (size_t)T * B;
  p.N = N;
  for (int i = 0; i < 3; ++i) {
    const StridedConv& c = n->conv[i];
    p.col[i] = b.take(N * c.hout * c.wout * (size_t)(c.k * c.k * c.cin) * 4);
    p.act[i] = b.take(N * c.hout * c.wout * (size_t)c.cout * 4);
    p.g[i] = b.take(N * c.hout * c.wout * (size_t)c.cout * 4);
  }
  p.core = core_plan(n->core, b, T, B);
  p.vh = b.take(N * kRH * 4);
  p.ah = b.take(N * kRH * 4);
  p.v = b.take(N * 4);
  p.adv = b.take(N * (size_t)n->A * 4);
  p.dv = b.take(N * 4);
  p.dadv = b.take(N * (size_t)n->A * 4);
  p.dvh = b.take(N * kRH * 4);
  p.dah = b.take(N * kRH * 4);
  p.gemm_ws = b.take(gemm_tc_workspace_bytes());
  p.tcerr = b.take(256);
  p.total = b.off;
  return p;
}

static GemmExec r_exec(const seedrl_r2d2_net* n, const RPlan& pl, void* ws, cudaStream_t st) {
  return GemmExec{n->mode, gemm_tc_gather_enabled(), W<float>(ws, pl.gemm_ws), gemm_tc_workspace_bytes(),
                  W<int>(ws, pl.tcerr), st};
}
static inline const float* RP(const seedrl_r2d2_net* n, const float* arena, int idx) {
  return arena + n->params.offset(idx);
}
static inline float* RG(const seedrl_r2d2_net* n, float* arena, int idx) { return arena + n->params.offset(idx); }

// _head (networks.py:275-288): q = value + advantage - mean(advantage); action = argmax_a q (first
// maximum, tf.argmax).  Thread per row.
__global__ void dueling_fwd_kernel(int Nrows, int A, const float* __restrict__ v, const float* __restrict__ adv,
                                   float* __restrict__ q, int32_t* __restrict__ action) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nrows) return;
  const float* a = adv + (size_t)n * A;
  float s = 0.f;
  for (int j = 0; j < A; ++j) s += a[j];
  const float mean = s / (float)A, val = v[n];
  float best = -INFINITY;
  int arg = 0;
  for (int j = 0; j < A; ++j) {
    const float x = val + (a[j] - mean);
    q[(size_t)n * A + j] = x;
    if (x > best) { best = x; arg = j; }
  }
  if (action) action[n] = arg;
}
// dvalue = sum_a dq ; dadvantage = dq - mean_a dq
__global__ void dueling_bwd_kernel(int Nrows, int A, const float* __restrict__ dq, float* __restrict__ dv,
                                   float* __restrict__ dadv) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= Nrows) return;
  const float* d = dq + (size_t)n * A;
  float s = 0.f;
  for (int j = 0; j < A; ++j) s += d[j];
  dv[n] = s;
  const float mean = s / (float)A;
  for (int j = 0; j < A; ++j) dadv[(size_t)n * A + j] = d[j] - mean;
}

}  // namespace seedrl

using namespace seedrl;

extern "C" int seedrl_r2d2_net_create(int num_actions, int obs_h, int obs_w, int channels, seedrl_r2d2_net** out) {
  SEEDRL_CHECK_ARG(out, "null pointer");
  SEEDRL_CHECK_ARG(num_actions >= 1 && channels >= 1, "bad shape");
  SEEDRL_CHECK_ARG(obs_h >= 36 && obs_w >= 36, "frames too small for the 8x8/4, 4x4/2, 3x3/1 body");
  seedrl_r2d2_net* n = new seedrl_r2d2_net();
  n->A = num_actions; n->H = obs_h; n->W = obs_w; n->C = channels;
  n->mode = 2;
  const int spec[3][3] = {{32, 8, 4}, {64, 4, 2}, {64, 3, 1}};     // (filters, kernel, stride) :233-238
  int h = obs_h, w = obs_w, c = channels;
  for (int i = 0; i < 3; ++i) {
    const StridedConv& k = n->conv[i] = StridedConv(spec[i][1], spec[i][2], c, spec[i][0], h, w);
    h = k.hout; w = k.wout; c = k.cout;
  }
  ParamTable& t = n->params;
  // tf.Module attribute order: _advantage, _body, _core, _value
  n->p_ah_w = t.add("advantage/hidden/kernel", {kRH, 512});
  n->p_ah_b = t.add("advantage/hidden/bias", {512});
  n->p_a_w = t.add("advantage/head/kernel", {512, num_actions});
  for (int i = 0; i < 3; ++i) {
    const StridedConv& k = n->conv[i];
    const std::string pre = "body/conv" + std::to_string(i);
    n->conv_w[i] = t.add(pre + "/kernel", {k.k, k.k, k.cin, k.cout});
    n->conv_b[i] = t.add(pre + "/bias", {k.cout});
  }
  // _torso tail (networks.py:262-273): the reward is NOT clipped, unlike ImpalaDeep
  n->core = core_create(t, "body/dense", kRH, h * w * c, num_actions, false, false);
  n->p_vh_w = t.add("value/hidden/kernel", {kRH, 512});
  n->p_vh_b = t.add("value/hidden/bias", {512});
  n->p_v_w = t.add("value/head/kernel", {512, 1});
  n->p_v_b = t.add("value/head/bias", {1});
  n->logical_params = 0;
  for (const ParamInfo& p : t.list) n->logical_params += p.size;
  *out = n;
  return SEEDRL_OK;
}

extern "C" void seedrl_r2d2_net_destroy(seedrl_r2d2_net* net) { delete net; }
extern "C" int seedrl_r2d2_net_num_param_tensors(const seedrl_r2d2_net* net) {
  return net ? (int)net->params.list.size() : 0;
}
extern "C" size_t seedrl_r2d2_net_num_params(const seedrl_r2d2_net* net) { return net ? net->logical_params : 0; }
extern "C" size_t seedrl_r2d2_net_arena_floats(const seedrl_r2d2_net* net) {
  return net ? net->params.arena_floats : 0;
}
extern "C" int seedrl_r2d2_net_set_mode(seedrl_r2d2_net* net, int mode) {
  SEEDRL_CHECK_ARG(net && (mode == 0 || mode == 2), "mode must be 0 (fp32 SIMT) or 2 (wgmma bf16x3)");
  net->mode = mode;
  return SEEDRL_OK;
}
extern "C" int seedrl_r2d2_net_set_lstm_mode(seedrl_r2d2_net* net, int mode) {
  SEEDRL_CHECK_ARG(net && (mode == 2 || mode == 3), "mode must be 2 (tiled) or 3 (tc3: tiled on wgmma bf16x3)");
  net->core.lstm_mode = mode;
  return SEEDRL_OK;
}
extern "C" int seedrl_r2d2_net_param_info(const seedrl_r2d2_net* net, int index, char* name_buf, size_t name_cap,
                                          int64_t* dims4, int* rank, size_t* offset_floats) {
  SEEDRL_CHECK_ARG(net && index >= 0 && index < (int)net->params.list.size(), "bad index");
  const ParamInfo* p = net->params.info(index, name_buf, name_cap, dims4, offset_floats);
  if (rank) *rank = p->rank;
  return SEEDRL_OK;
}
extern "C" size_t seedrl_r2d2_net_workspace_bytes(const seedrl_r2d2_net* net, int T, int B) {
  if (!net || T < 1 || B < 1) return 0;
  return r_plan(net, T, B).total;
}

extern "C" int seedrl_r2d2_net_forward(const seedrl_r2d2_net* n, const float* prm, int T, int B,
                                       const int64_t* prev_actions, const float* reward, const uint8_t* done,
                                       const uint8_t* frames, const float* h0, const float* c0, float* q_values,
                                       int32_t* action, float* h_out, float* c_out, void* ws, size_t ws_bytes,
                                       seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(n && prm && prev_actions && reward && done && frames && h0 && c0 && q_values && ws,
                   "null pointer");
  SEEDRL_CHECK_ARG(T >= 1 && B >= 1, "T, B must be >= 1");
  const RPlan pl = r_plan(n, T, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  SEEDRL_CHECK_ARG(pl.N * (size_t)n->conv[0].hout * n->conv[0].wout < (size_t)8000000,
                   "unroll batch too large (GEMM row count)");
  cudaStream_t st = (cudaStream_t)stream;
  const GemmExec ex = r_exec(n, pl, ws, st);
  const int N = (int)pl.N, A = n->A;
  SEEDRL_CUDA(cudaMemsetAsync(W<int>(ws, pl.tcerr), 0, sizeof(int), st));
  // ---- body: three convolutions as im2col + GEMM (bias + ReLU in the epilogue) ----------------
  const void* x = frames;
  for (int i = 0; i < 3; ++i) {
    const StridedConv& c = n->conv[i];
    float* act = W<float>(ws, pl.act[i]);
    SEEDRL_TRY(c.forward(ex, N, i == 0, x, RP(n, prm, n->conv_w[i]), RP(n, prm, n->conv_b[i]), W<float>(ws, pl.col[i]),
                         act, c.cout));
    x = act;
  }
  // Flatten (NHWC order) + Dense(512) + the LSTM core
  SEEDRL_TRY(core_forward(n->core, n->params, pl.core, ex, ws, prm, W<float>(ws, pl.act[2]), reward, prev_actions, done,
                          h0, c0));
  const float* hs = W<float>(ws, pl.core.hs);
  // dueling heads
  float* vh = W<float>(ws, pl.vh); float* ah = W<float>(ws, pl.ah);
  float* v = W<float>(ws, pl.v); float* adv = W<float>(ws, pl.adv);
  GemmEpi e = epi_none();
  e.bias = RP(n, prm, n->p_vh_b); e.relu = 1;
  SEEDRL_TRY(ex.gemm(false, false, N, 512, kRH, hs, kRH, RP(n, prm, n->p_vh_w), 512, vh, 512, e));
  e.bias = RP(n, prm, n->p_ah_b);
  SEEDRL_TRY(ex.gemm(false, false, N, 512, kRH, hs, kRH, RP(n, prm, n->p_ah_w), 512, ah, 512, e));
  e = epi_none();
  e.bias = RP(n, prm, n->p_v_b);
  SEEDRL_TRY(ex.gemm(false, false, N, 1, 512, vh, 512, RP(n, prm, n->p_v_w), 1, v, 1, e));
  e = epi_none();
  SEEDRL_TRY(ex.gemm(false, false, N, A, 512, ah, 512, RP(n, prm, n->p_a_w), A, adv, A, e));
  dueling_fwd_kernel<<<ceil_div(N, 128), 128, 0, st>>>(N, A, v, adv, q_values, action);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return core_final_state(n->core, pl.core, st, ws, h_out, c_out);
}

// Backward of the unroll whose forward last used `ws` (same T, B, frames).  grads = flat arena (overwritten).
extern "C" int seedrl_r2d2_net_backward(const seedrl_r2d2_net* n, const float* prm, int T, int B,
                                        const uint8_t* frames, const uint8_t* done, const float* dq, float* grd,
                                        void* ws, size_t ws_bytes, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(n && prm && frames && done && dq && grd && ws, "null pointer");
  const RPlan pl = r_plan(n, T, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const GemmExec ex = r_exec(n, pl, ws, st);
  const int N = (int)pl.N, A = n->A;
  const float* hs = W<float>(ws, pl.core.hs);
  float* vh = W<float>(ws, pl.vh); float* ah = W<float>(ws, pl.ah);
  float* dv = W<float>(ws, pl.dv); float* dadv = W<float>(ws, pl.dadv);
  float* dvh = W<float>(ws, pl.dvh); float* dah = W<float>(ws, pl.dah);
  float* dhs = W<float>(ws, pl.core.dhs);
  SEEDRL_CUDA(cudaMemsetAsync(grd, 0, n->params.arena_floats * sizeof(float), st));
  const GemmEpi e0 = epi_none();
  GemmEpi eacc = epi_none();
  eacc.accumulate = 1;
  // dueling combination
  dueling_bwd_kernel<<<ceil_div(N, 128), 128, 0, st>>>(N, A, dq, dv, dadv);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  // advantage stream
  SEEDRL_TRY(ex.gemm(true, false, 512, A, N, ah, 512, dadv, A, RG(n, grd, n->p_a_w), A, e0));
  GemmEpi em = epi_none();
  em.mask = ah; em.ldm = 512;
  SEEDRL_TRY(ex.gemm(false, true, N, 512, A, dadv, A, RP(n, prm, n->p_a_w), A, dah, 512, em));
  SEEDRL_TRY(ex.gemm(true, false, kRH, 512, N, hs, kRH, dah, 512, RG(n, grd, n->p_ah_w), 512, e0));
  SEEDRL_TRY(ex.colsum(N, 512, dah, 512, RG(n, grd, n->p_ah_b)));
  // value stream
  SEEDRL_TRY(ex.gemm(true, false, 512, 1, N, vh, 512, dv, 1, RG(n, grd, n->p_v_w), 1, e0));
  SEEDRL_TRY(ex.colsum(N, 1, dv, 1, RG(n, grd, n->p_v_b)));
  em.mask = vh;
  SEEDRL_TRY(ex.gemm(false, true, N, 512, 1, dv, 1, RP(n, prm, n->p_v_w), 1, dvh, 512, em));
  SEEDRL_TRY(ex.gemm(true, false, kRH, 512, N, hs, kRH, dvh, 512, RG(n, grd, n->p_vh_w), 512, e0));
  SEEDRL_TRY(ex.colsum(N, 512, dvh, 512, RG(n, grd, n->p_vh_b)));
  // d core output
  SEEDRL_TRY(ex.gemm(false, true, N, kRH, 512, dah, 512, RP(n, prm, n->p_ah_w), 512, dhs, kRH, e0));
  SEEDRL_TRY(ex.gemm(false, true, N, kRH, 512, dvh, 512, RP(n, prm, n->p_vh_w), 512, dhs, kRH, eacc));
  // BPTT, the core and Dense(512), down to d flat
  SEEDRL_TRY(core_backward(n->core, n->params, pl.core, ex, ws, prm, grd, done, W<float>(ws, pl.act[2]),
                           W<float>(ws, pl.g[2]), nullptr));
  // convolutions, last to first; the weight gradient reads the layer's input (gathered) or the im2col
  // matrix the forward kept
  for (int i = 2; i >= 0; --i) {
    const StridedConv& c = n->conv[i];
    float* col = W<float>(ws, pl.col[i]);
    const float* g = W<float>(ws, pl.g[i]);
    const void* xin = i == 0 ? (const void*)frames : (const void*)W<float>(ws, pl.act[i - 1]);
    SEEDRL_TRY(c.wgrad(ex, N, i == 0, xin, col, g, RG(n, grd, n->conv_w[i]), c.cout, RG(n, grd, n->conv_b[i])));
    if (i > 0)
      SEEDRL_TRY(c.dgrad(ex, N, g, RP(n, prm, n->conv_w[i]), col, W<float>(ws, pl.act[i - 1]),
                         W<float>(ws, pl.g[i - 1])));
  }
  return SEEDRL_OK;
}

extern "C" int seedrl_r2d2_net_check_error(const seedrl_r2d2_net* n, int T, int B, void* ws, size_t ws_bytes,
                                           seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(n && ws && T >= 1 && B >= 1, "bad arguments");
  const RPlan pl = r_plan(n, T, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  return read_error_flag(W<int>(ws, pl.tcerr), (cudaStream_t)stream, "unroll");
}

// Where the post-ReLU activations of the last forward sit in a (T, B) workspace (host arithmetic only).
extern "C" int seedrl_debug_r2d2_net_views(const seedrl_r2d2_net* n, int T, int B, int index, size_t* offset,
                                           size_t* bytes) {
  SEEDRL_CHECK_ARG(n && offset && bytes && T >= 1 && B >= 1, "bad arguments");
  SEEDRL_CHECK_ARG(index >= 0 && index <= 5, "index must be 0..5");
  const RPlan pl = r_plan(n, T, B);
  if (index <= 2) {
    const StridedConv& c = n->conv[index];
    *offset = pl.act[index];
    *bytes = pl.N * c.hout * c.wout * (size_t)c.cout * 4;
  } else if (index == 3) {
    *offset = pl.core.xc;
    *bytes = pl.N * (size_t)n->core.core_in * 4;
  } else {
    *offset = index == 4 ? pl.vh : pl.ah;
    *bytes = pl.N * kRH * 4;
  }
  return SEEDRL_OK;
}
