// (a5) Policy network graph: dmlab/networks.py:63-171 ImpalaDeep (and the IMPALA-paper
// shallow net) as a fixed schedule of this library's kernels -- forward unroll
// (_torso folded over T*B by batch_apply, utils.py:714-732; LSTM over T with
// done-resets; heads) and the matching backward (what tf.GradientTape computes at
// agents/vtrace/learner.py:261-264).
//
// Parameters: one flat fp32 arena, tensors in tf.Module.trainable_variables order
// (_baseline, _conv_to_linear, _core, _policy_logits, _stacks...), Keras layouts,
// every tensor start aligned to 64 floats (256 B), then the scalar entropy_cost_param
// (learner.py:225-234).
#include "schedule.h"

namespace seedrl {

constexpr int kHidden = 256;   // LSTMCell(256), Dense(256)

struct ConvLayer {
  int cin, cout;
  int w, b;        // param indices
};
struct Stack {
  int hin, win, cin, c, hout, wout;
  ConvLayer conv, r00, r01, r10, r11;
};

}  // namespace seedrl

struct seedrl_net {
  seedrl_net_config cfg;
  seedrl::ParamTable params;               // network tensors, then entropy_cost_param
  size_t logical_params;
  int p_base_w, p_base_b, p_pol_w, p_pol_b;
  seedrl::Core core;                       // Dense(256) + LSTM(256); lstm_mode 2 or 3 (schedule.h)
  std::vector<seedrl::Stack> stacks;       // deep
  seedrl::StridedConv sh[2];               // shallow: conv 8x8/4 -> 16, conv 4x4/2 -> 32
  int sh_w[2], sh_b[2];                    // their param indices
  int conv_mode = 0;                       // 0 = fp32 SIMT, 1 = wgmma bf16, 2 = wgmma bf16x3 (fp32-faithful)
};

namespace seedrl {

static ConvLayer add_conv(seedrl_net* n, const std::string& prefix, int k, int cin, int cout) {
  ConvLayer l;
  l.cin = cin; l.cout = cout;
  l.w = n->params.add(prefix + "/kernel", {k, k, cin, cout});
  l.b = n->params.add(prefix + "/bias", {cout});
  return l;
}

// ---- workspace plan -----------------------------------------------------------
// Where an activation x of the deep torso sits: its raw value (a conv input or residual operand) and relu(x)
// (a conv input, and in the backward the ReLU mask x > 0).  fp32 NHWC (conv modes 0-2): one buffer, raw == relu,
// and a conv that reads relu(x) applies the ReLU as it loads it (IN_RELU).  Plane tensors (conv mode 3,
// conv_planes.cu): relu(x) is a plane tensor of its own, and a copy that nothing reads is not kept (kNone).
// Gradients use the same description with their one buffer in `raw`.
constexpr size_t kNone = ~(size_t)0;
struct Act {
  size_t raw, relu;
  bool planes;
};
static Act f32_act(size_t off) { return Act{off, off, false}; }

struct StackBufs {
  Act a0;                  // the stack's first conv before the max-pool: fp32 NHWC, full resolution
  size_t idx;              // max-pool taps
  Act p, c0, o0, c1, o1;   // pooled resolution; the last stack's o1 is fp32 NHWC for the Dense layer
};

// packed-weight slot: (hi + lo) x 9 x 32 x 32 bf16; deferred weight-gradient partials of all
// 15 convs: at most one CTA per SM x 97 680 floats (51.6 MB on 132 SMs) rounded up
constexpr size_t kPackSlotBytes = 2 * 9 * 32 * 32 * 2;
constexpr size_t kPartialAllBytes = (size_t)64 << 20;

struct Plan {
  int N;                       // T1 * B frames
  std::vector<StackBufs> st;
  size_t sh_a1, sh_a2;         // shallow conv outputs (post-relu)
  size_t sh_col0, sh_col1;     // shallow net, tensor-core modes: im2col matrices (kept for the backward)
  CorePlan core;
  // backward scratch.  gA: d loss / d (torso output) from Dense, fp32; g: the deep torso's pooled-resolution
  // gradients (fp32: g[0] is gA); gPool: the gradient of the max-pool input of stacks 1 and 2; gFull: fp32 at
  // full resolution (the max-pool backward of the first layer's unfused paths)
  size_t gA, gFull, wt, partial, wq, tcerr, gemm_ws, wq_all, partial_all;
  Act g[3], gPool;
  size_t obs4, w0pad, dw0pad;  // 3-channel frames: zero-padded frames / first-conv weights / their gradient
  size_t total;
};

// Carves one activation: an fp32 NHWC buffer, or a plane tensor for each copy that is read.
static Act take_act(Bump& b, bool planes, size_t f32_bytes, size_t planes_bytes, bool raw, bool relu) {
  if (!planes) return f32_act(b.take(f32_bytes));
  Act a{kNone, kNone, true};
  if (raw) a.raw = b.take(planes_bytes);
  if (relu) a.relu = b.take(planes_bytes);
  return a;
}

static Plan make_plan(const seedrl_net* n, int T1, int B) {
  Plan p;
  Bump b;
  const size_t N = (size_t)T1 * B;
  p.N = (int)N;
  size_t pooled_max = 0, full_max = 0, pooled_planes_max = 0, full_planes_max = 0;
  const bool planes = n->conv_mode == 3 && n->cfg.net == SEEDRL_NET_DEEP;
  if (n->cfg.net == SEEDRL_NET_DEEP) {
    for (size_t si = 0; si < n->stacks.size(); ++si) {
      const Stack& s = n->stacks[si];
      StackBufs sb;
      const size_t full = N * s.hin * s.win * s.c, pooled = N * s.hout * s.wout * s.c;
      const size_t pb = planes_bytes((int)N, s.hout, s.wout, s.c);
      sb.a0 = f32_act(b.take(full * 4));
      sb.idx = b.take(pooled);
      // p and o0 are ReLU'd conv inputs and residuals, c0 and c1 only ReLU'd conv inputs, o1 the next stack's input
      sb.p = take_act(b, planes, pooled * 4, pb, true, true);
      sb.c0 = take_act(b, planes, pooled * 4, pb, false, true);
      sb.o0 = take_act(b, planes, pooled * 4, pb, true, true);
      sb.c1 = take_act(b, planes, pooled * 4, pb, false, true);
      sb.o1 = take_act(b, planes && si + 1 < n->stacks.size(), pooled * 4, pb, true, false);
      if (pb > pooled_planes_max) pooled_planes_max = pb;
      if (si > 0) {
        const size_t fb = planes_bytes((int)N, s.hin, s.win, s.c);
        if (fb > full_planes_max) full_planes_max = fb;
      }
      p.st.push_back(sb);
      if (pooled > pooled_max) pooled_max = pooled;
      if (full > full_max) full_max = full;
    }
    p.sh_a1 = p.sh_a2 = 0;
  } else {
    const StridedConv &l0 = n->sh[0], &l1 = n->sh[1];
    const size_t a1 = N * l0.hout * l0.wout * l0.cout, a2 = N * l1.hout * l1.wout * l1.cout;
    p.sh_a1 = b.take(a1 * 4);
    p.sh_a2 = b.take(a2 * 4);
    p.sh_col0 = p.sh_col1 = 0;
    if (n->conv_mode >= 1) {
      p.sh_col0 = b.take(N * l0.hout * l0.wout * (size_t)(l0.k * l0.k * l0.cin) * 4);
      p.sh_col1 = b.take(N * l1.hout * l1.wout * (size_t)(l1.k * l1.k * l1.cin) * 4);
    }
    pooled_max = a1 > a2 ? a1 : a2;
    full_max = 0;
  }
  p.core = core_plan(n->core, b, T1, B);
  p.obs4 = p.w0pad = p.dw0pad = 0;
  if (n->cfg.net == SEEDRL_NET_DEEP && n->cfg.obs_c == 3) {
    p.obs4 = b.take(N * n->cfg.obs_h * n->cfg.obs_w * 4);
    p.w0pad = b.take(9 * 4 * 16 * 4);
    p.dw0pad = b.take(9 * 4 * 16 * 4);
  }
  p.gA = b.take(pooled_max * 4);
  p.g[0] = planes ? take_act(b, true, 0, pooled_planes_max, true, false) : f32_act(p.gA);
  p.g[1] = take_act(b, planes, pooled_max * 4, pooled_planes_max, true, false);
  p.g[2] = take_act(b, planes, pooled_max * 4, pooled_planes_max, true, false);
  if (planes) p.gPool = take_act(b, true, 0, full_planes_max, true, false);
  p.gFull = b.take(full_max * 4);
  if (!planes) p.gPool = f32_act(p.gFull);
  p.wt = b.take(64 * 1024 * 4);
  p.wq = b.take(2 * 64 * 1024 * 2);
  p.gemm_ws = b.take(gemm_tc_workspace_bytes());
  p.wq_all = b.take((size_t)kMaxPackJobs * kPackSlotBytes);
  p.partial_all = b.take(kPartialAllBytes);
  p.tcerr = b.take(256);
  p.partial = b.take(conv3x3_wgrad_partial_bytes());
  p.total = b.off;
  return p;
}

// The torso's output, the flat features Dense(256) reads (the deep net's is ReLU'd as it is read).
static const float* flat_features(const seedrl_net* n, const Plan& pl, void* ws) {
  return W<float>(ws, n->cfg.net == SEEDRL_NET_DEEP ? pl.st.back().o1.raw : pl.sh_a2);
}

// The deep net's first layer (stack 0's conv + max-pool on the uint8 frames) runs one of three kernel paths.
// The forward and the backward pick theirs independently: the fused kernels' limits differ (conv_first.cu).
enum FirstPath {
  kFirstFused,     // conv0pool_forward / first_wgrad_pooled (plane tensors): no full-resolution tensor
  kFirstStaged,    // 4-channel frames: wgmma conv on staged uint8 tiles + max-pool, wgmma weight gradient
  kFirstGeneric,   // SIMT channel-generic conv3x3_u8_* (1 to 16 channels) + max-pool
};

// test hook: 1 = conv mode 3 keeps the dense (full-resolution) first-layer paths
static int g_first_dense = 0;

// Channels of the frames the deep net's first layer reads: 3-channel frames run on their zero-padded
// 4-channel copy (pad_first_layer); every other count (1..16) is read as it is, zero-filled in shared memory.
static inline int first_c(const seedrl_net* n) { return n->cfg.obs_c == 3 ? 4 : n->cfg.obs_c; }
// frames that only the channel-generic first-layer kernels take (conv modes 0 and 3)
static inline bool generic_first(const seedrl_net* n) {
  return n->cfg.net == SEEDRL_NET_DEEP && first_c(n) != 4;
}

// The first layer's path for a forward or a backward call of the deep net, or the refusal of frames that no
// path of this conv mode takes.
static int first_layer(const seedrl_net* n, bool backward, FirstPath* path) {
  const Stack& k = n->stacks[0];
  const bool fused = n->conv_mode == 3 && !g_first_dense &&
                     (backward ? first_wgrad_pooled_supported(first_c(n), k.c, k.hin, k.win)
                               : conv0pool_supported(first_c(n), k.c, k.hin, k.win));
  if (n->conv_mode == 3 && !fused && generic_first(n))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT,
                     g_first_dense || backward
                         ? "the dense first-layer path takes 3- or 4-channel frames; switch it off for these frames"
                         : "conv mode 3: the fused first layer takes frames up to 107 pixels wide");
  *path = fused ? kFirstFused : n->conv_mode >= 1 && !generic_first(n) ? kFirstStaged : kFirstGeneric;
  return SEEDRL_OK;
}

// State of one forward or backward call, passed down the schedule: the GEMM execution, the weights
// pre-packed for this call, the deferred weight-gradient reductions, the first layer's path, and for
// 3-channel frames the zero-padded first-conv weights and their gradient (pad_first_layer), which stand
// in for that one parameter in P() / G().
struct Call {
  const seedrl_net* n;
  const Plan& pl;
  const float* prm;
  float* grd;                        // backward only
  void* ws;
  GemmExec ex;
  PackTable packed;
  WgradBatch wb;
  FirstPath first = kFirstGeneric;   // deep net: first_layer() of this call's direction
  int w0_index = -1;
  const float* w0_pad = nullptr;
  float* dw0_pad = nullptr;

  Call(const seedrl_net* n_, const Plan& pl_, const float* prm_, float* grd_, void* ws_, cudaStream_t st)
      : n(n_), pl(pl_), prm(prm_), grd(grd_), ws(ws_),
        ex{n_->conv_mode >= 2 ? 2 : n_->conv_mode, gemm_tc_gather_enabled(), W<float>(ws_, pl_.gemm_ws),
           gemm_tc_workspace_bytes(), W<int>(ws_, pl_.tcerr), st},
        wb{nullptr, 0, 0, 0, {}} {
    packed.n = 0;
  }
  const float* P(int idx) const { return idx == w0_index && w0_pad ? w0_pad : prm + n->params.offset(idx); }
  float* G(int idx) const { return idx == w0_index && dw0_pad ? dw0_pad : grd + n->params.offset(idx); }
  template <typename T = void>
  T* at(size_t off) const { return off == kNone ? nullptr : W<T>(ws, off); }   // a workspace buffer, or null
};

__global__ void pad_frames3_kernel(size_t npix, const uint8_t* __restrict__ src, uchar4* __restrict__ dst) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix) return;
  dst[i] = make_uchar4(src[3 * i], src[3 * i + 1], src[3 * i + 2], 0);
}
// w[tap][3][co] <-> wp[tap][4][co]
__global__ void pad_w0_kernel(int cout, const float* __restrict__ w, float* __restrict__ wp) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * 4 * cout) return;
  const int co = i % cout, ci = (i / cout) % 4, tap = i / (4 * cout);
  wp[i] = ci < 3 ? w[(tap * 3 + ci) * cout + co] : 0.f;
}
__global__ void unpad_dw0_kernel(int cout, const float* __restrict__ dwp, float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * 3 * cout) return;
  const int co = i % cout, ci = (i / cout) % 3, tap = i / (3 * cout);
  dw[i] = dwp[(tap * 4 + ci) * cout + co];
}

// Packs the weights of every conv of the deep torso with one launch: forward forms, or the
// flipped/transposed forms of the data-gradient convolutions (all but the first layer).  The first
// conv is packed only for the staged kernel, in that kernel's layout.
static int pack_all_weights(Call& c, int flip) {
  const seedrl_net* n = c.n;
  c.packed.n = 0;
  if (n->conv_mode < 1 || n->cfg.net != SEEDRL_NET_DEEP) return SEEDRL_OK;
  char* base = W<char>(c.ws, c.pl.wq_all);
  for (size_t s = 0; s < n->stacks.size(); ++s) {
    const Stack& k = n->stacks[s];
    const ConvLayer* ls[5] = {&k.conv, &k.r00, &k.r01, &k.r10, &k.r11};
    for (int i = 0; i < 5; ++i) {
      const ConvLayer& l = *ls[i];
      const bool first = s == 0 && i == 0;
      if (first && (flip || c.first != kFirstStaged)) continue;   // no data gradient into the frames
      const int cin = flip ? l.cout : l.cin, cout = flip ? l.cin : l.cout;
      if (c.packed.n >= kMaxPackJobs) return SEEDRL_OK;
      PackJob j;
      j.w = c.P(l.w);
      j.wq = base + (size_t)c.packed.n * kPackSlotBytes;
      j.ck = cin < 16 ? 16 : cin; j.cout = cout; j.cin_src = cin; j.flip = flip;
      j.legacy = first;
      c.packed.jobs[c.packed.n++] = j;
    }
  }
  return conv3x3_tc_pack_weights_batch(c.packed, n->conv_mode == 3 ? 2 : (n->conv_mode >= 2 ? 1 : 0), c.ex.st);
}
// The packed form of `w` from this call's table, or packed into the single-layer scratch slot.
static int packed_weights(const Call& c, int cin, int cout, const float* w, int flip, int split, const void** wq) {
  for (int i = 0; i < c.packed.n; ++i)
    if (c.packed.jobs[i].w == w && c.packed.jobs[i].flip == flip) {
      *wq = c.packed.jobs[i].wq;
      return SEEDRL_OK;
    }
  void* scratch = W<void>(c.ws, c.pl.wq);
  SEEDRL_TRY(conv3x3_tc_pack_weights(cin, cout, flip, split, w, scratch, c.ex.st));
  *wq = scratch;
  return SEEDRL_OK;
}

// ---- the operations of the stack schedule, on either storage format ----------------------------
// One 3x3 'same' convolution of layer l: out = conv(x) + bias + res, x = relu(in) (in_mode IN_RELU) or in
// (IN_F32), res the raw value of `res`.  flip != 0: the data gradient (weights flipped and transposed, no
// bias), out = 0 where `mask` <= 0 (the ReLU'd copy of the forward input).  Plane tensors run convp; fp32
// NHWC runs the wgmma kernel when the net runs in tensor-core mode and the shape is supported, else fp32
// SIMT.  out may be fp32 NHWC in either format.
static int run_conv(const Call& c, const ConvLayer& l, int H, int Wd, int in_mode, const Act& in, const Act* res,
                    const Act& out, int flip = 0, const Act* mask = nullptr) {
  cudaStream_t st = c.ex.st;
  const int N = c.pl.N, cin = flip ? l.cout : l.cin, cout = flip ? l.cin : l.cout;
  const float* w = c.P(l.w);
  const float* bias = flip ? nullptr : c.P(l.b);
  const void* x = c.at(in_mode == IN_RELU ? in.relu : in.raw);
  const float* m = mask ? c.at<float>(mask->relu) : nullptr;
  const float* r = res ? c.at<float>(res->raw) : nullptr;
  const void* wq;
  if (in.planes) {
    SEEDRL_TRY(packed_weights(c, cin, cout, w, flip, 2, &wq));
    PlaneConv pc;
    pc.N = N; pc.H = H; pc.W = Wd; pc.in = x; pc.wq = wq; pc.bias = bias; pc.mask = m; pc.res = r;
    pc.out_raw = out.planes ? c.at(out.raw) : nullptr; pc.out_relu = out.planes ? c.at(out.relu) : nullptr;
    pc.out_nhwc = out.planes ? nullptr : c.at<float>(out.raw); pc.err = c.ex.err;
    return convp_forward(cin, cout, pc, st);
  }
  if (c.n->conv_mode >= 1 && conv3x3_tc_supported(cin, cout, in_mode)) {
    const int split = c.n->conv_mode >= 2;
    SEEDRL_TRY(packed_weights(c, cin, cout, w, flip, split, &wq));
    return conv3x3_tc_forward(cin, cout, in_mode, split, N, H, Wd, x, wq, bias, m, r, c.at<float>(out.raw),
                              c.ex.err, st);
  }
  if (flip) {
    float* wt = W<float>(c.ws, c.pl.wt);
    SEEDRL_TRY(conv3x3_flip_weights(cout, cin, w, wt, st));   // source layout is [tap][cout][cin]
    w = wt;
  }
  return conv3x3_forward(cin, cout, in_mode, N, H, Wd, x, w, bias, m, r, c.at<float>(out.raw), st);
}

// Backward of run_conv(l, in_mode, x) -> dy: the weight and bias gradient, then the data gradient
// dx = flipped conv of dy, masked by x > 0 where the forward read relu(x), plus dres.
static int conv_bwd(Call& c, const ConvLayer& l, int H, int Wd, int x_mode, const Act& x, const Act& dy,
                    const Act* dres, const Act& dx) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl; cudaStream_t st = c.ex.st;
  const void* xin = c.at(x_mode == IN_RELU ? x.relu : x.raw);
  if (x.planes) {
    SEEDRL_TRY(wgradp(l.cin, l.cout, pl.N, H, Wd, xin, c.at(dy.raw), c.G(l.w), c.G(l.b), c.ex.err, &c.wb, st));
  } else if (n->conv_mode >= 1 && conv3x3_wgrad_tc_supported(l.cin, l.cout, x_mode)) {
    SEEDRL_TRY(conv3x3_wgrad_tc(l.cin, l.cout, x_mode, n->conv_mode >= 2, pl.N, H, Wd, xin, c.at<float>(dy.raw),
                                c.G(l.w), c.G(l.b), W<float>(c.ws, pl.partial), conv3x3_wgrad_partial_bytes(),
                                c.ex.err, &c.wb, st));
  } else {
    SEEDRL_TRY(conv3x3_wgrad(l.cin, l.cout, x_mode, pl.N, H, Wd, xin, c.at<float>(dy.raw), c.G(l.w), c.G(l.b),
                             W<float>(c.ws, pl.partial), conv3x3_wgrad_partial_bytes(), st));
  }
  g_conv_cat = PC_CONV_DGRAD;
  const int rc = run_conv(c, l, H, Wd, IN_F32, dy, dres, dx, 1, x_mode == IN_RELU ? &x : nullptr);
  g_conv_cat = PC_CONV_FWD;
  return rc;
}

// max-pool 3x3/2 'SAME' of the stack's first conv output a0 into p, recording the taps
static int pool_forward(const Call& c, const Stack& k, const StackBufs& b) {
  const float* a0 = c.at<float>(b.a0.raw);
  uint8_t* idx = c.at<uint8_t>(b.idx);
  if (b.p.planes) return poolp_forward(c.pl.N, k.hin, k.win, k.c, a0, c.at(b.p.raw), c.at(b.p.relu), idx, c.ex.st);
  return maxpool3s2_forward(c.pl.N, k.hin, k.win, k.c, a0, c.at<float>(b.p.raw), idx, c.ex.st);
}
// its backward: the pooled gradient dy -> dx at full resolution
static int pool_backward(const Call& c, const Stack& k, size_t idx, const Act& dy, const Act& dx) {
  const uint8_t* taps = c.at<uint8_t>(idx);
  if (dy.planes)
    return poolp_backward(c.pl.N, k.hin, k.win, k.c, c.at(dy.raw), taps, dx.planes ? c.at(dx.raw) : nullptr,
                          dx.planes ? nullptr : c.at<float>(dx.raw), c.ex.st);
  return maxpool3s2_backward(c.pl.N, k.hin, k.win, k.c, c.at<float>(dy.raw), taps, c.at<float>(dx.raw), c.ex.st);
}

// d loss / d o1 of the last stack, which Dense's backward leaves in gA (fp32 NHWC), into g[0]
static int gradient_from_dense(const Call& c) {
  const Act& g = c.pl.g[0];
  if (!g.planes) return SEEDRL_OK;   // g[0] is gA
  const Stack& k = c.n->stacks.back();
  return to_planes(c.pl.N, k.hout, k.wout, k.c, 0, W<float>(c.ws, c.pl.gA), c.at(g.raw), c.ex.st);
}

// 3-channel frames (DMLab's 72x96x3, dmlab/env.py:44-54): the first convolution's kernels are built
// for 4 input channels, so a forward/backward call works on a zero-padded copy of the frames and of
// the first conv's weights ([3,3,3,16] -> [3,3,4,16]); its weight gradient is computed in the padded
// shape and copied back without the 4th channel.  Builds both copies in the workspace, points *obs at
// the padded frames and redirects the first conv's parameter of this call; no-op for other frames.
static int pad_first_layer(Call& c, const uint8_t** obs) {
  const seedrl_net* n = c.n;
  if (n->cfg.net != SEEDRL_NET_DEEP || n->cfg.obs_c != 3) return SEEDRL_OK;
  const Plan& pl = c.pl;
  cudaStream_t st = c.ex.st;
  const size_t npix = (size_t)pl.N * n->cfg.obs_h * n->cfg.obs_w;
  pad_frames3_kernel<<<(unsigned)((npix + 255) / 256), 256, 0, st>>>(npix, *obs, W<uchar4>(c.ws, pl.obs4));
  count_launch(PC_MISC, st);
  const int wi = n->stacks[0].conv.w;
  pad_w0_kernel<<<ceil_div(9 * 4 * 16, 128), 128, 0, st>>>(16, c.prm + n->params.offset(wi), W<float>(c.ws, pl.w0pad));
  count_launch(PC_MISC, st);
  if (cudaGetLastError() != cudaSuccess) return set_error(SEEDRL_ERR_INTERNAL, "3-channel padding launch failed");
  *obs = W<uint8_t>(c.ws, pl.obs4);
  c.w0_index = wi; c.w0_pad = W<float>(c.ws, pl.w0pad); c.dw0_pad = W<float>(c.ws, pl.dw0pad);
  return SEEDRL_OK;
}

// The first layer forward: frames -> stack 0's pooled activation p and the max-pool taps.
static int first_forward(const Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; cudaStream_t st = c.ex.st;
  const Stack& k = n->stacks[0];
  const StackBufs& b = c.pl.st[0];
  const int N = c.pl.N, split = n->conv_mode >= 2;
  const float *w = c.P(k.conv.w), *bias = c.P(k.conv.b);
  float* a0 = c.at<float>(b.a0.raw);
  const void* wq;
  if (c.first == kFirstFused)   // conv + bias + max-pool in one kernel
    return conv0pool_forward(N, k.hin, k.win, first_c(n), obs, w, bias, c.at(b.p.raw), c.at(b.p.relu),
                             c.at<uint8_t>(b.idx), c.ex.err, st);
  if (c.first == kFirstStaged) {
    SEEDRL_TRY(packed_weights(c, k.cin, k.c, w, 0, split, &wq));
    SEEDRL_TRY(conv3x3_tc_forward(k.cin, k.c, IN_U8, split, N, k.hin, k.win, obs, wq, bias, nullptr, nullptr, a0,
                                  c.ex.err, st));
  } else {
    SEEDRL_TRY(conv3x3_u8_forward(first_c(n), N, k.hin, k.win, obs, w, bias, a0, st));
  }
  return pool_forward(c, k, b);
}

// The first layer backward: stack 0's pooled gradient g[0] -> the first conv's weight and bias gradient (no
// gradient flows into the frames).
static int first_backward(Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl; cudaStream_t st = c.ex.st;
  const Stack& k = n->stacks[0];
  const int N = pl.N;
  float *dw = c.G(k.conv.w), *db = c.G(k.conv.b);
  if (c.first == kFirstFused)   // straight from the pooled gradient and the pool's taps
    return first_wgrad_pooled(N, k.hin, k.win, first_c(n), obs, c.at(pl.g[0].raw), c.at<uint8_t>(pl.st[0].idx), dw,
                              db, &c.wb, st);
  SEEDRL_TRY(pool_backward(c, k, pl.st[0].idx, pl.g[0], f32_act(pl.gFull)));
  const float* gF = W<float>(c.ws, pl.gFull);
  float* partial = W<float>(c.ws, pl.partial);
  const size_t pbytes = conv3x3_wgrad_partial_bytes();
  if (c.first == kFirstStaged)
    return conv3x3_wgrad_tc(k.cin, k.c, IN_U8, n->conv_mode >= 2, N, k.hin, k.win, obs, gF, dw, db, partial, pbytes,
                            c.ex.err, &c.wb, st);
  return conv3x3_u8_wgrad(first_c(n), N, k.hin, k.win, obs, gF, dw, db, partial, pbytes, st);
}

}  // namespace seedrl

using namespace seedrl;

extern "C" int seedrl_net_create(const seedrl_net_config* cfg, seedrl_net** out) {
  SEEDRL_CHECK_ARG(cfg && out, "null pointer");
  SEEDRL_CHECK_ARG(cfg->net == SEEDRL_NET_DEEP || cfg->net == SEEDRL_NET_SHALLOW, "unknown net");
  SEEDRL_CHECK_ARG(cfg->num_actions >= 1 && cfg->obs_h > 0 && cfg->obs_w > 0, "bad shape");
  seedrl_net* n = new seedrl_net();
  n->cfg = *cfg;
  const int A = cfg->num_actions;
  // tf.Module order: _baseline, _conv_to_linear, _core, _policy_logits, _stacks
  n->p_base_w = n->params.add("baseline/kernel", {kHidden, 1});
  n->p_base_b = n->params.add("baseline/bias", {1});
  int flat = 0;
  if (cfg->net == SEEDRL_NET_DEEP) {
    if (cfg->obs_c < 1 || cfg->obs_c > 16) {
      delete n;
      return set_error(SEEDRL_ERR_INVALID_ARGUMENT,
                       "seedrl_net_create: the deep net takes uint8 frames with 1 to 16 channels");
    }
    int h = cfg->obs_h, w = cfg->obs_w;
    const int chans[3] = {16, 32, 32};
    for (int s = 0; s < 3; ++s) { h = (h + 1) / 2; w = (w + 1) / 2; }
    flat = h * w * chans[2];
  } else {
    n->sh[0] = StridedConv(8, 4, cfg->obs_c, 16, cfg->obs_h, cfg->obs_w);
    n->sh[1] = StridedConv(4, 2, 16, 32, n->sh[0].hout, n->sh[0].wout);
    flat = n->sh[1].hout * n->sh[1].wout * 32;
  }
  // the reward is clipped (networks.py:111); the deep torso's output is ReLU'd as Dense reads it (:105), the
  // shallow one's already is
  n->core = core_create(n->params, "conv_to_linear", kHidden, flat, A, true, cfg->net == SEEDRL_NET_DEEP);
  n->p_pol_w = n->params.add("policy_logits/kernel", {kHidden, A});
  n->p_pol_b = n->params.add("policy_logits/bias", {A});
  if (cfg->net == SEEDRL_NET_DEEP) {
    int h = cfg->obs_h, w = cfg->obs_w, c = cfg->obs_c;
    const int chans[3] = {16, 32, 32};
    for (int s = 0; s < 3; ++s) {
      Stack st;
      const std::string pre = "stack" + std::to_string(s);
      // stack 0: the kernels see the frame's channels zero-padded to 4, 8 or 16
      st.hin = h; st.win = w; st.cin = s == 0 ? (c <= 4 ? 4 : (c <= 8 ? 8 : 16)) : c; st.c = chans[s];
      st.hout = (h + 1) / 2; st.wout = (w + 1) / 2;
      st.conv = add_conv(n, pre + "/conv", 3, c, st.c);      // the parameter keeps the frame's channel count
      st.conv.cin = st.cin;                                  // ... the kernels see the padded one
      // tf.Module order inside _Stack: _conv, _res_convs0[0..1], _res_convs1[0..1]
      st.r00 = add_conv(n, pre + "/res_0/conv2d_0", 3, st.c, st.c);
      st.r10 = add_conv(n, pre + "/res_1/conv2d_0", 3, st.c, st.c);
      st.r01 = add_conv(n, pre + "/res_0/conv2d_1", 3, st.c, st.c);
      st.r11 = add_conv(n, pre + "/res_1/conv2d_1", 3, st.c, st.c);
      n->stacks.push_back(st);
      h = st.hout; w = st.wout; c = st.c;
    }
  } else {
    for (int i = 0; i < 2; ++i) {
      const StridedConv& l = n->sh[i];
      const ConvLayer cl = add_conv(n, "conv" + std::to_string(i), l.k, l.cin, l.cout);
      n->sh_w[i] = cl.w; n->sh_b[i] = cl.b;
    }
  }
  n->logical_params = 0;
  for (const ParamInfo& p : n->params.list) n->logical_params += p.size;
  n->params.add("entropy_cost_param", {});
  *out = n;
  return SEEDRL_OK;
}

extern "C" void seedrl_net_destroy(seedrl_net* net) { delete net; }
extern "C" int seedrl_net_num_param_tensors(const seedrl_net* net) {
  return net ? (int)net->params.list.size() - 1 : 0;
}
extern "C" size_t seedrl_net_num_params(const seedrl_net* net) { return net ? net->logical_params : 0; }
extern "C" size_t seedrl_net_arena_floats(const seedrl_net* net) { return net ? net->params.arena_floats : 0; }
extern "C" int seedrl_net_set_lstm_mode(seedrl_net* net, int mode) {
  SEEDRL_CHECK_ARG(net && (mode == 2 || mode == 3), "mode must be 2 (tiled) or 3 (tc3: tiled on wgmma bf16x3)");
  net->core.lstm_mode = mode;
  return SEEDRL_OK;
}
extern "C" int seedrl_net_set_conv_mode(seedrl_net* net, int mode) {
  SEEDRL_CHECK_ARG(net && mode >= 0 && mode <= 3,
                   "mode must be 0 (fp32 SIMT), 1 (wgmma bf16), 2 (wgmma bf16x3) or 3 (bf16x3 plane tensors)");
  SEEDRL_CHECK_ARG(mode != 3 || net->cfg.net == SEEDRL_NET_DEEP, "mode 3 is built for the deep net");
  SEEDRL_CHECK_ARG(!generic_first(net) || (mode != 1 && mode != 2),
                   "conv modes 1 (tc) and 2 (tc3) take 3- or 4-channel frames in the deep net; use 0 (simt) or 3 (tc3p)");
  SEEDRL_CHECK_ARG(!generic_first(net) || mode != 3 ||
                       conv0pool_supported(first_c(net), 16, net->cfg.obs_h, net->cfg.obs_w),
                   "conv mode 3 (tc3p) takes frames of 3 to 107 pixels per side for this channel count; use 0 (simt)");
  net->conv_mode = mode;
  return SEEDRL_OK;
}

extern "C" int seedrl_net_param_info(const seedrl_net* net, int index, char* name_buf,
                                     size_t name_buf_len, int64_t* dims, size_t* offset) {
  const ParamInfo* p = net ? net->params.info(index, name_buf, name_buf_len, dims, offset) : nullptr;
  return p ? p->rank : -1;
}

extern "C" size_t seedrl_net_workspace_bytes(const seedrl_net* net, int T1, int B) {
  if (!net || T1 <= 0 || B <= 0) return 0;
  return make_plan(net, T1, B).total;
}

// ---- forward --------------------------------------------------------------------
// _Stack.__call__, dmlab/networks.py:46-60, for every stack: conv, max-pool 3x3/2, two residual blocks.
static int torso_forward(const Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl;
  for (size_t s = 0; s < n->stacks.size(); ++s) {
    const Stack& k = n->stacks[s];
    const StackBufs& b = pl.st[s];
    const int H = k.hout, Wd = k.wout;
    if (s == 0) {
      SEEDRL_TRY(first_forward(c, obs));
    } else {
      SEEDRL_TRY(run_conv(c, k.conv, k.hin, k.win, IN_F32, pl.st[s - 1].o1, nullptr, b.a0));
      SEEDRL_TRY(pool_forward(c, k, b));
    }
    // res block 0: c0 = conv00(relu(p)); o0 = conv01(relu(c0)) + p        (networks.py:52-58)
    SEEDRL_TRY(run_conv(c, k.r00, H, Wd, IN_RELU, b.p, nullptr, b.c0));
    SEEDRL_TRY(run_conv(c, k.r01, H, Wd, IN_RELU, b.c0, &b.p, b.o0));
    // res block 1: c1 = conv10(relu(o0)); o1 = conv11(relu(c1)) + o0
    SEEDRL_TRY(run_conv(c, k.r10, H, Wd, IN_RELU, b.o0, nullptr, b.c1));
    SEEDRL_TRY(run_conv(c, k.r11, H, Wd, IN_RELU, b.c1, &b.o0, b.o1));
  }
  return SEEDRL_OK;
}

static int torso_forward_shallow(const Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl; void* ws = c.ws; cudaStream_t st = c.ex.st;
  const int N = pl.N;
  float* a1 = W<float>(ws, pl.sh_a1);
  float* a2 = W<float>(ws, pl.sh_a2);
  if (n->conv_mode >= 1 && n->cfg.obs_c % 4 == 0) {
    // tensor-core modes: the R2D2 body's im2col + GEMM layers (strided_conv.cu)
    SEEDRL_TRY(n->sh[0].forward(c.ex, N, true, obs, c.P(n->sh_w[0]), c.P(n->sh_b[0]), W<float>(ws, pl.sh_col0), a1,
                                16));
    return n->sh[1].forward(c.ex, N, false, a1, c.P(n->sh_w[1]), c.P(n->sh_b[1]), W<float>(ws, pl.sh_col1), a2, 32);
  }
  SEEDRL_TRY(convgen_forward(N, n->cfg.obs_h, n->cfg.obs_w, n->cfg.obs_c, 16, 8, 4, 1, obs,
                             c.P(n->sh_w[0]), c.P(n->sh_b[0]), 1, a1, st));
  SEEDRL_TRY(convgen_forward(N, n->sh[0].hout, n->sh[0].wout, 16, 32, 4, 2, 0, a1, c.P(n->sh_w[1]),
                             c.P(n->sh_b[1]), 1, a2, st));
  return SEEDRL_OK;
}

extern "C" int seedrl_net_forward(const seedrl_net* n, const float* prm, int T1, int B,
                                  const int64_t* prev_actions, const float* reward,
                                  const uint8_t* done, const uint8_t* observation,
                                  const float* h0, const float* c0, float* policy_logits,
                                  float* baseline, float* h_out, float* c_out, void* ws,
                                  size_t ws_bytes, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(n && prm && prev_actions && reward && done && observation && h0 && c0 &&
                       policy_logits && baseline && ws, "null pointer");
  SEEDRL_CHECK_ARG(T1 >= 1 && B >= 1, "T1, B must be >= 1");
  const Plan pl = make_plan(n, T1, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  Call c(n, pl, prm, nullptr, ws, st);
  const int N = pl.N, A = n->cfg.num_actions;
  // bounded-wait error flag of the wgmma / persistent kernels: cleared here, set by any kernel of
  // this forward or the matching backward, read back by seedrl_net_check_error
  SEEDRL_CUDA(cudaMemsetAsync(W<int>(ws, pl.tcerr), 0, sizeof(int), st));
  if (n->cfg.net == SEEDRL_NET_DEEP) {
    SEEDRL_TRY(first_layer(n, false, &c.first));
    SEEDRL_TRY(pad_first_layer(c, &observation));
    SEEDRL_TRY(pack_all_weights(c, 0));
    SEEDRL_TRY(torso_forward(c, observation));
  } else {
    SEEDRL_TRY(torso_forward_shallow(c, observation));
  }
  SEEDRL_TRY(core_forward(n->core, n->params, pl.core, c.ex, ws, prm, flat_features(n, pl, ws), reward, prev_actions,
                          done, h0, c0));
  const float* hs = W<float>(ws, pl.core.hs);
  // heads, networks.py:116-118
  GemmEpi e = epi_none();
  e.bias = c.P(n->p_pol_b);
  SEEDRL_TRY(c.ex.gemm(false, false, N, A, kHidden, hs, kHidden, c.P(n->p_pol_w), A, policy_logits,
                   A, e));
  e.bias = c.P(n->p_base_b);
  SEEDRL_TRY(c.ex.gemm(false, false, N, 1, kHidden, hs, kHidden, c.P(n->p_base_w), 1, baseline, 1,
                   e));
  return core_final_state(n->core, pl.core, st, ws, h_out, c_out);
}

extern "C" int seedrl_net_check_error(const seedrl_net* n, int T1, int B, void* ws, size_t ws_bytes,
                                      seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(n && ws && T1 >= 1 && B >= 1, "bad arguments");
  const Plan pl = make_plan(n, T1, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  return read_error_flag(W<int>(ws, pl.tcerr), (cudaStream_t)stream, "step");
}

// Where the ReLU and max-pool decisions of the last forward sit in a (T1, B) workspace (host arithmetic only).
extern "C" int seedrl_debug_net_views(const seedrl_net* n, int T1, int B, int index, size_t* offset, size_t* bytes,
                                      int* format) {
  SEEDRL_CHECK_ARG(n && offset && bytes && format && T1 >= 1 && B >= 1, "bad arguments");
  const Plan pl = make_plan(n, T1, B);
  const size_t N = pl.N;
  const bool deep = n->cfg.net == SEEDRL_NET_DEEP;
  const int last = deep ? 16 : 2;
  SEEDRL_CHECK_ARG(index >= 0 && index <= last, deep ? "index must be 0..16" : "index must be 0..2");
  if (index == last) {
    *offset = pl.core.xc; *bytes = N * (size_t)n->core.core_in * 4; *format = 0;
  } else if (!deep) {
    const StridedConv& l = n->sh[index];
    *offset = index == 0 ? pl.sh_a1 : pl.sh_a2; *bytes = N * l.hout * l.wout * (size_t)l.cout * 4; *format = 0;
  } else {
    // stack s, j = 0..3: p, c0, o0, c1, j = 4: the taps; index 15: the last stack's o1 (j = 5)
    const size_t s = index == 15 ? n->stacks.size() - 1 : index / 5;
    const int j = index == 15 ? 5 : index % 5;
    const Stack& k = n->stacks[s];
    const StackBufs& b = pl.st[s];
    const size_t pooled = N * k.hout * k.wout * (size_t)k.c;
    const Act* acts[6] = {&b.p, &b.c0, &b.o0, &b.c1, nullptr, &b.o1};
    if (j == 4) {
      *offset = b.idx; *bytes = pooled; *format = 2;
    } else {
      // p and o1 before their ReLU; c0, o0 and c1 as the buffer the next conv reads relu(x) from
      const Act& a = *acts[j];
      *offset = j == 0 || j == 5 ? a.raw : a.relu;
      *bytes = a.planes ? planes_bytes(pl.N, k.hout, k.wout, k.c) : pooled * 4;
      *format = a.planes ? 1 : 0;
    }
  }
  return SEEDRL_OK;
}

// ---- backward -------------------------------------------------------------------
// The mirror image of torso_forward.  On entry gA holds d loss / d o1 of the last stack.
static int torso_backward(Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl;
  const Act* g = pl.g;
  SEEDRL_TRY(gradient_from_dense(c));
  for (int s = (int)n->stacks.size() - 1; s >= 0; --s) {
    const Stack& k = n->stacks[s];
    const StackBufs& b = pl.st[s];
    const int H = k.hout, Wd = k.wout;
    // block 1: o1 = conv11(relu(c1)) + o0 ; c1 = conv10(relu(o0))
    SEEDRL_TRY(conv_bwd(c, k.r11, H, Wd, IN_RELU, b.c1, g[0], nullptr, g[1]));
    SEEDRL_TRY(conv_bwd(c, k.r10, H, Wd, IN_RELU, b.o0, g[1], &g[0], g[2]));
    // block 0: o0 = conv01(relu(c0)) + p ; c0 = conv00(relu(p))
    SEEDRL_TRY(conv_bwd(c, k.r01, H, Wd, IN_RELU, b.c0, g[2], nullptr, g[1]));
    SEEDRL_TRY(conv_bwd(c, k.r00, H, Wd, IN_RELU, b.p, g[1], &g[2], g[0]));
    // max-pool, then the stack's first conv
    if (s > 0) {
      SEEDRL_TRY(pool_backward(c, k, b.idx, g[0], pl.gPool));
      SEEDRL_TRY(conv_bwd(c, k.conv, k.hin, k.win, IN_F32, pl.st[s - 1].o1, pl.gPool, nullptr, g[0]));
    }
  }
  return first_backward(c, obs);
}

static int torso_backward_shallow(Call& c, const uint8_t* obs) {
  const seedrl_net* n = c.n; const Plan& pl = c.pl; void* ws = c.ws; cudaStream_t st = c.ex.st;
  // On entry gA holds d loss / d a2 (already masked by a2 > 0).
  const int N = pl.N;
  float* gA = W<float>(ws, pl.gA); float* gB = W<float>(ws, pl.g[1].raw);
  const float* a1 = W<float>(ws, pl.sh_a1);
  if (n->conv_mode >= 1 && n->cfg.obs_c % 4 == 0) {
    const StridedConv &l0 = n->sh[0], &l1 = n->sh[1];
    float* col1 = W<float>(ws, pl.sh_col1);
    SEEDRL_TRY(l1.wgrad(c.ex, N, false, a1, col1, gA, c.G(n->sh_w[1]), 32, c.G(n->sh_b[1])));
    SEEDRL_TRY(l1.dgrad(c.ex, N, gA, c.P(n->sh_w[1]), col1, a1, gB));
    return l0.wgrad(c.ex, N, true, obs, W<float>(ws, pl.sh_col0), gB, c.G(n->sh_w[0]), 16, c.G(n->sh_b[0]));
  }
  SEEDRL_TRY(convgen_wgrad(N, n->sh[0].hout, n->sh[0].wout, 16, 32, 4, 2, 0, a1, gA, c.G(n->sh_w[1]),
                           c.G(n->sh_b[1]), W<float>(ws, pl.partial),
                           conv3x3_wgrad_partial_bytes(), st));
  SEEDRL_TRY(convgen_dgrad(N, n->sh[0].hout, n->sh[0].wout, 16, 32, 4, 2, gA, c.P(n->sh_w[1]), a1, gB, st));
  SEEDRL_TRY(convgen_wgrad(N, n->cfg.obs_h, n->cfg.obs_w, n->cfg.obs_c, 16, 8, 4, 1, obs, gB,
                           c.G(n->sh_w[0]), c.G(n->sh_b[0]), W<float>(ws, pl.partial),
                           conv3x3_wgrad_partial_bytes(), st));
  return SEEDRL_OK;
}

// seedrl_net_backward; head_ready (may be null) is recorded once the first arena bucket's gradients are final.
static int net_backward(const seedrl_net* n, const float* prm, int T1, int B, const uint8_t* done,
                        const uint8_t* observation, const float* dlogits, const float* dbaseline, float* grd,
                        void* ws, size_t ws_bytes, cudaEvent_t head_ready, cudaStream_t st) {
  SEEDRL_CHECK_ARG(n && prm && done && observation && dlogits && dbaseline && grd && ws,
                   "null pointer");
  const Plan pl = make_plan(n, T1, B);
  SEEDRL_CHECK_ARG(ws_bytes >= pl.total, "workspace too small");
  Call c(n, pl, prm, grd, ws, st);
  const int N = pl.N, A = n->cfg.num_actions;
  const float* hs = W<float>(ws, pl.core.hs);
  float* dhs = W<float>(ws, pl.core.dhs);
  // padding floats and the entropy_cost_param slot must not carry garbage into Adam / all-reduce
  SEEDRL_CUDA(cudaMemsetAsync(grd, 0, n->params.arena_floats * sizeof(float), st));

  // heads
  GemmEpi e = epi_none();
  SEEDRL_TRY(c.ex.gemm(true, false, kHidden, A, N, hs, kHidden, dlogits, A, c.G(n->p_pol_w), A, e));
  SEEDRL_TRY(c.ex.colsum(N, A, dlogits, A, c.G(n->p_pol_b)));
  SEEDRL_TRY(c.ex.gemm(true, false, kHidden, 1, N, hs, kHidden, dbaseline, 1, c.G(n->p_base_w), 1, e));
  SEEDRL_TRY(c.ex.colsum(N, 1, dbaseline, 1, c.G(n->p_base_b)));
  SEEDRL_TRY(c.ex.gemm(false, true, N, kHidden, A, dlogits, A, c.P(n->p_pol_w), A, dhs, kHidden, e));
  GemmEpi eacc = epi_none();
  eacc.accumulate = 1;
  SEEDRL_TRY(c.ex.gemm(false, true, N, kHidden, 1, dbaseline, 1, c.P(n->p_base_w), 1, dhs, kHidden,
                   eacc));
  // BPTT, the core and Dense(256).  head_ready: every gradient of the arena's first bucket (heads, Dense,
  // LSTM: floats [0, seedrl_net_grad_split)) is final before dflat -- the conv torso's backward below only
  // writes the second bucket
  SEEDRL_TRY(core_backward(n->core, n->params, pl.core, c.ex, ws, prm, grd, done, flat_features(n, pl, ws),
                           W<float>(ws, pl.gA), head_ready));
  if (n->cfg.net == SEEDRL_NET_DEEP) {
    SEEDRL_TRY(first_layer(n, true, &c.first));
    c.wb = WgradBatch{W<float>(ws, pl.partial_all), kPartialAllBytes / sizeof(float), 0, 0, {}};
    SEEDRL_TRY(pad_first_layer(c, &observation));
    SEEDRL_TRY(pack_all_weights(c, 1));
    SEEDRL_TRY(torso_backward(c, observation));
    SEEDRL_TRY(wgrad_reduce_batch(&c.wb, st));
    if (c.dw0_pad) {        // padded [3,3,4,16] gradient -> the [3,3,3,16] parameter slot
      unpad_dw0_kernel<<<ceil_div(9 * 3 * 16, 128), 128, 0, st>>>(16, c.dw0_pad,
                                                                   grd + n->params.offset(n->stacks[0].conv.w));
      count_launch(PC_MISC, st);
    }
    return SEEDRL_OK;
  }
  return torso_backward_shallow(c, observation);
}

extern "C" int seedrl_net_backward(const seedrl_net* n, const float* prm, int T1, int B,
                                   const int64_t* prev_actions, const float* reward,
                                   const uint8_t* done, const uint8_t* observation,
                                   const float* dlogits, const float* dbaseline, float* grd,
                                   void* ws, size_t ws_bytes, seedrl_stream_t stream) {
  (void)prev_actions; (void)reward;
  return net_backward(n, prm, T1, B, done, observation, dlogits, dbaseline, grd, ws, ws_bytes, nullptr,
                      (cudaStream_t)stream);
}

// Data-parallel overlap (SURVEY 8e: the one exchange step): same as seedrl_net_backward, and
// `head_ready_event` (a cudaEvent_t) is recorded on `stream` as soon as the gradients of the first
// arena bucket -- floats [0, seedrl_net_grad_split(net)): baseline, conv_to_linear, core,
// policy_logits = 94 % of ImpalaDeep's parameters -- are final, i.e. before the convolution torso's
// backward (about half of the backward's time): the caller all-reduces that bucket on a side
// stream while the torso runs, then the remaining bucket.
extern "C" int seedrl_net_backward_overlap(const seedrl_net* n, const float* prm, int T1, int B,
                                           const int64_t* prev_actions, const float* reward, const uint8_t* done,
                                           const uint8_t* observation, const float* dlogits, const float* dbaseline,
                                           float* grd, void* ws, size_t ws_bytes, void* head_ready_event,
                                           seedrl_stream_t stream) {
  (void)prev_actions; (void)reward;
  return net_backward(n, prm, T1, B, done, observation, dlogits, dbaseline, grd, ws, ws_bytes,
                      (cudaEvent_t)head_ready_event, (cudaStream_t)stream);
}
extern "C" size_t seedrl_net_grad_split(const seedrl_net* n) {
  if (!n) return 0;
  const int first_conv = n->cfg.net == SEEDRL_NET_DEEP ? n->stacks[0].conv.w : n->sh_w[0];
  return n->params.offset(first_conv);
}

// ---- single-kernel test hooks (exported so the GPU parity tests can localise a
// failure to one kernel; not used by the product path) ------------------------------
extern "C" int seedrl_debug_conv3x3(int cin, int cout, int in_mode, int N, int H, int W,
                                    const void* in, const float* w, const float* bias,
                                    const float* mask, const float* res, float* out,
                                    seedrl_stream_t stream) {
  return conv3x3_forward(cin, cout, in_mode, N, H, W, in, w, bias, mask, res, out,
                         (cudaStream_t)stream);
}
extern "C" int seedrl_debug_conv3x3_flip(int cin, int cout, const float* w, float* wt,
                                         seedrl_stream_t stream) {
  return conv3x3_flip_weights(cin, cout, w, wt, (cudaStream_t)stream);
}
extern "C" size_t seedrl_debug_wgrad_partial_bytes(void) { return conv3x3_wgrad_partial_bytes(); }
extern "C" int seedrl_debug_conv3x3_wgrad(int cin, int cout, int in_mode, int N, int H, int W,
                                          const void* x, const float* dy, float* dw, float* db,
                                          float* partial, size_t partial_bytes,
                                          seedrl_stream_t stream) {
  return conv3x3_wgrad(cin, cout, in_mode, N, H, W, x, dy, dw, db, partial, partial_bytes,
                       (cudaStream_t)stream);
}
extern "C" int seedrl_debug_maxpool(int backward, int N, int H, int W, int C, const float* x_or_dy,
                                    float* y_or_dx, uint8_t* idx, seedrl_stream_t stream) {
  if (backward) return maxpool3s2_backward(N, H, W, C, x_or_dy, idx, y_or_dx, (cudaStream_t)stream);
  return maxpool3s2_forward(N, H, W, C, x_or_dy, y_or_dx, idx, (cudaStream_t)stream);
}
// wgmma GEMM test hook (same contract as seedrl_debug_sgemm; split != 0: bf16x3 operands;
// ws: >= ws_bytes of scratch for split-K partials, may be null).
extern "C" int seedrl_debug_gemm_tc(int ta, int tb, int split, int M, int N, int K, const float* A, int lda,
                                    const float* B, int ldb, float* C, int ldc, const float* bias,
                                    const float* mask, int ldm, int relu, int accumulate, int a_relu,
                                    float* ws, size_t ws_bytes, int* error_flag, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(M >= 1 && N >= 1 && K >= 1 && A && B && C, "bad arguments");
  GemmEpi e{bias, mask, ldm, relu, accumulate, a_relu};
  return gemm_tc(ta != 0, tb != 0, split, M, N, K, A, lda, B, ldb, C, ldc, e, ws, ws_bytes, error_flag,
                 (cudaStream_t)stream);
}

extern "C" int seedrl_debug_sgemm(int ta, int tb, int M, int N, int K, const float* A, int lda,
                                  const float* B, int ldb, float* C, int ldc, const float* bias,
                                  const float* mask, int ldm, int relu, int accumulate, int a_relu,
                                  seedrl_stream_t stream) {
  GemmEpi e{bias, mask, ldm, relu, accumulate, a_relu};
  return sgemm(ta != 0, tb != 0, M, N, K, A, lda, B, ldb, C, ldc, e, (cudaStream_t)stream);
}

// 0: the im2col convolutions (shallow net, R2D2 body) materialise their matrices instead of gathering
// them inside the GEMM (A/B parity tests; results are bit-identical).
extern "C" int seedrl_debug_set_gemm_gather(int on) {
  gemm_tc_set_gather(on);
  return SEEDRL_OK;
}

// Column-sum test hook (bias gradients): out[n] = sum_m X[m*ld + n]; `ws` enables the row-slab path.
extern "C" int seedrl_debug_colsum(int M, int N, const float* X, int ld, float* out, float* ws, size_t ws_bytes,
                                   seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(M >= 1 && N >= 1 && X && out && ld >= N, "bad arguments");
  return colsum(M, N, X, ld, out, (cudaStream_t)stream, ws, ws_bytes);
}

// Host evaluation of the tall-image position -> pixel maps the conv kernels use (multiply-high
// division): which = 0 padded-input position, 1 output position.  No GPU involved.
extern "C" int seedrl_debug_conv_pixels(int N, int H, int W, int which, int start, int count, int* out) {
  SEEDRL_CHECK_ARG(N >= 1 && H >= 1 && W >= 1 && start >= 0 && count >= 0 && out, "bad arguments");
  const ConvGeom g = make_geom(N, H, W);
  for (int i = 0; i < count; ++i) out[i] = which ? out_pixel(g, start + i) : in_pixel(g, start + i);
  return SEEDRL_OK;
}

// Bench knob: K positions per pipeline stage of the tensor-core weight-gradient kernel
// (the largest of 512/256/128 not above `kc` whose stages fit shared memory is used; default 512).
extern "C" int seedrl_debug_set_wgrad_chunk(int kc) {
  SEEDRL_CHECK_ARG(kc == 128 || kc == 256 || kc == 512, "chunk must be 128, 256 or 512");
  conv3x3_wgrad_tc_set_chunk(kc);
  return SEEDRL_OK;
}

extern "C" int seedrl_debug_conv3x3_wgrad_tc(int cin, int cout, int in_mode, int split, int N, int H, int W,
                                             const void* x, const float* dy, float* dw, float* db,
                                             float* partial, size_t partial_bytes, int* error_flag,
                                             seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(conv3x3_wgrad_tc_supported(cin, cout, in_mode), "unsupported (cin,cout,mode)");
  return conv3x3_wgrad_tc(cin, cout, in_mode, split, N, H, W, x, dy, dw, db, partial, partial_bytes,
                          error_flag, nullptr, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_conv0pool(int N, int H, int W, const uint8_t* frames, const float* w, const float* bias,
                                      void* praw, void* prelu, uint8_t* idx, int* err, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(frames && w && bias && praw && prelu && idx && err, "null pointer");
  SEEDRL_CHECK_ARG(conv0pool_supported(4, 16, H, W), "unsupported frame size");
  return conv0pool_forward(N, H, W, 4, frames, w, bias, praw, prelu, idx, err, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_conv0pool_c(int N, int H, int W, int C, const uint8_t* frames, const float* w,
                                        const float* bias, void* praw, void* prelu, uint8_t* idx, int* err,
                                        seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(frames && w && bias && praw && prelu && idx && err, "null pointer");
  SEEDRL_CHECK_ARG(N >= 1 && conv0pool_supported(C, 16, H, W), "unsupported frame shape");
  return conv0pool_forward(N, H, W, C, frames, w, bias, praw, prelu, idx, err, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_first_wgrad_pooled_c(int N, int H, int W, int C, const uint8_t* frames,
                                                 const void* g_planes, const uint8_t* idx, float* dw, float* db,
                                                 float* partial, size_t partial_bytes, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(frames && g_planes && idx && dw && db && partial, "null pointer");
  SEEDRL_CHECK_ARG(N >= 1 && first_wgrad_pooled_supported(C, 16, H, W), "unsupported frame shape");
  WgradBatch wb{partial, partial_bytes / sizeof(float), 0, 0, {}};
  SEEDRL_TRY(first_wgrad_pooled(N, H, W, C, frames, g_planes, idx, dw, db, &wb, (cudaStream_t)stream));
  return wgrad_reduce_batch(&wb, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_set_first_layer_dense(int on) {
  g_first_dense = on ? 1 : 0;
  return SEEDRL_OK;
}
// Bench knob: output positions per tile of the tensor-core forward / data-gradient kernel
// (the largest of 512/256/128 not above `mt` that keeps >= 2 CTAs per SM is used; default 512).
extern "C" int seedrl_debug_set_conv_tile(int mt) {
  SEEDRL_CHECK_ARG(mt == 128 || mt == 256 || mt == 512, "tile must be 128, 256 or 512");
  conv3x3_tc_set_tile(mt);
  return SEEDRL_OK;
}

// wgmma conv test hook: packs fp32 HWIO weights (optionally flipped/transposed for the
// data-gradient) into `wq_scratch` (>= 2*9*max(cin,16)*cout*2 bytes) and runs the tensor-core conv.
// `variant` must be 0 (the argument is kept for ABI compatibility); the kernel has no bounded waits, so
// *error_flag is left unchanged.
extern "C" int seedrl_debug_conv3x3_tc(int cin, int cout, int in_mode, int split, int N, int H, int W,
                                       const void* in, const float* w, const float* bias,
                                       const float* mask, const float* res, float* out, int flip,
                                       int variant, void* wq_scratch, int* error_flag,
                                       seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(variant == 0, "variant must be 0");
  SEEDRL_CHECK_ARG(conv3x3_tc_supported(cin, cout, in_mode), "unsupported (cin,cout,mode)");
  SEEDRL_TRY(conv3x3_tc_pack_weights(cin, cout, flip, split, w, wq_scratch, (cudaStream_t)stream));
  return conv3x3_tc_forward(cin, cout, in_mode, split, N, H, W, in, wq_scratch, bias, mask, res, out,
                            error_flag, (cudaStream_t)stream);
}

// ---- plane-tensor path test hooks (conv_planes.cu) ---------------------------------------------
extern "C" size_t seedrl_debug_planes_bytes(int N, int H, int W, int C) {
  if (N < 1 || H < 1 || W < 1 || C < 8 || C % 8) return 0;
  return planes_bytes(N, H, W, C);
}
extern "C" int seedrl_debug_to_planes(int N, int H, int W, int C, int relu, const float* x, void* out,
                                      seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0 && x && out, "bad arguments");
  return to_planes(N, H, W, C, relu, x, out, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_from_planes(int N, int H, int W, int C, const void* in, float* y,
                                        seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0 && in && y, "bad arguments");
  return from_planes(N, H, W, C, in, y, (cudaStream_t)stream);
}
// 3x3 'same' conv on plane tensors.  w: fp32 HWIO of the FORWARD layer; flip != 0 runs the data
// gradient (cin/cout are those of the gradient convolution).  wq_scratch >= 2*9*cin*cout*2 bytes.
extern "C" int seedrl_debug_convp(int cin, int cout, int N, int H, int W, const void* in, const float* w,
                                  const float* bias, const void* mask, const void* res, int flip,
                                  void* out_raw, void* out_relu, float* out_nhwc, void* wq_scratch,
                                  int* error_flag, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(convp_supported(cin, cout) && in && w && wq_scratch, "unsupported (cin,cout) or null pointer");
  SEEDRL_TRY(conv3x3_tc_pack_weights(cin, cout, flip, 2, w, wq_scratch, (cudaStream_t)stream));
  PlaneConv c;
  c.N = N; c.H = H; c.W = W; c.in = in; c.wq = wq_scratch; c.bias = bias; c.mask = mask; c.res = res;
  c.out_raw = out_raw; c.out_relu = out_relu; c.out_nhwc = out_nhwc; c.err = error_flag;
  return convp_forward(cin, cout, c, (cudaStream_t)stream);
}
extern "C" int seedrl_debug_wgradp(int cin, int cout, int N, int H, int W, const void* x, const void* dy,
                                   float* dw, float* db, float* partial, size_t partial_bytes,
                                   int* error_flag, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(x && dy && dw && db && partial, "null pointer");
  WgradBatch wb{partial, partial_bytes / sizeof(float), 0, 0, {}};
  SEEDRL_TRY(wgradp(cin, cout, N, H, W, x, dy, dw, db, error_flag, &wb, (cudaStream_t)stream));
  return wgrad_reduce_batch(&wb, (cudaStream_t)stream);
}
// max-pool 3x3/2 'SAME' on the plane path.  forward: x fp32 NHWC -> out_raw / out_relu plane tensors
// + idx; backward: dy plane tensor (pooled) + idx -> dx plane tensor (out_raw) or fp32 NHWC (out_nhwc).
extern "C" int seedrl_debug_poolp(int backward, int N, int H, int W, int C, const void* in, void* out_raw,
                                  void* out_relu, float* out_nhwc, uint8_t* idx, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 1 && H >= 1 && W >= 1 && C >= 8 && C % 8 == 0 && in && idx, "bad arguments");
  if (backward) return poolp_backward(N, H, W, C, in, idx, out_raw, out_nhwc, (cudaStream_t)stream);
  SEEDRL_CHECK_ARG(out_raw && out_relu, "null pointer");
  return poolp_forward(N, H, W, C, reinterpret_cast<const float*>(in), out_raw, out_relu, idx,
                       (cudaStream_t)stream);
}
