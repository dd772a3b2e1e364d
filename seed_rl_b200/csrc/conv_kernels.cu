// Convolution / pooling kernels (fp32 SIMT path) for the ImpalaDeep torso,
// dmlab/networks.py:26-60 (_Stack: Conv2D 3x3 'same' + MaxPool 3/2 'same' +
// residual blocks) -- forward, data-gradient and weight-gradient.
//
// Layout: activations NHWC (as the reference), weights HWIO = [tap][ci][co].
//
// "Tall image" formulation.  The N images of a layer are treated as ONE tall,
// zero-padded image: padded width PW = W+2, image n occupies padded rows
// n*(H+1)+1 .. n*(H+1)+H, and padded row n*(H+1) is a shared zero row (bottom
// pad of image n-1 == top pad of image n).  With positions flattened as
// p = R*PW + c, the 3x3 'same' convolution becomes
//     out[p] = sum_{kh,kw} in_pad[p + kh*PW + kw] . W[kh,kw]
// for EVERY p, so a CTA simply owns a contiguous chunk of QC positions: no
// per-image tails, unit-stride (bank-conflict-free) shared-memory reads, and
// the same code serves every feature-map size.  Positions that land on a pad
// column or separator row are computed and dropped (3.5% at 84x84 .. 22% at
// 11x11).
#include "kernels.h"

namespace seedrl {

// channels 4*c4 .. 4*c4+3 of pixel pix of [.., C] uint8 frames, zero at and above C
__device__ __forceinline__ uchar4 load_u8_padded(const void* frames, int pix, int C, int c4) {
  const uint8_t* p = reinterpret_cast<const uint8_t*>(frames) + (size_t)pix * C + 4 * c4;
  const int c = 4 * c4;
  return make_uchar4(c < C ? __ldg(p) : 0, c + 1 < C ? __ldg(p + 1) : 0, c + 2 < C ? __ldg(p + 2) : 0,
                     c + 3 < C ? __ldg(p + 3) : 0);
}

// ---------------------------------------------------------------------------
// conv3x3 (forward, and data-gradient with flipped/transposed weights).
//   out[pix, co] = epi( sum_{tap,ci} tin(in)[pix+tap, ci] * w[tap][ci][co] )
//   epi(v) = v (+ bias[co]) ; if mask: v = mask[pix,co] > 0 ? v : 0 ; (+ res[pix,co])
// 128 threads; warp = (position-warp, output-channel group of 16).
// IN_U8 with cin_src < CIN: frames of cin_src channels, zero-filled to CIN in shared memory, and
// weights [3,3,cin_src,COUT] with zero rows for the padding channels (first conv of C-channel frames).
template <int CIN, int COUT, int IN_MODE>
struct Conv3x3Cfg {
  static constexpr int kThreads = 128;
  static constexpr int CO = 16;
  static constexpr int NCOG = COUT / CO;
  static constexpr int NPW = (kThreads / 32) / NCOG;
  static constexpr int PXT = 4;
  static constexpr int QC = NPW * PXT * 32;
};

template <int CIN, int COUT, int IN_MODE>
__global__ void __launch_bounds__(128)
conv3x3_kernel(ConvGeom g, int cin_src, const void* __restrict__ in_, const float* __restrict__ w,
               const float* __restrict__ bias, const float* __restrict__ mask,
               const float* __restrict__ res, float* __restrict__ out) {
  using Cfg = Conv3x3Cfg<CIN, COUT, IN_MODE>;
  constexpr int QC = Cfg::QC, CO = Cfg::CO, PXT = Cfg::PXT;
  extern __shared__ float smem[];
  const int PW = g.PW;
  const int L = QC + 2 * PW + 2;
  const int LP = L | 1;                      // odd plane stride: conflict-free transposing stores
  float* s_in = smem;                        // [CIN][LP]
  float* s_w = smem + (size_t)CIN * LP;      // [9][CIN][COUT]
  const int tid = threadIdx.x;
  const int q0 = blockIdx.x * QC;

  // weights -> smem (vectorised, L2-resident)
  if (IN_MODE == IN_U8 && cin_src != CIN) {
    for (int i = tid; i < 9 * CIN * COUT; i += Cfg::kThreads) {
      const int co = i % COUT, ci = (i / COUT) % CIN, tap = i / (CIN * COUT);
      s_w[i] = ci < cin_src ? __ldg(w + (tap * cin_src + ci) * COUT + co) : 0.f;
    }
  } else {
    const float4* w4 = reinterpret_cast<const float4*>(w);
    float4* s4 = reinterpret_cast<float4*>(s_w);
    for (int i = tid; i < 9 * CIN * COUT / 4; i += Cfg::kThreads) s4[i] = __ldg(w4 + i);
  }
  // input tile -> smem, channel-planar.  One thread moves 4 channels of a position.
  {
    constexpr int C4 = CIN / 4;
    for (int i = tid; i < L * C4; i += Cfg::kThreads) {
      const int s = i / C4, c4 = i - s * C4;
      const int pix = in_pixel(g, q0 + s);
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (pix >= 0) {
        if (IN_MODE == IN_U8) {
          const uchar4 u = cin_src == CIN ? __ldg(reinterpret_cast<const uchar4*>(in_) + (size_t)pix * C4 + c4)
                                          : load_u8_padded(in_, pix, cin_src, c4);
          const float k = 1.0f / 255.0f;     // dmlab/networks.py:98-100
          v = make_float4(u.x * k, u.y * k, u.z * k, u.w * k);
          // NOTE: x/255 and x*(1/255) differ by <=1 ulp; tolerance documented in tests.
        } else {
          v = __ldg(reinterpret_cast<const float4*>(in_) + (size_t)pix * C4 + c4);
          if (IN_MODE == IN_RELU) {
            v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f);
            v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
          }
        }
      }
      float* d = s_in + (size_t)(c4 * 4) * LP + s;
      d[0] = v.x; d[LP] = v.y; d[2 * LP] = v.z; d[3 * LP] = v.w;
    }
  }
  __syncthreads();

  const int warp = tid >> 5, lane = tid & 31;
  const int cog = warp % Cfg::NCOG;
  const int pw = warp / Cfg::NCOG;
  const int pbase = pw * PXT * 32 + lane;    // positions pbase + 32*j
  float acc[PXT][CO];
#pragma unroll
  for (int j = 0; j < PXT; ++j)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[j][c] = 0.f;

#pragma unroll 1
  for (int ci = 0; ci < CIN; ++ci) {
    const float* xin = s_in + (size_t)ci * LP + pbase;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const float4* wp = reinterpret_cast<const float4*>(
            s_w + ((size_t)((kh * 3 + kw) * CIN + ci)) * COUT + cog * CO);
        float wv[CO];
#pragma unroll
        for (int c4 = 0; c4 < CO / 4; ++c4) {
          const float4 t = wp[c4];
          wv[c4 * 4 + 0] = t.x; wv[c4 * 4 + 1] = t.y; wv[c4 * 4 + 2] = t.z; wv[c4 * 4 + 3] = t.w;
        }
        const int off = kh * PW + kw;
#pragma unroll
        for (int j = 0; j < PXT; ++j) {
          const float x = xin[off + 32 * j];
#pragma unroll
          for (int c = 0; c < CO; ++c) acc[j][c] = fmaf(x, wv[c], acc[j][c]);
        }
      }
    }
  }

  // epilogue
  float bv[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) bv[c] = bias ? __ldg(bias + cog * CO + c) : 0.f;
#pragma unroll
  for (int j = 0; j < PXT; ++j) {
    const int p = q0 + pbase + 32 * j;
    const int pix = out_pixel(g, p);
    if (pix < 0) continue;
    const size_t o = (size_t)pix * COUT + cog * CO;
#pragma unroll
    for (int c4 = 0; c4 < CO / 4; ++c4) {
      float4 v = make_float4(acc[j][c4 * 4 + 0] + bv[c4 * 4 + 0], acc[j][c4 * 4 + 1] + bv[c4 * 4 + 1],
                             acc[j][c4 * 4 + 2] + bv[c4 * 4 + 2], acc[j][c4 * 4 + 3] + bv[c4 * 4 + 3]);
      if (mask) {
        const float4 m = __ldg(reinterpret_cast<const float4*>(mask + o) + c4);
        v.x = m.x > 0.f ? v.x : 0.f; v.y = m.y > 0.f ? v.y : 0.f;
        v.z = m.z > 0.f ? v.z : 0.f; v.w = m.w > 0.f ? v.w : 0.f;
      }
      if (res) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(res + o) + c4);
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      reinterpret_cast<float4*>(out + o)[c4] = v;
    }
  }
}

template <int CIN, int COUT, int IN_MODE>
static int launch_conv3x3(int N, int H, int W, const void* in, const float* w, const float* bias,
                          const float* mask, const float* res, float* out, cudaStream_t st, int cin_src = CIN) {
  using Cfg = Conv3x3Cfg<CIN, COUT, IN_MODE>;
  const ConvGeom g = make_geom(N, H, W);
  const int L = Cfg::QC + 2 * g.PW + 2;
  const size_t smem = ((size_t)CIN * (L | 1) + 9 * CIN * COUT) * sizeof(float);
  SEEDRL_CUDA(allow_smem<conv3x3_kernel<CIN, COUT, IN_MODE>>(200 * 1024));
  if (smem > 200 * 1024) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3: image too wide");
  if (g.Q + Cfg::QC + 4 * g.PW >= (1LL << 31))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3: batch too large for 32-bit positions");
  const long long grid = (g.Q + Cfg::QC - 1) / Cfg::QC;
  conv3x3_kernel<CIN, COUT, IN_MODE><<<(unsigned)grid, Cfg::kThreads, smem, st>>>(g, cin_src, in, w, bias,
                                                                                 mask, res, out);
  count_launch(g_conv_cat, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int conv3x3_forward(int cin, int cout, int in_mode, int N, int H, int W, const void* in,
                    const float* w, const float* bias, const float* mask, const float* res,
                    float* out, cudaStream_t st) {
#define SEEDRL_CONV_CASE(CI, CO_, MODE)                                              \
  if (cin == CI && cout == CO_ && in_mode == MODE)                                   \
    return launch_conv3x3<CI, CO_, MODE>(N, H, W, in, w, bias, mask, res, out, st);
  SEEDRL_CONV_CASE(4, 16, IN_U8)
  SEEDRL_CONV_CASE(4, 16, IN_F32)
  SEEDRL_CONV_CASE(16, 16, IN_F32)
  SEEDRL_CONV_CASE(16, 16, IN_RELU)
  SEEDRL_CONV_CASE(16, 32, IN_F32)
  SEEDRL_CONV_CASE(32, 16, IN_F32)
  SEEDRL_CONV_CASE(32, 32, IN_F32)
  SEEDRL_CONV_CASE(32, 32, IN_RELU)
#undef SEEDRL_CONV_CASE
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3: unsupported (cin,cout,mode)");
}

// First conv of the deep net on [N,H,W,C] uint8 frames, C in 1..16, 16 output channels: the 4-, 8- or
// 16-channel kernel with the frames and weights zero-filled to that width in shared memory.
int conv3x3_u8_forward(int C, int N, int H, int W, const uint8_t* frames, const float* w, const float* bias,
                       float* out, cudaStream_t st) {
  if (C >= 1 && C <= 4) return launch_conv3x3<4, 16, IN_U8>(N, H, W, frames, w, bias, nullptr, nullptr, out, st, C);
  if (C >= 5 && C <= 8) return launch_conv3x3<8, 16, IN_U8>(N, H, W, frames, w, bias, nullptr, nullptr, out, st, C);
  if (C >= 9 && C <= 16) return launch_conv3x3<16, 16, IN_U8>(N, H, W, frames, w, bias, nullptr, nullptr, out, st, C);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3_u8: channels must be 1..16");
}

// w[tap][ci][co] -> wt[8-tap][co][ci]   (data-gradient weights)
__global__ void flip_transpose_w_kernel(int cin, int cout, const float* __restrict__ w,
                                        float* __restrict__ wt) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * cin * cout) return;
  const int co = i % cout;
  const int ci = (i / cout) % cin;
  const int tap = i / (cout * cin);
  wt[((size_t)(8 - tap) * cout + co) * cin + ci] = w[i];
}

int conv3x3_flip_weights(int cin, int cout, const float* w, float* wt, cudaStream_t st) {
  const int n = 9 * cin * cout;
  flip_transpose_w_kernel<<<ceil_div(n, 256), 256, 0, st>>>(cin, cout, w, wt);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// ---------------------------------------------------------------------------
// conv3x3 weight gradient:  dW[tap][ci][co] = sum_p tin(x)[p+tap][ci] * dy[p][co],
// db[co] = sum_p dy[p][co].  Persistent CTAs (grid = k * 148) loop over position
// chunks; each thread owns dW[0..8][ci][co4..co4+3] in registers and walks its
// share of the chunk sequentially with a rolling 3x3 register window (3 new x
// loads + 1 float4 dy load per 36 FMAs).  Per-CTA partials are reduced by
// wgrad_reduce_kernel in fixed order (deterministic, no atomics).
template <int CIN, int COUT>
struct WgradCfg {
  static constexpr int kThreads = 256;
  static constexpr int TPG = CIN * (COUT / 4);       // threads per position-group
  static constexpr int G = kThreads / TPG;           // position groups
  static constexpr int QC = 256;                     // positions per chunk
  static constexpr int PPG = QC / G;                 // positions per group per chunk
};

template <int CIN, int COUT, int IN_MODE>
__global__ void __launch_bounds__(256)
conv3x3_wgrad_kernel(ConvGeom g, int cin_src, const void* __restrict__ x_, const float* __restrict__ dy,
                     float* __restrict__ partial /* [grid][9*cin_src*COUT + COUT] */) {
  using Cfg = WgradCfg<CIN, COUT>;
  constexpr int QC = Cfg::QC, G = Cfg::G, PPG = Cfg::PPG, TPG = Cfg::TPG;
  extern __shared__ float smem[];
  const int PW = g.PW;
  const int L = QC + 2 * PW + 2;
  constexpr int XS = CIN + 1;                        // padded position stride (odd-ish)
  float* s_x = smem;                                 // [L][XS]
  float* s_dy = smem + (((size_t)L * XS + 3) & ~(size_t)3);   // [QC][COUT], 16B aligned
  const int tid = threadIdx.x;
  const int grp = tid / TPG;
  const int r = tid - grp * TPG;
  const int ci = r % CIN;
  const int cog = r / CIN;                           // float4 group of output channels

  float acc[9][4];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < 4; ++c) acc[t][c] = 0.f;
  float4 bacc = make_float4(0.f, 0.f, 0.f, 0.f);

  const long long nchunks = (g.Q + QC - 1) / QC;
  for (long long ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const int q0 = (int)(ch * QC);
    __syncthreads();   // previous chunk fully consumed
    {
      constexpr int C4 = CIN / 4;
      for (int i = tid; i < L * C4; i += Cfg::kThreads) {
        const int s = i / C4, c4 = i - s * C4;
        const int pix = in_pixel(g, q0 + s);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (pix >= 0) {
          if (IN_MODE == IN_U8) {
            const uchar4 u = cin_src == CIN ? __ldg(reinterpret_cast<const uchar4*>(x_) + (size_t)pix * C4 + c4)
                                            : load_u8_padded(x_, pix, cin_src, c4);
            const float k = 1.0f / 255.0f;
            v = make_float4(u.x * k, u.y * k, u.z * k, u.w * k);
          } else {
            v = __ldg(reinterpret_cast<const float4*>(x_) + (size_t)pix * C4 + c4);
            if (IN_MODE == IN_RELU) {
              v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f);
              v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
            }
          }
        }
        float* d = s_x + (size_t)s * XS + c4 * 4;
        d[0] = v.x; d[1] = v.y; d[2] = v.z; d[3] = v.w;
      }
      constexpr int O4 = COUT / 4;
      for (int i = tid; i < QC * O4; i += Cfg::kThreads) {
        const int s = i / O4, c4 = i - s * O4;
        const int pix = out_pixel(g, q0 + s);
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (pix >= 0) v = __ldg(reinterpret_cast<const float4*>(dy) + (size_t)pix * O4 + c4);
        reinterpret_cast<float4*>(s_dy)[i] = v;
      }
    }
    __syncthreads();
    // rolling window over this group's PPG consecutive positions
    const int p0 = grp * PPG;
    float xw[3][3];
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      xw[kh][1] = s_x[(size_t)(p0 + kh * PW + 0) * XS + ci];
      xw[kh][2] = s_x[(size_t)(p0 + kh * PW + 1) * XS + ci];
    }
#pragma unroll 4
    for (int pp = 0; pp < PPG; ++pp) {
      const int p = p0 + pp;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        xw[kh][0] = xw[kh][1];
        xw[kh][1] = xw[kh][2];
        xw[kh][2] = s_x[(size_t)(p + kh * PW + 2) * XS + ci];
      }
      const float4 d = reinterpret_cast<const float4*>(s_dy)[p * (COUT / 4) + cog];
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const float x = xw[kh][kw];
          acc[kh * 3 + kw][0] = fmaf(x, d.x, acc[kh * 3 + kw][0]);
          acc[kh * 3 + kw][1] = fmaf(x, d.y, acc[kh * 3 + kw][1]);
          acc[kh * 3 + kw][2] = fmaf(x, d.z, acc[kh * 3 + kw][2]);
          acc[kh * 3 + kw][3] = fmaf(x, d.w, acc[kh * 3 + kw][3]);
        }
      if (ci == 0) { bacc.x += d.x; bacc.y += d.y; bacc.z += d.z; bacc.w += d.w; }
    }
  }
  // cross-group reduction in shared memory (fixed order), then one partial per CTA
  __syncthreads();
  float* s_red = smem;   // [G][9*CIN*COUT + COUT]  (reuses tile memory)
  constexpr int NW = 9 * CIN * COUT + COUT;
  float* mine = s_red + (size_t)grp * NW;
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < 4; ++c) mine[((size_t)t * CIN + ci) * COUT + cog * 4 + c] = acc[t][c];
  if (ci == 0) {
    mine[9 * CIN * COUT + cog * 4 + 0] = bacc.x; mine[9 * CIN * COUT + cog * 4 + 1] = bacc.y;
    mine[9 * CIN * COUT + cog * 4 + 2] = bacc.z; mine[9 * CIN * COUT + cog * 4 + 3] = bacc.w;
  }
  __syncthreads();
  // partial in the real [3][3][cin_src][COUT] order (rows of the padding channels are dropped)
  const int nwr = 9 * cin_src * COUT;
  float* dst = partial + (size_t)blockIdx.x * (nwr + COUT);
  for (int i = tid; i < nwr + COUT; i += Cfg::kThreads) {
    int j = i;
    if (cin_src != CIN) {
      const int co = i % COUT, cr = i / COUT, tap = cr / cin_src;
      j = i < nwr ? (tap * CIN + cr - tap * cin_src) * COUT + co : 9 * CIN * COUT + i - nwr;
    }
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < G; ++k) s += s_red[(size_t)k * NW + j];
    dst[i] = s;
  }
}

// out[i] = sum_k partial[k][i]  (k in fixed order).  dW -> dw, db -> db.
__global__ void wgrad_reduce_kernel(int nparts, int nw, int nb, const float* __restrict__ partial,
                                    float* __restrict__ dw, float* __restrict__ db) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nw + nb) return;
  float s = 0.f;
  for (int k = 0; k < nparts; ++k) s += partial[(size_t)k * (nw + nb) + i];
  if (i < nw) dw[i] = s; else db[i - nw] = s;
}

template <int CIN, int COUT, int IN_MODE>
static int launch_wgrad(int N, int H, int W, const void* x, const float* dy, float* dw, float* db,
                        float* partial, size_t partial_bytes, cudaStream_t st, int cin_src = CIN) {
  using Cfg = WgradCfg<CIN, COUT>;
  const ConvGeom g = make_geom(N, H, W);
  const int L = Cfg::QC + 2 * g.PW + 2;
  constexpr int NW = 9 * CIN * COUT + COUT;
  size_t smem = ((((size_t)L * (CIN + 1) + 3) & ~(size_t)3) + (size_t)Cfg::QC * COUT) * sizeof(float);
  const size_t red = (size_t)Cfg::G * NW * sizeof(float);
  if (red > smem) smem = red;
  SEEDRL_CUDA(allow_smem<conv3x3_wgrad_kernel<CIN, COUT, IN_MODE>>(200 * 1024));
  if (smem > 200 * 1024) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad: tile too large");
  if (g.Q + Cfg::QC + 4 * g.PW >= (1LL << 31))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad: batch too large for 32-bit positions");
  const long long nchunks = (g.Q + Cfg::QC - 1) / Cfg::QC;
  int grid = kNumSMs * 2;
  if (grid > nchunks) grid = (int)nchunks;
  if ((size_t)grid * NW * sizeof(float) > partial_bytes)
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad: partial buffer too small");
  conv3x3_wgrad_kernel<CIN, COUT, IN_MODE><<<grid, Cfg::kThreads, smem, st>>>(g, cin_src, x, dy, partial);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  wgrad_reduce_kernel<<<ceil_div(9 * cin_src * COUT + COUT, 256), 256, 0, st>>>(grid, 9 * cin_src * COUT, COUT,
                                                                                 partial, dw, db);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int wgrad_reduce(int nparts, int nw, int nb, const float* partial, float* dw, float* db,
                 cudaStream_t st) {
  wgrad_reduce_kernel<<<ceil_div(nw + nb, 256), 256, 0, st>>>(nparts, nw, nb, partial, dw, db);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

size_t conv3x3_wgrad_partial_bytes() {
  return (size_t)kNumSMs * 2 * (9 * 32 * 32 + 32) * sizeof(float);
}

int conv3x3_wgrad(int cin, int cout, int in_mode, int N, int H, int W, const void* x,
                  const float* dy, float* dw, float* db, float* partial, size_t partial_bytes,
                  cudaStream_t st) {
#define SEEDRL_WG_CASE(CI, CO_, MODE)                                               \
  if (cin == CI && cout == CO_ && in_mode == MODE)                                  \
    return launch_wgrad<CI, CO_, MODE>(N, H, W, x, dy, dw, db, partial, partial_bytes, st);
  SEEDRL_WG_CASE(4, 16, IN_U8)
  SEEDRL_WG_CASE(4, 16, IN_F32)
  SEEDRL_WG_CASE(16, 16, IN_RELU)
  SEEDRL_WG_CASE(16, 32, IN_F32)
  SEEDRL_WG_CASE(32, 32, IN_F32)
  SEEDRL_WG_CASE(32, 32, IN_RELU)
#undef SEEDRL_WG_CASE
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad: unsupported (cin,cout,mode)");
}

// Weight gradient of conv3x3_u8_forward: dw in the real [3,3,C,16] layout.
int conv3x3_u8_wgrad(int C, int N, int H, int W, const uint8_t* frames, const float* dy, float* dw, float* db,
                     float* partial, size_t partial_bytes, cudaStream_t st) {
  if (C >= 1 && C <= 4)
    return launch_wgrad<4, 16, IN_U8>(N, H, W, frames, dy, dw, db, partial, partial_bytes, st, C);
  if (C >= 5 && C <= 8)
    return launch_wgrad<8, 16, IN_U8>(N, H, W, frames, dy, dw, db, partial, partial_bytes, st, C);
  if (C >= 9 && C <= 16)
    return launch_wgrad<16, 16, IN_U8>(N, H, W, frames, dy, dw, db, partial, partial_bytes, st, C);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad_u8: channels must be 1..16");
}

// ---------------------------------------------------------------------------
// MaxPool 3x3 stride 2, TF 'SAME' (asymmetric) padding, dmlab/networks.py:32-33,49.
// pad_before = total/2 where total = max((Ho-1)*2+3-H, 0): (0 before, 1 after) for
// 84->42 and 42->21, (1,1) for 21->11.  Stores the argmax tap (0..8) per element
// so that the backward is a gather.  One thread = 4 channels of one output pixel.
// One CTA per output row (n, ho) [blockIdx.x], threads over (wo, c4) [+ blockIdx.y chunks]:
// no per-thread division, 32-bit indexing (host checks the element counts fit).
__global__ void maxpool3s2_fwd_kernel(int N, int H, int W, int C, int Ho, int Wo, int pt, int pl,
                                      const float* __restrict__ x, float* __restrict__ y,
                                      uint8_t* __restrict__ idx) {
  const int C4 = C >> 2;
  const int row = blockIdx.x;                 // n * Ho + ho
  const int n = row / Ho, ho = row - n * Ho;
  const int j = blockIdx.y * blockDim.x + threadIdx.x;   // wo * C4 + c4
  if (j >= Wo * C4) return;
  const int wo = (C4 & (C4 - 1)) == 0 ? j >> (31 - __clz(C4)) : j / C4, c4 = j - wo * C4;
  float4 best = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
  uchar4 arg = make_uchar4(0, 0, 0, 0);
  const float4* xn = reinterpret_cast<const float4*>(x) + (size_t)n * H * W * C4;
#pragma unroll
  for (int kh = 0; kh < 3; ++kh) {
    const int h = ho * 2 - pt + kh;
    if (h < 0 || h >= H) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int w = wo * 2 - pl + kw;
      if (w < 0 || w >= W) continue;
      const float4 v = __ldg(xn + (h * W + w) * C4 + c4);
      const unsigned char t = (unsigned char)(kh * 3 + kw);
      if (v.x > best.x) { best.x = v.x; arg.x = t; }
      if (v.y > best.y) { best.y = v.y; arg.y = t; }
      if (v.z > best.z) { best.z = v.z; arg.z = t; }
      if (v.w > best.w) { best.w = v.w; arg.w = t; }
    }
  }
  const size_t o = (size_t)row * Wo * C4 + j;
  reinterpret_cast<float4*>(y)[o] = best;
  reinterpret_cast<uchar4*>(idx)[o] = arg;
}

// dx[n,h,w,c] = sum over the <=4 windows containing (h,w) whose argmax is (h,w).
// A thread owns a 2x2 block of input pixels (padded coordinates hp in {2a, 2a+1}, wp in
// {2b, 2b+1}) x 4 channels: the block is covered by exactly the four windows (a-1..a, b-1..b),
// each loaded once (argmax byte + gradient) and scattered to the <= 9 (pixel, tap) pairs it
// owns inside the block -- 2 loads per output instead of up to 8.  One CTA per row pair.
__global__ void maxpool3s2_bwd_kernel(int N, int H, int W, int C, int Ho, int Wo, int pt, int pl,
                                      const float* __restrict__ dy, const uint8_t* __restrict__ idx,
                                      float* __restrict__ dx) {
  const int C4 = C >> 2;
  const int npairs = (H + pt + 1) >> 1;
  const int row = blockIdx.x;                 // n * npairs + a
  const int n = row / npairs, a = row - n * npairs;
  const int j = blockIdx.y * blockDim.x + threadIdx.x;   // b * C4 + c4
  const int nbw = (W + pl + 1) >> 1;
  if (j >= nbw * C4) return;
  const int b = (C4 & (C4 - 1)) == 0 ? j >> (31 - __clz(C4)) : j / C4, c4 = j - b * C4;
  const float4* dyn = reinterpret_cast<const float4*>(dy) + (size_t)n * Ho * Wo * C4;
  const uchar4* idn = reinterpret_cast<const uchar4*>(idx) + (size_t)n * Ho * Wo * C4;
  // acc[r][s]: pixel (hp = 2a + r, wp = 2b + s)
  float4 acc[2][2];
#pragma unroll
  for (int r = 0; r < 2; ++r)
#pragma unroll
    for (int q = 0; q < 2; ++q) acc[r][q] = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int dh = 0; dh < 2; ++dh) {
    const int ho = a - 1 + dh;
    if (ho < 0 || ho >= Ho) continue;
#pragma unroll
    for (int dw = 0; dw < 2; ++dw) {
      const int wo = b - 1 + dw;
      if (wo < 0 || wo >= Wo) continue;
      const int o = (ho * Wo + wo) * C4 + c4;
      const uchar4 t = __ldg(idn + o);
      const float4 g = __ldg(dyn + o);
      // window (ho, wo) covers hp = 2ho..2ho+2: inside the block that is kh = 2 (row 0) for
      // ho = a-1, kh = 0 (row 0) and 1 (row 1) for ho = a; same along w.
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        const int kh = dh == 0 ? (r == 0 ? 2 : -1) : r;
        if (kh < 0) continue;
#pragma unroll
        for (int q = 0; q < 2; ++q) {
          const int kw = dw == 0 ? (q == 0 ? 2 : -1) : q;
          if (kw < 0) continue;
          const unsigned char tap = (unsigned char)(kh * 3 + kw);
          if (t.x == tap) acc[r][q].x += g.x;
          if (t.y == tap) acc[r][q].y += g.y;
          if (t.z == tap) acc[r][q].z += g.z;
          if (t.w == tap) acc[r][q].w += g.w;
        }
      }
    }
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int h = 2 * a + r - pt;
    if (h < 0 || h >= H) continue;
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      const int w = 2 * b + q - pl;
      if (w < 0 || w >= W) continue;
      reinterpret_cast<float4*>(dx)[((size_t)(n * H + h) * W + w) * C4 + c4] = acc[r][q];
    }
  }
}

int maxpool3s2_forward(int N, int H, int W, int C, const float* x, float* y, uint8_t* idx,
                       cudaStream_t st) {
  int Ho, Wo, pt, pl;
  same_pad3s2(H, &Ho, &pt);
  same_pad3s2(W, &Wo, &pl);
  const long long total = (long long)N * Ho * Wo * (C / 4);
  (void)total;
  const int per_row = Wo * (C / 4);
  const int threads = per_row >= 256 ? 256 : ((per_row + 31) / 32) * 32;
  maxpool3s2_fwd_kernel<<<dim3((unsigned)(N * Ho), (unsigned)ceil_div(per_row, threads)), threads, 0, st>>>(
      N, H, W, C, Ho, Wo, pt, pl, x, y, idx);
  count_launch(PC_POOL, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int maxpool3s2_backward(int N, int H, int W, int C, const float* dy, const uint8_t* idx, float* dx,
                        cudaStream_t st) {
  int Ho, Wo, pt, pl;
  same_pad3s2(H, &Ho, &pt);
  same_pad3s2(W, &Wo, &pl);
  const long long total = (long long)N * H * W * (C / 4);
  (void)total;
  const int per_row = ((W + pl + 1) / 2) * (C / 4);
  const int threads = per_row >= 256 ? 256 : ((per_row + 31) / 32) * 32;
  const int npairs = (H + pt + 1) / 2;
  maxpool3s2_bwd_kernel<<<dim3((unsigned)(N * npairs), (unsigned)ceil_div(per_row, threads)), threads, 0, st>>>(
      N, H, W, C, Ho, Wo, pt, pl, dy, idx, dx);
  count_launch(PC_POOL, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

}  // namespace seedrl
