// 'valid' strided convolutions as im2col + GEMM (schedule.h StridedConv): the R2D2 body's 8x8/4, 4x4/2 and
// 3x3/1 layers and the shallow IMPALA net's 8x8/4 and 4x4/2 layers in tensor-core modes.
#include "schedule.h"

namespace seedrl {

// im2col: col[(n*Ho + ho)*Wo + wo][(kh*K + kw)*C + c] = x[n][ho*S + kh][wo*S + kw][c]  (* 1/255 for
// uint8 frames).  Thread = VEC consecutive channels of one col element (VEC = 4 when C % 4 == 0).
template <bool U8, int VEC>
__global__ void __launch_bounds__(256)
im2col_kernel(long long total, int H, int W, int C, int K, int S, int Ho, int Wo, const void* __restrict__ x_,
              float* __restrict__ col) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int CV = C / VEC;
  const int KK = K * K * CV;
  const long long row = i / KK;
  const int e = (int)(i - row * KK);
  const int cv = e % CV, kk = e / CV, kw = kk % K, kh = kk / K;
  const int wo = (int)(row % Wo);
  const long long r2 = row / Wo;
  const int ho = (int)(r2 % Ho);
  const long long n = r2 / Ho;
  const size_t src = (((size_t)n * H + (ho * S + kh)) * W + (wo * S + kw)) * C + (size_t)cv * VEC;
  float* dst = col + (size_t)row * (K * K * C) + (size_t)kk * C + cv * VEC;
  if (VEC == 4) {
    float4 v;
    if (U8) {
      const uchar4 u = __ldg(reinterpret_cast<const uchar4*>(reinterpret_cast<const uint8_t*>(x_) + src));
      const float k = 1.0f / 255.0f;
      v = make_float4(u.x * k, u.y * k, u.z * k, u.w * k);
    } else {
      v = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(x_) + src));
    }
    *reinterpret_cast<float4*>(dst) = v;
  } else {
    if (U8) *dst = (float)__ldg(reinterpret_cast<const uint8_t*>(x_) + src) * (1.0f / 255.0f);
    else *dst = __ldg(reinterpret_cast<const float*>(x_) + src);
  }
}

// col2im (gather form): dx[n][h][w][c] = sum over (kh, kw) with (h - kh) % S == 0, (w - kw) % S == 0,
// ho = (h - kh) / S < Ho, wo < Wo of dcol[(n, ho, wo)][(kh, kw, c)], masked by x > 0 (x = the ReLU'd
// activation this gradient flows into).  Thread = 4 channels of one input pixel.
__global__ void __launch_bounds__(256)
col2im_kernel(long long total, int H, int W, int C, int K, int S, int Ho, int Wo, const float* __restrict__ dcol,
              const float* __restrict__ xmask, float* __restrict__ dx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int C4 = C >> 2;
  const int c4 = (int)(i % C4);
  long long r = i / C4;
  const int w = (int)(r % W); r /= W;
  const int h = (int)(r % H);
  const long long n = r / H;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  const int KC = K * K * C;
  for (int kh = h % S; kh < K; kh += S) {
    const int ho = (h - kh) / S;
    if (h - kh < 0) break;
    if (ho >= Ho) continue;
    for (int kw = w % S; kw < K; kw += S) {
      const int wo = (w - kw) / S;
      if (w - kw < 0) break;
      if (wo >= Wo) continue;
      const float4 d = __ldg(reinterpret_cast<const float4*>(
          dcol + (((size_t)n * Ho + ho) * Wo + wo) * KC + (size_t)(kh * K + kw) * C + c4 * 4));
      acc.x += d.x; acc.y += d.y; acc.z += d.z; acc.w += d.w;
    }
  }
  const float4 m = __ldg(reinterpret_cast<const float4*>(xmask) + i);
  acc.x = m.x > 0.f ? acc.x : 0.f; acc.y = m.y > 0.f ? acc.y : 0.f;
  acc.z = m.z > 0.f ? acc.z : 0.f; acc.w = m.w > 0.f ? acc.w : 0.f;
  reinterpret_cast<float4*>(dx)[i] = acc;
}

// Both the forward shape and the weight-gradient shape must suit gemm_tc.
bool StridedConv::gathered(const GemmExec& ex, int N, bool u8, const void* x, ConvGather* cg) const {
  const int K = k * k * cin, M = N * hout * wout;
  return ex.mode >= 1 && ex.gather && gemm_tc_supported(M, cout, K) && gemm_tc_supported(K, cout, M) &&
         conv_gather_setup(x, u8 ? 1 : 0, N, hin, win, cin, k, s, cg);
}

int StridedConv::im2col(int N, bool u8, const void* x, float* col, cudaStream_t st) const {
  // 4-channel vectors need uchar4 / float4-aligned input and float4-aligned columns
  const uintptr_t xa = reinterpret_cast<uintptr_t>(x), ca = reinterpret_cast<uintptr_t>(col);
  const int vec = (cin % 4 == 0 && (xa & (u8 ? 3 : 15)) == 0 && (ca & 15) == 0) ? 4 : 1;
  const long long total = (long long)N * hout * wout * k * k * (cin / vec);
  const unsigned grid = (unsigned)((total + 255) / 256);
#define SEEDRL_I2C(U8_, V_) \
  im2col_kernel<U8_, V_><<<grid, 256, 0, st>>>(total, hin, win, cin, k, s, hout, wout, x, col)
  if (u8) { if (vec == 4) SEEDRL_I2C(true, 4); else SEEDRL_I2C(true, 1); }
  else    { if (vec == 4) SEEDRL_I2C(false, 4); else SEEDRL_I2C(false, 1); }
#undef SEEDRL_I2C
  count_launch(PC_CONV_FWD, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int StridedConv::forward(const GemmExec& ex, int N, bool u8, const void* x, const float* w, const float* b,
                         float* col, float* y, int ldy) const {
  const int K = k * k * cin, M = N * hout * wout;
  GemmEpi e = epi_none();
  e.bias = b; e.relu = 1;
  ConvGather cg;
  if (gathered(ex, N, u8, x, &cg)) return ex.gemm_gather(false, M, cout, K, cg, w, cout, y, ldy, e);
  SEEDRL_TRY(im2col(N, u8, x, col, ex.st));
  return ex.gemm(false, false, M, cout, K, col, K, w, cout, y, ldy, e);
}

int StridedConv::wgrad(const GemmExec& ex, int N, bool u8, const void* x, const float* col, const float* dy,
                       float* dw, int lddw, float* db) const {
  const int K = k * k * cin, M = N * hout * wout;
  ConvGather cg;
  if (gathered(ex, N, u8, x, &cg))
    SEEDRL_TRY(ex.gemm_gather(true, K, cout, M, cg, dy, cout, dw, lddw, epi_none()));
  else
    SEEDRL_TRY(ex.gemm(true, false, K, cout, M, col, K, dy, cout, dw, lddw, epi_none()));
  return ex.colsum(M, cout, dy, cout, db);
}

int StridedConv::dgrad(const GemmExec& ex, int N, const float* dy, const float* w, float* col, const float* xmask,
                       float* dx) const {
  const int K = k * k * cin, M = N * hout * wout;
  SEEDRL_TRY(ex.gemm(false, true, M, K, cout, dy, cout, w, cout, col, K, epi_none()));
  const long long total = (long long)N * hin * win * (cin / 4);
  col2im_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ex.st>>>(total, hin, win, cin, k, s, hout, wout, col,
                                                                    xmask, dx);
  count_launch(PC_CONV_DGRAD, ex.st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

}  // namespace seedrl

using namespace seedrl;

// One layer through StridedConv, the code the networks run: op 0 forward, 1 weight + bias gradient,
// 2 data gradient (include/seedrl_b200.h).
extern "C" int seedrl_debug_strided_conv(int op, int mode, int gather, int in_u8, int N, int H, int W, int C, int K,
                                         int S, int cout, const void* x, const float* w, const float* bias,
                                         const float* dy, const float* mask, float* out, int ldo, float* dbias,
                                         float* col, size_t col_bytes, float* ws, size_t ws_bytes, int* error_flag,
                                         int* gathered, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(op >= 0 && op <= 2 && mode >= 0 && mode <= 2, "op and mode must be in 0..2");
  SEEDRL_CHECK_ARG(N >= 1 && C >= 1 && K >= 1 && S >= 1 && H >= K && W >= K && cout >= 1, "bad shape");
  SEEDRL_CHECK_ARG(w && out && (op == 2 || ldo >= cout), "null output / weights or ldo < cout");
  const StridedConv c(K, S, C, cout, H, W);
  const long long Ml = (long long)N * c.hout * c.wout;
  SEEDRL_CHECK_ARG(Ml * (K * K * C > cout ? K * K * C : cout) < (1ll << 31), "problem too large");
  const bool col_ok = col && col_bytes >= (size_t)Ml * K * K * C * sizeof(float);
  const GemmExec ex{mode, gather != 0, ws, ws_bytes, error_flag, (cudaStream_t)stream};
  if (gathered) *gathered = 0;
  if (op == 0 || op == 1) {
    SEEDRL_CHECK_ARG(x && (op == 0 || (dy && dbias)), "null pointer");
    ConvGather cg;
    const bool g = c.gathered(ex, N, in_u8 != 0, x, &cg);
    if (gathered) *gathered = g ? 1 : 0;
    SEEDRL_CHECK_ARG(g || col_ok, "column scratch too small");
    if (op == 0) return c.forward(ex, N, in_u8 != 0, x, w, bias, col, out, ldo);
    if (!g) SEEDRL_TRY(c.im2col(N, in_u8 != 0, x, col, ex.st));   // the matrix the network's forward leaves
    return c.wgrad(ex, N, in_u8 != 0, x, col, dy, out, ldo, dbias);
  }
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  SEEDRL_CHECK_ARG(dy && mask && col_ok && C % 4 == 0 && al16(col) && al16(mask) && al16(out),
                   "data gradient: null pointer, column scratch too small, C % 4 != 0 or unaligned buffers");
  return c.dgrad(ex, N, dy, w, col, mask, out);
}
