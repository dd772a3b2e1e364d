// First layer of ImpalaDeep (dmlab/networks.py:31-37: Conv2D(16, 3, 'same') on the uint8 frames,
// then MaxPool 3x3 / 2 'same'), fused: backward here, forward (conv0pool_kernel) at the end of the file.
//
// The gradient that reaches the convolution output is the max-pool's scatter of the pooled gradient
// g: at most one position per (pooled pixel, channel) is non-zero.  Materialising that full-
// resolution tensor (607 MB fp32 at 1 344 frames) and running a dense weight-gradient convolution over
// it costs a full-resolution write, two full-resolution reads and the dense MACs.  Here each
// (pooled pixel q, channel co) adds  g[q][co] * x[argmax(q, co) + tap]  to dW[tap][:][co] directly:
//     dW[kh][kw][ci][co] = sum_{n,q} g[n,q,co] * x[n][p(q,co) + (kh-1, kw-1)][ci] / 255,
//     db[co]            = sum_{n,q} g[n,q,co],
// p(q, co) = the window position stored by the forward pool (idx).  4x fewer MACs than the dense
// form, no full-resolution gradient, fp32 accumulation (exact products: frames are integers).
// A CTA stages one frame at a time in shared memory as bf16 (exact for 0..255) with a zero border, CP
// channels per pixel (the frame's C channels zero-filled to CP = 4, 8 or 16);
// thread = (channel co, 4-channel group, pooled-pixel lane): 9 x 8-byte patch loads + 36 FMAs per
// (q, co) into 36 register accumulators; per-CTA partials, in the parameter's own [3][3][C][16] order,
// go through the deterministic deferred reduce.
#include <cuda.h>

#include <cstring>

#include "kernels.h"
#include "tc_common.cuh"

namespace seedrl {

constexpr int kFwThreads = 256;
constexpr int kFwCo = 16;
constexpr int kFwLanes = kFwThreads / kFwCo;   // (4-channel group, pooled-pixel lane) slots per channel

// channels per staged pixel: the frame's C rounded up to 4, 8 or 16
static inline int first_layer_cp(int c) { return c <= 4 ? 4 : (c <= 8 ? 8 : 16); }
// pooled rows per work unit of the weight gradient (16 channels: fewer, to keep 3 CTAs / SM)
static inline int fw_rows_per_band(int cp) { return cp == 16 ? 4 : 6; }
// staged pixels: [2*rb+3][W+2][cp/4] x 8 B, rounded up to 16 B (the fp32 gradient stage behind them
// is read and written as float4)
static inline size_t fw_pixels_8b(int cp, int rb, int W) { return ((size_t)(2 * rb + 3) * (W + 2) * (cp / 4) + 1) & ~(size_t)1; }
static inline size_t fw_smem(int cp, int rb, int W) {
  const int wo = (W + 1) / 2;
  return fw_pixels_8b(cp, rb, W) * 8 + (size_t)rb * wo * kFwCo * 5;
}

struct FirstWgradArgs {
  int N, H, W, C, Ho, Wo, pt, pl;
  int Lpp, PWp, RHp;             // pooled plane-tensor geometry
  int rb;                        // pooled rows per work unit
  const uint8_t* frames;         // [N,H,W,C]
  const uint4* g;                // pooled gradient planes: 2 hi planes then 2 lo planes, [Lpp] x 16 B
  const uint8_t* idx;            // [N,Ho,Wo,16] window tap kh*3+kw of the forward arg-max
  float* partial;                // [grid][9*C*16 + 16]
};

// 4 bytes (channels c0 .. c0+3 of a pixel, zero at and above C) -> one little-endian word
__device__ __forceinline__ uint32_t load_u8x4(const uint8_t* px, int c0, int C) {
  uint32_t v = 0u;
#pragma unroll
  for (int j = 0; j < 4; ++j)
    if (c0 + j < C) v |= (uint32_t)__ldg(px + c0 + j) << (8 * j);
  return v;
}

// kU32: 4-channel frames, one 32-bit load per pixel, 3 CTAs / SM; otherwise C <= CP channels, byte
// loads, 2 CTAs / SM (the loader's extra registers would spill under the 3-CTA bound)
template <int CP, bool kU32>
__global__ void __launch_bounds__(kFwThreads, kU32 ? 3 : 2) first_wgrad_pooled_kernel(const FirstWgradArgs a) {
  constexpr int G = CP / 4;                                      // 4-channel groups per pixel
  constexpr int NL = kFwLanes / G;                               // pooled-pixel lanes
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x;
  const int co = tid & (kFwCo - 1), grp = (tid >> 4) & (G - 1), ql = (tid >> 4) / G;
  const int SW = a.W + 2;
  const int RB = a.rb;                                           // pooled rows per band
  const int SR = 2 * RB + 3;                                     // staged frame rows (incl. the two border rows)
  uint2* s_x = reinterpret_cast<uint2*>(smem_raw);               // [SR][SW][G] pixels x CP bf16
  float* s_g = reinterpret_cast<float*>(s_x + ((SR * SW * G + 1) & ~1));   // [RB*Wo][16] pooled gradient (hi + lo), 16-B aligned
  uint8_t* s_t = reinterpret_cast<uint8_t*>(s_g + RB * a.Wo * kFwCo);   // [RB*Wo][16] arg-max taps
  float acc[36];
#pragma unroll
  for (int i = 0; i < 36; ++i) acc[i] = 0.f;
  float accb = 0.f;
  const int bands = (a.Ho + RB - 1) / RB;
  const int units = a.N * bands;
  // work unit = (frame, band of pooled rows): keeps the static schedule balanced and the staged
  // working set small enough for 3+ CTAs per SM
  for (int u = blockIdx.x; u < units; u += gridDim.x) {
    const int n = u / bands, band = u - n * bands;
    const int r0 = band * RB, r1 = min(a.Ho, r0 + RB);
    const int nq = (r1 - r0) * a.Wo;
    // ---- stage: frame rows f0 .. f0+SR-1 (zero outside the frame / at the two border columns) ----
    const int f0 = 2 * r0 - a.pt - 1;
    for (int i = tid; i < SR * SW * G; i += kFwThreads) {
      const int px = i / G, gi = i - px * G;
      const int lr = px / SW, bc = px - lr * SW, fr = f0 + lr;
      uint32_t w32 = 0u;
      if (fr >= 0 && fr < a.H && bc >= 1 && bc <= a.W) {
        const size_t pix = ((size_t)n * a.H + fr) * a.W + bc - 1;
        if (kU32) w32 = __ldg(reinterpret_cast<const uint32_t*>(a.frames) + pix);
        else w32 = load_u8x4(a.frames + pix * a.C, 4 * gi, a.C);
      }
      // bf16 x 4 (exact for 0..255): the consumer turns them back into floats with one shift / mask each
      const uint32_t f0_ = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7540)) - 8388608.0f);
      const uint32_t f1_ = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7541)) - 8388608.0f);
      const uint32_t f2_ = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7542)) - 8388608.0f);
      const uint32_t f3_ = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7543)) - 8388608.0f);
      s_x[i] = make_uint2(__byte_perm(f0_, f1_, 0x7632), __byte_perm(f2_, f3_, 0x7632));
    }
    // ---- stage: the band's pooled gradient (hi + lo planes -> fp32) and arg-max taps: coalesced
    //      16-byte loads, all independent (the main loop then touches shared memory only) ----
    for (int i = tid; i < nq * 2; i += kFwThreads) {
      const int gq = i & 1, qq = i >> 1;
      const int qr = qq / a.Wo, qw = qq - qr * a.Wo;
      const size_t sp = (size_t)(n * a.RHp + r0 + qr + 1) * a.PWp + qw + 1;
      const uint4 hh = __ldg(a.g + (size_t)gq * a.Lpp + sp), ll = __ldg(a.g + (size_t)(2 + gq) * a.Lpp + sp);
      float4* dst = reinterpret_cast<float4*>(s_g + (size_t)qq * kFwCo + gq * 8);
      dst[0] = make_float4(__uint_as_float(hh.x << 16) + __uint_as_float(ll.x << 16),
                           __uint_as_float(hh.x & 0xFFFF0000u) + __uint_as_float(ll.x & 0xFFFF0000u),
                           __uint_as_float(hh.y << 16) + __uint_as_float(ll.y << 16),
                           __uint_as_float(hh.y & 0xFFFF0000u) + __uint_as_float(ll.y & 0xFFFF0000u));
      dst[1] = make_float4(__uint_as_float(hh.z << 16) + __uint_as_float(ll.z << 16),
                           __uint_as_float(hh.z & 0xFFFF0000u) + __uint_as_float(ll.z & 0xFFFF0000u),
                           __uint_as_float(hh.w << 16) + __uint_as_float(ll.w << 16),
                           __uint_as_float(hh.w & 0xFFFF0000u) + __uint_as_float(ll.w & 0xFFFF0000u));
    }
    {
      const uint4* isrc = reinterpret_cast<const uint4*>(a.idx + ((size_t)n * a.Ho + r0) * a.Wo * kFwCo);
      for (int i = tid; i < nq; i += kFwThreads) reinterpret_cast<uint4*>(s_t)[i] = __ldg(isrc + i);
    }
    __syncthreads();
    // ---- thread = (channel co, channel group, pooled-pixel lane): 9 x 8-byte patch loads + 36 FMAs
    //      per pixel ----
    int qh = ql / a.Wo, qw = ql - qh * a.Wo;                    // band-local pooled row / column
    for (int q = ql; q < nq; q += NL) {
      const int t = s_t[q * kFwCo + co];
      const float gv = s_g[q * kFwCo + co];
      const int kh = t / 3, kw = t - kh * 3;
      // arg-max position (frame row 2*(r0+qh) - pt + kh); its 3x3 patch starts one row / column
      // earlier = staged row 2*qh + kh, band column 2*qw - pl + kw
      const uint2* patch = s_x + ((2 * qh + kh) * SW + (2 * qw - a.pl + kw)) * G + grp;
      accb += gv;
#pragma unroll
      for (int dh = 0; dh < 3; ++dh) {             // one patch row at a time: fewer live registers
        uint2 v[3];
#pragma unroll
        for (int dw = 0; dw < 3; ++dw) v[dw] = patch[(dh * SW + dw) * G];
#pragma unroll
        for (int dw = 0; dw < 3; ++dw) {
          float* c = acc + (dh * 3 + dw) * 4;
          c[0] = fmaf(gv, __uint_as_float(v[dw].x << 16), c[0]);
          c[1] = fmaf(gv, __uint_as_float(v[dw].x & 0xFFFF0000u), c[1]);
          c[2] = fmaf(gv, __uint_as_float(v[dw].y << 16), c[2]);
          c[3] = fmaf(gv, __uint_as_float(v[dw].y & 0xFFFF0000u), c[3]);
        }
      }
      qw += NL;
      while (qw >= a.Wo) { qw -= a.Wo; ++qh; }
    }
    __syncthreads();                       // the staged band is rewritten by the next unit
  }
  // ---- reduce the pooled-pixel lanes per (channel group, co) (fixed order) -> this CTA's partial ----
  float* s_red = reinterpret_cast<float*>(smem_raw);              // [NL ql][G][37][16 co] (staging buffers are free)
  const int slot = ql * G + grp;
#pragma unroll
  for (int i = 0; i < 36; ++i) s_red[(slot * 37 + i) * kFwCo + co] = acc[i];
  s_red[(slot * 37 + 36) * kFwCo + co] = accb;
  __syncthreads();
  const int nw = 9 * a.C;                                         // (tap, ci) rows of the real HWIO kernel
  float* dst = a.partial + (size_t)blockIdx.x * ((nw + 1) * kFwCo);
  for (int e = tid; e < (nw + 1) * kFwCo; e += kFwThreads) {
    const int i = e / kFwCo, c = e - i * kFwCo;
    const int tap = i / a.C, ci = i - tap * a.C;
    // (channel group, accumulator) of row i; the bias row sums group 0's copies
    const int gi = i < nw ? ci >> 2 : 0, k = i < nw ? tap * 4 + (ci & 3) : 36;
    float s = 0.f;
#pragma unroll
    for (int l = 0; l < NL; ++l) s += s_red[((l * G + gi) * 37 + k) * kFwCo + c];
    if (i < nw) dst[i * kFwCo + c] = s * (1.0f / 255.0f);        // (tap, ci) x co: HWIO order
    else dst[nw * kFwCo + c] = s;
  }
}

bool first_wgrad_pooled_supported(int cin, int cout, int H, int W) {
  if (cin < 1 || cin > 16 || cout != 16 || H < 3 || W < 3) return false;
  const int cp = first_layer_cp(cin);
  return fw_smem(cp, fw_rows_per_band(cp), W) <= 70 * 1024;
}

template <int CP, bool kU32>
static int launch_first_wgrad(const FirstWgradArgs& a, int grid, size_t smem, cudaStream_t st) {
  SEEDRL_CUDA(allow_smem<first_wgrad_pooled_kernel<CP, kU32>>(72 * 1024));
  first_wgrad_pooled_kernel<CP, kU32><<<grid, kFwThreads, smem, st>>>(a);
  return SEEDRL_OK;
}

// dW / db of the first convolution from the POOLED gradient planes + the pool's arg-max taps.
// frames: [N,H,W,C] uint8; dw: [3,3,C,16].
int first_wgrad_pooled(int N, int H, int W, int C, const uint8_t* frames, const void* g_planes, const uint8_t* idx,
                       float* dw, float* db, WgradBatch* batch, cudaStream_t st) {
  if (!first_wgrad_pooled_supported(C, 16, H, W))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "first_wgrad_pooled: unsupported frame shape");
  int Ho, Wo, pt, pl;
  same_pad3s2(H, &Ho, &pt);
  same_pad3s2(W, &Wo, &pl);
  const int cp = first_layer_cp(C);
  FirstWgradArgs a;
  a.N = N; a.H = H; a.W = W; a.C = C; a.Ho = Ho; a.Wo = Wo; a.pt = pt; a.pl = pl;
  a.Lpp = (int)planes_positions(N, Ho, Wo); a.PWp = Wo + 2; a.RHp = Ho + 1;
  a.frames = frames; a.g = reinterpret_cast<const uint4*>(g_planes); a.idx = idx;
  a.rb = fw_rows_per_band(cp) < Ho ? fw_rows_per_band(cp) : Ho;
  size_t smem = fw_smem(cp, a.rb, W);
  const size_t red = (size_t)kFwLanes * 37 * kFwCo * 4;
  if (red > smem) smem = red;
  smem = (smem + 127) / 128 * 128;
  const int NW = 9 * C * kFwCo + kFwCo;
  const int units = N * ((Ho + a.rb - 1) / a.rb);
  int grid = (C == 4 ? 3 : 2) * kNumSMs;
  if (grid > units) grid = units;
  if (!batch || batch->n >= kMaxReduceJobs || batch->used + (size_t)grid * NW > batch->cap_floats)
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "first_wgrad_pooled: partial buffer too small");
  a.partial = batch->buf + batch->used;
  batch->used += (size_t)grid * NW;
  const int rc = C == 4    ? launch_first_wgrad<4, true>(a, grid, smem, st)
                 : cp == 4 ? launch_first_wgrad<4, false>(a, grid, smem, st)
                 : cp == 8 ? launch_first_wgrad<8, false>(a, grid, smem, st)
                           : launch_first_wgrad<16, false>(a, grid, smem, st);
  if (rc != SEEDRL_OK) return rc;
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  batch->jobs[batch->n++] = ReduceJob{a.partial, dw, db, grid, 9 * C * kFwCo, kFwCo};
  return SEEDRL_OK;
}

// =================================================================================================
// First layer, forward, fused: Conv2D(16, 3, 'same') on the uint8 frames + bias + MaxPool 3x3/2
// 'same' (dmlab/networks.py:31-37,47-48) -> the pooled activation as plane tensors (raw and ReLU'd)
// + the arg-max taps.  The full-resolution conv output (607 MB fp32 at 1 344 frames, which a separate
// pool kernel would write once and read once) never leaves the SM.
//
// Work unit = (frame, band of kCpRows pooled rows).  Per unit:
//   1. the band's frame rows -> shared memory as a PAIR array: entry e = [pixel e, pixel e+1] of the
//      zero-bordered band (row pitch SW = W + 2), 4 channels each, bf16 (exact for 0..255) = 16 bytes.
//      That array IS a K-major wgmma operand whose row p reads, for kernel row kh, the 16 bytes at
//      e = p + kh*SW (taps kw = 0, 1) and at e + 2 (taps kw = 2 and a 4th, zero-weight, tap): the two
//      K-groups of one K = 16 instruction are the same array 32 bytes apart (LBO = 32 B).  A whole
//      kernel row per MMA: 3 MMAs of 64 x 32 x 16 per 64 positions, no im2col pass.
//   2. warpgroup wg issues them for position blocks wg, wg + 2, ...: D[64, 0:16] = A hi(W),
//      D[64, 16:32] = A lo(W) (frames are exact in bf16, so two products make the fp32-faithful result);
//   3. epilogue: accumulator registers -> (hi + lo) / 255 + bias -> fp32 tile in shared memory;
//   4. pooling from shared memory, TF-SAME windows, first maximum wins; hi/lo split; coalesced
//      16-byte plane stores; padding positions of the plane tensors written as zeros.
// 2 CTAs / SM: the phases of one CTA overlap the other's.
//
// Frames of C != 4 channels (C in 1..16) are zero-filled to CP = 4, 8 or 16 channels on the way into
// shared memory (the weights' padding rows of B are zero; no padded copy exists in HBM):
//   CP = 4  (C = 1..3): the pair array above;
//   CP = 8  (C = 5..8): entry e = ONE pixel (8 channels = one 16-byte K-group); a kernel row takes two
//           K = 16 MMAs: taps 0-1 (LBO = 16 B), then tap 2 and a zero-weight group;
//   CP = 16 (C = 9..16): two such arrays (channels 0-7, 8-15; LBO = the array stride), one MMA per tap.
// Such frames are read with plain loads straight from HBM (their W*C-byte row pitch rarely meets the
// TMA's 16-byte rule, and a W*C-byte box row exceeds its 256-element limit).
constexpr int kCpThreadsF = 256;
constexpr int kCpRows = 3;          // pooled rows per unit: 7 conv rows ...
constexpr int kCpMaxBlocks = 6;     // ... in at most 6 blocks of 128 positions
constexpr int kCpOutStride = 20;    // floats per position in the fp32 tile (16 + 4: pool reads 2-way conflict)

struct Conv0PoolArgs {
  int N, H, W, Ho, Wo, pt, pl;
  int Lpp, PWp, RHp;                 // pooled plane-tensor geometry
  int C;                             // channels per frame pixel
  unsigned int sw_mul; int sw_sh;    // division by SW = W + 2
  const uint8_t* frames;             // [N,H,W,C]
  const float* w;                    // [3,3,C,16]
  const float* bias;                 // [16]
  uint4* praw; uint4* prelu;         // plane tensors, 16 channels (2 hi planes, 2 lo planes)
  uint8_t* idx;                      // [N,Ho,Wo,16]
  int* err;
};

__device__ __forceinline__ uint2 u8x4_to_bf16x4(uint32_t w32) {
  // byte -> float without I2F: 0x4B0000kk is 2^23 + kk; the high half of the float is its bf16
  const uint32_t f0 = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7540)) - 8388608.0f);
  const uint32_t f1 = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7541)) - 8388608.0f);
  const uint32_t f2 = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7542)) - 8388608.0f);
  const uint32_t f3 = __float_as_uint(__uint_as_float(__byte_perm(w32, 0x4B000000u, 0x7543)) - 8388608.0f);
  return make_uint2(__byte_perm(f0, f1, 0x7632), __byte_perm(f2, f3, 0x7632));
}

// The observation tile of a unit -- frame rows cr0-1 .. cr0+7 of frame n, all W pixels x 4 channels --
// arrives by ONE TMA tensor copy (cp.async.bulk.tensor.3d over the [N][H][W] uint32 view of the
// frames; rows above / below the frame are zero-filled by the TMA unit: the 'same' padding costs
// nothing) into one of two raw stages; the copy of the NEXT unit's tile is in flight while this
// unit converts, multiplies and pools.
// CP = 4 with kTma: 4-channel frames (the tile copy above); otherwise plain loads, C <= CP channels.
template <int CP, bool kTma>
__global__ void __launch_bounds__(kCpThreadsF, 2) conv0pool_kernel(const __grid_constant__ CUtensorMap tm_frames,
                                                                    const Conv0PoolArgs a) {
  static_assert(CP == 4 || !kTma, "the tile copy reads 4-channel pixels");
  constexpr int kPlanes = CP == 16 ? 2 : 1;                   // 16-byte arrays of the A operand
  constexpr int KH = CP == 16 ? 48 : 4 * CP;                  // B rows (K) per kernel row
  constexpr int KT = 3 * KH;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const int W = a.W, H = a.H, SW = W + 2;
  const int npair = kCpMaxBlocks * 128 + 2 * SW + 8;          // pair entries an MMA may touch
  uint4* s_p = reinterpret_cast<uint4*>(smem_raw);            // pair array (or [kPlanes][npair] pixels), 16 B per entry
  float* s_out = reinterpret_cast<float*>(smem_raw + (size_t)kPlanes * npair * 16);  // [positions][20] fp32
  uint8_t* s_bq = reinterpret_cast<uint8_t*>(s_out + (size_t)kCpMaxBlocks * 128 * kCpOutStride);
  s_bq = reinterpret_cast<uint8_t*>(((uintptr_t)s_bq + 127) & ~(uintptr_t)127);     // B: KT x 32 bf16 (3 KB at CP = 4)
  float* s_bias = reinterpret_cast<float*>(s_bq + KT * 32 * 2);
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_bias + 16);   // [2] TMA stage filled
  constexpr int kRawRows = 2 * kCpRows + 3;                   // frame rows per tile (incl. the halo rows)
  uint32_t* s_raw = reinterpret_cast<uint32_t*>(((uintptr_t)(s_full + 4) + 127) & ~(uintptr_t)127);   // [2][kRawRows][W]
  const uint32_t raw_bytes = (uint32_t)(kRawRows * W) * 4u;
  const uint32_t raw_stride = (raw_bytes + 127u) & ~127u;     // stage pitch (TMA destinations are 128-byte aligned)

  // ---- one-time setup: B operand (K-major, [N = 32][K = KT]: hi(w) | lo(w); k = kh*KH + kw*CP + ci,
  //      the 4th tap of a row (CP < 16) and channels ci >= C have zero weights), bias, barriers ------
  for (int i = tid; i < KT * 32; i += kCpThreadsF) {
    const int k = i / 32, nn = i - k * 32;
    const int kh = k / KH, kw = (k - kh * KH) / CP, ci = k - kh * KH - kw * CP;
    float v = 0.f;
    if (kw < 3 && ci < a.C) {
      const float wv = __ldg(a.w + ((kh * 3 + kw) * a.C + ci) * 16 + (nn & 15));
      v = nn < 16 ? wv : bf16_resid(wv);
    }
    const uint32_t off = (uint32_t)(k >> 3) * 512u + (uint32_t)(nn >> 3) * 128u + (uint32_t)(nn & 7) * 16u +
                         (uint32_t)(k & 7) * 2u;
    *reinterpret_cast<__nv_bfloat16*>(s_bq + off) = __float2bfloat16_rn(v);
  }
  if (tid < 16) s_bias[tid] = __ldg(a.bias + tid);
  for (int i = tid; i < kPlanes * npair; i += kCpThreadsF) s_p[i] = make_uint4(0u, 0u, 0u, 0u);
  if (kTma && tid == 0) {
    mbar_init(s_full, 1);
    mbar_init(s_full + 1, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_frames)) : "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  __syncthreads();
  const uint32_t a_base = smem_u32(s_p), b_base = smem_u32(s_bq);

  const int bands = (a.Ho + kCpRows - 1) / kCpRows;
  const int units = a.N * bands;
  bool timed_out = false;
  auto unit_geom = [&](int u, int* n, int* r0, int* r1, int* cr0, int* cr1) {
    *n = u / bands;
    const int band = u - *n * bands;
    *r0 = band * kCpRows; *r1 = min(a.Ho, *r0 + kCpRows);
    *cr0 = max(0, 2 * *r0 - a.pt); *cr1 = min(H - 1, 2 * (*r1 - 1) - a.pt + 2);
  };
  // one thread issues the tile copy of unit u into stage st: box = W pixels x kRawRows rows x 1 frame
  // starting one row above the band's first conv row (negative / >= H rows come back as zeros)
  auto issue_tile = [&](int u, int st) {
    int n, r0, r1, cr0, cr1;
    unit_geom(u, &n, &r0, &r1, &cr0, &cr1);
    const uint32_t dst = smem_u32(s_raw) + (uint32_t)st * raw_stride, bar = smem_u32(s_full + st);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(raw_bytes) : "memory");
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::
            "r"(dst), "l"(reinterpret_cast<uint64_t>(&tm_frames)), "r"(0), "r"(cr0 - 1), "r"(n), "r"(bar)
        : "memory");
  };
  if (kTma && tid == 0 && (int)blockIdx.x < units) issue_tile(blockIdx.x, 0);
  int it = 0;
  for (int u = blockIdx.x; u < units; u += gridDim.x, ++it) {
    int n, r0, r1, cr0, cr1;
    unit_geom(u, &n, &r0, &r1, &cr0, &cr1);
    const int band = u - n * bands;
    const int CR = cr1 - cr0 + 1, npos = CR * SW, nblk = (npos + 127) >> 7;
    const int st = it & 1;
    if constexpr (kTma) {
      // the next unit's tile goes into the other stage (its previous contents were converted one unit ago)
      if (tid == 0 && u + (int)gridDim.x < units) issue_tile(u + gridDim.x, st ^ 1);
      if (!mbar_wait_bounded(s_full + st, (uint32_t)((it >> 1) & 1))) timed_out = true;
      // ---- 1. raw tile (row lr = frame row cr0-1+lr, W pixels) -> pair array: entry (lr, bc) =
      //      [pixel bc-1, pixel bc] of that row as bf16 x 4 each, zero at the two border columns ----
      const uint32_t* raw = s_raw + (size_t)st * (raw_stride / 4);
      for (int e = tid; e < (CR + 2) * SW; e += kCpThreadsF) {
        const int lr = (int)(__umulhi((unsigned)e, a.sw_mul) >> a.sw_sh), bc = e - lr * SW;
        const uint32_t w0 = (bc >= 1 && bc <= W) ? raw[lr * W + bc - 1] : 0u;
        const uint32_t w1 = (bc + 1 <= W) ? raw[lr * W + bc] : 0u;
        const uint2 p0 = u8x4_to_bf16x4(w0), p1 = u8x4_to_bf16x4(w1);
        s_p[e] = make_uint4(p0.x, p0.y, p1.x, p1.y);
      }
    } else {
      // ---- 1. frame rows cr0-1 .. cr0+CR straight from HBM (zero outside the frame and at the two
      //      border columns), C channels zero-filled to CP: the pair array (CP = 4) or pixel arrays ----
      const uint8_t* fb = a.frames + (size_t)n * H * W * a.C;
      for (int e = tid; e < (CR + 2) * SW; e += kCpThreadsF) {
        const int lr = (int)(__umulhi((unsigned)e, a.sw_mul) >> a.sw_sh), bc = e - lr * SW;
        const int fr = cr0 - 1 + lr;
        const bool in_row = fr >= 0 && fr < H;
        const uint8_t* row = fb + (size_t)(in_row ? fr : 0) * W * a.C;
        if constexpr (CP == 4) {
          const uint32_t w0 = (in_row && bc >= 1 && bc <= W) ? load_u8x4(row + (size_t)(bc - 1) * a.C, 0, a.C) : 0u;
          const uint32_t w1 = (in_row && bc + 1 <= W) ? load_u8x4(row + (size_t)bc * a.C, 0, a.C) : 0u;
          const uint2 p0 = u8x4_to_bf16x4(w0), p1 = u8x4_to_bf16x4(w1);
          s_p[e] = make_uint4(p0.x, p0.y, p1.x, p1.y);
        } else {
          const bool in = in_row && bc >= 1 && bc <= W;
          const uint8_t* px = row + (size_t)(bc - 1) * a.C;
#pragma unroll
          for (int g = 0; g < kPlanes; ++g) {
            const uint2 p0 = u8x4_to_bf16x4(in ? load_u8x4(px, 8 * g, a.C) : 0u);
            const uint2 p1 = u8x4_to_bf16x4(in ? load_u8x4(px, 8 * g + 4, a.C) : 0u);
            s_p[(size_t)g * npair + e] = make_uint4(p0.x, p0.y, p1.x, p1.y);
          }
        }
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    // ---- 2. MMAs: one per kernel row and 64-position block; 3. epilogue: accumulators -> fp32 tile
    //      [position o = lr*SW + c][16 (+4 pad)] -------------------------------------------------------
    for (int m = wg; m < 2 * nblk; m += kCpThreadsF / 128) {
      float acc[16];
#pragma unroll
      for (int i = 0; i < 16; ++i) acc[i] = 0.f;
      wgmma_fence_acc<16>(acc);
      wgmma_fence();
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        if constexpr (CP == 4) {
          const uint64_t da = gmma_desc(a_base + (uint32_t)(m * 64 + kh * SW) * 16u, 32u, 128u);
          const uint64_t db = gmma_desc(b_base + (uint32_t)(2 * kh) * 512u, 512u, 128u);
          Wgmma<32>::mma<0, 0>(acc, da, db, 1u);
        } else if constexpr (CP == 8) {
          // taps (0, 1), then (2, zero-weight 3): K-groups are adjacent pixels, 16 B apart
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const uint64_t da = gmma_desc(a_base + (uint32_t)(m * 64 + kh * SW + 2 * j) * 16u, 16u, 128u);
            const uint64_t db = gmma_desc(b_base + (uint32_t)(4 * kh + 2 * j) * 512u, 512u, 128u);
            Wgmma<32>::mma<0, 0>(acc, da, db, 1u);
          }
        } else {
          // one tap per MMA: K-group 0 = channels 0-7 (array 0), K-group 1 = channels 8-15 (array 1)
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const uint64_t da = gmma_desc(a_base + (uint32_t)(m * 64 + kh * SW + kw) * 16u, (uint32_t)npair * 16u, 128u);
            const uint64_t db = gmma_desc(b_base + (uint32_t)(6 * kh + 2 * kw) * 512u, 512u, 128u);
            Wgmma<32>::mma<0, 0>(acc, da, db, 1u);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc<16>(acc);
      // a thread holds channels c, c+1 of two positions; columns 16.. are the lo(W) products
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int o = m * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h;
        if (o < npos) {
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            *reinterpret_cast<float2*>(s_out + (size_t)o * kCpOutStride + c) =
                make_float2(fmaf(acc[4 * j + 2 * h] + acc[4 * (j + 2) + 2 * h], 1.0f / 255.0f, s_bias[c]),
                            fmaf(acc[4 * j + 2 * h + 1] + acc[4 * (j + 2) + 2 * h + 1], 1.0f / 255.0f, s_bias[c + 1]));
          }
        }
      }
    }
    __syncthreads();
    // ---- 4. max-pool 3x3 / 2 from the tile; thread = (pooled pixel, 8-channel group) ----------------
    const int nout = (r1 - r0) * a.Wo * 2;
    for (int i = tid; i < nout; i += kCpThreadsF) {
      const int gq = i & 1, qq = i >> 1;
      const int qr = qq / a.Wo, qw = qq - qr * a.Wo, qh = r0 + qr;
      float best[8];
      unsigned char arg[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) { best[e] = -INFINITY; arg[e] = 0; }
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int h = qh * 2 - a.pt + kh;
        if (h < 0 || h >= H) continue;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int w = qw * 2 - a.pl + kw;
          if (w < 0 || w >= W) continue;
          const float4* s4 = reinterpret_cast<const float4*>(s_out + (size_t)((h - cr0) * SW + w) * kCpOutStride + gq * 8);
          const float4 x0 = s4[0], x1 = s4[1];
          const float vv[8] = {x0.x, x0.y, x0.z, x0.w, x1.x, x1.y, x1.z, x1.w};
          const unsigned char t = (unsigned char)(kh * 3 + kw);
#pragma unroll
          for (int e = 0; e < 8; ++e)
            if (vv[e] > best[e]) { best[e] = vv[e]; arg[e] = t; }
        }
      }
      const size_t pix = ((size_t)n * a.Ho + qh) * a.Wo + qw;
      uint2 packed;
      packed.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | ((uint32_t)arg[3] << 24);
      packed.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | ((uint32_t)arg[7] << 24);
      *reinterpret_cast<uint2*>(a.idx + pix * 16 + gq * 8) = packed;
      const size_t sp = (size_t)(n * a.RHp + qh + 1) * a.PWp + qw + 1;
      const float4 va = make_float4(best[0], best[1], best[2], best[3]), vb = make_float4(best[4], best[5], best[6], best[7]);
      a.praw[(size_t)gq * a.Lpp + sp] = pack8_bf16(va, vb);
      a.praw[(size_t)(2 + gq) * a.Lpp + sp] = pack8_bf16(bf16_resid4(va), bf16_resid4(vb));
      const float4 ra = make_float4(fmaxf(va.x, 0.f), fmaxf(va.y, 0.f), fmaxf(va.z, 0.f), fmaxf(va.w, 0.f));
      const float4 rb = make_float4(fmaxf(vb.x, 0.f), fmaxf(vb.y, 0.f), fmaxf(vb.z, 0.f), fmaxf(vb.w, 0.f));
      a.prelu[(size_t)gq * a.Lpp + sp] = pack8_bf16(ra, rb);
      a.prelu[(size_t)(2 + gq) * a.Lpp + sp] = pack8_bf16(bf16_resid4(ra), bf16_resid4(rb));
    }
    // ---- padding positions of the plane tensors owned by this unit: zeros -------------------------
    {
      // per pooled row: columns 0 and Wo+1; band 0 also the separator row above the image; the last
      // unit also the tail [N*RHp*PWp, Lpp)
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      const int rows = r1 - r0;
      for (int i = tid; i < rows * 2 * 4; i += kCpThreadsF) {
        const int pl_ = i & 3, side = (i >> 2) & 1, rr = i >> 3;
        const size_t sp = (size_t)(n * a.RHp + r0 + rr + 1) * a.PWp + (side ? a.Wo + 1 : 0);
        a.praw[(size_t)pl_ * a.Lpp + sp] = z;
        a.prelu[(size_t)pl_ * a.Lpp + sp] = z;
      }
      if (band == 0) {
        for (int i = tid; i < a.PWp * 4; i += kCpThreadsF) {
          const int pl_ = i & 3, cc = i >> 2;
          const size_t sp = (size_t)(n * a.RHp) * a.PWp + cc;
          a.praw[(size_t)pl_ * a.Lpp + sp] = z;
          a.prelu[(size_t)pl_ * a.Lpp + sp] = z;
        }
      }
      if (u == units - 1) {
        const int t0 = a.N * a.RHp * a.PWp;
        for (int i = tid; i < (a.Lpp - t0) * 4; i += kCpThreadsF) {
          const int pl_ = i & 3, cc = i >> 2;
          a.praw[(size_t)pl_ * a.Lpp + t0 + cc] = z;
          a.prelu[(size_t)pl_ * a.Lpp + t0 + cc] = z;
        }
      }
    }
    __syncthreads();      // s_out and the pair array are rewritten by the next unit
  }
  if (timed_out && a.err) atomicExch(a.err, 1);
}

bool conv0pool_supported(int cin, int cout, int H, int W) {
  // 7 conv rows of the widest band in 6 blocks of 128 positions: W <= 107
  if (cout != 16 || H < 3 || W < 3 || 7 * (W + 2) > 6 * 128) return false;
  // 4 channels: the tile copy's row pitch W*4 bytes must be a multiple of 16
  if (cin == 4) return W % 4 == 0 && W <= 256;
  return cin >= 1 && cin <= 16;
}

template <int CP, bool TMA>
static int launch_conv0pool(Conv0PoolArgs a, const uint8_t* frames, cudaStream_t st) {
  constexpr int KT = 3 * (CP == 16 ? 48 : 4 * CP);
  const int N = a.N, H = a.H, W = a.W;
  const size_t raw_stride = TMA ? (((size_t)(2 * kCpRows + 3) * W * 4) + 127) / 128 * 128 : 0;
  const size_t smem = (size_t)(CP == 16 ? 2 : 1) * (kCpMaxBlocks * 128 + 2 * (W + 2) + 8) * 16 +
                      (size_t)kCpMaxBlocks * 128 * kCpOutStride * 4 + 128 + KT * 32 * 2 + 16 * 4 + 64 + 128 +
                      2 * raw_stride;
  SEEDRL_CUDA(allow_smem<conv0pool_kernel<CP, TMA>>(112 * 1024));
  if (smem > 112 * 1024) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv0pool: image too wide");
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));                    // plain-load variants never read it
  if (TMA) {
    // [N][H][W] view of the frames with one uint32 (= 4 uint8 channels) per pixel
    const EncodeTiledFn enc = encode_tiled_fn();
    if (!enc) return set_error(SEEDRL_ERR_INTERNAL, "cuTensorMapEncodeTiled is not available");
    const cuuint64_t gdim[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)N};
    const cuuint64_t gstr[2] = {(cuuint64_t)W * 4, (cuuint64_t)H * W * 4};
    const cuuint32_t box[3] = {(cuuint32_t)W, (cuuint32_t)(2 * kCpRows + 3), 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT32, 3, const_cast<uint8_t*>(frames), gdim, gstr, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return set_error(SEEDRL_ERR_INTERNAL, "conv0pool: cuTensorMapEncodeTiled failed");
  }
  const int units = N * ((a.Ho + kCpRows - 1) / kCpRows);
  const int grid = units < 2 * kNumSMs ? units : 2 * kNumSMs;       // 2 CTAs / SM
  conv0pool_kernel<CP, TMA><<<grid, kCpThreadsF, smem, st>>>(tm, a);
  count_launch(PC_CONV_FWD, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// frames: [N,H,W,C] uint8, w: [3,3,C,16].  4-channel frames take the TMA-fed kernel; other channel
// counts the plain-load kernels.
int conv0pool_forward(int N, int H, int W, int C, const uint8_t* frames, const float* w, const float* bias,
                      void* praw, void* prelu, uint8_t* idx, int* err, cudaStream_t st) {
  if (!conv0pool_supported(C, 16, H, W))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv0pool: unsupported frame shape");
  Conv0PoolArgs a;
  a.N = N; a.H = H; a.W = W; a.C = C;
  same_pad3s2(H, &a.Ho, &a.pt);
  same_pad3s2(W, &a.Wo, &a.pl);
  a.Lpp = (int)planes_positions(N, a.Ho, a.Wo); a.PWp = a.Wo + 2; a.RHp = a.Ho + 1;
  fast_div_setup((unsigned int)(W + 2), &a.sw_mul, &a.sw_sh);
  a.frames = frames; a.w = w; a.bias = bias;
  a.praw = reinterpret_cast<uint4*>(praw); a.prelu = reinterpret_cast<uint4*>(prelu); a.idx = idx; a.err = err;
  if (C == 4) return launch_conv0pool<4, true>(a, frames, st);
  const int cp = first_layer_cp(C);
  return cp == 4 ? launch_conv0pool<4, false>(a, frames, st)
                 : (cp == 8 ? launch_conv0pool<8, false>(a, frames, st) : launch_conv0pool<16, false>(a, frames, st));
}

}  // namespace seedrl
