// conv3x3 'same' on the Hopper tensor cores (wgmma), bf16 (or bf16x3) operands,
// fp32 accumulation -- forward, data-gradient and weight-gradient of every convolution of
// dmlab/networks.py:26-60, the uint8 4->16 first layer included.
//
// Implicit GEMM on the "tall image" (see conv_kernels.cu): a CTA owns tiles of MT = 128..512
// consecutive flattened output positions (MT / 64 wgmma row blocks).  Activations are staged in shared memory as
// channel-group planes [CIN/8][positions][8 ch] bf16 (16 B per position per plane), which
// IS the canonical no-swizzle K-major wgmma layout:
//     8 consecutive positions x 8 channels  = one 128-byte core matrix
//     SBO (next 8 rows)            = 128 B
//     LBO (next 8 K-elements)      = plane stride
// and filter tap (kh,kw) is nothing but the descriptor START ADDRESS moved by
// (kh*PW + kw) * 16 bytes.  So the 3x3 conv is 9 * CIN/16 back-to-back
// wgmma.mma_async (64 x COUT x 16) per row block into one register accumulator -- no im2col,
// no per-tap data movement.
// Weights are pre-packed (prep kernel) to the K-major core-matrix layout
// [tap][slab][kchunk][COUT/8][8 co][8 ci] bf16; the data-gradient uses the same kernel
// with flipped/transposed packing.
// Epilogue straight from the accumulator registers (a thread holds 2 adjacent channels of 2
// positions per 8-channel group) -> bias / ReLU-mask / residual -> fp32 NHWC.
#include <cuda_bf16.h>

#include "kernels.h"
#include "tc_common.cuh"

namespace seedrl {

// w fp32 [tap][ci_src][co_src]  ->  packed bf16 for an implicit GEMM with CIN x COUT:
//   forward: element (tap, ci, co)   = w[tap][ci][co]
//   flipped: element (tap, ci, co)   = w[8-tap][co][ci]     (data-gradient; src is [tap][COUT][CIN])
// split != 0 (bf16x3): the lo parts (w - bf16(w), rounded to bf16) follow at wq[9*CIN*COUT + i].
// cin_src < CIN (first conv: 4 of 16): the missing input channels are packed as zeros.
__global__ void pack_w_tc_kernel(int CIN, int COUT, int cin_src, int flip, int split, const float* __restrict__ w,
                                 __nv_bfloat16* __restrict__ wq) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * CIN * COUT) return;
  const int e = i & 7;                       // ci % 8
  const int r = (i >> 3) & 7;                // co % 8
  int rest = i >> 6;
  const int cog = rest % (COUT / 8); rest /= (COUT / 8);
  const int kc = rest & 1; rest >>= 1;
  const int NS = CIN / 16;
  const int slab = rest % NS;
  const int tap = rest / NS;
  const int ci = slab * 16 + kc * 8 + e, co = cog * 8 + r;
  const float v = ci >= cin_src ? 0.f
                  : (flip ? w[((size_t)(8 - tap) * COUT + co) * CIN + ci] : w[((size_t)tap * cin_src + ci) * COUT + co]);
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  if (split == 2) {
    // merged layout of the plane-tensor kernels (conv_planes.cu): per (tap, slab, kchunk) the hi
    // c_out groups are followed by the lo c_out groups, so ONE MMA with N = 2*COUT computes
    // a*hi(w) and a*lo(w) from a single read of the activation tile
    const int GOc = COUT / 8;
    const size_t j = ((((size_t)(tap * NS + slab) * 2 + kc) * (2 * GOc) + cog) * 8 + r) * 8 + e;
    wq[j] = hi;
    wq[j + (size_t)GOc * 64] = __float2bfloat16_rn(v - __bfloat162float(hi));
    return;
  }
  wq[i] = hi;
  if (split) wq[9 * CIN * COUT + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

// All layers' weights packed by ONE launch (blockIdx.y = job) instead of one small launch per conv.
__global__ void pack_w_tc_batch_kernel(const __grid_constant__ PackTable t, int split) {
  const PackJob j = t.jobs[blockIdx.y];
  const int CIN = j.ck, COUT = j.cout;
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 9 * CIN * COUT) return;
  const int e = i & 7;                       // ci % 8
  const int r = (i >> 3) & 7;                // co % 8
  int rest = i >> 6;
  const int cog = rest % (COUT / 8); rest /= (COUT / 8);
  const int kc = rest & 1; rest >>= 1;
  const int NS = CIN / 16;
  const int slab = rest % NS;
  const int tap = rest / NS;
  const int ci = slab * 16 + kc * 8 + e, co = cog * 8 + r;
  const float v = ci >= j.cin_src ? 0.f
                  : (j.flip ? j.w[((size_t)(8 - tap) * COUT + co) * CIN + ci]
                            : j.w[((size_t)tap * j.cin_src + ci) * COUT + co]);
  __nv_bfloat16* wq = reinterpret_cast<__nv_bfloat16*>(j.wq);
  const __nv_bfloat16 hi = __float2bfloat16_rn(v);
  if (split == 2 && !j.legacy) {          // merged hi|lo layout (see pack_w_tc_kernel)
    const int GOc = COUT / 8;
    const size_t q = ((((size_t)(tap * NS + slab) * 2 + kc) * (2 * GOc) + cog) * 8 + r) * 8 + e;
    wq[q] = hi;
    wq[q + (size_t)GOc * 64] = __float2bfloat16_rn(v - __bfloat162float(hi));
    return;
  }
  wq[i] = hi;
  if (split) wq[9 * CIN * COUT + i] = __float2bfloat16_rn(v - __bfloat162float(hi));
}

int conv3x3_tc_pack_weights_batch(const PackTable& t, int split, cudaStream_t st) {
  if (t.n == 0) return SEEDRL_OK;
  pack_w_tc_batch_kernel<<<dim3(ceil_div(9 * 32 * 32, 256), t.n), 256, 0, st>>>(t, split);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

constexpr int kTcThreads = 256;
constexpr int kTcM = 128;
#ifndef SEEDRL_TC_ITEMS_U8
#define SEEDRL_TC_ITEMS_U8 4
#endif
#ifndef SEEDRL_TC_ITEMS_G2
#define SEEDRL_TC_ITEMS_G2 4
#endif
#ifndef SEEDRL_TC_MIN_BLOCKS
#define SEEDRL_TC_MIN_BLOCKS 4
#endif
constexpr int kTcMinBlocks = SEEDRL_TC_MIN_BLOCKS;   // resident CTAs per SM the register budget targets
                                                     // (one fewer for 32 input channels)

// One tile = MT consecutive output positions (MT / 64 wgmma row blocks); the staged input covers
// MT + 2*PW + 2 positions, so the halo re-read and the per-tile barriers shrink with MT.
// 8 warps: all stage; warpgroup wg multiplies row blocks wg, wg + 2, ... one at a time and
// stores each from its registers.
// SPLIT = bf16x3: activations and weights are split v = hi + lo (two bf16 planes / two packed
// weight sets) and each K-step issues hi*hi + lo*hi + hi*lo -- an fp32-faithful (~2^-16
// relative) contraction on the tensor cores; SPLIT = false is plain bf16 operands.
// IN_U8 (first conv, CIN = 4): one staged plane [x0 x1 x2 x3 0 0 0 0]; the MMA's second
// K-group re-reads it (LBO = 0) against zero weights; exact in bf16 (no lo plane); the 1/255
// scale is applied to the accumulator.
template <int CIN, int COUT, int IN_MODE, bool SPLIT, int MT>
__global__ void __launch_bounds__(kTcThreads, CIN >= 32 ? kTcMinBlocks - 1 : kTcMinBlocks)
conv3x3_tc_kernel(ConvGeom g, const void* __restrict__ in_, const uint4* __restrict__ wq,
                  const float* __restrict__ bias, const float* __restrict__ mask,
                  const float* __restrict__ res, float* __restrict__ out) {
  constexpr int CK = CIN < 16 ? 16 : CIN;   // channels the MMAs contract over
  constexpr int G = CIN < 8 ? 1 : CIN / 8;  // staged channel-group planes
  constexpr int NS = CK / 16;               // K slabs per tap
  constexpr bool ASPLIT = SPLIT && IN_MODE != IN_U8;
  constexpr int SA = ASPLIT ? 2 : 1, SB = SPLIT ? 2 : 1;
  constexpr int NBLK = MT / 64;
  constexpr int IT = IN_MODE == IN_U8 ? SEEDRL_TC_ITEMS_U8 : (G == 2 ? SEEDRL_TC_ITEMS_G2 : 4);
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int PW = g.PW;
  const int L = MT + 2 * PW + 2;      // staged input positions
  const int LPl = L | 1;              // plane stride in 16-byte units (odd: conflict-free stores)
  uint4* s_a = reinterpret_cast<uint4*>(smem_raw);                       // [SA][G][LPl] x 16 B
  uint4* s_b = s_a + (size_t)SA * G * LPl;                               // [SB] 9*CK*COUT bf16
  float* s_bias = reinterpret_cast<float*>(s_b + SB * 9 * CK * COUT / 8); // [COUT]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wg = tid >> 7;
  const float* inf = reinterpret_cast<const float*>(in_);
  const uint32_t* inu = reinterpret_cast<const uint32_t*>(in_);          // IN_U8: 4 channels = one word

  // ---- one-time setup: weights -> smem ------------------------------------------------
  for (int i = tid; i < SB * 9 * CK * COUT / 8; i += kTcThreads) s_b[i] = __ldg(wq + i);
  if (tid < COUT) s_bias[tid] = bias ? __ldg(bias + tid) : 0.f;
  __syncthreads();
  const uint32_t a_base = smem_u32(s_a), b_base = smem_u32(s_b);
  // K-major descriptors (header comment): A's LBO is the plane stride (0 for the one IN_U8 plane), B's
  // the COUT/8 core matrices of one K-group; SBO is one 128-byte core matrix for both
  const uint32_t a_lbo = CIN < 16 ? 0u : (uint32_t)LPl * 16u;
  constexpr uint32_t a_sbo = 128u, b_lbo = (uint32_t)(COUT / 8) * 128u, b_sbo = 128u;
  const float oscale = IN_MODE == IN_U8 ? (1.0f / 255.0f) : 1.0f;

  const int nchunks = (int)((g.Q + MT - 1) / MT);
  for (int ch = blockIdx.x; ch < nchunks; ch += gridDim.x) {
    const int q0 = ch * MT;
    // ---- stage the input tile: NHWC -> bf16 channel-group planes ---------------------------
    // IT items per thread per round: all loads of a round are issued before any is consumed;
    // with several CTAs per SM the round latency is hidden by the other CTAs
    for (int i0 = tid; i0 < L * G; i0 += IT * kTcThreads) {
      float4 va[IN_MODE == IN_U8 ? 1 : IT], vb[IN_MODE == IN_U8 ? 1 : IT];
      uint32_t vw[IN_MODE == IN_U8 ? IT : 1];
#pragma unroll
      for (int k = 0; k < IT; ++k) {
        const int i = i0 + k * kTcThreads;
        constexpr bool U8 = IN_MODE == IN_U8;
        va[U8 ? 0 : k] = make_float4(0.f, 0.f, 0.f, 0.f);
        vb[U8 ? 0 : k] = va[U8 ? 0 : k];
        vw[U8 ? k : 0] = 0u;
        if (i < L * G) {
          const int s = i / G, gch = i - s * G;
          const int pix = in_pixel(g, q0 + s);
          if (pix >= 0) {
            if (IN_MODE == IN_U8) {
              vw[IN_MODE == IN_U8 ? k : 0] = __ldg(inu + pix);
            } else {
              const float4* src = reinterpret_cast<const float4*>(inf + (size_t)pix * CIN + gch * 8);
              va[IN_MODE == IN_U8 ? 0 : k] = __ldg(src);
              vb[IN_MODE == IN_U8 ? 0 : k] = __ldg(src + 1);
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < IT; ++k) {
        const int i = i0 + k * kTcThreads;
        if (i < L * G) {
          const int s = i / G, gch = i - s * G;
          if (IN_MODE == IN_U8) {
            const uint32_t w = vw[IN_MODE == IN_U8 ? k : 0];     // byte k -> float without I2F: 0x4B0000kk is 2^23 + kk
            s_a[s] = pack8_bf16(make_float4(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540)) - 8388608.0f,
                                            __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7541)) - 8388608.0f,
                                            __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7542)) - 8388608.0f,
                                            __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7543)) - 8388608.0f),
                                make_float4(0.f, 0.f, 0.f, 0.f));
          } else {
            float4 a = va[IN_MODE == IN_U8 ? 0 : k], b = vb[IN_MODE == IN_U8 ? 0 : k];
            if (IN_MODE == IN_RELU) {
              a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
              b.x = fmaxf(b.x, 0.f); b.y = fmaxf(b.y, 0.f); b.z = fmaxf(b.z, 0.f); b.w = fmaxf(b.w, 0.f);
            }
            s_a[(size_t)gch * LPl + s] = pack8_bf16(a, b);
            if (ASPLIT) s_a[(size_t)(G + gch) * LPl + s] = pack8_bf16(bf16_resid4(a), bf16_resid4(b));
          }
        }
      }
    }
    // generic-proxy smem writes -> visible to the tensor core's async proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();

    // ---- warpgroup wg: row blocks wg, wg + 2, ...: 9 * NS (x3 when SPLIT) MMAs, then the epilogue
#pragma unroll 1
    for (int m = wg; m < NBLK; m += kTcThreads / 128) {
      float acc[COUT / 2];
#pragma unroll
      for (int i = 0; i < COUT / 2; ++i) acc[i] = 0.f;
      wgmma_fence_acc<COUT / 2>(acc);
      wgmma_fence();
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int off = m * 64 + (tap / 3) * PW + (tap % 3);
#pragma unroll
        for (int sl = 0; sl < NS; ++sl) {
          const uint64_t da = gmma_desc(a_base + ((uint32_t)(sl * 2) * LPl + off) * 16u, a_lbo, a_sbo);
          const uint64_t db = gmma_desc(b_base + (uint32_t)(tap * NS + sl) * (COUT * 32u), b_lbo, b_sbo);
          Wgmma<COUT>::template mma<0, 0>(acc, da, db, 1u);
          if (SPLIT) {   // + lo(a)*hi(b) + hi(a)*lo(b); the address field counts 16-byte units
            if (ASPLIT) Wgmma<COUT>::template mma<0, 0>(acc, da + (uint64_t)(G * LPl), db, 1u);
            Wgmma<COUT>::template mma<0, 0>(acc, da, db + (uint64_t)(9 * CK * COUT / 8), 1u);
          }
        }
      }
      wgmma_commit();
      wgmma_wait<0>();
      wgmma_fence_acc<COUT / 2>(acc);
      // ---- epilogue: (position, 2 channels) pairs of the accumulator -> fp32 NHWC ---------------
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int pix = out_pixel(g, q0 + m * 64 + 16 * (warp & 3) + (lane >> 2) + 8 * h);
        if (pix >= 0) {
#pragma unroll
          for (int j = 0; j < COUT / 8; ++j) {
            const int c = 8 * j + 2 * (lane & 3);
            const size_t o = (size_t)pix * COUT + c;
            float2 v = make_float2(fmaf(acc[4 * j + 2 * h], oscale, s_bias[c]),
                                   fmaf(acc[4 * j + 2 * h + 1], oscale, s_bias[c + 1]));
            if (mask) {
              const float2 mk = __ldg(reinterpret_cast<const float2*>(mask + o));
              v.x = mk.x > 0.f ? v.x : 0.f; v.y = mk.y > 0.f ? v.y : 0.f;
            }
            if (res) {
              const float2 r = __ldg(reinterpret_cast<const float2*>(res + o));
              v.x += r.x; v.y += r.y;
            }
            *reinterpret_cast<float2*>(out + o) = v;
          }
        }
      }
    }
    // every MMA of this tile has read the staged input before the next tile overwrites it
    __syncthreads();
  }
}

static int g_tc_mt = 512;   // output positions per tile to try first (bench/debug knob)
void conv3x3_tc_set_tile(int mt) { g_tc_mt = mt; }
constexpr int kTcTryNext = -12346;

template <int CIN, int COUT, int IN_MODE, bool SPLIT, int MT>
static int launch_tc(int N, int H, int W, const void* in, const uint4* wq, const float* bias,
                     const float* mask, const float* res, float* out, int* err, cudaStream_t st) {
  const ConvGeom g = make_geom(N, H, W);
  const int L = MT + 2 * g.PW + 2;
  constexpr int CK = CIN < 16 ? 16 : CIN;
  constexpr int G = CIN < 8 ? 1 : CIN / 8;
  constexpr int SA = (SPLIT && IN_MODE != IN_U8) ? 2 : 1, SB = SPLIT ? 2 : 1;
  const size_t smem = SA * (size_t)G * (L | 1) * 16 + SB * (size_t)9 * CK * COUT * 2 + 16 + COUT * 4 + 64;
  if (smem > 200 * 1024) {
    if (MT > kTcM) return kTcTryNext;
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3_tc: image too wide");
  }
  SEEDRL_CUDA(allow_smem<conv3x3_tc_kernel<CIN, COUT, IN_MODE, SPLIT, MT>>(200 * 1024));
  // resident CTAs per SM: registers (64K, allocated in units of 8 per thread), shared memory
  // (228 KB, 1 KB reserved per CTA), threads
  static int regs = 0, static_smem = 0;
  if (regs == 0) {
    cudaFuncAttributes fa;
    SEEDRL_CUDA(cudaFuncGetAttributes(&fa, conv3x3_tc_kernel<CIN, COUT, IN_MODE, SPLIT, MT>));
    regs = fa.numRegs > 0 ? fa.numRegs : 255;
    static_smem = (int)fa.sharedSizeBytes;
  }
  int per_sm = 65536 / (((regs + 7) & ~7) * kTcThreads);
  const int by_smem = (int)((size_t)(228 * 1024) / (smem + (size_t)static_smem + 1024));
  if (per_sm > by_smem) per_sm = by_smem;
  if (per_sm > 2048 / kTcThreads) per_sm = 2048 / kTcThreads;
  if (per_sm > 6) per_sm = 6;
  if (per_sm < 2 && MT > kTcM) return kTcTryNext;          // a smaller tile keeps >= 2 CTAs / SM
  if (per_sm < 1) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3_tc: image too wide");
  if (g.Q + MT + 4 * g.PW >= (1LL << 31))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3_tc: batch too large for 32-bit positions");
  const long long nchunks = (g.Q + MT - 1) / MT;
  long long grid = (long long)kNumSMs * per_sm;
  if (grid > nchunks) grid = nchunks;
  conv3x3_tc_kernel<CIN, COUT, IN_MODE, SPLIT, MT><<<(unsigned)grid, kTcThreads, smem, st>>>(
      g, in, wq, bias, mask, res, out);
  count_launch(g_conv_cat, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// ---------------------------------------------------------------------------------------
// Weight gradient on the tensor cores.
//   dW[kh][kw][ci][co] = sum_p x~[p + kh*PW + kw][ci] * dy[p][co]   (x~ = relu(x) for the res convs,
//                                                                    frame/255 for the first conv)
// as a GEMM with M = co, N = (kw, ci), K = positions, one accumulator per kernel row kh.
// Both operands are MN-major: for a fixed position (K index) the 8 channels of a group are
// contiguous -- the channel-group plane layout of the forward kernel:
//     core matrix = 8 positions (K) x 8 channels (MN), 128 B;  K-group stride (LBO) = 128 B;
//     MN-group stride (SBO) = plane stride.
// A = dy planes [COUT/8][128].  B = x planes [3][CP/8][Lk]: plane (kw, g) holds x shifted by kw
// positions (the producers store every x unit three times), so that the three taps of a
// kernel row are consecutive N-groups of ONE MMA (N = 3*CP instead of three N = CP MMAs);
// kh is a descriptor start-address offset of kh*PW positions.  wgmma M is 64, rows >= COUT of
// the accumulators are junk (they read whatever follows the dy planes in shared memory) and are
// never stored.  Warpgroup kh (warps 4kh .. 4kh+3) owns kernel row kh: its 64 x 3*CP accumulator
// lives in registers across ALL chunks of a persistent CTA (1 CTA / SM).  Pipeline over `nb` stages:
//     warps 12..19 producers: global -> registers (prefetched two chunks ahead when registers
//                  allow) -> bf16 planes in smem -> fence.proxy.async -> arrive on full[stage]
//     warps 0..11  wait full[stage], issue KC/16 (x3 when SPLIT) MMAs, keep one chunk in flight
//                  (wgmma.wait_group 1) and release the previous chunk's stage on empty[stage]
// SPLIT = bf16x3: operands are split v = hi + lo (two bf16 planes) and the product is
// hi*hi + lo*hi + hi*lo, i.e. fp32-faithful (~2^-16 relative) contraction on tensor cores.
// uint8 frames (first conv, CIN = 4 padded to one 8-channel group) are exact in bf16: no lo
// plane; the 1/255 scale is applied to the accumulators.
// Per-CTA partial dW/db are reduced in fixed order by wgrad_reduce (deterministic).

// x items per producer per chunk (compile-time bound on ceil(L * G / producers); L = KC + 2*PW + 2
// with PW <= 86 for 8-channel, <= 44 for 16-channel and <= 23 for 32-channel inputs)
__host__ __device__ constexpr int wg_ix(int G, int KC) {
  return KC <= 128 ? (G == 4 ? 3 : 2) : (KC <= 256 ? (G == 1 ? 2 : (G == 2 ? 3 : 5)) : 3);
}
// Longest chunk per input width: beyond it the producers' prefetch registers spill under the
// 640-thread launch bound.
__host__ __device__ constexpr int wg_max_chunk(int CP) { return CP == 8 ? 512 : (CP == 16 ? 256 : 128); }
static int g_wgrad_kc = 256;   // K positions per pipeline stage to try first (bench/debug knob)
void conv3x3_wgrad_tc_set_chunk(int kc) { g_wgrad_kc = kc; }

constexpr int kWgMmaThreads = 3 * 128;          // one warpgroup per kernel row
constexpr int kWgProducers = 256;
constexpr int kWgThreads = kWgMmaThreads + kWgProducers;
constexpr int kWgMaxBufs = 3;

__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity, bool* timed_out) {
  if (!mbar_wait_bounded(bar, parity)) *timed_out = true;
}

template <int CIN, int COUT, int IN_MODE, bool SPLIT, int KC>
__global__ void __launch_bounds__(kWgThreads, 1)
conv3x3_wgrad_tc_kernel(ConvGeom g, const void* __restrict__ x_, const float* __restrict__ dy,
                        float* __restrict__ partial, const int nb, int* __restrict__ error_flag) {
  constexpr int CP = CIN < 8 ? 8 : CIN;                   // channels per position in the x planes
  constexpr int G = CP / 8, GO = COUT / 8;
  constexpr bool XSPLIT = SPLIT && IN_MODE != IN_U8;
  constexpr int SX = XSPLIT ? 2 : 1, SD = SPLIT ? 2 : 1;
  constexpr int NN = 3 * CP;                              // wgmma N: (kw, ci)
  constexpr int NW = 9 * CIN * COUT + COUT;
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int PW = g.PW;
  const int L = KC + 2 * PW + 2;                        // x positions a chunk touches
  const int Lk = KC + 2 * PW;                           // positions per shifted plane
  const int LPk = Lk | 1;                                 // x plane stride (16-byte units)
  // one stage: [x hi planes | x lo planes | dy hi planes | dy lo planes]
  const uint32_t xs_units = (uint32_t)(3 * G) * LPk, ds_units = (uint32_t)GO * KC;
  const uint32_t buf_units = SX * xs_units + SD * ds_units;
  uint4* s_buf = reinterpret_cast<uint4*>(smem_raw);
  // (whatever follows the last stage is only ever READ, by the junk rows of A)
  uint64_t* s_full = reinterpret_cast<uint64_t*>(smem_raw + (size_t)nb * buf_units * 16);
  uint64_t* s_empty = s_full + kWgMaxBufs;
  float* s_bias = reinterpret_cast<float*>(smem_raw);     // reused after the pipeline drains
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < kWgMaxBufs; ++i) {
      mbar_init(s_full + i, kWgProducers / 32);
      mbar_init(s_empty + i, kWgMmaThreads / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int nchunks = (int)((g.Q + KC - 1) / KC);
  const int my_chunks = ((int)blockIdx.x < nchunks) ? (nchunks - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  bool timed_out = false;
  float bsum[8];
#pragma unroll
  for (int c = 0; c < 8; ++c) bsum[c] = 0.f;
  float* dst = partial + (size_t)blockIdx.x * NW;

  if (tid < kWgMmaThreads) {
    // ================================ MMA warpgroups ========================================
    const int kh = warp >> 2;
    float acc[NN / 2];
#pragma unroll
    for (int i = 0; i < NN / 2; ++i) acc[i] = 0.f;
    wgmma_fence_acc<NN / 2>(acc);
    for (int it = 0; it < my_chunks; ++it) {
      const int b = it % nb;
      mbar_wait(s_full + b, (uint32_t)((it / nb) & 1), &timed_out);
      const uint32_t xbase = smem_u32(s_buf + (size_t)b * buf_units);
      const uint32_t dbase = xbase + SX * xs_units * 16u;
      // descriptors with start address 0; the address field counts 16-byte units
      const uint64_t bx = gmma_desc(0u, 128u, (uint32_t)LPk * 16u);
      const uint64_t ad = gmma_desc(0u, 128u, (uint32_t)KC * 16u);
      const uint64_t xh = bx + (xbase >> 4) + (uint64_t)(kh * PW), xl = xh + xs_units;
      const uint64_t dh = ad + (dbase >> 4), dl = dh + ds_units;
      wgmma_fence();
#pragma unroll
      for (int ks = 0; ks < KC / 16; ++ks) {
        const uint32_t ko = (uint32_t)(ks * 16);
        Wgmma<NN>::template mma<1, 1>(acc, dh + ko, xh + ko, 1u);
        if (SPLIT) Wgmma<NN>::template mma<1, 1>(acc, dl + ko, xh + ko, 1u);
        if (XSPLIT) Wgmma<NN>::template mma<1, 1>(acc, dh + ko, xl + ko, 1u);
      }
      wgmma_commit();
      wgmma_wait<1>();                     // the previous chunk's MMAs have read their stage
      if (it > 0 && lane == 0) mbar_arrive(s_empty + (it - 1) % nb);
    }
    wgmma_wait<0>();
    wgmma_fence_acc<NN / 2>(acc);
    // ---- rows 0..COUT-1 of this kernel row's accumulator -> this CTA's partial ----------------
    const float scale = IN_MODE == IN_U8 ? (1.0f / 255.0f) : 1.0f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int co = 16 * (warp & 3) + (lane >> 2) + 8 * h;
      if (co < COUT) {
#pragma unroll
        for (int j = 0; j < NN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int n = 8 * j + 2 * (lane & 3) + e, kw = n / CP, ci = n - kw * CP;
            if (ci < CIN) dst[((size_t)(kh * 3 + kw) * CIN + ci) * COUT + co] = acc[4 * j + 2 * h + e] * scale;
          }
        }
      }
    }
  } else {
    // ================================ producers ============================================
    // Two register sets: while chunk i is converted into shared memory, the global loads of
    // chunks i+1 and i+2 are already in flight (the producers are pure latency hiding).
    const int pt = tid - kWgMmaThreads;
    constexpr int IX = wg_ix(G, KC);                                  // host checks L*G <= IX*producers
    constexpr int ID = (KC * GO + kWgProducers - 1) / kWgProducers;
    constexpr int DEPTH = (IX + ID <= 4) ? 2 : 1;                     // register sets of prefetched chunks
    const float* xf = reinterpret_cast<const float*>(x_);
    const uint32_t* xu = reinterpret_cast<const uint32_t*>(x_);       // IN_U8: 4 channels = one word
    struct Regs { float4 xa[IX], xb[IX], dya[ID], dyb[ID]; uint32_t xw[IX]; };
    auto issue_loads = [&](Regs& r, int q0) {
#pragma unroll
      for (int k = 0; k < IX; ++k) {
        const int i = pt + k * kWgProducers;
        r.xa[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        r.xb[k] = r.xa[k];
        r.xw[k] = 0u;
        if (i < L * G) {
          const int s = i / G, gch = i - s * G;
          const int pix = in_pixel(g, q0 + s);
          if (pix >= 0) {
            if (IN_MODE == IN_U8) {
              r.xw[k] = __ldg(xu + pix);
            } else {
              const float4* src = reinterpret_cast<const float4*>(xf + (size_t)pix * CIN + gch * 8);
              r.xa[k] = __ldg(src);
              r.xb[k] = __ldg(src + 1);
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < ID; ++k) {
        const int i = pt + k * kWgProducers;
        r.dya[k] = make_float4(0.f, 0.f, 0.f, 0.f);
        r.dyb[k] = r.dya[k];
        if (i < KC * GO) {
          const int s = i / GO, go = i - s * GO;
          const int pix = out_pixel(g, q0 + s);
          if (pix >= 0) {
            const float4* src = reinterpret_cast<const float4*>(dy + (size_t)pix * COUT + go * 8);
            r.dya[k] = __ldg(src);
            r.dyb[k] = __ldg(src + 1);
          }
        }
      }
    };
    auto chunk_q0 = [&](int it) { return ((int)blockIdx.x + it * (int)gridDim.x) * KC; };
    auto stage = [&](Regs& r, int it) {
      const int pb = it % nb;
      uint4* s_x = s_buf + (size_t)pb * buf_units;
      uint4* s_d = s_x + (size_t)SX * xs_units;
      if (it >= nb) mbar_wait(s_empty + pb, (uint32_t)(((it / nb) - 1) & 1), &timed_out);
#pragma unroll
      for (int k = 0; k < IX; ++k) {
        const int i = pt + k * kWgProducers;
        if (i < L * G) {
          const int s = i / G, gch = i - s * G;
          uint4 hi, lo = make_uint4(0u, 0u, 0u, 0u);
          if (IN_MODE == IN_U8) {
            const uint32_t w = r.xw[k];     // exact in bf16; channels 4..7 are zero padding
            // byte k -> float without I2F: 0x4B0000kk is 2^23 + kk
            hi = pack8_bf16(make_float4(__uint_as_float(__byte_perm(w, 0x4B000000u, 0x7540)) - 8388608.0f,
                                        __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7541)) - 8388608.0f,
                                        __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7542)) - 8388608.0f,
                                        __uint_as_float(__byte_perm(w, 0x4B000000u, 0x7543)) - 8388608.0f),
                            make_float4(0.f, 0.f, 0.f, 0.f));
          } else {
            float4 a = r.xa[k], c = r.xb[k];
            if (IN_MODE == IN_RELU) {
              a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
              c.x = fmaxf(c.x, 0.f); c.y = fmaxf(c.y, 0.f); c.z = fmaxf(c.z, 0.f); c.w = fmaxf(c.w, 0.f);
            }
            hi = pack8_bf16(a, c);
            if (XSPLIT) lo = pack8_bf16(bf16_resid4(a), bf16_resid4(c));
          }
          // plane (kw, gch)[p] = x[p + kw]
#pragma unroll
          for (int kw = 0; kw < 3; ++kw) {
            const int p = s - kw;
            if (p >= 0 && p < Lk) {
              s_x[(size_t)(kw * G + gch) * LPk + p] = hi;
              if (XSPLIT) s_x[xs_units + (size_t)(kw * G + gch) * LPk + p] = lo;
            }
          }
        }
      }
      // a thread always stages the same co-group (kWgProducers % GO == 0) => bsum[] is per
      // (thread, channel-in-group) and the final reduction order is fixed (deterministic).
#pragma unroll
      for (int k = 0; k < ID; ++k) {
        const int i = pt + k * kWgProducers;
        if (i < KC * GO) {
          const int s = i / GO, go = i - s * GO;
          const float4 a = r.dya[k], c = r.dyb[k];
          bsum[0] += a.x; bsum[1] += a.y; bsum[2] += a.z; bsum[3] += a.w;
          bsum[4] += c.x; bsum[5] += c.y; bsum[6] += c.z; bsum[7] += c.w;
          s_d[(size_t)go * KC + s] = pack8_bf16(a, c);
          if (SPLIT) s_d[ds_units + (size_t)go * KC + s] = pack8_bf16(bf16_resid4(a), bf16_resid4(c));
        }
      }
      if (it + DEPTH < my_chunks) issue_loads(r, chunk_q0(it + DEPTH));   // refill this register set
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0)
        asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}\n" ::"r"(
                         smem_u32(s_full + pb))
                     : "memory");
    };
    if (DEPTH == 2) {
      Regs r0, r1;
      if (my_chunks > 0) issue_loads(r0, chunk_q0(0));
      if (my_chunks > 1) issue_loads(r1, chunk_q0(1));
      for (int it = 0; it < my_chunks; it += 2) {
        stage(r0, it);
        if (it + 1 < my_chunks) stage(r1, it + 1);
      }
    } else {
      Regs r0;
      if (my_chunks > 0) issue_loads(r0, chunk_q0(0));
      for (int it = 0; it < my_chunks; ++it) stage(r0, it);
    }
  }
  if (timed_out && error_flag) atomicExch(error_flag, 1);
  __syncthreads();                          // every MMA has completed: the stages are free

  // ---- bias partial: fixed-order reduction over the producers that staged each co-group -------
  if (tid >= kWgMmaThreads) {
#pragma unroll
    for (int c = 0; c < 8; ++c) s_bias[(tid - kWgMmaThreads) * 8 + c] = bsum[c];
  }
  __syncthreads();
  if (tid < COUT) {
    const int go = tid >> 3, c = tid & 7;
    float sum = 0.f;
    for (int t = go; t < kWgProducers; t += GO) sum += s_bias[t * 8 + c];   // producer t staged group t % GO
    dst[9 * CIN * COUT + tid] = sum;
  }
}

// rc: SEEDRL_OK, an error, or kWgTryNext when this chunk length does not fit the geometry
constexpr int kWgTryNext = -12345;
template <int CIN, int COUT, int IN_MODE, bool SPLIT, int KC>
static int launch_wgrad_tc(int N, int H, int W, const void* x, const float* dy, float* dw, float* db,
                           float* partial, size_t partial_bytes, int* err, WgradBatch* batch,
                           cudaStream_t st) {
  const ConvGeom g = make_geom(N, H, W);
  constexpr int CP = CIN < 8 ? 8 : CIN;
  constexpr int SX = (SPLIT && IN_MODE != IN_U8) ? 2 : 1, SD = SPLIT ? 2 : 1;
  const int L = KC + 2 * g.PW + 2;
  const size_t plane = (size_t)((KC + 2 * g.PW) | 1) * 16;
  const size_t buf = SX * 3 * (size_t)(CP / 8) * plane + SD * (size_t)(COUT / 8) * KC * 16;
  // A's junk rows reach 8 dy-plane strides (16 KB) past the start of the last stage's dy planes
  const size_t tail = 8 * (size_t)KC * 16 + 256;
  const size_t budget = 224 * 1024;
  int nb = kWgMaxBufs;
  while (nb > 1 && nb * buf + tail > budget) --nb;
  if (nb < 2 || (size_t)L * (CP / 8) > (size_t)wg_ix(CP / 8, KC) * kWgProducers) return kWgTryNext;
  size_t smem = nb * buf + tail;
  if (smem < (size_t)kWgProducers * 8 * 4) smem = (size_t)kWgProducers * 8 * 4;
  SEEDRL_CUDA(allow_smem<conv3x3_wgrad_tc_kernel<CIN, COUT, IN_MODE, SPLIT, KC>>((int)budget));
  if (g.Q + KC + 4 * g.PW >= (1LL << 31))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad_tc: batch too large for 32-bit positions");
  constexpr int NW = 9 * CIN * COUT + COUT;
  const long long nchunks = (g.Q + KC - 1) / KC;
  int grid = kNumSMs;                       // 1 CTA per SM (register-resident accumulators)
  if (grid > nchunks) grid = (int)nchunks;
  // deferred reduction: this layer's partials get their own slice of the batch buffer and are
  // reduced together with every other layer's by ONE launch at the end of the backward pass
  const bool defer = batch && batch->n < kMaxReduceJobs &&
                     batch->used + (size_t)grid * NW <= batch->cap_floats;
  if (defer) {
    partial = batch->buf + batch->used;
    batch->used += (size_t)grid * NW;
  } else if ((size_t)grid * NW * sizeof(float) > partial_bytes) {
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad_tc: partial buffer too small");
  }
  conv3x3_wgrad_tc_kernel<CIN, COUT, IN_MODE, SPLIT, KC><<<grid, kWgThreads, smem, st>>>(g, x, dy, partial, nb, err);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  if (defer) {
    batch->jobs[batch->n++] = ReduceJob{partial, dw, db, grid, 9 * CIN * COUT, COUT};
    return SEEDRL_OK;
  }
  return wgrad_reduce(grid, 9 * CIN * COUT, COUT, partial, dw, db, st);
}

// launch_wgrad_tc for the chunk lengths wg_max_chunk allows; longer ones are never instantiated
template <int CIN, int COUT, int IN_MODE, int KC>
static int try_wgrad_tc(int split, int N, int H, int W, const void* x, const float* dy, float* dw, float* db,
                        float* partial, size_t partial_bytes, int* err, WgradBatch* batch, cudaStream_t st) {
  if constexpr (KC > wg_max_chunk(CIN < 8 ? 8 : CIN)) {
    return kWgTryNext;
  } else {
    return split ? launch_wgrad_tc<CIN, COUT, IN_MODE, true, KC>(N, H, W, x, dy, dw, db, partial, partial_bytes,
                                                                 err, batch, st)
                 : launch_wgrad_tc<CIN, COUT, IN_MODE, false, KC>(N, H, W, x, dy, dw, db, partial, partial_bytes,
                                                                  err, batch, st);
  }
}

__global__ void wgrad_reduce_batch_kernel(const __grid_constant__ ReduceTable t) {
  const ReduceJob j = t.jobs[blockIdx.y];
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= j.nw + j.nb) return;
  // fixed-order sum over the CTAs' partials; the loads of 8 partials are issued together (they are
  // independent), the adds stay sequential => same result as the plain loop, ~4x less latency
  float s = 0.f;
  const size_t stride = (size_t)(j.nw + j.nb);
  const float* src = j.partial + i;
  int k = 0;
  for (; k + 8 <= j.nparts; k += 8) {
    float v[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) v[q] = __ldcs(src + (size_t)(k + q) * stride);
#pragma unroll
    for (int q = 0; q < 8; ++q) s += v[q];
  }
  for (; k < j.nparts; ++k) s += __ldcs(src + (size_t)k * stride);
  if (i < j.nw) j.dw[i] = s; else j.db[i - j.nw] = s;
}

int wgrad_reduce_batch(WgradBatch* b, cudaStream_t st) {
  if (!b || b->n == 0) return SEEDRL_OK;
  ReduceTable t;
  int maxn = 0;
  for (int i = 0; i < b->n; ++i) {
    t.jobs[i] = b->jobs[i];
    if (b->jobs[i].nw + b->jobs[i].nb > maxn) maxn = b->jobs[i].nw + b->jobs[i].nb;
  }
  wgrad_reduce_batch_kernel<<<dim3(ceil_div(maxn, 256), b->n), 256, 0, st>>>(t);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  b->n = 0;
  b->used = 0;
  return SEEDRL_OK;
}

int conv3x3_wgrad_tc(int cin, int cout, int in_mode, int split, int N, int H, int W, const void* x,
                     const float* dy, float* dw, float* db, float* partial, size_t partial_bytes,
                     int* err, WgradBatch* batch, cudaStream_t st) {
#define SEEDRL_WGTC_ARGS N, H, W, x, dy, dw, db, partial, partial_bytes, err, batch, st
#define SEEDRL_WGTC_CASE(CI, CO_, MODE)                                                          \
  if (cin == CI && cout == CO_ && in_mode == MODE) {                                             \
    int rc = kWgTryNext;                                                                         \
    if (g_wgrad_kc >= 512) rc = try_wgrad_tc<CI, CO_, MODE, 512>(split, SEEDRL_WGTC_ARGS);         \
    if (rc == kWgTryNext && g_wgrad_kc >= 256)                                                   \
      rc = try_wgrad_tc<CI, CO_, MODE, 256>(split, SEEDRL_WGTC_ARGS);                            \
    if (rc == kWgTryNext) rc = try_wgrad_tc<CI, CO_, MODE, 128>(split, SEEDRL_WGTC_ARGS);          \
    if (rc == kWgTryNext) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad_tc: image too wide"); \
    return rc;                                                                                   \
  }
  SEEDRL_WGTC_CASE(4, 16, IN_U8)
  SEEDRL_WGTC_CASE(16, 16, IN_RELU)
  SEEDRL_WGTC_CASE(16, 32, IN_F32)
  SEEDRL_WGTC_CASE(32, 32, IN_F32)
  SEEDRL_WGTC_CASE(32, 32, IN_RELU)
#undef SEEDRL_WGTC_CASE
#undef SEEDRL_WGTC_ARGS
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgrad_tc: unsupported (cin,cout,mode)");
}

bool conv3x3_wgrad_tc_supported(int cin, int cout, int in_mode) {
  return (cin == 4 && cout == 16 && in_mode == IN_U8) || (cin == 16 && cout == 16 && in_mode == IN_RELU) ||
         (cin == 16 && cout == 32 && in_mode == IN_F32) ||
         (cin == 32 && cout == 32 && (in_mode == IN_F32 || in_mode == IN_RELU));
}

bool conv3x3_tc_supported(int cin, int cout, int in_mode) {
  return ((cin == 16 || cin == 32) && (cout == 16 || cout == 32) && (in_mode == IN_F32 || in_mode == IN_RELU)) ||
         (cin == 4 && cout == 16 && in_mode == IN_U8);
}

int conv3x3_tc_pack_weights(int cin, int cout, int flip, int split, const float* w, void* wq,
                            cudaStream_t st) {
  const int ck = cin < 16 ? 16 : cin;     // wq holds (split ? 2 : 1) * 9 * ck * cout bf16
  const int n = 9 * ck * cout;
  pack_w_tc_kernel<<<ceil_div(n, 256), 256, 0, st>>>(ck, cout, cin, flip, split, w,
                                                     reinterpret_cast<__nv_bfloat16*>(wq));
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int conv3x3_tc_forward(int cin, int cout, int in_mode, int split, int N, int H, int W, const void* in,
                       const void* wq, const float* bias, const float* mask, const float* res,
                       float* out, int* err, cudaStream_t st) {
  const uint4* q = reinterpret_cast<const uint4*>(wq);
#define SEEDRL_TC_ARGS N, H, W, in, q, bias, mask, res, out, err, st
#define SEEDRL_TC_CASE(CI, CO_, MODE)                                                               \
  if (cin == CI && cout == CO_ && in_mode == MODE) {                                                \
    int rc = kTcTryNext;                                                                            \
    if (g_tc_mt >= 512)                                                                             \
      rc = split ? launch_tc<CI, CO_, MODE, true, 512>(SEEDRL_TC_ARGS) : launch_tc<CI, CO_, MODE, false, 512>(SEEDRL_TC_ARGS); \
    if (rc == kTcTryNext && g_tc_mt >= 256)                                                         \
      rc = split ? launch_tc<CI, CO_, MODE, true, 256>(SEEDRL_TC_ARGS) : launch_tc<CI, CO_, MODE, false, 256>(SEEDRL_TC_ARGS); \
    if (rc == kTcTryNext)                                                                           \
      rc = split ? launch_tc<CI, CO_, MODE, true, 128>(SEEDRL_TC_ARGS) : launch_tc<CI, CO_, MODE, false, 128>(SEEDRL_TC_ARGS); \
    return rc;                                                                                      \
  }
  SEEDRL_TC_CASE(4, 16, IN_U8)
  SEEDRL_TC_CASE(16, 16, IN_F32)
  SEEDRL_TC_CASE(16, 16, IN_RELU)
  SEEDRL_TC_CASE(16, 32, IN_F32)
  SEEDRL_TC_CASE(32, 16, IN_F32)
  SEEDRL_TC_CASE(32, 32, IN_F32)
  SEEDRL_TC_CASE(32, 32, IN_RELU)
#undef SEEDRL_TC_CASE
#undef SEEDRL_TC_ARGS
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv3x3_tc: unsupported (cin,cout,mode)");
}

}  // namespace seedrl
