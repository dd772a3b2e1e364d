// "Planes" convolution path (conv_mode 3, 'tc3p'): activations and gradients of the 16/32-channel
// layers of dmlab/networks.py:26-60 live in HBM in the tensor core's own operand format, so that
// every 3x3 convolution (forward, data gradient, weight gradient) is
//      TMA tile (cp.async.bulk.tensor)  ->  wgmma  ->  epilogue
// with no thread ever touching an input element.
//
// HBM format of a [N, H, W, C] activation ("plane tensor"):
//   the N images form one zero-padded tall image (PW = W + 2 columns, RH = H + 1 rows per image,
//   one shared zero row between images); pixel (n, h, w) sits at storage position
//       s = (n * RH + h + 1) * PW + (w + 1),          0 <= s < Lp,
//   and the tensor is 2 * C/8 planes [Lp][8 ch] bf16 (16 bytes per position): first the C/8 "hi"
//   planes (bf16(v)), then the C/8 "lo" planes (bf16(v - hi)) -- v = hi + lo to ~2^-17 relative,
//   the bf16x3 operand split of the 'tc3' mode, done ONCE by the producing kernel's epilogue
//   instead of by every consumer.  Padding positions hold zeros.
//   One plane is exactly the canonical no-swizzle wgmma layout (core matrix = 8 positions x 16 B):
//   K-major A operand of the forward / data-gradient GEMM (M = positions, K = channels: LBO = plane
//   stride, SBO = 128 B) and MN-major operand of the weight-gradient GEMM (K = positions: LBO =
//   128 B, SBO = plane stride); a filter tap (kh, kw) is the descriptor start address moved by
//   (kh * PW + kw) * 16 bytes.
//
// Kernels (all persistent, 1 CTA / SM, warp-specialised, mbarrier pipelines, bounded waits):
//   convp_kernel<CIN, COUT, NSUB>   forward / data gradient.  warp 16 = TMA producer (one
//       cp.async.bulk.tensor.3d per tile: box = chunks of positions x (2 * CIN/8 planes), 2..4
//       smem stages), warps 0..15 = four warpgroups that take the CTA's 64-position blocks
//       round-robin: 9*CIN/16*2 wgmma 64 x {2 COUT, COUT} x 16 into registers, release the stage
//       on its empty barrier, then the epilogue straight from the accumulator registers (quad
//       shuffles -> bias / ReLU-mask / residual -> hi/lo split -> coalesced 16-byte plane stores;
//       optionally a second, ReLU'd copy for the next conv, or fp32 NHWC for the max-pool / Dense
//       consumers) while the other warpgroups' MMAs keep the tensor pipe busy.
//   wgradp_kernel<CP, COUT, KC>     weight + bias gradient: one TMA copy of x and of dy per K chunk
//       (+ halo); M = (kw, ci) rows (+ a constant row whose accumulator is the bias gradient) built
//       in registers by ldmatrix with the kw shift in each lane's address, N = (hi | lo, c_out) per
//       kh as a descriptor offset into dy, K = positions; three warpgroups per 64 rows (one per kh)
//       for 16-channel inputs, one for 32; every warpgroup takes every chunk of the CTA in order;
//       per-CTA partials reduced in fixed order by the deferred reduce of conv_tc_kernels.cu.
//   poolp_fwd / poolp_bwd / to_planes / from_planes: elementwise format kernels.
#include <cuda.h>
#include <cuda_bf16.h>

#include <cstdio>

#include "kernels.h"
#include "tc_common.cuh"

namespace seedrl {

// ------------------------------------------------------------------------------------------------
// geometry
long long planes_positions(int N, int H, int W) {
  const long long Q = (long long)N * (H + 1) * (W + 2);
  // every storage position a consumer's TMA box can touch inside its declared extent is written
  // (zeros) by the producer: tiles read up to 2*PW+2 past Q, shifted maps drop up to 64 positions
  return ((Q + 2 * (W + 2) + 2 + 256 + 127) / 128) * 128;
}
size_t planes_bytes(int N, int H, int W, int C) {
  return (size_t)planes_positions(N, H, W) * 16 * 2 * (C / 8);
}

// Positions per TMA box row.  The TMA engine pays a fixed cost per box row, so rows are as long as
// the 256-element box limit allows: 128 positions x 16 B = 256 x uint64.  Tiles start on multiples of it.
constexpr int kPlanesChunk = 128;

// 3-D view of a plane tensor starting `shift` positions in: {one chunk of CH positions as 2*CH
// uint64, chunks, planes}; box = {2*CH, box_chunks, box_planes}.  Out-of-extent chunks read as zeros.
static int make_plane_map(CUtensorMap* tm, const void* base, long long Lp, int planes, int shift,
                          int CH, int box_chunks, int box_planes) {
  EncodeTiledFn enc = encode_tiled_fn();
  if (!enc) return set_error(SEEDRL_ERR_INTERNAL, "cuTensorMapEncodeTiled is not available");
  if (box_chunks < 1 || box_chunks > 256 || box_planes < 1 || box_planes > planes)
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "conv planes: TMA box out of range");
  const cuuint64_t gdim[3] = {(cuuint64_t)(2 * CH), (cuuint64_t)((Lp - shift) / CH), (cuuint64_t)planes};
  const cuuint64_t gstr[2] = {(cuuint64_t)CH * 16, (cuuint64_t)Lp * 16};
  const cuuint32_t box[3] = {(cuuint32_t)(2 * CH), (cuuint32_t)box_chunks, (cuuint32_t)box_planes};
  const cuuint32_t estr[3] = {1, 1, 1};
  void* addr = const_cast<char*>(reinterpret_cast<const char*>(base)) + (size_t)shift * 16;
  const CUresult r = enc(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 3, addr, gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                         CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[128];
    snprintf(msg, sizeof msg, "cuTensorMapEncodeTiled failed (%d) Lp=%lld planes=%d shift=%d box=%dx%d", (int)r, Lp,
             planes, shift, box_chunks, box_planes);
    return set_error(SEEDRL_ERR_INTERNAL, msg);
  }
  return SEEDRL_OK;
}

__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* dst, const CUtensorMap* tm, int c0, int c1, int c2,
                                            uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];" ::
          "r"(smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(tm)), "r"(c0), "r"(c1), "r"(c2), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ float bf16lo(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float bf16hi(uint32_t w) { return __uint_as_float(w & 0xFFFF0000u); }

// ------------------------------------------------------------------------------------------------
// forward / data gradient
struct ConvpArgs {
  ConvGeom g;
  int Lp;                      // storage positions per plane (input and output share the geometry)
  int nch;                     // chunks per staged tile (box_chunks of the map)
  int chunk;                   // positions per chunk
  int ntiles;
  int nb;                      // smem stages
  const uint4* wq;             // packed weights [hi | lo], conv_tc_kernels.cu layout
  const float* bias;           // [COUT] or null
  const uint4* mask;           // hi planes of the ReLU'd forward activation (COUT/8 planes) or null
  const uint4* res;            // residual plane tensor (COUT channels) or null
  uint4* out_raw;              // plane tensor or null
  uint4* out_relu;             // plane tensor (ReLU applied) or null
  float* out_nhwc;             // fp32 [N,H,W,COUT] or null
  int* err;
};

constexpr int kCpWarpgroups = 4;                         // MMA + epilogue warpgroups: warps 0 .. 15
constexpr int kCpThreads = 128 * kCpWarpgroups + 32;     // + the TMA producer warp
constexpr int kCpM = 128;
constexpr int kCpMaxStages = 4;

// 4 x 4 transpose of float2 elements across the lanes of a quad (q = lane & 3): on entry slot u of
// lane s holds element (s, u), on exit slot s of lane u holds it.  Two butterfly stages; in stage b
// an element moves iff bit b of its lane and of its slot differ.
__device__ __forceinline__ void quad_transpose(float2 (&t)[4], int q) {
#pragma unroll
  for (int b = 1; b <= 2; b <<= 1) {
    const bool up = (q & b) != 0;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (u & b) continue;
      const float2 send = up ? t[u] : t[u | b];
      const float2 r = make_float2(__shfl_xor_sync(0xffffffffu, send.x, b), __shfl_xor_sync(0xffffffffu, send.y, b));
      if (up) t[u] = r; else t[u | b] = r;
    }
  }
}

template <int CIN, int COUT, int NSUB>
__global__ void __launch_bounds__(kCpThreads, 1)
convp_kernel(const __grid_constant__ CUtensorMap tm_in, const ConvpArgs a) {
  constexpr int G = CIN / 8, GO = COUT / 8, NS = CIN / 16;
  constexpr int MT = NSUB * kCpM;
  constexpr int NBLK = 2 * NSUB;                         // 64-position blocks per tile
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int PW = a.g.PW, nb = a.nb;
  const uint32_t P = (uint32_t)(a.nch * a.chunk) * 16u;  // plane stride in a stage (bytes)
  const uint32_t stage_bytes = 2u * G * P;
  uint8_t* s_stage = smem_raw;                           // [nb][hi G planes | lo G planes]
  uint4* s_b = reinterpret_cast<uint4*>(smem_raw + (size_t)nb * stage_bytes);   // 2 * 9*CIN*COUT bf16
  float* s_bias = reinterpret_cast<float*>(s_b + 2 * 9 * CIN * COUT / 8);
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_bias + COUT);
  uint64_t* s_empty = s_full + kCpMaxStages;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  for (int i = tid; i < 2 * 9 * CIN * COUT / 8; i += kCpThreads) s_b[i] = __ldg(a.wq + i);
  if (tid < COUT) s_bias[tid] = a.bias ? __ldg(a.bias + tid) : 0.f;
  if (tid == 0) {
    for (int i = 0; i < nb; ++i) {
      mbar_init(s_full + i, 1);
      mbar_init(s_empty + i, 4 * kCpWarpgroups);       // every consumer warp, once per tile
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_in)) : "memory");
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // weights: generic -> async proxy
  __syncthreads();

  const int my_tiles = ((int)blockIdx.x < a.ntiles) ? (a.ntiles - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  bool timed_out = false;

  if (warp == 4 * kCpWarpgroups) {
    // ================================ TMA producer ============================================
    if (elect_one()) {
      for (int it = 0; it < my_tiles; ++it) {
        const int s = it % nb;
        if (it >= nb && !mbar_wait_bounded(s_empty + s, (uint32_t)(((it / nb) - 1) & 1))) { timed_out = true; break; }
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        mbar_expect_tx(s_full + s, stage_bytes);
        tma_load_3d(s_stage + (size_t)s * stage_bytes, &tm_in, 0, tile * MT / a.chunk, 0, s_full + s);
      }
    }
    __syncwarp();
  } else {
    // ============================ MMA + epilogue warpgroups ===================================
    // The tensor core reads the A tile (positions x 16 channels) from shared memory for EVERY
    // instruction -- that, not the FLOP rate, bounds small-N MMAs.  So the bf16x3 product is issued
    // as TWO reads of the activations per (tap, slab): hi(a) x [hi(w) | lo(w)] as one N = 2*COUT
    // instruction, lo(a) x hi(w) accumulated onto its first half; the epilogue adds the halves.
    // Each warpgroup runs one block's MMAs and then its epilogue; the epilogue overlaps the MMAs of
    // the other warpgroups, which take the next blocks.
    const int cw = warp >> 2;
    const size_t plane_u = (size_t)a.Lp;          // plane stride in 16-byte units (global)
    if (blockIdx.x == 0) {                        // head margin s in [0, PW + 1): zeros
      const uint4 z = make_uint4(0u, 0u, 0u, 0u);
      for (int i = tid; i < (PW + 1) * 2 * GO; i += 128 * kCpWarpgroups) {
        const int pl = i / (PW + 1), s = i - pl * (PW + 1);
        if (a.out_raw) a.out_raw[(size_t)pl * plane_u + s] = z;
        if (a.out_relu) a.out_relu[(size_t)pl * plane_u + s] = z;
      }
    }
    // epilogue thread = (position row, every other channel group).  In the accumulator the 4 lanes
    // of a quad hold rows r and r + 8, two channels of every group each; after the quad transposes
    // lane l holds all 8 channels of row r + 8 (l & 1) in channel groups (l & 3) / 2 + 2k.
    const int q = lane & 3;
    const int row = 16 * (warp & 3) + (lane >> 2) + 8 * (q & 1);
    const uint32_t b_base = smem_u32(s_b);
    const uint64_t db0 = gmma_desc(b_base, (uint32_t)(2 * GO) * 128u, 128u);
    for (int it = 0; it < my_tiles; ++it) {
      const int s = it % nb;
      const int tile = (int)blockIdx.x + it * (int)gridDim.x;
      if (!mbar_wait_bounded(s_full + s, (uint32_t)((it / nb) & 1))) { timed_out = true; break; }
      // the CTA's blocks, concatenated over its tiles, go round-robin to the warpgroups; one with
      // no block in this tile releases the stage at once
      const int m0 = (cw - it * NBLK) & (kCpWarpgroups - 1);
      if (m0 >= NBLK && lane == 0) mbar_arrive(s_empty + s);
      const uint32_t a_base = smem_u32(s_stage + (size_t)s * stage_bytes);
      // descriptors are advanced by adding to their address field (16-byte units)
      const uint64_t da0 = gmma_desc(a_base, P, 128u);
      const uint64_t lo_off = (uint64_t)((G * P) >> 4), slab_off = (uint64_t)((2 * P) >> 4);
#pragma unroll 1
      for (int m = m0; m < NBLK; m += kCpWarpgroups) {
        float acc[COUT];                          // 64 x 2*COUT: [a*hi(w) + lo(a)*hi(w) | hi(a)*lo(w)]
#pragma unroll
        for (int i = 0; i < COUT; ++i) acc[i] = 0.f;
        wgmma_fence_acc<COUT>(acc);
        wgmma_fence();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const uint64_t off = (uint64_t)(m * 64 + (tap / 3) * PW + (tap % 3));
#pragma unroll
          for (int sl = 0; sl < NS; ++sl) {
            const uint64_t da = da0 + off + (uint64_t)sl * slab_off;
            const uint64_t db = db0 + (uint64_t)((tap * NS + sl) * (COUT * 64 / 16));
            Wgmma<2 * COUT>::template mma<0, 0>(acc, da, db, 1u);
            Wgmma<COUT>::template mma<0, 0>(acc, da + lo_off, db, 1u);
          }
        }
        wgmma_commit();
        // the mask / residual operands are loaded while the MMAs run, so their latency is not
        // added after the wait
        const int p = tile * MT + m * 64 + row;
        const int sp = p + PW + 1;
        const int pix = out_pixel(a.g, p);
        uint4 mk[GO / 2], rh[GO / 2], rl[GO / 2];
        if (pix >= 0) {
#pragma unroll
          for (int k = 0; k < GO / 2; ++k) {
            const int go = (q >> 1) + 2 * k;
            if (a.mask) mk[k] = __ldg(a.mask + (size_t)go * plane_u + sp);
            if (a.res) {
              rh[k] = __ldg(a.res + (size_t)go * plane_u + sp);
              rl[k] = __ldg(a.res + (size_t)(GO + go) * plane_u + sp);
            }
          }
        }
        wgmma_wait<0>();
        wgmma_fence_acc<COUT>(acc);
        // this warpgroup's last block of the tile: its MMAs no longer read the stage
        if (m + kCpWarpgroups >= NBLK && lane == 0) mbar_arrive(s_empty + s);
        // bias / mask / residual -> stores
        const bool in_store = sp < a.Lp;
#pragma unroll
        for (int k = 0; k < GO / 2; ++k) {
          const int go = (q >> 1) + 2 * k;
          // slot u: hi + lo halves of channel group 2k + u/2, row r + 8 (u & 1), channels 2q, 2q + 1
          float2 t[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const int j = 2 * k + (u >> 1), h = u & 1;
            t[u] = make_float2(acc[4 * j + 2 * h] + acc[4 * (j + GO) + 2 * h],
                               acc[4 * j + 2 * h + 1] + acc[4 * (j + GO) + 2 * h + 1]);
          }
          quad_transpose(t, q);
          float x[8];
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            x[2 * e] = t[e].x + s_bias[go * 8 + 2 * e];
            x[2 * e + 1] = t[e].y + s_bias[go * 8 + 2 * e + 1];
          }
          if (pix >= 0 && a.mask) {
            const uint32_t mw[4] = {mk[k].x, mk[k].y, mk[k].z, mk[k].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              x[2 * e] = bf16lo(mw[e]) > 0.f ? x[2 * e] : 0.f;
              x[2 * e + 1] = bf16hi(mw[e]) > 0.f ? x[2 * e + 1] : 0.f;
            }
          }
          if (pix >= 0 && a.res) {
            const uint32_t hw[4] = {rh[k].x, rh[k].y, rh[k].z, rh[k].w};
            const uint32_t lw[4] = {rl[k].x, rl[k].y, rl[k].z, rl[k].w};
#pragma unroll
            for (int e = 0; e < 4; ++e) {
              x[2 * e] += bf16lo(hw[e]) + bf16lo(lw[e]);
              x[2 * e + 1] += bf16hi(hw[e]) + bf16hi(lw[e]);
            }
          }
          if (pix < 0) {
#pragma unroll
            for (int e = 0; e < 8; ++e) x[e] = 0.f;
          }
          const float4 xa = make_float4(x[0], x[1], x[2], x[3]), xb = make_float4(x[4], x[5], x[6], x[7]);
          if (a.out_raw && in_store) {
            a.out_raw[(size_t)go * plane_u + sp] = pack8_bf16(xa, xb);
            a.out_raw[(size_t)(GO + go) * plane_u + sp] = pack8_bf16(bf16_resid4(xa), bf16_resid4(xb));
          }
          if (a.out_relu && in_store) {
            const float4 ra = make_float4(fmaxf(xa.x, 0.f), fmaxf(xa.y, 0.f), fmaxf(xa.z, 0.f), fmaxf(xa.w, 0.f));
            const float4 rb = make_float4(fmaxf(xb.x, 0.f), fmaxf(xb.y, 0.f), fmaxf(xb.z, 0.f), fmaxf(xb.w, 0.f));
            a.out_relu[(size_t)go * plane_u + sp] = pack8_bf16(ra, rb);
            a.out_relu[(size_t)(GO + go) * plane_u + sp] = pack8_bf16(bf16_resid4(ra), bf16_resid4(rb));
          }
          if (a.out_nhwc && pix >= 0) {
            float4* o = reinterpret_cast<float4*>(a.out_nhwc + (size_t)pix * COUT + go * 8);
            o[0] = xa; o[1] = xb;
          }
        }
      }
    }
  }
  if (timed_out && a.err) atomicExch(a.err, 1);
}

template <int CIN, int COUT, int NSUB>
static int launch_convp(const PlaneConv& c, cudaStream_t st) {
  const ConvGeom g = make_geom(c.N, c.H, c.W);
  constexpr int MT = NSUB * kCpM;
  const long long Lp = planes_positions(c.N, c.H, c.W);
  if (Lp + MT + 4 * g.PW >= (1LL << 31))
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "convp: batch too large for 32-bit positions");
  const int L = MT + 2 * g.PW + 2;
  const int CH = kPlanesChunk;
  const int nch = (L + CH - 1) / CH;
  const size_t stage = (size_t)2 * (CIN / 8) * nch * CH * 16;
  const size_t fixed = (size_t)2 * 9 * CIN * COUT * 2 + COUT * 4 + 2 * kCpMaxStages * 8;
  int nb = kCpMaxStages;
  while (nb > 1 && nb * stage + fixed > 227 * 1024) --nb;
  if (nb < 2) return kPlanesTryNext;
  const size_t smem = nb * stage + fixed;
  CUtensorMap tm;
  SEEDRL_TRY(make_plane_map(&tm, c.in, Lp, 2 * (CIN / 8), 0, CH, nch, 2 * (CIN / 8)));
  SEEDRL_CUDA(allow_smem<convp_kernel<CIN, COUT, NSUB>>(227 * 1024));
  ConvpArgs a;
  a.g = g; a.Lp = (int)Lp; a.nch = nch; a.chunk = CH; a.nb = nb;
  a.ntiles = (int)((Lp - g.PW - 1 + MT - 1) / MT);       // every storage position >= PW + 1 is written
  a.wq = reinterpret_cast<const uint4*>(c.wq); a.bias = c.bias;
  a.mask = reinterpret_cast<const uint4*>(c.mask); a.res = reinterpret_cast<const uint4*>(c.res);
  a.out_raw = reinterpret_cast<uint4*>(c.out_raw); a.out_relu = reinterpret_cast<uint4*>(c.out_relu);
  a.out_nhwc = c.out_nhwc; a.err = c.err;
  const int grid = a.ntiles < kNumSMs ? a.ntiles : kNumSMs;
  convp_kernel<CIN, COUT, NSUB><<<grid, kCpThreads, smem, st>>>(tm, a);
  count_launch(g_conv_cat, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

bool convp_supported(int cin, int cout) {
  return (cin == 16 || cin == 32) && (cout == 16 || cout == 32);
}

int convp_forward(int cin, int cout, const PlaneConv& c, cudaStream_t st) {
  // big tiles amortise the halo; small problems (inference batches) take 128-position tiles so
  // that every SM still gets work
  const long long Lp = planes_positions(c.N, c.H, c.W);
  const bool small = Lp / 512 < 2 * kNumSMs;
#define SEEDRL_CP_CASE(CI, CO_)                                                   \
  if (cin == CI && cout == CO_) {                                                 \
    int rc = kPlanesTryNext;                                                      \
    if (!small) rc = launch_convp<CI, CO_, 4>(c, st);                             \
    if (rc == kPlanesTryNext) rc = launch_convp<CI, CO_, 2>(c, st);               \
    if (rc == kPlanesTryNext) rc = launch_convp<CI, CO_, 1>(c, st);               \
    if (rc == kPlanesTryNext) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "convp: image too wide"); \
    return rc;                                                                    \
  }
  SEEDRL_CP_CASE(16, 16)
  SEEDRL_CP_CASE(16, 32)
  SEEDRL_CP_CASE(32, 16)
  SEEDRL_CP_CASE(32, 32)
#undef SEEDRL_CP_CASE
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "convp: unsupported (cin,cout)");
}

// ------------------------------------------------------------------------------------------------
// weight + bias gradient
//   dW[kh][kw][ci][co] = sum_p x~[p + kh*PW + kw][ci] * dy[p][co]
//                      = sum_j x~[j + PW + kw][ci] * dy[j + (2 - kh)*PW + 1][co]      (storage positions,
//                                                                                    j = p + (kh-1)*PW)
// GEMM with K = positions j (chunks of KC), M = (kw, ci) rows (+ one row whose accumulator is the
// bias gradient), N = (hi | lo, co) columns, one MMA per kh.  Each operand is copied from L2 ONCE
// per chunk, plus a halo, and the nine tap shifts are made on chip:
//   x  hi + lo planes over [j0 + PW, j0 + PW + KC + 8)           -> A, built in registers:
//      ldmatrix.trans with each lane's row address moved by its kw; the bias row (1.0 in channel
//      0) and the rows past it are constant fragments
//   dy hi + lo planes over [j0 + 1, j0 + 1 + KC + T), T = 2*PW rounded up to 8   -> B, MN-major in
//      shared memory; kh is the descriptor start address moved by (2 - kh) * PW positions
// A stage is copied per plane as KC/CH rows of CH positions plus a halo of 8-position rows, so the
// halo is not rounded up to a whole CH-position row.  Per 16 positions and kh:
//   hi(x) x [hi(dy) | lo(dy)]   N = 2*COUT
//   lo(x) x  hi(dy)             N = COUT, accumulated onto the first half
// Terms with j < 0 pair the zero row above the first image with dy and vanish.  Warp 4*NCW issues
// the TMA copies.  Each 64-row M-tile has KSPL warpgroups that split the three kh between them (one
// each for 16-channel inputs, so one warpgroup's fragment loads and waits run under the others'
// MMAs; one for all three at 32 channels, where two M-tiles already give two warpgroups).  Every
// warpgroup multiplies every chunk of the CTA, in order, into its own accumulator columns: each
// output element is summed over the same positions, in the same order and in the same MMA
// groupings whichever warpgroup holds it, so the partials do not depend on the split.
struct WgradpArgs {
  int PW, T, nchunks, nb;               // dy halo positions per chunk; K chunks; stages
  int chunk;                            // positions per TMA box row of the main copies
  float* partial;                       // [grid][9*CIN*COUT + COUT]
  int* err;
};

constexpr int kWpMaxStages = 6;
constexpr int kWpHaloRow = 8;           // positions per TMA box row of the halo copies
__host__ __device__ constexpr int wgradp_mtiles(int CP) { return 3 * CP + 1 <= 64 ? 1 : 2; }
__host__ __device__ constexpr int wgradp_khsplit(int CP) { return CP == 16 ? 3 : 1; }   // warpgroups per M-tile
__host__ __device__ constexpr int wgradp_threads(int CP) { return 128 * wgradp_mtiles(CP) * wgradp_khsplit(CP) + 32; }

struct WgradMaps { CUtensorMap x, x_halo, dy, dy_halo; };

template <int CP, int COUT, int KC>
__global__ void __launch_bounds__(wgradp_threads(CP), 1)
wgradp_kernel(const __grid_constant__ WgradMaps tm, const WgradpArgs a) {
  constexpr int G = CP / 8, GO = COUT / 8;
  constexpr int MT = wgradp_mtiles(CP), KSPL = wgradp_khsplit(CP), NCW = MT * KSPL;
  constexpr int NKH = 3 / KSPL;                             // kh per warpgroup
  constexpr int NW = 9 * CP * COUT + COUT;
  constexpr uint32_t Px = (KC + kWpHaloRow) * 16;           // x plane stride in a stage (bytes)
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int nb = a.nb, PW = a.PW;
  const uint32_t Pd = (uint32_t)(KC + a.T) * 16u;           // dy plane stride
  const uint32_t x_bytes = 2u * G * Px;
  const uint32_t stage_bytes = x_bytes + 2u * GO * Pd;      // [x hi | x lo | dy hi | dy lo]
  uint64_t* s_full = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* s_empty = s_full + kWpMaxStages;
  uint8_t* s_stage = smem_raw + 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    for (int i = 0; i < kWpMaxStages; ++i) { mbar_init(s_full + i, 1); mbar_init(s_empty + i, 4 * NCW); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  const int my_chunks = ((int)blockIdx.x < a.nchunks) ? (a.nchunks - 1 - (int)blockIdx.x) / (int)gridDim.x + 1 : 0;
  bool timed_out = false;

  if (warp == 4 * NCW) {
    if (elect_one()) {
      for (int it = 0; it < my_chunks; ++it) {
        const int s = it % nb;
        if (it >= nb && !mbar_wait_bounded(s_empty + s, (uint32_t)(((it / nb) - 1) & 1))) { timed_out = true; break; }
        const int j0 = ((int)blockIdx.x + it * (int)gridDim.x) * KC;
        uint8_t* xs = s_stage + (size_t)s * stage_bytes;
        uint8_t* ds = xs + x_bytes;
        mbar_expect_tx(s_full + s, stage_bytes);
        for (int p = 0; p < 2 * G; ++p) {
          tma_load_3d(xs + p * Px, &tm.x, 0, j0 / a.chunk, p, s_full + s);
          tma_load_3d(xs + p * Px + KC * 16, &tm.x_halo, 0, (j0 + KC) / kWpHaloRow, p, s_full + s);
        }
        for (int p = 0; p < 2 * GO; ++p) {
          tma_load_3d(ds + p * Pd, &tm.dy, 0, j0 / a.chunk, p, s_full + s);
          tma_load_3d(ds + p * Pd + KC * 16, &tm.dy_halo, 0, (j0 + KC) / kWpHaloRow, p, s_full + s);
        }
      }
    }
    __syncwarp();
  } else {
    const int cw = warp >> 2, mt = cw % MT, kh0 = (cw / MT) * NKH;
    // M group m (8 rows) = (kw, g) = (m / G, m % G) for m < 3G.  This lane gives row (lane & 7) of
    // ldmatrix matrix lane >> 3: M group mg0 + ((lane >> 3) & 1), K half lane >> 4
    const int mg0 = 8 * mt + 2 * (warp & 3);
    const int mg = mg0 + ((lane >> 3) & 1);
    const uint32_t a_off = (mg < 3 * G ? (uint32_t)(mg % G) * Px + (uint32_t)(mg / G) * 16u : 0u) +
                           (uint32_t)((lane >> 4) * 8 + (lane & 7)) * 16u;
    // groups past the data: group 3G is the bias row (row 0 = 1.0, its lo part 0), the rest zeros
    const bool data0 = mg0 < 3 * G, data1 = mg0 + 1 < 3 * G;
    const uint32_t one = (lane >> 2) == 0 ? 0x3F803F80u : 0u;
    const uint32_t c0 = mg0 == 3 * G ? one : 0u, c1 = mg0 + 1 == 3 * G ? one : 0u;
    float acc[NKH][COUT];                         // per kh: 64 x 2*COUT [x * hi(dy) | hi(x) * lo(dy)]
#pragma unroll
    for (int i = 0; i < NKH * COUT; ++i) (&acc[0][0])[i] = 0.f;
    wgmma_fence_acc<NKH * COUT>(&acc[0][0]);
    // B descriptors: the start address is in the low word (beside LBO), so offsets are 32-bit adds
    const uint64_t desc0 = gmma_desc(0u, 128u, Pd);
    const uint32_t desc_lo = (uint32_t)desc0, desc_hi = (uint32_t)(desc0 >> 32);
    for (int it = 0; it < my_chunks; ++it) {
      const int s = it % nb;
      if (!mbar_wait_bounded(s_full + s, (uint32_t)((it / nb) & 1))) { timed_out = true; break; }
      const uint32_t sb = smem_u32(s_stage + (size_t)s * stage_bytes);
      const uint32_t xb = sb + a_off;
      const uint32_t db = desc_lo + ((sb + x_bytes) >> 4) + (uint32_t)((2 - kh0) * PW);     // kh = kh0
      uint32_t ah[2][4], al[2][4];                // fragments of 16 positions, double-buffered
#pragma unroll
      for (int ks = 0; ks < KC / 16; ++ks) {
        uint32_t(&h)[4] = ah[ks & 1];
        uint32_t(&l)[4] = al[ks & 1];
        ldsm_x4_trans(h, xb + ks * 256);
        ldsm_x4_trans(l, xb + G * Px + ks * 256);
        if (!data0) { h[0] = h[2] = c0; l[0] = l[2] = 0u; }
        if (!data1) { h[1] = h[3] = c1; l[1] = l[3] = 0u; }
        wgmma_fence();
#pragma unroll
        for (int kh = 0; kh < NKH; ++kh) {
          const uint64_t b = make_desc64(db - (uint32_t)(kh * PW) + (uint32_t)(ks * 16), desc_hi);
          WgmmaRA<2 * COUT>::template mma<1>(acc[kh], h, b, 1u);
          WgmmaRA<COUT>::template mma<1>(acc[kh], l, b, 1u);
        }
        wgmma_commit();
        wgmma_wait<1>();                          // ks - 1 is done: its fragment buffer is free
      }
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(s_empty + s);
    }
    wgmma_fence_acc<NKH * COUT>(&acc[0][0]);
    // ---- rows (kw, ci) of the accumulator -> this CTA's partial ------------------------------------
    float* dst = a.partial + (size_t)blockIdx.x * NW;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = 64 * mt + 16 * (warp & 3) + (lane >> 2) + 8 * h;
      const int kw = row / CP, ci = row - kw * CP;
#pragma unroll
      for (int k = 0; k < NKH; ++k) {
        const int kh = kh0 + k;
#pragma unroll
        for (int j = 0; j < GO; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int co = 8 * j + 2 * (lane & 3) + e;
            const float v = acc[k][4 * j + 2 * h + e] + acc[k][4 * j + 2 * h + e + COUT / 2];
            if (row < 3 * CP) dst[((size_t)(kh * 3 + kw) * CP + ci) * COUT + co] = v;
            else if (row == 3 * CP && kh == 1) dst[9 * CP * COUT + co] = v;   // bias row x the kh = 1 view
          }
        }
      }
    }
  }
  if (timed_out && a.err) atomicExch(a.err, 1);
}

template <int CP, int COUT, int KC>
static int launch_wgradp(int N, int H, int W, const void* x, const void* dy, float* dw, float* db, int* err,
                         WgradBatch* batch, cudaStream_t st) {
  const ConvGeom g = make_geom(N, H, W);
  const long long Lp = planes_positions(N, H, W);
  constexpr int G = CP / 8, GO = COUT / 8;
  const int CH = kPlanesChunk < KC ? kPlanesChunk : KC;    // K chunks start on multiples of KC
  if (KC % CH) return kPlanesTryNext;
  const int T = (2 * g.PW + kWpHaloRow - 1) / kWpHaloRow * kWpHaloRow;
  const size_t stage = (size_t)2 * G * (KC + kWpHaloRow) * 16 + (size_t)2 * GO * (KC + T) * 16;
  int nb = kWpMaxStages;
  while (nb > 1 && 128 + nb * stage > 227 * 1024) --nb;
  if (nb < 2) return kPlanesTryNext;
  const size_t smem = 128 + nb * stage;
  WgradMaps tm;
  SEEDRL_TRY(make_plane_map(&tm.x, x, Lp, 2 * G, g.PW, CH, KC / CH, 1));
  SEEDRL_TRY(make_plane_map(&tm.x_halo, x, Lp, 2 * G, g.PW, kWpHaloRow, 1, 1));
  SEEDRL_TRY(make_plane_map(&tm.dy, dy, Lp, 2 * GO, 1, CH, KC / CH, 1));
  SEEDRL_TRY(make_plane_map(&tm.dy_halo, dy, Lp, 2 * GO, 1, kWpHaloRow, T / kWpHaloRow, 1));
  SEEDRL_CUDA(allow_smem<wgradp_kernel<CP, COUT, KC>>(227 * 1024));
  constexpr int NW = 9 * CP * COUT + COUT;
  WgradpArgs a;
  a.PW = g.PW; a.T = T; a.nb = nb; a.err = err; a.chunk = CH;
  a.nchunks = (int)((g.Q + g.PW + KC - 1) / KC);        // j = p + (kh - 1) * PW ranges over [0, Q + PW)
  const int grid = a.nchunks < kNumSMs ? a.nchunks : kNumSMs;
  if (!batch || batch->n >= kMaxReduceJobs || batch->used + (size_t)grid * NW > batch->cap_floats)
    return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgradp: partial buffer too small");
  a.partial = batch->buf + batch->used;
  batch->used += (size_t)grid * NW;
  wgradp_kernel<CP, COUT, KC><<<grid, wgradp_threads(CP), smem, st>>>(tm, a);
  count_launch(PC_CONV_WGRAD, st);
  SEEDRL_CHECK_LAUNCH();
  batch->jobs[batch->n++] = ReduceJob{a.partial, dw, db, grid, 9 * CP * COUT, COUT};
  return SEEDRL_OK;
}

int wgradp(int cin, int cout, int N, int H, int W, const void* x, const void* dy, float* dw, float* db,
           int* err, WgradBatch* batch, cudaStream_t st) {
  // KC = 256 positions for 16 -> 16 and 128 for 32 output channels: the chunks, and so each CTA's
  // positions and their order, of the weight gradient this path has always computed, so the learner's
  // results stay bit-identical to it.  A shorter chunk only where two stages of the halo'd tiles do
  // not fit (very wide images).
#define SEEDRL_WP_CASE(CI, CO_, KC0)                                                                        \
  if (cin == CI && cout == CO_) {                                                                           \
    int rc = kPlanesTryNext;                                                                                \
    if constexpr (KC0 >= 256) rc = launch_wgradp<CI, CO_, 256>(N, H, W, x, dy, dw, db, err, batch, st);     \
    if (rc == kPlanesTryNext) rc = launch_wgradp<CI, CO_, 128>(N, H, W, x, dy, dw, db, err, batch, st);     \
    if (rc == kPlanesTryNext) rc = launch_wgradp<CI, CO_, 64>(N, H, W, x, dy, dw, db, err, batch, st);      \
    if (rc == kPlanesTryNext) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgradp: does not fit");        \
    return rc;                                                                                              \
  }
  SEEDRL_WP_CASE(16, 16, 256)
  SEEDRL_WP_CASE(16, 32, 128)
  SEEDRL_WP_CASE(32, 32, 128)
#undef SEEDRL_WP_CASE
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "wgradp: unsupported (cin,cout)");
}

// ------------------------------------------------------------------------------------------------
// format kernels (elementwise, HBM-bound; thread = one 16-byte unit = position x 8 channels)
__global__ void to_planes_kernel(ConvGeom g, int Lp, int G, int relu, const float* __restrict__ x,
                                 uint4* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Lp * G) return;
  const int s = (int)(i / G), go = (int)(i - (long long)s * G);     // group fastest: a warp reads whole pixels
  const int pix = in_pixel(g, s);
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  if (pix >= 0) {
    const float4* src = reinterpret_cast<const float4*>(x + (size_t)pix * (G * 8) + go * 8);
    a = __ldg(src); b = __ldg(src + 1);
    if (relu) {
      a.x = fmaxf(a.x, 0.f); a.y = fmaxf(a.y, 0.f); a.z = fmaxf(a.z, 0.f); a.w = fmaxf(a.w, 0.f);
      b.x = fmaxf(b.x, 0.f); b.y = fmaxf(b.y, 0.f); b.z = fmaxf(b.z, 0.f); b.w = fmaxf(b.w, 0.f);
    }
  }
  out[(size_t)go * Lp + s] = pack8_bf16(a, b);
  out[(size_t)(G + go) * Lp + s] = pack8_bf16(bf16_resid4(a), bf16_resid4(b));
}

__global__ void from_planes_kernel(ConvGeom g, int Lp, int G, const uint4* __restrict__ in, float* __restrict__ y) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Lp * G) return;
  const int s = (int)(i / G), go = (int)(i - (long long)s * G);     // group fastest: a warp reads whole pixels
  const int pix = in_pixel(g, s);
  if (pix < 0) return;
  const uint4 h = __ldg(in + (size_t)go * Lp + s), l = __ldg(in + (size_t)(G + go) * Lp + s);
  float4* dst = reinterpret_cast<float4*>(y + (size_t)pix * (G * 8) + go * 8);
  dst[0] = make_float4(bf16lo(h.x) + bf16lo(l.x), bf16hi(h.x) + bf16hi(l.x), bf16lo(h.y) + bf16lo(l.y),
                       bf16hi(h.y) + bf16hi(l.y));
  dst[1] = make_float4(bf16lo(h.z) + bf16lo(l.z), bf16hi(h.z) + bf16hi(l.z), bf16lo(h.w) + bf16lo(l.w),
                       bf16hi(h.w) + bf16hi(l.w));
}

int to_planes(int N, int H, int W, int C, int relu, const float* x, void* out, cudaStream_t st) {
  const ConvGeom g = make_geom(N, H, W);
  const long long Lp = planes_positions(N, H, W);
  const long long n = Lp * (C / 8);
  to_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, (int)Lp, C / 8, relu, x,
                                                                reinterpret_cast<uint4*>(out));
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}
int from_planes(int N, int H, int W, int C, const void* in, float* y, cudaStream_t st) {
  const ConvGeom g = make_geom(N, H, W);
  const long long Lp = planes_positions(N, H, W);
  const long long n = Lp * (C / 8);
  from_planes_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, (int)Lp, C / 8,
                                                                  reinterpret_cast<const uint4*>(in), y);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// Max-pool 3x3 / stride 2, TF 'SAME' (dmlab/networks.py:36-37): fp32 NHWC in -> plane tensors out
// (raw and ReLU'd: the two consumers of the pooled activation, networks.py:52-58) + argmax taps.
__global__ void poolp_fwd_kernel(ConvGeom go_, int Lp, int G, int H, int W, int pt, int pl,
                                 const float* __restrict__ x, uint4* __restrict__ out_raw,
                                 uint4* __restrict__ out_relu, uint8_t* __restrict__ idx) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (long long)Lp * G) return;
  const int s = (int)(i / G), gq = (int)(i - (long long)s * G);
  const int pix = in_pixel(go_, s);           // pooled pixel (n * Ho + ho) * Wo + wo
  float best[8];
  unsigned char arg[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { best[e] = 0.f; arg[e] = 0; }
  if (pix >= 0) {
    const int Wo = go_.W, Ho = go_.H, C = G * 8;
    const int n = pix / (Ho * Wo), r = pix - n * (Ho * Wo), ho = r / Wo, wo = r - ho * Wo;
#pragma unroll
    for (int e = 0; e < 8; ++e) best[e] = -INFINITY;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      const int h = ho * 2 - pt + kh;
      if (h < 0 || h >= H) continue;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const int w = wo * 2 - pl + kw;
        if (w < 0 || w >= W) continue;
        const float4* src = reinterpret_cast<const float4*>(x + ((size_t)(n * H + h) * W + w) * C + gq * 8);
        const float4 a = __ldg(src), b = __ldg(src + 1);
        const float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
        const unsigned char t = (unsigned char)(kh * 3 + kw);
#pragma unroll
        for (int e = 0; e < 8; ++e)
          if (v[e] > best[e]) { best[e] = v[e]; arg[e] = t; }
      }
    }
    uint2 packed;
    packed.x = arg[0] | (arg[1] << 8) | (arg[2] << 16) | ((uint32_t)arg[3] << 24);
    packed.y = arg[4] | (arg[5] << 8) | (arg[6] << 16) | ((uint32_t)arg[7] << 24);
    *reinterpret_cast<uint2*>(idx + (size_t)pix * C + gq * 8) = packed;
  }
  const float4 a = make_float4(best[0], best[1], best[2], best[3]), b = make_float4(best[4], best[5], best[6], best[7]);
  out_raw[(size_t)gq * Lp + s] = pack8_bf16(a, b);
  out_raw[(size_t)(G + gq) * Lp + s] = pack8_bf16(bf16_resid4(a), bf16_resid4(b));
  const float4 ra = make_float4(fmaxf(a.x, 0.f), fmaxf(a.y, 0.f), fmaxf(a.z, 0.f), fmaxf(a.w, 0.f));
  const float4 rb = make_float4(fmaxf(b.x, 0.f), fmaxf(b.y, 0.f), fmaxf(b.z, 0.f), fmaxf(b.w, 0.f));
  out_relu[(size_t)gq * Lp + s] = pack8_bf16(ra, rb);
  out_relu[(size_t)(G + gq) * Lp + s] = pack8_bf16(bf16_resid4(ra), bf16_resid4(rb));
}

// dx[n,h,w,c] = sum over the <= 4 windows containing (h, w) whose argmax is (h, w); dy is a plane
// tensor at the pooled resolution, dx either a plane tensor (full resolution) or fp32 NHWC.
template <bool OUT_PLANES>
__global__ void poolp_bwd_kernel(ConvGeom gf, int Lpf, ConvGeom gp, int Lpp, int G, int pt, int pl,
                                 const uint4* __restrict__ dy, const uint8_t* __restrict__ idx,
                                 uint4* __restrict__ dx_planes, float* __restrict__ dx_nhwc) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int H = gf.H, W = gf.W, Ho = gp.H, Wo = gp.W, C = G * 8;
  int gq, s = 0, pix;
  if (OUT_PLANES) {
    if (i >= (long long)Lpf * G) return;
    s = (int)(i / G); gq = (int)(i - (long long)s * G);
    pix = in_pixel(gf, s);
  } else {
    if (i >= (long long)gf.N * H * W * G) return;
    pix = (int)(i / G); gq = (int)(i - (long long)pix * G);
  }
  float acc[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) acc[e] = 0.f;
  if (pix >= 0) {
    const int n = pix / (H * W), r = pix - n * (H * W), h = r / W, w = r - h * W;
    const int hp = h + pt, wp = w + pl;
#pragma unroll
    for (int dh = 0; dh < 2; ++dh) {
      const int ho = (hp >> 1) - dh;
      const int kh = hp - 2 * ho;
      if (ho < 0 || ho >= Ho || kh > 2) continue;
#pragma unroll
      for (int dw = 0; dw < 2; ++dw) {
        const int wo = (wp >> 1) - dw;
        const int kw = wp - 2 * wo;
        if (wo < 0 || wo >= Wo || kw > 2) continue;
        const unsigned tap = (unsigned)(kh * 3 + kw);
        const size_t o = ((size_t)(n * Ho + ho) * Wo + wo) * C + gq * 8;
        const uint2 t = __ldg(reinterpret_cast<const uint2*>(idx + o));
        const int sp = (n * gp.RH + ho + 1) * gp.PW + wo + 1;
        const uint4 hh = __ldg(dy + (size_t)gq * Lpp + sp), ll = __ldg(dy + (size_t)(G + gq) * Lpp + sp);
        const float gv[8] = {bf16lo(hh.x) + bf16lo(ll.x), bf16hi(hh.x) + bf16hi(ll.x), bf16lo(hh.y) + bf16lo(ll.y),
                             bf16hi(hh.y) + bf16hi(ll.y), bf16lo(hh.z) + bf16lo(ll.z), bf16hi(hh.z) + bf16hi(ll.z),
                             bf16lo(hh.w) + bf16lo(ll.w), bf16hi(hh.w) + bf16hi(ll.w)};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const unsigned te = ((e < 4 ? t.x : t.y) >> (8 * (e & 3))) & 0xFFu;
          if (te == tap) acc[e] += gv[e];
        }
      }
    }
  }
  const float4 a = make_float4(acc[0], acc[1], acc[2], acc[3]), b = make_float4(acc[4], acc[5], acc[6], acc[7]);
  if (OUT_PLANES) {
    dx_planes[(size_t)gq * Lpf + s] = pack8_bf16(a, b);
    dx_planes[(size_t)(G + gq) * Lpf + s] = pack8_bf16(bf16_resid4(a), bf16_resid4(b));
  } else {
    float4* dst = reinterpret_cast<float4*>(dx_nhwc + (size_t)pix * C + gq * 8);
    dst[0] = a; dst[1] = b;
  }
}

int poolp_forward(int N, int H, int W, int C, const float* x, void* out_raw, void* out_relu, uint8_t* idx,
                  cudaStream_t st) {
  int Ho, Wo, pt, pl;
  same_pad3s2(H, &Ho, &pt);
  same_pad3s2(W, &Wo, &pl);
  const ConvGeom g = make_geom(N, Ho, Wo);
  const long long Lp = planes_positions(N, Ho, Wo);
  const long long n = Lp * (C / 8);
  poolp_fwd_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(g, (int)Lp, C / 8, H, W, pt, pl, x,
                                                                reinterpret_cast<uint4*>(out_raw),
                                                                reinterpret_cast<uint4*>(out_relu), idx);
  count_launch(PC_POOL, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

int poolp_backward(int N, int H, int W, int C, const void* dy, const uint8_t* idx, void* dx_planes,
                   float* dx_nhwc, cudaStream_t st) {
  int Ho, Wo, pt, pl;
  same_pad3s2(H, &Ho, &pt);
  same_pad3s2(W, &Wo, &pl);
  const ConvGeom gf = make_geom(N, H, W), gp = make_geom(N, Ho, Wo);
  const long long Lpf = planes_positions(N, H, W), Lpp = planes_positions(N, Ho, Wo);
  if (dx_planes) {
    const long long n = Lpf * (C / 8);
    poolp_bwd_kernel<true><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        gf, (int)Lpf, gp, (int)Lpp, C / 8, pt, pl, reinterpret_cast<const uint4*>(dy), idx,
        reinterpret_cast<uint4*>(dx_planes), nullptr);
  } else {
    const long long n = (long long)N * H * W * (C / 8);
    poolp_bwd_kernel<false><<<(unsigned)((n + 255) / 256), 256, 0, st>>>(
        gf, (int)Lpf, gp, (int)Lpp, C / 8, pt, pl, reinterpret_cast<const uint4*>(dy), idx, nullptr, dx_nhwc);
  }
  count_launch(PC_POOL, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

}  // namespace seedrl
