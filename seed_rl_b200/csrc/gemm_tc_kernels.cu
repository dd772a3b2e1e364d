// Dense-layer GEMMs on the Hopper tensor cores (wgmma): the Linear contractions of
// dmlab/networks.py:105-118,157-169 (Dense(256), LSTM input projection, their data and weight
// gradients) with fp32 storage, bf16 (or bf16x3) operands and fp32 accumulation.
//
//   C[M,N] (=|+=) op(A)[M,K] * op(B)[K,N]      row-major fp32, leading dims lda/ldb/ldc
//   TA: A is stored [K,M] (C = A^T B).   TB: B is stored [N,K] (C = A B^T).
//
// Either storage order of either operand is ALREADY a canonical no-swizzle wgmma layout once
// 8 contiguous elements are packed into one 16-byte bf16 unit:
//   contiguous along K  -> K-major :  planes [K/8][rows][8 k],  LBO = plane stride, SBO = 128 B
//   contiguous along MN -> MN-major:  planes [MN/8][k][8 mn],   LBO = 128 B, SBO = plane stride
// so there is no transpose anywhere: TA / TB only flip the transpose bits of the instruction.
// A CTA owns a 128 x BN tile of C (two warpgroups, 64 rows each, BN <= 128 columns of fp32
// accumulators in registers) and a slice of K (split-K over blockIdx.z); K is walked in blocks
// through two shared-memory stages: all 8 warps convert fp32 global -> bf16 units of stage s while
// the MMAs of stage s^1 run (wgmma.wait_group 1 keeps one K-block in flight).  Split = bf16x3:
// every operand is staged as hi and lo planes and each K-step issues hi*hi + lo*hi + hi*lo.
// Epilogue: accumulators -> fp32 tile in shared memory -> bias / relu / mask / accumulate -> C, or
// -> the split-K workspace, reduced in slice order by gemm_tc_reduce_kernel (deterministic).
#include "kernels.h"
#include "tc_common.cuh"

namespace seedrl {

constexpr int kGtThreads = 256;
constexpr int kGtBM = 128;
constexpr int kGtMaxBN = 128;   // tile width cap: a warpgroup holds 64 x 128 fp32 accumulators = 64 registers/thread
constexpr int kGtBK = 32;       // K elements per staged block

struct GemmTcParams {
  int M, N, K;
  const float* A; int lda;
  const float* B; int ldb;
  float* C; int ldc;            // final output (splits == 1) ...
  float* ws;                    // ... or split-K partials [splits][M][N]
  int BN;                       // tile width: multiple of 16, <= kGtMaxBN
  int kblocks_per_split;        // K blocks (of kGtBK) per blockIdx.z
  int vecA, vecB;               // 16-byte aligned rows: float4 loads
  GemmEpi e;
  int* error_flag;
  ConvGather cg;                // GATHER kernels: op(A) = im2col(cg.x)
};

// 8 consecutive elements along the contiguous direction of a row-major matrix (raw fp32, two
// float4).  `row` / `col0` are global coordinates; rows/cols outside [0,R) x [0,Cn) read as zero.
struct RawUnit { float4 a, b; };
__device__ __forceinline__ RawUnit load_raw(const float* __restrict__ P, int ld, int row, int col0, int R, int Cn,
                                            bool vec) {
  RawUnit r;
  r.a = make_float4(0.f, 0.f, 0.f, 0.f);
  r.b = r.a;
  if (row < R && col0 < Cn) {
    const float* src = P + (size_t)row * ld + col0;
    if (vec && col0 + 8 <= Cn) {
      r.a = __ldg(reinterpret_cast<const float4*>(src));
      r.b = __ldg(reinterpret_cast<const float4*>(src) + 1);
    } else {
      float v[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) v[j] = col0 + j < Cn ? __ldg(src + j) : 0.f;
      r.a = make_float4(v[0], v[1], v[2], v[3]);
      r.b = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
  return r;
}
// 8 consecutive columns (kh, kw, c) of row `pos` = (n, ho, wo) of the im2col matrix, read from the
// NHWC tensor itself: x[n][ho*S + kh][wo*S ...][...] is contiguous over (kw, c) for a fixed kh.
// kc0 % 8 == 0 and KC % 8 == 0 (host-checked), so a unit never straddles two kernel rows.
__device__ __forceinline__ RawUnit load_gather(const ConvGather& g, int pos, int kc0, int R, int Cn) {
  RawUnit r;
  r.a = make_float4(0.f, 0.f, 0.f, 0.f);
  r.b = r.a;
  if (pos < R && kc0 < Cn) {
    const unsigned int t = fast_div((unsigned int)pos, g.wo_mul, g.wo_sh);
    const int wo = pos - (int)t * g.Wo;
    const unsigned int n = fast_div(t, g.ho_mul, g.ho_sh);
    const int ho = (int)t - (int)n * g.Ho;
    const int kh = (int)fast_div((unsigned int)kc0, g.kc_mul, g.kc_sh);
    const int rem = kc0 - kh * g.KC;
    const size_t off = (((size_t)n * g.H + (size_t)(ho * g.S + kh)) * g.W + (size_t)(wo * g.S)) * g.C + rem;
    if (g.u8) {
      const uint2 v = __ldg(reinterpret_cast<const uint2*>(reinterpret_cast<const uint8_t*>(g.x) + off));
      const float k = 1.0f / 255.0f;
      r.a = make_float4((float)(v.x & 0xffu) * k, (float)((v.x >> 8) & 0xffu) * k,
                        (float)((v.x >> 16) & 0xffu) * k, (float)(v.x >> 24) * k);
      r.b = make_float4((float)(v.y & 0xffu) * k, (float)((v.y >> 8) & 0xffu) * k,
                        (float)((v.y >> 16) & 0xffu) * k, (float)(v.y >> 24) * k);
    } else {
      const float4* src = reinterpret_cast<const float4*>(reinterpret_cast<const float*>(g.x) + off);
      r.a = __ldg(src);
      r.b = __ldg(src + 1);
    }
  }
  return r;
}
// -> one bf16x8 unit (+ the residual unit for bf16x3)
template <bool SPLIT>
__device__ __forceinline__ void store_unit(RawUnit r, bool relu, uint4* hi_dst, uint4* lo_dst) {
  if (relu) {
    r.a.x = fmaxf(r.a.x, 0.f); r.a.y = fmaxf(r.a.y, 0.f); r.a.z = fmaxf(r.a.z, 0.f); r.a.w = fmaxf(r.a.w, 0.f);
    r.b.x = fmaxf(r.b.x, 0.f); r.b.y = fmaxf(r.b.y, 0.f); r.b.z = fmaxf(r.b.z, 0.f); r.b.w = fmaxf(r.b.w, 0.f);
  }
  *hi_dst = pack8_bf16(r.a, r.b);
  if (SPLIT) *lo_dst = pack8_bf16(bf16_resid4(r.a), bf16_resid4(r.b));
}

// D += A * B for one K = 16 step of a warpgroup: the tile width is a runtime value (a multiple of 16)
template <int TA, int TB>
__device__ __forceinline__ void gemm_tc_mma(int bn, float* acc, uint64_t a, uint64_t b) {
  switch (bn) {
    case 16: Wgmma<16>::mma<TA, TB>(acc, a, b, 1u); break;
    case 32: Wgmma<32>::mma<TA, TB>(acc, a, b, 1u); break;
    case 48: Wgmma<48>::mma<TA, TB>(acc, a, b, 1u); break;
    case 64: Wgmma<64>::mma<TA, TB>(acc, a, b, 1u); break;
    case 80: Wgmma<80>::mma<TA, TB>(acc, a, b, 1u); break;
    case 96: Wgmma<96>::mma<TA, TB>(acc, a, b, 1u); break;
    case 112: Wgmma<112>::mma<TA, TB>(acc, a, b, 1u); break;
    default: Wgmma<128>::mma<TA, TB>(acc, a, b, 1u); break;
  }
}

template <bool TA, bool TB, bool SPLIT, bool GATHER>
__global__ void __launch_bounds__(kGtThreads)
gemm_tc_kernel(const GemmTcParams p) {
  constexpr int S = SPLIT ? 2 : 1;
  constexpr int KG = kGtBK / 8;                 // 16-byte K-groups per row of a block
  extern __shared__ __align__(128) uint8_t smem_raw[];
  const int BN = p.BN;
  // one stage: [A hi | A lo | B hi | B lo].  Plane strides are padded by one 16-byte unit so
  // that the 8 lanes of a store phase (8 consecutive planes, same row) hit 8 different banks.
  constexpr uint32_t a_ps = TA ? (kGtBK + 1) : (kGtBM + 1);            // A plane stride (units)
  constexpr uint32_t a_units = TA ? (kGtBM / 8) * a_ps : (kGtBK / 8) * a_ps;
  const uint32_t b_ps = TB ? (uint32_t)BN + 1 : (uint32_t)kGtBK + 1;    // B plane stride (units)
  const uint32_t b_units = TB ? (kGtBK / 8) * b_ps : (uint32_t)(BN / 8) * b_ps;
  const int b_items = BN * kGtBK / 8;                                  // 16-byte units actually staged
  const uint32_t stage_units = S * (a_units + b_units);
  uint4* s_buf = reinterpret_cast<uint4*>(smem_raw);
  const int tid = threadIdx.x, wg = tid >> 7;
  const int m0 = blockIdx.y * kGtBM, n0 = blockIdx.x * BN;
  const int kb0 = blockIdx.z * p.kblocks_per_split;
  const int nkb_total = (p.K + kGtBK - 1) / kGtBK;
  const int nkb = min(p.kblocks_per_split, nkb_total - kb0);
  // warpgroup wg multiplies rows [64 wg, 64 wg + 64) of the tile: K-major A holds a row per 16-byte
  // unit of a plane, MN-major A 8 rows per plane
  const uint32_t a_wg = TA ? (uint32_t)wg * 8u * a_ps * 16u : (uint32_t)wg * 64u * 16u;
  float acc[kGtMaxBN / 2];
#pragma unroll
  for (int i = 0; i < kGtMaxBN / 2; ++i) acc[i] = 0.f;
  wgmma_fence_acc<kGtMaxBN / 2>(acc);

  for (int kb = 0; kb < nkb; ++kb) {
    const int st = kb & 1;
    const int k0 = (kb0 + kb) * kGtBK;
    uint4* sA = s_buf + (size_t)st * stage_units;
    uint4* sB = sA + (size_t)S * a_units;
    // ---- stage the K-block: every global load is issued before the first conversion -------
    // consecutive threads take consecutive 8-element groups of the SAME row (coalesced).
    constexpr int AI = (kGtBM * kGtBK / 8) / kGtThreads;       // A units per thread
    constexpr int BI = (kGtMaxBN * kGtBK / 8) / kGtThreads;    // <= BI B units per thread
    RawUnit ra[AI], rb[BI];
#pragma unroll
    for (int r = 0; r < AI; ++r) {
      const int u = tid + r * kGtThreads;
      if (GATHER) {           // rows of the im2col matrix are positions: M of the forward, K of the weight gradient
        if (!TA) ra[r] = load_gather(p.cg, m0 + u / KG, k0 + (u % KG) * 8, p.M, p.K);
        else     ra[r] = load_gather(p.cg, k0 + (u >> 4), m0 + (u & 15) * 8, p.K, p.M);
      } else {
        if (!TA) ra[r] = load_raw(p.A, p.lda, m0 + u / KG, k0 + (u % KG) * 8, p.M, p.K, p.vecA != 0);   // A[M,K]
        else     ra[r] = load_raw(p.A, p.lda, k0 + (u >> 4), m0 + (u & 15) * 8, p.K, p.M, p.vecA != 0);  // A stored [K,M]
      }
    }
    const int bng = BN >> 3;
#pragma unroll
    for (int r = 0; r < BI; ++r) {
      const int u = tid + r * kGtThreads;
      if (u < b_items) {
        if (TB) rb[r] = load_raw(p.B, p.ldb, n0 + u / KG, k0 + (u % KG) * 8, p.N, p.K, p.vecB != 0);  // B stored [N,K]
        else    rb[r] = load_raw(p.B, p.ldb, k0 + u / bng, n0 + (u % bng) * 8, p.K, p.N, p.vecB != 0); // B[K,N]
      }
    }
    // the MMAs that read this stage two K-blocks ago have completed, in both warpgroups
    if (kb >= 2) wgmma_wait<1>();
    __syncthreads();
#pragma unroll
    for (int r = 0; r < AI; ++r) {
      const int u = tid + r * kGtThreads;
      // K-major planes [8 kg][128 m] / MN-major planes [16 mg][64 k]
      const uint32_t o = !TA ? (uint32_t)(u % KG) * a_ps + u / KG : (uint32_t)(u & 15) * a_ps + (u >> 4);
      store_unit<SPLIT>(ra[r], p.e.a_relu != 0, sA + o, sA + a_units + o);
    }
#pragma unroll
    for (int r = 0; r < BI; ++r) {
      const int u = tid + r * kGtThreads;
      if (u < b_items) {
        // K-major planes [8 kg][BN n] / MN-major planes [BN/8 ng][64 k]
        const uint32_t o = TB ? (uint32_t)(u % KG) * b_ps + u / KG : (uint32_t)(u % bng) * b_ps + u / bng;
        store_unit<SPLIT>(rb[r], false, sB + o, sB + b_units + o);
      }
    }
    // generic-proxy smem writes -> visible to the tensor core's async proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    wgmma_fence();
    const uint32_t a_addr = smem_u32(sA) + a_wg, b_addr = smem_u32(sB);
#pragma unroll
    for (int ks = 0; ks < kGtBK / 16; ++ks) {
      // K-major: two K-groups = two planes (LBO = plane stride);  MN-major: 16 k-rows = 256 B
      const uint64_t da = TA ? gmma_desc(a_addr + ks * 256u, 128u, a_ps * 16u)
                             : gmma_desc(a_addr + ks * 2u * a_ps * 16u, a_ps * 16u, 128u);
      const uint64_t db = TB ? gmma_desc(b_addr + ks * 2u * b_ps * 16u, b_ps * 16u, 128u)
                             : gmma_desc(b_addr + ks * 256u, 128u, b_ps * 16u);
      gemm_tc_mma<TA ? 1 : 0, TB ? 0 : 1>(BN, acc, da, db);
      if (SPLIT) {   // + lo(a)*hi(b) + hi(a)*lo(b); the address field counts 16-byte units
        gemm_tc_mma<TA ? 1 : 0, TB ? 0 : 1>(BN, acc, da + a_units, db);
        gemm_tc_mma<TA ? 1 : 0, TB ? 0 : 1>(BN, acc, da, db + b_units);
      }
    }
    wgmma_commit();
  }
  wgmma_wait<0>();
  wgmma_fence_acc<kGtMaxBN / 2>(acc);

  // ---- epilogue: registers -> fp32 tile in shared memory (aliasing the operand stages, which no
  // MMA reads any more once both warpgroups are here) -> row-contiguous global accesses
  __syncthreads();
  {
    const int ld = BN + 4;
    float* tile = reinterpret_cast<float*>(smem_raw);
    const int w = (tid >> 5) & 3, l = tid & 31;
    const int r0 = wg * 64 + 16 * w + (l >> 2), c0 = 2 * (l & 3);
#pragma unroll
    for (int j = 0; j < kGtMaxBN / 8; ++j) {
      if (8 * j < BN) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          *reinterpret_cast<float2*>(tile + (size_t)(r0 + 8 * h) * ld + 8 * j + c0) =
              make_float2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1]);
      }
    }
    __syncthreads();
    const bool partial = p.ws != nullptr;
    for (int i = tid; i < kGtBM * BN; i += kGtThreads) {
      const int r = i / BN, c = i - r * BN;
      const int gm = m0 + r, gn = n0 + c;
      if (gm < p.M && gn < p.N) {
        float x = tile[(size_t)r * ld + c];
        if (partial) {
          p.ws[((size_t)blockIdx.z * p.M + gm) * p.N + gn] = x;
        } else {
          if (p.e.bias) x += __ldg(p.e.bias + gn);
          if (p.e.relu) x = fmaxf(x, 0.f);
          if (p.e.mask) x = __ldg(p.e.mask + (size_t)gm * p.e.ldm + gn) > 0.f ? x : 0.f;
          float* cp = p.C + (size_t)gm * p.ldc + gn;
          *cp = p.e.accumulate ? *cp + x : x;
        }
      }
    }
  }
}

// C = epilogue(sum_z ws[z]) in slice order.  VEC: four columns per thread (N % 4 == 0; the
// partial planes are then 16-byte aligned), all `splits` loads of a thread independent.
template <bool VEC>
__global__ void gemm_tc_reduce_kernel(int M, int N, int splits, const float* __restrict__ ws,
                                      float* __restrict__ C, int ldc, GemmEpi e) {
  constexpr int W = VEC ? 4 : 1;
  const int i = (blockIdx.x * blockDim.x + threadIdx.x) * W;
  if (i >= M * N) return;
  const int m = i / N, n = i - m * N;
  float x[W];
#pragma unroll
  for (int j = 0; j < W; ++j) x[j] = 0.f;
  const size_t plane = (size_t)M * N;
#pragma unroll 4
  for (int z = 0; z < splits; ++z) {
    if (VEC) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(ws + (size_t)z * plane + i));
      x[0] += v.x; x[W > 1 ? 1 : 0] += v.y; x[W > 2 ? 2 : 0] += v.z; x[W > 3 ? 3 : 0] += v.w;
    } else {
      x[0] += __ldcs(ws + (size_t)z * plane + i);
    }
  }
#pragma unroll
  for (int j = 0; j < W; ++j) {
    float v = x[j];
    if (e.bias) v += __ldg(e.bias + n + j);
    if (e.relu) v = fmaxf(v, 0.f);
    if (e.mask) v = __ldg(e.mask + (size_t)m * e.ldm + n + j) > 0.f ? v : 0.f;
    float* c = C + (size_t)m * ldc + n + j;
    *c = e.accumulate ? *c + v : v;
  }
}

// Same reduction for many slices (the im2col weight gradients: 64-128 slices of a small M x N): the slices
// of an output are spread over 8 lanes (lane zl sums z = zl, zl + 8, ... in order), the 8 partial sums are
// combined in lane order through shared memory => still a fixed summation order.  CTA = 32 float4 outputs.
__global__ void __launch_bounds__(256)
gemm_tc_reduce_wide_kernel(int M, int N, int splits, const float* __restrict__ ws, float* __restrict__ C, int ldc,
                           GemmEpi e) {
  __shared__ float4 part[8][32];
  const int o = threadIdx.x & 31, zl = threadIdx.x >> 5;
  const int i = (blockIdx.x * 32 + o) * 4;
  const bool in = i < M * N;
  const size_t plane = (size_t)M * N;
  float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
  if (in) {
    int z = zl;
    for (; z + 8 < splits; z += 16) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(ws + (size_t)z * plane + i));
      const float4 w = __ldcs(reinterpret_cast<const float4*>(ws + (size_t)(z + 8) * plane + i));
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
      b.x += w.x; b.y += w.y; b.z += w.z; b.w += w.w;
    }
    if (z < splits) {
      const float4 v = __ldcs(reinterpret_cast<const float4*>(ws + (size_t)z * plane + i));
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
  }
  part[zl][o] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
  __syncthreads();
  if (zl != 0 || !in) return;
  float x[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const float4 v = part[k][o];
    x[0] += v.x; x[1] += v.y; x[2] += v.z; x[3] += v.w;
  }
  const int m = i / N, n = i - m * N;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    float v = x[j];
    if (e.bias) v += __ldg(e.bias + n + j);
    if (e.relu) v = fmaxf(v, 0.f);
    if (e.mask) v = __ldg(e.mask + (size_t)m * e.ldm + n + j) > 0.f ? v : 0.f;
    float* c = C + (size_t)m * ldc + n + j;
    *c = e.accumulate ? *c + v : v;
  }
}

bool gemm_tc_supported(int M, int N, int K) { return M >= 64 && N >= 16 && K >= 32; }

size_t gemm_tc_workspace_bytes() { return (size_t)48 << 20; }

static int g_gemm_gather = 1;
void gemm_tc_set_gather(int on) { g_gemm_gather = on; }
bool gemm_tc_gather_enabled() { return g_gemm_gather != 0; }

bool conv_gather_setup(const void* x, int u8, int N, int H, int W, int C, int K, int S, ConvGather* g) {
  const int Ho = (H - K) / S + 1, Wo = (W - K) / S + 1, KC = K * C;
  if (Ho < 2 || Wo < 2 || KC < 8 || (KC & 7)) return false;
  if ((long long)N * Ho * Wo >= (1ll << 31)) return false;                 // fast_div domain
  if (u8 ? (((W * C) & 7) || ((S * C) & 7) || (reinterpret_cast<uintptr_t>(x) & 7))
         : ((C & 3) || (reinterpret_cast<uintptr_t>(x) & 15)))
    return false;                                                            // 8-byte / 16-byte loads
  g->x = x; g->u8 = u8; g->H = H; g->W = W; g->C = C; g->S = S; g->Ho = Ho; g->Wo = Wo; g->KC = KC;
  fast_div_setup((unsigned int)Wo, &g->wo_mul, &g->wo_sh);
  fast_div_setup((unsigned int)Ho, &g->ho_mul, &g->ho_sh);
  fast_div_setup((unsigned int)KC, &g->kc_mul, &g->kc_sh);
  return true;
}

int gemm_tc(bool ta, bool tb, int split, int M, int N, int K, const float* A, int lda, const float* B,
            int ldb, float* C, int ldc, const GemmEpi& e, float* ws, size_t ws_bytes, int* err,
            cudaStream_t st, const ConvGather* cg) {
  if (M <= 0 || N <= 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(!cg || (!tb && ((ta ? M : K) & 7) == 0), "gathered operand: tb or a ragged kernel row");
  GemmTcParams p;
  if (cg) p.cg = *cg; else p.cg = ConvGather{};
  p.M = M; p.N = N; p.K = K; p.A = A; p.lda = lda; p.B = B; p.ldb = ldb; p.C = C; p.ldc = ldc;
  p.e = e; p.error_flag = err;
  const int n16 = ((N + 15) / 16) * 16;
  int bn = kGtMaxBN;
  if (bn > n16) bn = n16;
  // narrower tiles until the grid can cover the SMs (with split-K below)
  const int nkb_all = ceil_div(K, kGtBK);
  const int kb256 = 256 / kGtBK;                        // K-blocks per 256 elements of K
  while (bn > 64 && ceil_div(M, kGtBM) * ceil_div(N, bn) * (nkb_all >= kb256 ? nkb_all / (kb256 / 2) : 1) < kNumSMs)
    bn >>= 1;
  p.BN = ((bn + 15) / 16) * 16;
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  p.vecA = al16(A) && (lda & 3) == 0;
  p.vecB = al16(B) && (ldb & 3) == 0;
  const int tiles = ceil_div(M, kGtBM) * ceil_div(N, p.BN);
  const int nkb = ceil_div(K, kGtBK);
  // split-K until the grid covers the SMs, keeping >= 128 elements of K per slice and the
  // partials inside the workspace
  int splits = 1;
  while (tiles * splits < kNumSMs && nkb / (splits * 2) >= 128 / kGtBK &&
         (size_t)(splits * 2) * M * N * sizeof(float) <= ws_bytes && ws)
    splits *= 2;
  p.kblocks_per_split = ceil_div(nkb, splits);
  splits = ceil_div(nkb, p.kblocks_per_split);
  p.ws = splits > 1 ? ws : nullptr;
  const int S = split ? 2 : 1;
  const size_t a_un = ta ? (size_t)(kGtBM / 8) * (kGtBK + 1) : (size_t)(kGtBK / 8) * (kGtBM + 1);
  const size_t b_un = tb ? (size_t)(kGtBK / 8) * (p.BN + 1) : (size_t)(p.BN / 8) * (kGtBK + 1);
  size_t smem = (size_t)2 * S * (a_un + b_un) * 16;
  const size_t epi = (size_t)kGtBM * (p.BN + 4) * 4;      // the epilogue's fp32 tile aliases the stages
  if (smem < epi) smem = epi;
  dim3 grid(ceil_div(N, p.BN), ceil_div(M, kGtBM), splits);
#define SEEDRL_GT_LAUNCH2(TA_, TB_, SP_, G_)                                                    \
  do {                                                                                          \
    SEEDRL_CUDA(allow_smem<gemm_tc_kernel<TA_, TB_, SP_, G_>>(200 * 1024));                     \
    gemm_tc_kernel<TA_, TB_, SP_, G_><<<grid, kGtThreads, smem, st>>>(p);                       \
  } while (0)
#define SEEDRL_GT_LAUNCH(TA_, TB_, SP_)                                                         \
  do {                                                                                          \
    if (cg && !(TB_)) SEEDRL_GT_LAUNCH2(TA_, false, SP_, true);                                 \
    else SEEDRL_GT_LAUNCH2(TA_, TB_, SP_, false);                                               \
  } while (0)
  if (split) {
    if (!ta && !tb) SEEDRL_GT_LAUNCH(false, false, true);
    else if (ta && !tb) SEEDRL_GT_LAUNCH(true, false, true);
    else if (!ta && tb) SEEDRL_GT_LAUNCH(false, true, true);
    else SEEDRL_GT_LAUNCH(true, true, true);
  } else {
    if (!ta && !tb) SEEDRL_GT_LAUNCH(false, false, false);
    else if (ta && !tb) SEEDRL_GT_LAUNCH(true, false, false);
    else if (!ta && tb) SEEDRL_GT_LAUNCH(false, true, false);
    else SEEDRL_GT_LAUNCH(true, true, false);
  }
#undef SEEDRL_GT_LAUNCH
#undef SEEDRL_GT_LAUNCH2
  count_launch(PC_GEMM, st);
  SEEDRL_CHECK_LAUNCH();
  if (splits > 1) {
    if ((N & 3) == 0 && splits >= 16)
      gemm_tc_reduce_wide_kernel<<<ceil_div(M * N / 4, 32), 256, 0, st>>>(M, N, splits, ws, C, ldc, e);
    else if ((N & 3) == 0)
      gemm_tc_reduce_kernel<true><<<ceil_div(M * N / 4, 256), 256, 0, st>>>(M, N, splits, ws, C, ldc, e);
    else
      gemm_tc_reduce_kernel<false><<<ceil_div(M * N, 256), 256, 0, st>>>(M, N, splits, ws, C, ldc, e);
    count_launch(PC_GEMM, st);
    SEEDRL_CHECK_LAUNCH();
  }
  return SEEDRL_OK;
}

}  // namespace seedrl
