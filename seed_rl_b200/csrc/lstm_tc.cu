// Persistent LSTM recurrence on the Hopper tensor cores ("tc3"): the Keras LSTMCell(H) of lstm_tiled.cu
// (same equations, same done-resets, same z / hs / cs / hp / dz layouts) with the recurrent products
// h[t-1] U (forward) and dZ[t+1] U^T (BPTT) computed by wgmma in bf16x3: hi*hi + lo*hi + hi*lo,
// fp32 accumulation.  One launch for the forward, one for the BPTT; CTA = (64-row batch tile,
// 16 hidden units), one warpgroup.
//
//   forward  D[64 x 128] = hi(h) [hi(U) | lo(U)]   (+)   D[64 x 64] += lo(h) hi(U)
//            B columns c = gate * 16 + unit (lo at c + 64), K = H.  In the accumulator fragment
//            (tc_common.cuh) columns c, c + 16, c + 32, c + 48 and c + 64 of one row are held by the
//            same thread, so the four gates of a unit and the lo product meet in registers and the cell
//            update runs there; c stays in registers for all T steps.
//   BPTT     D[64 x 32] = hi(dZ[t+1]) [hi(U_u^T) | lo(U_u^T)]  (+)  D[64 x 16] += lo(dZ) hi(U_u^T),
//            K = 4H; dc stays in registers.
//
// The CTA's slice of U is split into bf16 hi / lo planes once and stays in shared memory (forward
// H x 128 columns, BPTT 4H x 32 columns: 66 / 132 KB at H = 256 / 512).  Each step the CTA reads the
// fp32 rows of its batch tile (hp[t] / dz[t+1], which the dU / dW GEMMs need in fp32 anyway) in
// chunks of 128 K-elements, splits them into hi / lo planes in a two-stage ring and issues the MMAs of
// one chunk while the next chunk is loaded.  Rows past the batch are zero in the operand and never
// stored.  All operands are K-major no-swizzle planes [K/8][rows][8 k] (LBO = plane stride, SBO =
// 128 B); plane strides are padded by one 16-byte unit against bank conflicts.
//
// Synchronisation as in lstm_tiled.cu: one monotonic counter per batch tile with a bounded spin (sets
// *err, never hangs), batch tiles contiguous in blockIdx, cooperative launch when the grid fits.
// The MMA order is fixed and no floating-point atomics are used: results are bit-reproducible.
#include "kernels.h"
#include "tc_common.cuh"

namespace seedrl {

constexpr int kLtThreads = 128;      // one warpgroup
constexpr int kLtNU = 16;            // hidden units per CTA
constexpr int kLtM = 64;             // batch rows per CTA (wgmma M)
constexpr int kLtKC = 128;           // K-elements per staged chunk
constexpr int kLtAPS = kLtM + 1;     // A plane stride, 16-byte units
constexpr int kLtStageUnits = 2 * (kLtKC / 8) * kLtAPS;   // hi + lo planes of one chunk
constexpr int kLtUnitsPerThread = kLtM * kLtKC / 8 / kLtThreads;
constexpr int kLtSmemLimit = 227 * 1024;

struct LstmTcArgs {
  int T1, B, nug;
  const float* U;          // [H, 4H]
  const uint8_t* done;     // [T1, B]
  float* z;                // fwd: in x W + b, out activated gates; bwd: activated gates (in)
  const float* h0; const float* c0;
  float* hs; float* cs; float* hp;
  const float* dhs;        // bwd
  float* dz;               // bwd out
  unsigned int* counter;   // [nbt], zeroed by the launcher
  int* err;
};

__device__ __forceinline__ void lt_barrier_arrive(unsigned int* counter) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
  }
}
__device__ __forceinline__ void lt_barrier_wait(unsigned int* counter, unsigned int target, int* err) {
  if (threadIdx.x == 0) {
    int spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(counter) < target) {
      if (++spins > (1 << 24)) { if (err) atomicExch(err, 2); break; }
    }
    __threadfence();
  }
  __syncthreads();
}

// 8 consecutive fp32 of one row -> one hi unit and one lo unit (bf16)
__device__ __forceinline__ void lt_split_store(const float4 (&v)[2], uint4* hi, uint4* lo) {
  *hi = pack8_bf16(v[0], v[1]);
  *lo = pack8_bf16(bf16_resid4(v[0]), bf16_resid4(v[1]));
}

// Global loads of one chunk: rows [0, 64) of the tile x K-elements [k0, k0 + 128) of `src` (row
// stride ld floats, L2 reads: the rows were written by other CTAs of this launch).  Unit u = row *
// 16 + k-group, so 16 consecutive threads read one row's 512 contiguous bytes.
__device__ __forceinline__ void lt_load_chunk(float4 (&r)[kLtUnitsPerThread][2], const float* src, int ld,
                                              int nb, int k0) {
#pragma unroll
  for (int j = 0; j < kLtUnitsPerThread; ++j) {
    const int u = threadIdx.x + j * kLtThreads;
    const int row = u >> 4, kg = u & 15;
    if (row < nb) {
      const float4* p = reinterpret_cast<const float4*>(src + (size_t)row * ld + k0 + kg * 8);
      r[j][0] = __ldcg(p); r[j][1] = __ldcg(p + 1);
    } else {
      r[j][0] = r[j][1] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
}
__device__ __forceinline__ void lt_store_chunk(const float4 (&r)[kLtUnitsPerThread][2], uint4* stage) {
#pragma unroll
  for (int j = 0; j < kLtUnitsPerThread; ++j) {
    const int u = threadIdx.x + j * kLtThreads;
    const int o = (u & 15) * kLtAPS + (u >> 4);
    lt_split_store(r[j], stage + o, stage + (kLtKC / 8) * kLtAPS + o);
  }
}

// ------------------------------------------------------------------------------------------------
template <int H>
__global__ void __launch_bounds__(kLtThreads, 1) lstm_tc_fwd_kernel(const LstmTcArgs a) {
  constexpr int BPS = 2 * 4 * kLtNU + 1;       // B plane stride (units): 64 hi + 64 lo columns + pad
  constexpr int NCH = H / kLtKC;
  extern __shared__ __align__(128) uint4 smt[];
  uint4* s_b = smt;                            // [H/8][BPS]
  uint4* s_a = s_b + (H / 8) * BPS;            // [2 stages][hi | lo][16][kLtAPS]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const int bt = blockIdx.x / a.nug, ug = blockIdx.x - bt * a.nug;
  const int b0 = bt * kLtM, u0 = ug * kLtNU;
  const int nb = min(kLtM, a.B - b0);
  unsigned int* ctr = a.counter + bt;
  // U[:, gate * H + u0 + ul] -> hi at column gate * 16 + ul, lo at + 64
  for (int i = tid; i < (H / 8) * 64; i += kLtThreads) {
    const int kg = i >> 6, c = i & 63;
    const float* src = a.U + (size_t)(kg * 8) * 4 * H + (c >> 4) * H + u0 + (c & 15);
    float4 v[2];
    v[0] = make_float4(__ldg(src), __ldg(src + 4 * H), __ldg(src + 8 * H), __ldg(src + 12 * H));
    v[1] = make_float4(__ldg(src + 16 * H), __ldg(src + 20 * H), __ldg(src + 24 * H), __ldg(src + 28 * H));
    lt_split_store(v, s_b + kg * BPS + c, s_b + kg * BPS + 64 + c);
  }
  // this thread's cells: rows r0 + 8 rh, units 8 p + 2 q + j (rh, p, j in {0, 1})
  const int r0 = 16 * warp + (lane >> 2);
  float c_st[2][2][2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh)
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int row = r0 + 8 * rh;
        c_st[rh][p][j] = row < nb ? __ldg(a.c0 + (size_t)(b0 + row) * H + u0 + 8 * p + 2 * q + j) : 0.f;
      }
  const uint32_t a_base = smem_u32(s_a), b_base = smem_u32(s_b);
  const uint64_t lo_off = (uint64_t)((kLtKC / 8) * kLtAPS);   // descriptor units: hi -> lo planes

  for (int t = 0; t < a.T1; ++t) {
    const uint8_t* done_t = a.done + (size_t)t * a.B;
    const uint8_t* done_n = (t + 1 < a.T1) ? a.done + (size_t)(t + 1) * a.B : nullptr;
    if (t == 0) {
      // h0 with the resets of step 0 applied -> hp[0] (kept for the dU GEMM)
      if (ug == 0) {
        for (int i = tid; i < nb * (H / 4); i += kLtThreads) {
          const int b = i / (H / 4), k4 = i - b * (H / 4);
          float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
          if (!done_t[b0 + b]) v = __ldg(reinterpret_cast<const float4*>(a.h0 + (size_t)(b0 + b) * H) + k4);
          reinterpret_cast<float4*>(a.hp + (size_t)(b0 + b) * H)[k4] = v;
        }
      }
    } else {
      lt_barrier_wait(ctr, (unsigned int)t * a.nug, a.err);
    }
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    wgmma_fence_acc<64>(acc);
    for (int kc = 0; kc < NCH; ++kc) {
      float4 r[kLtUnitsPerThread][2];
      if (t == 0) {
        // step 0 reads h0 directly (every CTA), masked by done[0]
#pragma unroll
        for (int j = 0; j < kLtUnitsPerThread; ++j) {
          const int u = tid + j * kLtThreads;
          const int row = u >> 4, kg = u & 15;
          r[j][0] = r[j][1] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (row < nb && !done_t[b0 + row]) {
            const float4* p = reinterpret_cast<const float4*>(a.h0 + (size_t)(b0 + row) * H + kc * kLtKC + kg * 8);
            r[j][0] = __ldg(p); r[j][1] = __ldg(p + 1);
          }
        }
      } else {
        lt_load_chunk(r, a.hp + ((size_t)t * a.B + b0) * H, H, nb, kc * kLtKC);
      }
      if (kc >= 2) wgmma_wait<1>();              // the MMAs that read this stage have completed
      uint4* stage = s_a + (kc & 1) * kLtStageUnits;
      lt_store_chunk(r, stage);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncthreads();
      wgmma_fence();
      const uint32_t sa = a_base + (uint32_t)((kc & 1) * kLtStageUnits) * 16u;
#pragma unroll
      for (int ks = 0; ks < kLtKC / 16; ++ks) {
        const uint64_t da = gmma_desc(sa + (uint32_t)(2 * ks * kLtAPS) * 16u, kLtAPS * 16u, 128u);
        const uint64_t db = gmma_desc(b_base + (uint32_t)((kc * kLtKC / 8 + 2 * ks) * BPS) * 16u, BPS * 16u, 128u);
        Wgmma<128>::mma<0, 0>(acc, da, db, 1u);
        Wgmma<64>::mma<0, 0>(acc, da + lo_off, db, 1u);
      }
      wgmma_commit();
    }
    wgmma_wait<0>();
    wgmma_fence_acc<64>(acc);
    // ---- cell update from registers: acc[i] column 8 (i >> 2) + 2 q + (i & 1), row r0 + 8 ((i >> 1) & 1);
    // column c of hi(h) hi(U) + lo(h) hi(U) is acc[i], its hi(h) lo(U) partner (column c + 64) acc[i + 32]
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int row = r0 + 8 * rh;
      if (row >= nb) continue;
      const int gb = b0 + row;
      float* zrow = a.z + ((size_t)t * a.B + gb) * 4 * H;
      const bool reset = done_t[gb] != 0;
      const bool reset_n = done_n && done_n[gb];
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int u = u0 + 8 * p + 2 * q;
        float2 zin[4];
#pragma unroll
        for (int g = 0; g < 4; ++g) zin[g] = *reinterpret_cast<const float2*>(zrow + g * H + u);
        float gate[4][2], cn[2], hn[2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float zz[4];
#pragma unroll
          for (int g = 0; g < 4; ++g) {
            const int i = 4 * (2 * g + p) + 2 * rh + j;
            zz[g] = (acc[i] + acc[i + 32]) + (j ? zin[g].y : zin[g].x);
          }
          const float gi = sigmoidf_(zz[0]), gf = sigmoidf_(zz[1]), gg = tanhf(zz[2]), go = sigmoidf_(zz[3]);
          const float cp_ = reset ? 0.f : c_st[rh][p][j];
          const float c = gf * cp_ + gi * gg;
          const float h = go * tanhf(c);
          c_st[rh][p][j] = c;
          gate[0][j] = gi; gate[1][j] = gf; gate[2][j] = gg; gate[3][j] = go;
          cn[j] = c; hn[j] = h;
        }
#pragma unroll
        for (int g = 0; g < 4; ++g) *reinterpret_cast<float2*>(zrow + g * H + u) = make_float2(gate[g][0], gate[g][1]);
        const size_t o = ((size_t)t * a.B + gb) * H + u;
        *reinterpret_cast<float2*>(a.cs + o) = make_float2(cn[0], cn[1]);
        *reinterpret_cast<float2*>(a.hs + o) = make_float2(hn[0], hn[1]);
        if (done_n)
          *reinterpret_cast<float2*>(a.hp + o + (size_t)a.B * H) =
              reset_n ? make_float2(0.f, 0.f) : make_float2(hn[0], hn[1]);
      }
    }
    if (t + 1 < a.T1) lt_barrier_arrive(ctr);
  }
}

// ------------------------------------------------------------------------------------------------
template <int H>
__global__ void __launch_bounds__(kLtThreads, 1) lstm_tc_bwd_kernel(const LstmTcArgs a) {
  constexpr int BPS = 2 * kLtNU + 1;           // B plane stride (units): 16 hi + 16 lo rows + pad
  constexpr int NCH = 4 * H / kLtKC;
  extern __shared__ __align__(128) uint4 smt[];
  uint4* s_b = smt;                            // [4H/8][BPS]: row n = U[u0 + n, 8 kg .. 8 kg + 8)
  uint4* s_a = s_b + (4 * H / 8) * BPS;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const int bt = blockIdx.x / a.nug, ug = blockIdx.x - bt * a.nug;
  const int b0 = bt * kLtM, u0 = ug * kLtNU;
  const int nb = min(kLtM, a.B - b0);
  unsigned int* ctr = a.counter + bt;
  for (int i = tid; i < (4 * H / 8) * kLtNU; i += kLtThreads) {
    const int n = i / (4 * H / 8), kg = i - n * (4 * H / 8);     // coalesced along U's rows
    const float4* src = reinterpret_cast<const float4*>(a.U + (size_t)(u0 + n) * 4 * H + kg * 8);
    float4 v[2] = {__ldg(src), __ldg(src + 1)};
    lt_split_store(v, s_b + kg * BPS + n, s_b + kg * BPS + kLtNU + n);
  }
  const int r0 = 16 * warp + (lane >> 2);
  float dc_st[2][2][2];
#pragma unroll
  for (int rh = 0; rh < 2; ++rh)
#pragma unroll
    for (int p = 0; p < 2; ++p)
#pragma unroll
      for (int j = 0; j < 2; ++j) dc_st[rh][p][j] = 0.f;
  const uint32_t a_base = smem_u32(s_a), b_base = smem_u32(s_b);
  const uint64_t lo_off = (uint64_t)((kLtKC / 8) * kLtAPS);
  __syncthreads();

  unsigned int arrivals = 0;
  for (int t = a.T1 - 1; t >= 0; --t) {
    const bool last = (t + 1 == a.T1);
    const uint8_t* done_t = a.done + (size_t)t * a.B;
    const uint8_t* done_n = last ? nullptr : a.done + (size_t)(t + 1) * a.B;
    // ---- dh_rec[64 rows, 16 units] = dZ[t+1] U[u0 : u0 + 16, :]^T ------------------------------
    float acc[16];
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = 0.f;
    if (!last) {
      lt_barrier_wait(ctr, arrivals * a.nug, a.err);
      wgmma_fence_acc<16>(acc);
      const float* dzn = a.dz + ((size_t)(t + 1) * a.B + b0) * 4 * H;
      for (int kc = 0; kc < NCH; ++kc) {
        float4 r[kLtUnitsPerThread][2];
        lt_load_chunk(r, dzn, 4 * H, nb, kc * kLtKC);
        if (kc >= 2) wgmma_wait<1>();
        lt_store_chunk(r, s_a + (kc & 1) * kLtStageUnits);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
        wgmma_fence();
        const uint32_t sa = a_base + (uint32_t)((kc & 1) * kLtStageUnits) * 16u;
#pragma unroll
        for (int ks = 0; ks < kLtKC / 16; ++ks) {
          const uint64_t da = gmma_desc(sa + (uint32_t)(2 * ks * kLtAPS) * 16u, kLtAPS * 16u, 128u);
          const uint64_t db = gmma_desc(b_base + (uint32_t)((kc * kLtKC / 8 + 2 * ks) * BPS) * 16u, BPS * 16u, 128u);
          Wgmma<32>::mma<0, 0>(acc, da, db, 1u);
          Wgmma<16>::mma<0, 0>(acc, da + lo_off, db, 1u);
        }
        wgmma_commit();
      }
      wgmma_wait<0>();
      wgmma_fence_acc<16>(acc);
    }
    // ---- pointwise backward from registers: unit 8 p + 2 q + j of row r0 + 8 rh is acc[4 p + 2 rh + j]
    // (+ its hi(dZ) lo(U) partner acc[4 p + 2 rh + j + 8])
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int row = r0 + 8 * rh;
      if (row >= nb) continue;
      const int gb = b0 + row;
      const float* gr = a.z + ((size_t)t * a.B + gb) * 4 * H;
      const bool cut = done_n && done_n[gb];
      const bool reset = done_t[gb] != 0;
#pragma unroll
      for (int p = 0; p < 2; ++p) {
        const int u = u0 + 8 * p + 2 * q;
        const size_t o = ((size_t)t * a.B + gb) * H + u;
        const float2 gi2 = *reinterpret_cast<const float2*>(gr + u);
        const float2 gf2 = *reinterpret_cast<const float2*>(gr + H + u);
        const float2 gg2 = *reinterpret_cast<const float2*>(gr + 2 * H + u);
        const float2 go2 = *reinterpret_cast<const float2*>(gr + 3 * H + u);
        const float2 dh2 = *reinterpret_cast<const float2*>(a.dhs + o);
        const float2 cs2 = *reinterpret_cast<const float2*>(a.cs + o);
        float2 cp2 = make_float2(0.f, 0.f);
        if (!reset)
          cp2 = *reinterpret_cast<const float2*>(t == 0 ? a.c0 + (size_t)gb * H + u : a.cs + o - (size_t)a.B * H);
        float dzv[4][2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const float gi = j ? gi2.y : gi2.x, gf = j ? gf2.y : gf2.x, gg = j ? gg2.y : gg2.x, go = j ? go2.y : go2.x;
          float dh = j ? dh2.y : dh2.x;
          const int i = 4 * p + 2 * rh + j;
          if (!last && !cut) dh += acc[i] + acc[i + 8];
          const float tc = tanhf(j ? cs2.y : cs2.x);
          float dc = dh * go * (1.f - tc * tc);
          if (!last && !cut) dc += dc_st[rh][p][j];
          const float cprev = j ? cp2.y : cp2.x;
          dzv[0][j] = dc * gg * gi * (1.f - gi);
          dzv[1][j] = dc * cprev * gf * (1.f - gf);
          dzv[2][j] = dc * gi * (1.f - gg * gg);
          dzv[3][j] = dh * tc * go * (1.f - go);
          dc_st[rh][p][j] = dc * gf;
        }
        float* dzr = a.dz + ((size_t)t * a.B + gb) * 4 * H;
#pragma unroll
        for (int g = 0; g < 4; ++g) *reinterpret_cast<float2*>(dzr + g * H + u) = make_float2(dzv[g][0], dzv[g][1]);
      }
    }
    if (t > 0) { lt_barrier_arrive(ctr); ++arrivals; }
  }
}

// ------------------------------------------------------------------------------------------------
static size_t tc_smem(bool bwd, int H) {
  const size_t b_units = bwd ? (size_t)(4 * H / 8) * (2 * kLtNU + 1) : (size_t)(H / 8) * (8 * kLtNU + 1);
  return (b_units + 2 * (size_t)kLtStageUnits) * 16;
}

template <int H>
static int launch_lstm_tc(bool bwd, LstmTcArgs a, cudaStream_t st) {
  const size_t smem = tc_smem(bwd, H);
  if (smem > (size_t)kLtSmemLimit) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm (tc3): does not fit shared memory");
  const int nbt = (a.B + kLtM - 1) / kLtM;
  a.nug = H / kLtNU;
  if (nbt > 64) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm (tc3): batch too large");
  const void* fn = bwd ? (const void*)lstm_tc_bwd_kernel<H> : (const void*)lstm_tc_fwd_kernel<H>;
  SEEDRL_CUDA(bwd ? allow_smem<lstm_tc_bwd_kernel<H>>((int)smem) : allow_smem<lstm_tc_fwd_kernel<H>>((int)smem));
  SEEDRL_CUDA(cudaMemsetAsync(a.counter, 0, 64 * sizeof(unsigned int), st));
  const int grid = nbt * a.nug;
  void* args[] = {&a};
  if (grid <= kNumSMs) {
    SEEDRL_CUDA(cudaLaunchCooperativeKernel(fn, dim3(grid), dim3(kLtThreads), args, smem, st));
  } else {
    // batch tiles are contiguous in blockIdx: resident tiles finish and make room for the next ones
    SEEDRL_CUDA(cudaLaunchKernel(fn, dim3(grid), dim3(kLtThreads), args, smem, st));
  }
  count_launch(PC_LSTM_PW, st);
  return SEEDRL_OK;
}

int lstm_forward_tc(int H, int T1, int B, const float* U, const uint8_t* done, float* z, const float* h0,
                    const float* c0, float* hs, float* cs, float* hp, unsigned int* counter, int* err,
                    cudaStream_t st) {
  LstmTcArgs a;
  a.T1 = T1; a.B = B; a.U = U; a.done = done; a.z = z; a.h0 = h0; a.c0 = c0; a.hs = hs; a.cs = cs; a.hp = hp;
  a.dhs = nullptr; a.dz = nullptr; a.counter = counter; a.err = err;
  if (H == 256) return launch_lstm_tc<256>(false, a, st);
  if (H == 512) return launch_lstm_tc<512>(false, a, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: hidden size must be 256 or 512");
}

int lstm_backward_tc(int H, int T1, int B, const float* U, const uint8_t* done, const float* gates,
                     const float* cs, const float* c0, const float* dhs, float* dz, unsigned int* counter,
                     int* err, cudaStream_t st) {
  LstmTcArgs a;
  a.T1 = T1; a.B = B; a.U = U; a.done = done; a.z = const_cast<float*>(gates); a.h0 = nullptr; a.c0 = c0;
  a.hs = nullptr; a.cs = const_cast<float*>(cs); a.hp = nullptr; a.dhs = dhs; a.dz = dz; a.counter = counter;
  a.err = err;
  if (H == 256) return launch_lstm_tc<256>(true, a, st);
  if (H == 512) return launch_lstm_tc<512>(true, a, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: hidden size must be 256 or 512");
}

}  // namespace seedrl
