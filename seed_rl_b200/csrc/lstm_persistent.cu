// Persistent LSTM recurrence (Keras LSTMCell(256) unrolled over time with done-resets,
// dmlab/networks.py:157-169) -- forward and BPTT -- as ONE cooperative kernel each.
//
// The recurrence is latency-bound: per step only B x 256 x 1024 MACs (B = 64) but 2 x T
// dependent steps.  Launching a GEMM + a pointwise kernel per step pays two launches per step;
// here 128 CTAs stay resident for all T steps, each owning 2 hidden units (8 gate
// columns): its slice of the recurrent matrix U stays in shared memory, the cell state
// (forward) / cell-state gradient (backward) of its units stays on chip, and the only
// per-step global traffic is the [B,256] hidden state (forward) or the [B,1024] gate
// gradient (backward) exchanged through L2 between two grid-wide barriers.
//   forward : z[t] (+)= hprev[t] U ; gates ; c,h ; emits hprev[t+1] = done[t+1] ? 0 : h
//   backward: dh = dH[t] + (done[t+1] ? 0 : dZ[t+1] U^T) ; gate gradients dZ[t]
// Launched with cudaLaunchCooperativeKernel (co-residency guaranteed or the launch fails);
// the grid barrier is a monotonic atomic counter with a bounded spin (sets *err, never hangs).
#include "kernels.h"

namespace seedrl {

// Templated on <H, NU>: H hidden units, NU units per CTA (grid = H / NU = 128 CTAs for both
// LSTMCell(256) of ImpalaDeep (NU = 2) and LSTMCell(512) of DuelingLSTMDQNNet (NU = 4,
// atari/networks.py:252)).  A CTA owns 4*NU gate columns; thread = (batch row, gate).
constexpr int kLThreads = 256;
constexpr int kLBt = 64;            // batch tile

__device__ __forceinline__ void grid_barrier(unsigned int* counter, unsigned int nblocks,
                                             unsigned int* gen, int* err) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned int target = (*gen + 1u) * nblocks;
    atomicAdd(counter, 1u);
    int spins = 0;
    while (*reinterpret_cast<volatile unsigned int*>(counter) < target) {
      if (++spins > (1 << 24)) { if (err) atomicExch(err, 2); break; }
    }
    __threadfence();
  }
  *gen += 1u;
  __syncthreads();
}

struct LstmFwdArgs {
  int T1, B;
  const float* U;          // [H, 4H]
  const uint8_t* done;     // [T1, B]
  float* z;                // [T1, B, 4H]  in: x W + b ; out: activated gates (i,f,g,o)
  const float* h0;         // [B, H]
  const float* c0;         // [B, H]
  float* hs;               // [T1, B, H]
  float* cs;               // [T1, B, H]
  float* hp;               // [T1, B, H]  masked recurrent inputs (kept for dU)
  unsigned int* counter;   // zeroed by the host before launch
  int* err;
};

template <int H, int NU>
__global__ void __launch_bounds__(kLThreads, 1) lstm_fwd_persistent_kernel(const LstmFwdArgs a) {
  constexpr int NC = 4 * NU;                     // gate columns of this CTA: column g*NU + ul
  extern __shared__ float sm[];
  float* s_U = sm;                               // [H][NC]
  float* s_h = s_U + H * NC;                     // [64][H+4]
  float* s_z = s_h + kLBt * (H + 4);             // [64][NC]
  float* s_c = s_z + kLBt * NC;                  // [B][NU] cell state of this CTA's units
  const int tid = threadIdx.x;
  const int u0 = blockIdx.x * NU;
  const int B = a.B;
  unsigned int gen = 0;
  for (int i = tid; i < H * NC; i += kLThreads) {
    const int k = i / NC, c = i - k * NC;
    s_U[i] = __ldg(a.U + (size_t)k * 4 * H + (c / NU) * H + u0 + (c % NU));
  }
  for (int i = tid; i < B * NU; i += kLThreads)
    s_c[i] = __ldg(a.c0 + (size_t)(i / NU) * H + u0 + (i % NU));
  __syncthreads();

  for (int t = 0; t < a.T1; ++t) {
    const uint8_t* done_t = a.done + (size_t)t * B;
    const uint8_t* done_n = (t + 1 < a.T1) ? a.done + (size_t)(t + 1) * B : nullptr;
    float* hp_t = a.hp + (size_t)t * B * H;
    for (int b0 = 0; b0 < B; b0 += kLBt) {
      const int nb = min(kLBt, B - b0);
      // ---- recurrent input of step t for this batch tile -> smem --------------------------
      // (8 independent 16-byte loads in flight per thread: the step is latency-bound)
      for (int i0 = tid; i0 < nb * (H / 4); i0 += 8 * kLThreads) {
        float4 v[8];
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int i = i0 + r * kLThreads;
          v[r] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (i < nb * (H / 4)) {
            const int b = i / (H / 4), k4 = i - b * (H / 4);
            if (t == 0) {
              if (!done_t[b0 + b]) v[r] = __ldg(reinterpret_cast<const float4*>(a.h0 + (size_t)(b0 + b) * H) + k4);
            } else {
              v[r] = __ldcg(reinterpret_cast<const float4*>(hp_t + (size_t)(b0 + b) * H) + k4);
            }
          }
        }
#pragma unroll
        for (int r = 0; r < 8; ++r) {
          const int i = i0 + r * kLThreads;
          if (i < nb * (H / 4)) {
            const int b = i / (H / 4), k4 = i - b * (H / 4);
            if (t == 0 && blockIdx.x == 0) reinterpret_cast<float4*>(hp_t + (size_t)(b0 + b) * H)[k4] = v[r];
            *reinterpret_cast<float4*>(s_h + b * (H + 4) + k4 * 4) = v[r];
          }
        }
      }
      __syncthreads();
      // ---- z[b, NC cols] = x-part + h . U : thread = (b, gate), NU units each ---------------
      {
        const int b = tid >> 2, g = tid & 3;
        if (b < nb) {
          float acc[NU];
#pragma unroll
          for (int j = 0; j < NU; ++j) acc[j] = 0.f;
          const float* hrow = s_h + b * (H + 4);
#pragma unroll 8
          for (int k = 0; k < H; ++k) {
            const float hv = hrow[k];
            const float* ur = s_U + k * NC + g * NU;
#pragma unroll
            for (int j = 0; j < NU; ++j) acc[j] = fmaf(hv, ur[j], acc[j]);
          }
          const float* zrow = a.z + ((size_t)t * B + b0 + b) * 4 * H;
#pragma unroll
          for (int j = 0; j < NU; ++j) s_z[b * NC + g * NU + j] = acc[j] + __ldg(zrow + g * H + u0 + j);
        }
      }
      __syncthreads();
      // ---- pointwise: thread = (b, unit) -----------------------------------------------------
      if (tid < nb * NU) {
        const int b = tid / NU, ul = tid % NU;
        const float gi = sigmoidf_(s_z[b * NC + 0 * NU + ul]);
        const float gf = sigmoidf_(s_z[b * NC + 1 * NU + ul]);
        const float gg = tanhf(s_z[b * NC + 2 * NU + ul]);
        const float go = sigmoidf_(s_z[b * NC + 3 * NU + ul]);
        const int gb = b0 + b, u = u0 + ul;
        const float cp_ = done_t[gb] ? 0.f : s_c[gb * NU + ul];
        const float c = gf * cp_ + gi * gg;
        const float h = go * tanhf(c);
        s_c[gb * NU + ul] = c;
        float* zrow = a.z + ((size_t)t * B + gb) * 4 * H;
        zrow[u] = gi; zrow[H + u] = gf; zrow[2 * H + u] = gg; zrow[3 * H + u] = go;
        a.cs[((size_t)t * B + gb) * H + u] = c;
        a.hs[((size_t)t * B + gb) * H + u] = h;
        if (done_n) a.hp[((size_t)(t + 1) * B + gb) * H + u] = done_n[gb] ? 0.f : h;
      }
      __syncthreads();
    }
    if (t + 1 < a.T1) grid_barrier(a.counter, gridDim.x, &gen, a.err);
  }
}

struct LstmBwdArgs {
  int T1, B;
  const float* U;          // [H, 4H]
  const uint8_t* done;     // [T1, B]
  const float* gates;      // [T1, B, 4H] activated gates from the forward
  const float* cs;         // [T1, B, H]
  const float* c0;         // [B, H]
  const float* dhs;        // [T1, B, H]  d loss / d h_t from the heads
  float* dz;               // [T1, B, 4H] out: gate pre-activation gradients
  unsigned int* counter;
  int* err;
};

template <int H, int NU>
__global__ void __launch_bounds__(kLThreads, 1) lstm_bwd_persistent_kernel(const LstmBwdArgs a) {
  extern __shared__ float sm[];
  constexpr int KC = 128, KS = KC + 4;           // dZ chunk width (+pad)
  float* s_Ur = sm;                              // [NU][4H] rows u0.. of U
  float* s_dz = s_Ur + NU * 4 * H;               // [2][64][KS] double-buffered
  float* s_dh = s_dz + 2 * kLBt * KS;            // [64][NU] recurrent part of dh
  float* s_dc = s_dh + kLBt * NU;                // [B][NU] dc flowing to the previous step
  const int tid = threadIdx.x;
  const int u0 = blockIdx.x * NU;
  const int B = a.B;
  unsigned int gen = 0;
  for (int i = tid; i < NU * 4 * H; i += kLThreads)
    s_Ur[i] = __ldg(a.U + (size_t)(u0 + i / (4 * H)) * 4 * H + (i % (4 * H)));
  for (int i = tid; i < B * NU; i += kLThreads) s_dc[i] = 0.f;
  __syncthreads();

  for (int t = a.T1 - 1; t >= 0; --t) {
    const bool last = (t + 1 == a.T1);
    const uint8_t* done_t = a.done + (size_t)t * B;
    const uint8_t* done_n = last ? nullptr : a.done + (size_t)(t + 1) * B;
    for (int b0 = 0; b0 < B; b0 += kLBt) {
      const int nb = min(kLBt, B - b0);
      // ---- dh_rec[b, NU units] = dZ[t+1][b, :] . U[u, :]^T, streamed in K chunks of 128 ------
      const int b = tid >> 2, part = tid & 3;
      float acc[NU];
#pragma unroll
      for (int j = 0; j < NU; ++j) acc[j] = 0.f;
      if (!last) {
        const float* dzn = a.dz + ((size_t)(t + 1) * B + b0) * 4 * H;
        // chunk c+1 travels L2 -> registers while chunk c is consumed from shared memory
        constexpr int NL = (kLBt * (KC / 4)) / kLThreads;   // 8 x 16-byte loads per thread per chunk
        float4 pre[NL];
        auto load_chunk = [&](int k0) {
#pragma unroll
          for (int r = 0; r < NL; ++r) {
            const int i = tid + r * kLThreads;
            const int rr = i / (KC / 4), k4 = i - rr * (KC / 4);
            pre[r] = rr < nb ? __ldcg(reinterpret_cast<const float4*>(dzn + (size_t)rr * 4 * H + k0) + k4)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
          }
        };
        load_chunk(0);
        for (int c = 0; c < (4 * H) / KC; ++c) {
          const int k0 = c * KC;
          float* buf = s_dz + (c & 1) * (kLBt * KS);
#pragma unroll
          for (int r = 0; r < NL; ++r) {
            const int i = tid + r * kLThreads;
            const int rr = i / (KC / 4), k4 = i - rr * (KC / 4);
            *reinterpret_cast<float4*>(buf + rr * KS + k4 * 4) = pre[r];
          }
          __syncthreads();
          if (c + 1 < (4 * H) / KC) load_chunk(k0 + KC);
          if (b < nb) {
            const float* drow = buf + b * KS + part * (KC / 4);
            const float* ur = s_Ur + k0 + part * (KC / 4);
#pragma unroll 8
            for (int k = 0; k < KC / 4; ++k) {
              const float d = drow[k];
#pragma unroll
              for (int j = 0; j < NU; ++j) acc[j] = fmaf(d, ur[j * 4 * H + k], acc[j]);
            }
          }
        }
        __syncthreads();   // the last chunk's buffer is free before the next batch tile / step
        // reduce the 4 K-parts (adjacent lanes)
#pragma unroll
        for (int j = 0; j < NU; ++j) {
          acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 1);
          acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], 2);
        }
      }
      if (part == 0 && b < nb) {
#pragma unroll
        for (int j = 0; j < NU; ++j) s_dh[b * NU + j] = acc[j];
      }
      __syncthreads();
      // ---- pointwise backward: thread = (b, unit) ------------------------------------------
      if (tid < nb * NU) {
        const int bb = tid / NU, ul = tid % NU;
        const int gb = b0 + bb, u = u0 + ul;
        const float* gr = a.gates + ((size_t)t * B + gb) * 4 * H;
        const float gi = __ldg(gr + u), gf = __ldg(gr + H + u), gg = __ldg(gr + 2 * H + u),
                    go = __ldg(gr + 3 * H + u);
        const bool cut = done_n && done_n[gb];
        float dh = __ldg(a.dhs + ((size_t)t * B + gb) * H + u);
        if (!last && !cut) dh += s_dh[bb * NU + ul];
        const float tc = tanhf(__ldg(a.cs + ((size_t)t * B + gb) * H + u));
        float dc = dh * go * (1.f - tc * tc);
        if (!last && !cut) dc += s_dc[gb * NU + ul];
        const float cprev = done_t[gb] ? 0.f
                            : (t == 0 ? __ldg(a.c0 + (size_t)gb * H + u)
                                      : __ldg(a.cs + ((size_t)(t - 1) * B + gb) * H + u));
        float* dzr = a.dz + ((size_t)t * B + gb) * 4 * H;
        dzr[u] = dc * gg * gi * (1.f - gi);
        dzr[H + u] = dc * cprev * gf * (1.f - gf);
        dzr[2 * H + u] = dc * gi * (1.f - gg * gg);
        dzr[3 * H + u] = dh * tc * go * (1.f - go);
        s_dc[gb * NU + ul] = dc * gf;
      }
      __syncthreads();
    }
    if (t > 0) grid_barrier(a.counter, gridDim.x, &gen, a.err);
  }
}

static size_t lstm_fwd_smem(int H, int NU, int B) {
  return ((size_t)H * 4 * NU + (size_t)kLBt * (H + 4) + kLBt * 4 * NU + (size_t)B * NU) * sizeof(float);
}
static size_t lstm_bwd_smem(int H, int NU, int B) {
  return ((size_t)NU * 4 * H + (size_t)2 * kLBt * 132 + kLBt * NU + (size_t)B * NU) * sizeof(float);
}

template <int H, int NU>
static int launch_lstm_fwd(const LstmFwdArgs& a_, cudaStream_t st) {
  LstmFwdArgs a = a_;
  const size_t smem = lstm_fwd_smem(H, NU, a.B);
  if (smem > 200 * 1024) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: batch too large");
  static bool attr = false;
  if (!attr) {
    SEEDRL_CUDA(cudaFuncSetAttribute(lstm_fwd_persistent_kernel<H, NU>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     200 * 1024));
    attr = true;
  }
  SEEDRL_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), st));
  void* args[] = {&a};
  SEEDRL_CUDA(cudaLaunchCooperativeKernel((const void*)lstm_fwd_persistent_kernel<H, NU>, dim3(H / NU),
                                          dim3(kLThreads), args, smem, st));
  count_launch(PC_LSTM_PW, st);
  return SEEDRL_OK;
}

template <int H, int NU>
static int launch_lstm_bwd(const LstmBwdArgs& a_, cudaStream_t st) {
  LstmBwdArgs a = a_;
  const size_t smem = lstm_bwd_smem(H, NU, a.B);
  if (smem > 200 * 1024) return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: batch too large");
  static bool attr = false;
  if (!attr) {
    SEEDRL_CUDA(cudaFuncSetAttribute(lstm_bwd_persistent_kernel<H, NU>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     200 * 1024));
    attr = true;
  }
  SEEDRL_CUDA(cudaMemsetAsync(a.counter, 0, sizeof(unsigned int), st));
  void* args[] = {&a};
  SEEDRL_CUDA(cudaLaunchCooperativeKernel((const void*)lstm_bwd_persistent_kernel<H, NU>, dim3(H / NU),
                                          dim3(kLThreads), args, smem, st));
  count_launch(PC_LSTM_PW, st);
  return SEEDRL_OK;
}

int lstm_forward_persistent(int H, int T1, int B, const float* U, const uint8_t* done, float* z,
                            const float* h0, const float* c0, float* hs, float* cs, float* hp,
                            unsigned int* counter, int* err, cudaStream_t st) {
  const LstmFwdArgs a{T1, B, U, done, z, h0, c0, hs, cs, hp, counter, err};
  if (H == 256) return launch_lstm_fwd<256, 2>(a, st);
  if (H == 512) return launch_lstm_fwd<512, 4>(a, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: hidden size must be 256 or 512");
}

int lstm_backward_persistent(int H, int T1, int B, const float* U, const uint8_t* done, const float* gates,
                             const float* cs, const float* c0, const float* dhs, float* dz,
                             unsigned int* counter, int* err, cudaStream_t st) {
  const LstmBwdArgs a{T1, B, U, done, gates, cs, c0, dhs, dz, counter, err};
  if (H == 256) return launch_lstm_bwd<256, 2>(a, st);
  if (H == 512) return launch_lstm_bwd<512, 4>(a, st);
  return set_error(SEEDRL_ERR_INVALID_ARGUMENT, "lstm: hidden size must be 256 or 512");
}

}  // namespace seedrl
