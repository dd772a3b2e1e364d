// Dense / LSTM kernels (fp32 SIMT path) for dmlab/networks.py:105-118,157-169:
// Dense(256)+ReLU, the Keras LSTMCell(256) unrolled over time with done-resets,
// policy/baseline heads -- forward and backward.
#include "kernels.h"

namespace seedrl {

// ---------------------------------------------------------------------------
// C[M,N] (=|+=) op(A)[M,K] * op(B)[K,N]   row-major, leading dims lda/ldb/ldc.
//   TA: A is stored [K,M] (C = A^T B).   TB: B is stored [N,K] (C = A B^T).
//   a_relu: relu applied to A elements on load.
//   epilogue: + bias[n]; relu; keep only where mask[m*ldm+n] > 0; accumulate.
// 64x64x16 tiles, 256 threads, 4x4 outputs per thread.
template <bool TA, bool TB>
__global__ void __launch_bounds__(256)
sgemm_kernel(int M, int N, int K, const float* __restrict__ A, int lda,
             const float* __restrict__ B, int ldb, float* __restrict__ C, int ldc, GemmEpi e) {
  constexpr int BM = 64, BN = 64, BK = 16;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int tid = threadIdx.x;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int tx = tid & 15, ty = tid >> 4;   // 16 x 16 threads, each 4x4
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  for (int k0 = 0; k0 < K; k0 += BK) {
    // load A tile (BM x BK): 1024 elements, 4 per thread
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * 256;
      int m, k;
      if (TA) { m = idx & 63; k = idx >> 6; }       // m fastest (contiguous in memory)
      else    { k = idx & 15; m = idx >> 4; }       // k fastest
      const int gm = m0 + m, gk = k0 + k;
      float v = 0.f;
      if (gm < M && gk < K) v = TA ? A[(size_t)gk * lda + gm] : A[(size_t)gm * lda + gk];
      if (e.a_relu) v = fmaxf(v, 0.f);
      As[k][m] = v;
    }
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int idx = tid + r * 256;
      int n, k;
      if (TB) { k = idx & 15; n = idx >> 4; }       // B stored [N,K]: k fastest
      else    { n = idx & 63; k = idx >> 6; }       // B stored [K,N]: n fastest
      const int gn = n0 + n, gk = k0 + k;
      float v = 0.f;
      if (gn < N && gk < K) v = TB ? B[(size_t)gn * ldb + gk] : B[(size_t)gk * ldb + gn];
      Bs[k][n] = v;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float av[4] = {a.x, a.y, a.z, a.w};
      const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int gm = m0 + ty * 4 + i;
    if (gm >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int gn = n0 + tx * 4 + j;
      if (gn >= N) continue;
      float v = acc[i][j];
      if (e.bias) v += e.bias[gn];
      if (e.relu) v = fmaxf(v, 0.f);
      if (e.mask) v = e.mask[(size_t)gm * e.ldm + gn] > 0.f ? v : 0.f;
      float* c = C + (size_t)gm * ldc + gn;
      *c = e.accumulate ? *c + v : v;
    }
  }
}

__global__ void colsum_kernel(int M, int N, const float* __restrict__ X, int ld, const float* __restrict__ w,
                              int ldw, float* __restrict__ out);

// C[m] = bias + A[m, :] . b   (N == 1: the baseline / value heads).  One warp per row, fixed-order
// shuffle reduction; the tiled kernel would run M/64 CTAs whose threads each loop over all of K.
__global__ void __launch_bounds__(256) rowdot_kernel(int M, int K, const float* __restrict__ A, int lda,
                                                      const float* __restrict__ b, const float* __restrict__ bias,
                                                      float* __restrict__ C) {
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  const float* a = A + (size_t)row * lda;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) s = fmaf(a[k], __ldg(b + k), s);
  s = warp_sum(s);
  if (lane == 0) C[row] = s + (bias ? __ldg(bias) : 0.f);
}

int sgemm(bool ta, bool tb, int M, int N, int K, const float* A, int lda, const float* B, int ldb,
          float* C, int ldc, const GemmEpi& e, cudaStream_t st) {
  if (M <= 0 || N <= 0) return SEEDRL_OK;
  if (!ta && !tb && N == 1 && ldb == 1 && ldc == 1 && !e.mask && !e.relu && !e.accumulate && !e.a_relu) {
    rowdot_kernel<<<ceil_div(M, 8), 256, 0, st>>>(M, K, A, lda, B, e.bias, C);
    count_launch(PC_GEMM, st);
    SEEDRL_CHECK_LAUNCH();
    return SEEDRL_OK;
  }
  if (ta && N == 1 && ldc == 1 && !e.bias && !e.mask && !e.relu && !e.accumulate && !e.a_relu) {
    // C[M,1] = A^T b: a weighted column sum spread over M/32 CTAs (the tiled kernel would run 4 CTAs)
    colsum_kernel<<<ceil_div(M, 32), 1024, 0, st>>>(K, M, A, lda, B, ldb, C);
    count_launch(PC_GEMM, st);
    SEEDRL_CHECK_LAUNCH();
    return SEEDRL_OK;
  }
  // grid.y is capped at 65535 tiles of 64 rows: taller products (the im2col convolutions past 4.19 M output
  // positions) run as several launches over row slabs
  constexpr int kRowsPerLaunch = 65535 * 64;
  for (int r0 = 0; r0 < M; r0 += kRowsPerLaunch) {
    const int m = M - r0 < kRowsPerLaunch ? M - r0 : kRowsPerLaunch;
    const float* Ar = ta ? A + r0 : A + (size_t)r0 * lda;
    float* Cr = C + (size_t)r0 * ldc;
    GemmEpi er = e;
    if (e.mask) er.mask = e.mask + (size_t)r0 * e.ldm;
    dim3 grid(ceil_div(N, 64), ceil_div(m, 64));
    if (!ta && !tb) sgemm_kernel<false, false><<<grid, 256, 0, st>>>(m, N, K, Ar, lda, B, ldb, Cr, ldc, er);
    else if (ta && !tb) sgemm_kernel<true, false><<<grid, 256, 0, st>>>(m, N, K, Ar, lda, B, ldb, Cr, ldc, er);
    else if (!ta && tb) sgemm_kernel<false, true><<<grid, 256, 0, st>>>(m, N, K, Ar, lda, B, ldb, Cr, ldc, er);
    else sgemm_kernel<true, true><<<grid, 256, 0, st>>>(m, N, K, Ar, lda, B, ldb, Cr, ldc, er);
    count_launch(PC_GEMM, st);
    SEEDRL_CHECK_LAUNCH();
  }
  return SEEDRL_OK;
}

// out[n] = sum_m X[m*ld + n], m < M, n < N.  One CTA per 32 columns; fixed-order
// (deterministic) reduction.
// w != nullptr: out[n] = sum_m X[m*ld + n] * w[m*ldw]  (= X^T w, the N == 1 weight gradient).
// 32 warps stride the rows, four independent loads in flight per lane.
__global__ void __launch_bounds__(1024)
colsum_kernel(int M, int N, const float* __restrict__ X, int ld, const float* __restrict__ w, int ldw,
              float* __restrict__ out) {
  __shared__ float red[32][33];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;   // 32 warps
  const int n = blockIdx.x * 32 + lane;
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  if (n < N) {
    int m = wid;
    for (; m + 96 < M; m += 128) {
      const float x0 = X[(size_t)m * ld + n], x1 = X[(size_t)(m + 32) * ld + n];
      const float x2 = X[(size_t)(m + 64) * ld + n], x3 = X[(size_t)(m + 96) * ld + n];
      if (w) {
        s0 = fmaf(x0, w[(size_t)m * ldw], s0); s1 = fmaf(x1, w[(size_t)(m + 32) * ldw], s1);
        s2 = fmaf(x2, w[(size_t)(m + 64) * ldw], s2); s3 = fmaf(x3, w[(size_t)(m + 96) * ldw], s3);
      } else {
        s0 += x0; s1 += x1; s2 += x2; s3 += x3;
      }
    }
    for (; m < M; m += 32) s0 += X[(size_t)m * ld + n] * (w ? w[(size_t)m * ldw] : 1.f);
  }
  red[wid][lane] = (s0 + s1) + (s2 + s3);
  __syncthreads();
  if (wid == 0 && n < N) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < 32; ++k) t += red[k][lane];
    out[n] = t;
  }
}

// Stage 1 of the tall column sum (bias gradients of the im2col convolutions: M = frames x positions
// rows, N = 16..64 columns -- one CTA per 32 columns would leave a single CTA walking the whole
// matrix).  CTA s reduces rows [s*rps, (s+1)*rps) of a dense [M][N] matrix (ld == N, N a power of two
// <= 2048).  512 threads sweep 2048 consecutive floats per step and rps*N is a multiple of 2048, so a
// thread meets the same four columns every step; four 16-byte streaming loads in flight per thread.
// Fixed slab map and fixed-order adds => deterministic.
__global__ void __launch_bounds__(512)
colsum_slab_kernel(int M, int N, int rps, const float* __restrict__ X, float* __restrict__ part) {
  __shared__ float4 red[512];
  const int t = threadIdx.x;
  const size_t r0 = (size_t)blockIdx.x * rps;
  const size_t r1 = r0 + rps < (size_t)M ? r0 + rps : (size_t)M;
  const float4* x4 = reinterpret_cast<const float4*>(X);
  const size_t e4 = r1 * N / 4;
  size_t j = r0 * N / 4 + t;
  float4 a0 = make_float4(0.f, 0.f, 0.f, 0.f), a1 = a0, a2 = a0, a3 = a0;
  for (; j + 3 * 512 < e4; j += 4 * 512) {
    const float4 v0 = __ldcs(x4 + j), v1 = __ldcs(x4 + j + 512), v2 = __ldcs(x4 + j + 1024), v3 = __ldcs(x4 + j + 1536);
    a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
    a1.x += v1.x; a1.y += v1.y; a1.z += v1.z; a1.w += v1.w;
    a2.x += v2.x; a2.y += v2.y; a2.z += v2.z; a2.w += v2.w;
    a3.x += v3.x; a3.y += v3.y; a3.z += v3.z; a3.w += v3.w;
  }
  for (; j < e4; j += 512) {
    const float4 v0 = __ldcs(x4 + j);
    a0.x += v0.x; a0.y += v0.y; a0.z += v0.z; a0.w += v0.w;
  }
  red[t] = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y),
                       (a0.z + a1.z) + (a2.z + a3.z), (a0.w + a1.w) + (a2.w + a3.w));
  __syncthreads();
  const int G = N >> 2;            // column groups; thread t owns group t % G
  if (t < G) {
    float4 s = red[t];
    for (int k = t + G; k < 512; k += G) {
      const float4 v = red[k];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4*>(part + (size_t)blockIdx.x * N)[t] = s;
  }
}

int colsum(int M, int N, const float* X, int ld, float* out, cudaStream_t st, float* ws, size_t ws_bytes) {
  // tall dense matrices: row slabs over ~4 CTAs per SM, then the column sum of the slab partials
  const bool pow2 = N >= 4 && N <= 2048 && (N & (N - 1)) == 0;
  if (ws && pow2 && ld == N && (size_t)M * N >= ((size_t)1 << 20) && (reinterpret_cast<uintptr_t>(X) & 15) == 0) {
    const int sweep = 2048 / N;                                   // rows per 512-thread sweep
    int rps = ceil_div(ceil_div(M, 4 * kNumSMs), sweep) * sweep;   // rows per slab
    if (rps < 8 * sweep) rps = 8 * sweep;
    const int S = ceil_div(M, rps);
    if ((size_t)S * N * sizeof(float) <= ws_bytes && S > 1) {
      colsum_slab_kernel<<<S, 512, 0, st>>>(M, N, rps, X, ws);
      count_launch(PC_GEMM, st);
      SEEDRL_CHECK_LAUNCH();
      colsum_kernel<<<ceil_div(N, 32), 1024, 0, st>>>(S, N, ws, N, nullptr, 0, out);
      count_launch(PC_GEMM, st);
      SEEDRL_CHECK_LAUNCH();
      return SEEDRL_OK;
    }
  }
  colsum_kernel<<<ceil_div(N, 32), 1024, 0, st>>>(M, N, X, ld, nullptr, 0, out);
  count_launch(PC_GEMM, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// generic helpers ------------------------------------------------------------
__global__ void fill_kernel(size_t n, float* p, float v) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}
int fill(size_t n, float* p, float v, cudaStream_t st) {
  if (n == 0) return SEEDRL_OK;
  fill_kernel<<<(unsigned)ceil_div_sz(n, 256), 256, 0, st>>>(n, p, v);
  count_launch(PC_MISC, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// out[n] = baseline column of heads? (kept simple: strided copy)  dst[i] = src[i*ld + col]
__global__ void copy_col_kernel(int n, const float* __restrict__ src, int ld, int col,
                                float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[(size_t)i * ld + col];
}

}  // namespace seedrl
