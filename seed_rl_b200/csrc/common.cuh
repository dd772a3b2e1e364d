// Shared helpers for libseedrl_b200 (sm_90a only).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include <atomic>
#include <string>

#include "../../include/seedrl_b200.h"

namespace seedrl {

extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launch_count;

inline int set_error(int code, const std::string& msg) {
  g_last_error = msg;
  return code;
}

#define SEEDRL_TRY(expr)                \
  do {                                  \
    const int rc__ = (expr);            \
    if (rc__ != SEEDRL_OK) return rc__; \
  } while (0)

#define SEEDRL_CHECK_ARG(cond, msg)                                         \
  do {                                                                      \
    if (!(cond))                                                            \
      return ::seedrl::set_error(SEEDRL_ERR_INVALID_ARGUMENT,               \
                                 std::string(__func__) + ": " + (msg));     \
  } while (0)

#define SEEDRL_CHECK_LAUNCH()                                               \
  do {                                                                      \
    cudaError_t e__ = cudaGetLastError();                                   \
    if (e__ != cudaSuccess)                                                 \
      return ::seedrl::set_error(                                           \
          SEEDRL_ERR_INTERNAL, std::string(__func__) + ": CUDA launch: " +  \
                                   cudaGetErrorString(e__));                \
  } while (0)

// variadic so that the call may name a template with several arguments
#define SEEDRL_CUDA(...)                                                    \
  do {                                                                      \
    cudaError_t e__ = (__VA_ARGS__);                                        \
    if (e__ != cudaSuccess)                                                 \
      return ::seedrl::set_error(                                           \
          SEEDRL_ERR_INTERNAL,                                              \
          std::string(__func__) + ": " #__VA_ARGS__ ": " + cudaGetErrorString(e__)); \
  } while (0)

// Optional per-category kernel timing (CUDA events on the launching stream), used by
// bench.py's separate profiling pass -- never inside a timed region.
enum ProfCat { PC_CONV_FWD = 0, PC_CONV_DGRAD, PC_CONV_WGRAD, PC_POOL, PC_GEMM, PC_LSTM_PW,
               PC_LOSS, PC_ADAM, PC_VTRACE, PC_MISC, PC_COUNT };
extern bool g_prof_on;
extern int g_conv_cat;
// One event AFTER each launch; a kernel's time = gap to the previous event on the stream.
void prof_mark_(int cat, cudaStream_t st);

inline void count_launch(int cat = PC_MISC, cudaStream_t st = 0) {
  g_launch_count.fetch_add(1, std::memory_order_relaxed);
  if (g_prof_on) prof_mark_(cat, st);
}

constexpr int kNumSMs = 132;  // H100 SXM

// Opts kernel K into `bytes` of dynamic shared memory (more than the 48 KB default).  The attribute is
// set on the kernel's first launch only; the function-local static is initialised exactly once even when
// the inference and learner threads reach that launch together.
template <auto K>
cudaError_t allow_smem(int bytes) {
  static const cudaError_t e = cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
  return e;
}

// cuTensorMapEncodeTiled of the driver the runtime loaded (the library does not link libcuda), looked up
// once; null when that driver does not have it.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline EncodeTiledFn encode_tiled_fn() {
  static const EncodeTiledFn fn = [] {
    void* q = nullptr;
    cudaDriverEntryPointQueryResult qr;
    const bool found = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &q, cudaEnableDefault, &qr) == cudaSuccess &&
                       qr == cudaDriverEntryPointSuccess;
    (void)cudaGetLastError();
    return found ? reinterpret_cast<EncodeTiledFn>(q) : nullptr;
  }();
  return fn;
}

__host__ __device__ inline int ceil_div(int a, int b) { return (a + b - 1) / b; }
__host__ __device__ inline size_t ceil_div_sz(size_t a, size_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }

// Philox4x32-10 (Salmon et al. 2011).  The categorical sampler and the R2D2 epsilon-greedy draw
// from it; each states the counter layout it uses.
__device__ __forceinline__ uint4 philox4x32_10(uint4 ctr, uint2 key) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(M0, ctr.x), lo0 = M0 * ctr.x;
    const uint32_t hi1 = __umulhi(M1, ctr.z), lo1 = M1 * ctr.z;
    ctr = make_uint4(hi1 ^ ctr.y ^ key.x, lo1, hi0 ^ ctr.w ^ key.y, lo0);
    key.x += W0;
    key.y += W1;
  }
  return ctr;
}

}  // namespace seedrl
