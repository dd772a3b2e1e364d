// V-trace kernels for sm_90a.
//
//  vtrace_kernel            (a1)  common/vtrace.py:34-148
//  categorical_*_kernel     (a3)  common/parametric_distribution.py:66-74
//  vtrace_loss_kernel       (a2)  agents/vtrace/learner.py:82-157 + its gradient
//
// Layout is the reference's time-major [T, B(, A)].  All of these are HBM-bound
// streaming kernels (no reuse beyond one column's time scan), so the design is:
// coalesced loads across B, the T-scan sequential in registers per column,
// logits tiles staged through shared memory so that HBM sees only full-line
// coalesced traffic in both directions.
#include <cuda.h>
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace seedrl {

// ---------------------------------------------------------------------------
// (a1) one thread per column b; reverse scan over t with loads issued CH steps
// ahead of use (memory-level parallelism: 5*CH independent loads in flight).
template <int CH>
__global__ void __launch_bounds__(128)
vtrace_kernel(int T, int B, const float* __restrict__ tlp, const float* __restrict__ blp,
              const float* __restrict__ disc, const float* __restrict__ rew,
              const float* __restrict__ val, const float* __restrict__ boot,
              float clip_rho, float clip_pg, float lambda_, int has_clip_rho,
              int has_clip_pg, float* __restrict__ vs, float* __restrict__ pg) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float acc = 0.f;
  const float bootv = boot[b];
  float vs_next = bootv, v_next = bootv;
  int t_hi = T;  // exclusive
  while (t_hi > 0) {
    const int t_lo = t_hi - CH > 0 ? t_hi - CH : 0;
    float a_t[CH], a_b[CH], a_d[CH], a_r[CH], a_v[CH];
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      const int t = t_hi - 1 - k;
      if (t >= t_lo) {
        const size_t o = (size_t)t * B + b;
        a_t[k] = __ldg(tlp + o); a_b[k] = __ldg(blp + o); a_d[k] = __ldg(disc + o);
        a_r[k] = __ldg(rew + o); a_v[k] = __ldg(val + o);
      }
    }
#pragma unroll
    for (int k = 0; k < CH; ++k) {
      const int t = t_hi - 1 - k;
      if (t >= t_lo) {
        const float rho = expf(a_t[k] - a_b[k]);                       // vtrace.py:84,110
        const float crho = has_clip_rho ? fminf(clip_rho, rho) : rho;  // :111-114
        const float c = fminf(1.0f, rho) * lambda_;                    // :116-117
        const float v = a_v[k], d = a_d[k], r = a_r[k];
        const float delta = crho * (r + d * v_next - v);               // :122
        acc = delta + d * c * acc;                                     // :128
        const float vs_t = acc + v;                                    // :133
        const float cpg = has_clip_pg ? fminf(clip_pg, rho) : rho;     // :138-142
        const size_t o = (size_t)t * B + b;
        vs[o] = vs_t;
        pg[o] = cpg * (r + d * vs_next - v);                           // :143-144
        vs_next = vs_t;
        v_next = v;
      }
    }
    t_hi = t_lo;
  }
}

// ---------------------------------------------------------------------------
// (a3) one warp per row, lanes strided over A.
__global__ void categorical_logprob_entropy_kernel(int N, int A, const float* __restrict__ logits,
                                                   const int64_t* __restrict__ actions,
                                                   float* __restrict__ logp,
                                                   float* __restrict__ entropy) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (warp >= N) return;
  const float* l = logits + (size_t)warp * A;
  float m = -INFINITY;
  for (int j = lane; j < A; j += 32) m = fmaxf(m, l[j]);
  m = warp_max(m);
  float se = 0.f, sel = 0.f;
  for (int j = lane; j < A; j += 32) {
    const float e = expf(l[j] - m);
    se += e;
    sel += e * (l[j] - m);
  }
  se = warp_sum(se);
  sel = warp_sum(sel);
  if (lane == 0) {
    if (logp) {
      int64_t a = actions[warp];
      a = a < 0 ? 0 : (a >= A ? A - 1 : a);
      logp[warp] = (l[a] - m) - logf(se);   // not l[a] - (m + log se): m + log se rounds to ulp(m)
    }
    if (entropy) entropy[warp] = logf(se) - sel / se;   // H = lse - sum p*l
  }
}

// one thread per row (A is small); first max wins ties like np.argmax.  Philox counter =
// (offset lo, offset hi, row, block of 4 actions), key = seed (philox4x32_10, common.cuh).
__global__ void categorical_sample_kernel(int N, int A, const float* __restrict__ logits,
                                          const float* __restrict__ noise, uint64_t seed,
                                          uint64_t offset, const uint64_t* __restrict__ offset_dev,
                                          int64_t* __restrict__ actions) {
  const int n = blockIdx.x * blockDim.x + threadIdx.x;
  if (n >= N) return;
  if (offset_dev) offset = *offset_dev;      // device-resident call counter (CUDA-graph replays)
  const float* l = logits + (size_t)n * A;
  float best = -INFINITY;
  int arg = 0;
  if (noise) {
    const float* g = noise + (size_t)n * A;
    for (int j = 0; j < A; ++j) {
      const float s = l[j] + g[j];
      if (s > best) { best = s; arg = j; }
    }
  } else {
    const uint2 key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    for (int j0 = 0; j0 < A; j0 += 4) {
      const uint4 r = philox4x32_10(
          make_uint4((uint32_t)offset, (uint32_t)(offset >> 32), (uint32_t)n, (uint32_t)(j0 >> 2)), key);
      const uint32_t rr[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const int j = j0 + k;
        if (j < A) {
          // u in (0,1): (x + 0.5) * 2^-32 ; g = -log(-log u)
          const float u = ((float)rr[k] + 0.5f) * 2.3283064365386963e-10f;
          const float uu = fminf(fmaxf(u, 1e-10f), 0.99999994f);
          const float s = l[j] - logf(-logf(uu));
          if (s > best) { best = s; arg = j; }
        }
      }
    }
  }
  actions[n] = arg;
}

// ---------------------------------------------------------------------------
// (a2) fused log-softmax + V-trace + losses + analytic gradient.
// One CTA owns BB batch columns for all T steps.
//   phase A  behaviour logits tile -> smem, thread-per-row: beh_logp
//   phase B  learner   logits tile -> smem (same buffer), thread-per-row:
//            lse, target logp, entropy
//   phase C  thread-per-column reverse scan (vs, pg_adv) + loss partial sums
//   phase D  thread-per-row gradient in place, written back with float4 stores
// Per-CTA partial sums go to scratch[cta][8]; the last CTA to finish (ticket)
// reduces them in index order (deterministic) and writes loss_terms.  The loss sums are
// float64 wherever they run long (the small kernel's per-thread sums, every block and grid
// reduction): the means they make (mean value, policy loss, mean kl) are near zero against
// terms of order one, so an fp32 running sum over T x B rows would decide their leading digits.
constexpr int kLossThreads = 256;
constexpr int kLossPartials = 8;

struct LossParams {
  int T, B, A, BB, AP;
  const float* ll;   // learner logits [T+1,B,A]
  const float* lb;   // learner baseline [T+1,B]
  const float* bl;   // behaviour logits [T+1,B,A]
  const int64_t* act;
  const float* rew;
  const uint8_t* done;
  seedrl_loss_config cfg;
  const float* ecp;
  float* loss_terms;
  float* dlogits;
  float* dbaseline;
  float* d_ecp;
  float* vs_out;
  float* pg_out;
  double* partials;       // [grid][8]
  unsigned int* ticket;   // self-resetting
  // PopArt instantiations only (phase 1 of seedrl_vtrace_popart_loss_fwd)
  const float* pop_mom;   // [2] EMA moments mu1, mu2
  const float* pop_comp;  // [2] compensation sigma, mu
  float* pop_td;          // [T,B] (vs - u) / s
  float* pop_sums;        // [2] sum vs, sum vs^2 over this replica's T x B
  // [T+1,B] or null (= none).  Transition t is masked iff abandoned[t+1]: its delta_t and clipped pg
  // rho are 0, so vs_t = V_t, pg_adv_t = 0 and vs_{t-1} bootstraps from V_t (done[t+1] already zeroes
  // the discount, which cuts the trace).  Every other row's arithmetic is unchanged.
  const uint8_t* abandoned = nullptr;
  // Multi-task PopArt (seedrl_vtrace_popart_tasks_loss_fwd): column b is normalised with the state of task
  // task_ids[b]; pop_mom / pop_comp are then [K,2].  An id outside [0, K) sets *task_error and the column
  // takes the identity state (s = 1, m = 0, sigma = 1, mu = 0).  The tasks kernels write each column's
  // (sum_t vs, sum_t vs^2) to col_sums [B,2]; vtrace_popart_task_moments_kernel reduces them by task.
  // The single-task kernels only check the ids when task_ids is set (every id must be 0).
  const int* task_ids = nullptr;
  int num_tasks = 0;
  int* task_error = nullptr;
  double* col_sums = nullptr;
  double* pop_sums_d = nullptr;   // single-task kernels: [3] (sum vs, sum vs^2, rows) instead of pop_sums
};

// loss kernel instantiations
constexpr int kPlain = 0, kPopArt = 1, kPopArtTasks = 2;
constexpr int kMaxTasks = 64;

// ---- PopArt (agents/policy_gradient/modules/popart.py, running_statistics.py EMAMeanStd) ----
// s = clip(sqrt(mu2 - mu1^2), 1e-6, 1e6) (running_statistics.py:149-153), evaluated in float64 and
// rounded once; every kernel that needs s calls this, so the two phases agree bit for bit.
__device__ __forceinline__ float popart_std(float mu1, float mu2) {
  const double var = (double)mu2 - (double)mu1 * (double)mu1;
  return (float)fmin(fmax(sqrt(var), 1e-6), 1e6);
}
// u = s (sigma V + mu) + m: correct_prediction, then unnormalize_prediction (popart.py)
__device__ __forceinline__ float popart_u(float V, float s, float m, float sigma, float mu) {
  return fmaf(s, fmaf(sigma, V, mu), m);
}

// Multi-task PopArt: the task of column b, or num_tasks (the identity entry of the kernels' state tables) for
// an id outside [0, num_tasks), which sets *task_error when `report`.
__device__ __forceinline__ int task_slot(const int* task_ids, int num_tasks, int* task_error, int b, bool report) {
  const int id = __ldg(task_ids + b);
  if ((unsigned)id < (unsigned)num_tasks) return id;
  if (report) atomicOr(task_error, 1);
  return num_tasks;
}
// (s, m, sigma, mu) of task k (k = num_tasks: the identity)
__device__ __forceinline__ void task_state(const LossParams& p, int k, float* q) {
  if (k < p.num_tasks) {
    q[1] = __ldg(p.pop_mom + 2 * k);
    q[0] = popart_std(q[1], __ldg(p.pop_mom + 2 * k + 1));
    q[2] = __ldg(p.pop_comp + 2 * k);
    q[3] = __ldg(p.pop_comp + 2 * k + 1);
  } else {
    q[0] = 1.f; q[1] = 0.f; q[2] = 1.f; q[3] = 0.f;
  }
}

__device__ __forceinline__ float block_reduce_sum(float v, float* red) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = 0.f;
  if (w == 0) {
    r = l < (blockDim.x >> 5) ? red[l] : 0.f;
    r = warp_sum(r);
  }
  return r;  // valid in warp 0
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double block_reduce_sum_d(double v) {
  __shared__ double red[32];
  v = warp_sum_d(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  double r = 0.0;
  if (w == 0) {
    r = l < (blockDim.x >> 5) ? red[l] : 0.0;
    r = warp_sum_d(r);
  }
  return r;  // valid in warp 0
}
__device__ __forceinline__ float block_reduce_max(float v, float* red) {
  v = warp_max(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) red[w] = v;
  __syncthreads();
  float r = 0.f;
  if (w == 0) {
    r = l < (blockDim.x >> 5) ? red[l] : -INFINITY;
    r = warp_max(r);
  }
  return r;
}


// ---- thread-per-row softmax pieces over a row of A logits in shared memory -----------------
// Rows are dense (stride A floats).  Even A: rows are 8-byte aligned and read with 64-bit
// loads, which a half-warp serves conflict-free for A/2 odd (A = 18: word index 9r + k);
// odd A: the row stride is odd, 32-bit loads are conflict-free.  AS > 0 is a compile-time
// number of actions (loops fully unrolled), AS == 0 takes it at run time.  Four independent
// accumulators keep four loads / MUFU ops in flight per thread.  exp() is one FFMA/FMUL into
// ex2.approx.ftz (<= 2 ulp plus 6e-8 |x| relative): the only terms it perturbs visibly are
// the already-negligible ones; log() stays the accurate logf (two per row).
//
// A row's log-probabilities are log p_j = (l_j - a) - b for a pair (a, b) of the row maximum m
// and lg = log sum_j exp(l_j - m) in [0, log A] (lse_pair).  Rows whose maximum is below
// kSplitLseAbove in magnitude take a = m + lg, b = 0, and their exponents exp2(l_j log2 e -
// m log2 e): one rounding each, the arithmetic of earlier versions bit for bit (a learner step's
// result, and so a training run, is unchanged for ordinary logits).  Those forms round to an ulp
// of m, 1e-5..1e-4 of every probability for logits of magnitude 1e2..1e3 (a peaked policy, a
// large common offset), so larger maxima, and single-action rows (exactly log p = 0), take a = m,
// b = lg and exp2((l_j - m) log2 e): l_j - m is exact for every entry that matters.
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kSplitLseAbove = 16.f;
__device__ __forceinline__ bool split_lse(float m, int A) { return !(fabsf(m) < kSplitLseAbove && A > 1); }
__device__ __forceinline__ void lse_pair(float m, float lg, int A, float* a, float* b) {
  if (split_lse(m, A)) {
    *a = m; *b = lg;
  } else {
    *a = m + lg; *b = 0.f;
  }
}
__device__ __forceinline__ float ex2_ftz(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

template <int AS, typename F4, typename F1>
__device__ __forceinline__ void row_foreach(const float* l, int A_rt, F4 f4, F1 f1) {
  const int A = AS ? AS : A_rt;
  int j = 0;
  if ((A & 1) == 0) {
    const float2* l2 = reinterpret_cast<const float2*>(l);
    if (AS > 0) {
#pragma unroll
      for (int jj = 0; jj + 3 < AS; jj += 4) {
        const float2 a = l2[jj >> 1], b = l2[(jj >> 1) + 1];
        f4(jj, a.x, a.y, b.x, b.y);
      }
      j = AS & ~3;
    } else {
#pragma unroll 1
      for (; j + 3 < A; j += 4) {
        const float2 a = l2[j >> 1], b = l2[(j >> 1) + 1];
        f4(j, a.x, a.y, b.x, b.y);
      }
    }
    if (j < A) {
      const float2 a = l2[j >> 1];
      f1(j, a.x);
      f1(j + 1, a.y);
    }
  } else {
    if (AS > 0) {
#pragma unroll
      for (int jj = 0; jj + 3 < AS; jj += 4) f4(jj, l[jj], l[jj + 1], l[jj + 2], l[jj + 3]);
      j = AS & ~3;
    } else {
#pragma unroll 1
      for (; j + 3 < A; j += 4) f4(j, l[j], l[j + 1], l[j + 2], l[j + 3]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
      if (j + k < A) f1(j + k, l[j + k]);
  }
}

template <int AS>
__device__ __forceinline__ float row_max(const float* l, int A) {
  float m0 = -INFINITY, m1 = -INFINITY, m2 = -INFINITY, m3 = -INFINITY;
  row_foreach<AS>(l, A,
      [&](int, float x0, float x1, float x2, float x3) {
        m0 = fmaxf(m0, x0); m1 = fmaxf(m1, x1); m2 = fmaxf(m2, x2); m3 = fmaxf(m3, x3);
      },
      [&](int, float x0) { m0 = fmaxf(m0, x0); });
  return fmaxf(fmaxf(m0, m1), fmaxf(m2, m3));
}
// sum_j exp(l_j - m)
template <int AS>
__device__ __forceinline__ float row_sumexp(const float* l, int A, float m) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
  auto sum = [&](auto ex) {
    row_foreach<AS>(l, A,
        [&](int, float x0, float x1, float x2, float x3) {
          s0 += ex2_ftz(ex(x0)); s1 += ex2_ftz(ex(x1)); s2 += ex2_ftz(ex(x2)); s3 += ex2_ftz(ex(x3));
        },
        [&](int, float x0) { s0 += ex2_ftz(ex(x0)); });
  };
  if (split_lse(m, AS ? AS : A)) {
    sum([&](float x) { return (x - m) * kLog2e; });         // m split off exactly
  } else {
    const float nm2 = -m * kLog2e;
    sum([&](float x) { return fmaf(x, kLog2e, nm2); });     // m log2 e rounded: see lse_residual
  }
  return (s0 + s1) + (s2 + s3);
}
// log sum_j exp(l_j - m) from the log of row_sumexp: rows that do not split off m summed
// exp2(l_j log2 e - round(m log2 e)), which carries the factor 2^r of the rounding residual
// r = m log2 e - round(m log2 e) (exact by one FMA); the split form removes it.
__device__ __forceinline__ float lse_residual_free(float m, float lg, int A) {
  return split_lse(m, A) ? lg : fmaf(-fmaf(m, kLog2e, -m * kLog2e), 0.6931471805599453f, lg);
}
// se = sum_j exp(d_j), sel = sum_j exp(d_j) d_j with d_j = l_j - m
template <int AS>
__device__ __forceinline__ void row_sumexp_ent(const float* l, int A, float m, float* se, float* sel) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f, q0 = 0.f, q1 = 0.f, q2 = 0.f, q3 = 0.f;
  auto one = [&](float x, float& s, float& q) {
    const float d = x - m, e = ex2_ftz(d * kLog2e);
    s += e;
    q = fmaf(e, d, q);
  };
  row_foreach<AS>(l, A,
      [&](int, float x0, float x1, float x2, float x3) { one(x0, s0, q0); one(x1, s1, q1); one(x2, s2, q2); one(x3, s3, q3); },
      [&](int, float x0) { one(x0, s0, q0); });
  *se = (s0 + s1) + (s2 + s3);
  *sel = (q0 + q1) + (q2 + q3);
}
// in place: l_j <- wpg (1[j=a] - p_j) + wec p_j (log p_j + H),  log p_j = (l_j - la) - lb  (lse_pair)
//   d(-mean(tlp*pg))/dl_j = -pg/N (1[j=a]-p_j); d(kc*mean(blp-tlp)) = -kc/N (1[j=a]-p_j)
//   d(-ec*mean(H))/dl_j  = ec/N * p_j (log p_j + H)
// evaluated as p_j (wec (log p_j + H) - wpg), then + wpg on the taken action.
template <int AS>
__device__ __forceinline__ void row_grad(float* l, int A_rt, int a, float la, float lb, float ent, float wpg,
                                         float wec) {
  const int A = AS ? AS : A_rt;
  auto run = [&](auto logp_of) {
  auto g1 = [&](float x) {
    const float logp = logp_of(x);
    const float pj = ex2_ftz(logp * kLog2e);
    return pj * fmaf(wec, logp + ent, -wpg);
  };
  int j = 0;
  if ((A & 1) == 0) {
    float2* l2 = reinterpret_cast<float2*>(l);
    auto two = [&](int k) {
      float2 u = l2[k];
      u.x = g1(u.x); u.y = g1(u.y);
      l2[k] = u;
    };
    if (AS > 0) {
#pragma unroll
      for (int k = 0; k < AS / 2; ++k) two(k);
    } else {
#pragma unroll 1
      for (int k = 0; k < (A >> 1); ++k) two(k);
    }
  } else {
    if (AS > 0) {
#pragma unroll
      for (int jj = 0; jj < AS; ++jj) l[jj] = g1(l[jj]);
    } else {
#pragma unroll 1
      for (; j < A; ++j) l[j] = g1(l[j]);
    }
  }
  };
  if (lb == 0.f)
    run([&](float x) { return x - la; });              // (x - la) - 0, one rounding
  else
    run([&](float x) { return (x - la) - lb; });
  l[a] += wpg;
}

// Last CTA to arrive (ticket) reduces the per-CTA partials in index order and writes the
// loss terms; deterministic for a given grid.  POPART: partials 6 and 7 are sum vs and sum vs^2,
// written to pop_sums; the value-loss terms are left to seedrl_vtrace_popart_update.
template <bool POPART>
__device__ __forceinline__ void loss_finalize(const LossParams& p, float* s_red, float ec) {
  const int tid = threadIdx.x;
  const float mul = p.cfg.entropy_cost_adjustment_speed;
  const float kc = p.cfg.kl_cost;
  __shared__ bool s_last;
  if (tid == 0) {
    __threadfence();
    const unsigned int prev = atomicAdd(p.ticket, 1u);
    s_last = (prev == gridDim.x - 1);
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double acc5[5] = {0.0, 0.0, 0.0, 0.0, 0.0};
  float amax = 0.f;
  // deterministic: thread k sums slices k, k+256, ... then a fixed-order tree.
  for (unsigned int g = tid; g < gridDim.x; g += blockDim.x) {
    const volatile double* q = p.partials + (size_t)g * kLossPartials;
#pragma unroll
    for (int k = 0; k < 5; ++k) acc5[k] += q[k];
    amax = fmaxf(amax, (float)q[5]);
  }
  double tot[5];
#pragma unroll
  for (int k = 0; k < 5; ++k) tot[k] = block_reduce_sum_d(acc5[k]);
  const float max_a = block_reduce_max(amax, s_red);
  if (POPART) {
    double s1 = 0.0, s2 = 0.0;
    for (unsigned int g = tid; g < gridDim.x; g += blockDim.x) {
      const volatile double* q = p.partials + (size_t)g * kLossPartials;
      s1 += q[6];
      s2 += q[7];
    }
    s1 = block_reduce_sum_d(s1);
    s2 = block_reduce_sum_d(s2);
    if (tid == 0) {
      if (p.pop_sums_d) {   // rounded as pop_sums are, so phase 2 sees the same fp32 sums
        p.pop_sums_d[0] = (double)(float)s1;
        p.pop_sums_d[1] = (double)(float)s2;
        p.pop_sums_d[2] = (double)p.T * (double)p.B;
      } else {
        p.pop_sums[0] = (float)s1;
        p.pop_sums[1] = (float)s2;
      }
    }
  }
  if (tid == 0) {
    const double n = (double)p.T * (double)p.B;
    const float policy_loss = (float)(-tot[0] / n);
    const float mse = (float)(tot[1] / n);
    const float v_loss = p.cfg.baseline_cost * 0.5f * mse;
    const float mean_h = (float)(tot[2] / n);
    const float entropy_loss = -ec * mean_h;
    const float mean_kl = (float)(tot[3] / n);
    const float kl_loss = kc * mean_kl;
    float adj = 0.f, dparam = 0.f;
    if (p.cfg.has_target_entropy) {                        // :128-132
      adj = ec * (mean_h - p.cfg.target_entropy);
      dparam = mul * ec * (mean_h - p.cfg.target_entropy);
    }
    float* L = p.loss_terms;
    L[SEEDRL_LT_TOTAL] = policy_loss + v_loss + entropy_loss + kl_loss + adj;  // :134-135
    L[SEEDRL_LT_POLICY] = policy_loss;
    L[SEEDRL_LT_V] = v_loss;
    L[SEEDRL_LT_ENTROPY] = entropy_loss;
    L[SEEDRL_LT_KL] = kl_loss;
    L[SEEDRL_LT_ENTROPY_ADJ] = adj;
    L[SEEDRL_LT_V_MEAN] = (float)(tot[4] / n);
    L[SEEDRL_LT_V_L2_ERROR] = sqrtf(mse);
    L[SEEDRL_LT_MEAN_ENTROPY] = mean_h;
    L[SEEDRL_LT_ENTROPY_COST] = ec;
    L[SEEDRL_LT_MEAN_KL] = mean_kl;
    L[SEEDRL_LT_MAX_ACTION_ABS] = max_a;
    for (int k = 12; k < SEEDRL_LOSS_TERMS; ++k) L[k] = 0.f;
    *p.d_ecp = dparam;
    *p.ticket = 0u;   // self-reset for the next launch
  }
}

// Moves the CTA's logits tile between global memory ([T, B, A], columns b0..b0+nb) and
// shared memory ([T][BB][A], dense).  For each t the slice is nb*A contiguous floats; warp w
// takes rows t = w, w+8, ... and its lanes stride the row with float4 (all of a thread's
// loads are independent => several 16-byte requests in flight per thread).
template <bool LOAD>
__device__ __forceinline__ void tile_copy(float* s_tile, typename std::conditional<LOAD, const float*, float*>::type g,
                                          int T, int B, int A, int BB, int nb, int tid) {
  const int warp = tid >> 5, lane = tid & 31, nwarps = kLossThreads >> 5;
  const int n = nb * A;
  const bool vec = ((n & 3) == 0) && (((BB * A) & 3) == 0) && ((((size_t)B * A) & 3) == 0) &&
                   ((reinterpret_cast<uintptr_t>(g) & 15) == 0);
  for (int t = warp; t < T; t += nwarps) {
    float* sr = s_tile + (size_t)t * BB * A;
    auto gr = g + (size_t)t * B * A;
    if (vec) {
      for (int v = lane; v < (n >> 2); v += 32) {
        if (LOAD) reinterpret_cast<float4*>(sr)[v] = __ldg(reinterpret_cast<const float4*>(gr) + v);
        else reinterpret_cast<float4*>(const_cast<float*>(gr))[v] = reinterpret_cast<const float4*>(sr)[v];
      }
    } else {
      for (int e = lane; e < n; e += 32) {
        if (LOAD) sr[e] = __ldg(gr + e);
        else const_cast<float*>(gr)[e] = sr[e];
      }
    }
  }
}

// POPART: the values V are replaced by u = s (sigma V + mu) + m before the scan, the policy gradient
// takes pg_adv / s, and the value loss is left to seedrl_vtrace_popart_update: it gets (vs - u) / s
// in pop_td and sum vs, sum vs^2 in pop_sums.  TASKS: (s, m, sigma, mu) are those of the column's task,
// and the moment sums go to col_sums per column.
template <int MODE>
__device__ __forceinline__ void loss_small_body(const LossParams& p) {
  constexpr bool POPART = MODE != kPlain, TASKS = MODE == kPopArtTasks;
  extern __shared__ float smem[];
  __shared__ float s_cpop[TASKS ? 16 * 4 : 1];   // TASKS: (s, m, sigma, mu) of each column (BB <= 16)
  const int T = p.T, B = p.B, A = p.A, BB = p.BB;
  const int b0 = blockIdx.x * BB;
  const int nb = min(BB, B - b0);
  const int rows = T * BB;
  float* s_logits = smem;                      // [T][BB][A] dense, 16B-aligned rows of BB*A
  float* s_tlp = s_logits + (((size_t)rows * A + 3) & ~(size_t)3); // [rows] target logp -> later pg_adv
  float* s_blp = s_tlp + rows;                 // [rows] behaviour logp -> later v_err
  float* s_la = s_blp + rows;                  // [rows] lse_pair a
  float* s_lb = s_la + rows;                   // [rows] lse_pair b
  float* s_ent = s_lb + rows;                  // [rows]
  float* s_rew = s_ent + rows;                 // [rows] clipped reward r_{t+1}
  float* s_dis = s_rew + rows;                 // [rows] discount
  float* s_val = s_dis + rows;                 // [(T+1)*BB]
  int* s_act = reinterpret_cast<int*>(s_val + (T + 1) * BB);  // [rows]
  float* s_red = reinterpret_cast<float*>(s_act + rows);      // [32]
  uint8_t* s_ab = reinterpret_cast<uint8_t*>(s_red + 32);     // [rows] abandoned[t+1], iff p.abandoned
  const int tid = threadIdx.x;
  const float mul = p.cfg.entropy_cost_adjustment_speed;
  const float ec = expf(mul * __ldg(p.ecp));   // agent.entropy_cost(), learner.py:234

  // ---- small per-row inputs ------------------------------------------------
  for (int i = tid; i < rows; i += kLossThreads) {
    const int t = i / BB, c = i - t * BB;
    if (c < nb) {
      const size_t g1 = (size_t)(t + 1) * B + b0 + c;      // env_outputs[1:], learner.py:87
      float r = __ldg(p.rew + g1);
      if (p.cfg.max_abs_reward != 0.f)                     // :90-92
        r = fminf(fmaxf(r, -p.cfg.max_abs_reward), p.cfg.max_abs_reward);
      s_rew[i] = r;
      s_dis[i] = p.done[g1] ? 0.f : p.cfg.discounting;     // :93
      if (p.abandoned) s_ab[i] = p.abandoned[g1];
      int64_t a = p.act[(size_t)t * B + b0 + c];           // agent_outputs[:-1], :86
      s_act[i] = (int)a;
    } else {
      s_rew[i] = 0.f; s_dis[i] = 0.f; s_act[i] = 0;
      if (p.abandoned) s_ab[i] = 0;
    }
  }
  float pop_s = 1.f, pop_m = 0.f, pop_sigma = 1.f, pop_mu = 0.f;
  if (TASKS) {
    if (tid < BB)
      task_state(p, tid < nb ? task_slot(p.task_ids, p.num_tasks, p.task_error, b0 + tid, true) : p.num_tasks,
                 s_cpop + tid * 4);
    __syncthreads();
  } else if (POPART) {
    pop_m = __ldg(p.pop_mom);
    pop_s = popart_std(pop_m, __ldg(p.pop_mom + 1));
    pop_sigma = __ldg(p.pop_comp);
    pop_mu = __ldg(p.pop_comp + 1);
    if (p.task_ids && tid < nb && __ldg(p.task_ids + b0 + tid) != 0) atomicOr(p.task_error, 1);
  }
  for (int i = tid; i < (T + 1) * BB; i += kLossThreads) {
    const int t = i / BB, c = i - t * BB;
    if (TASKS) {
      const float* q = s_cpop + c * 4;
      s_val[i] = c < nb ? popart_u(__ldg(p.lb + (size_t)t * B + b0 + c), q[0], q[1], q[2], q[3]) : 0.f;
    } else if (POPART)
      s_val[i] = c < nb ? popart_u(__ldg(p.lb + (size_t)t * B + b0 + c), pop_s, pop_m, pop_sigma, pop_mu) : 0.f;
    else
      s_val[i] = c < nb ? __ldg(p.lb + (size_t)t * B + b0 + c) : 0.f;
  }

  double sum_tp = 0.0, sum_ve2 = 0.0, sum_h = 0.0, sum_kl = 0.0, sum_v = 0.0;
  double sum_vs = 0.0, sum_vs2 = 0.0;

  // ---- phase A: behaviour logits ------------------------------------------
  tile_copy<true>(s_logits, p.bl + (size_t)b0 * A, T, B, A, BB, nb, tid);
  __syncthreads();
  for (int i = tid; i < rows; i += kLossThreads) {
    const int c = i % BB;
    if (c < nb) {
      const float* l = s_logits + (size_t)i * A;
      const float m = row_max<0>(l, A);
      const float se = row_sumexp<0>(l, A, m);
      int a = s_act[i];
      a = a < 0 ? 0 : (a >= A ? A - 1 : a);
      const float lg = logf(se);
      float la, lb;
      lse_pair(m, lg, A, &la, &lb);
      s_blp[i] = (l[a] - la) - lb;                         // :97-98, for rho
      s_la[i] = (l[a] - m) - lse_residual_free(m, lg, A);  // split form, for the kl sum (until phase B)
    }
  }
  __syncthreads();
  // ---- phase B: learner logits --------------------------------------------
  tile_copy<true>(s_logits, p.ll + (size_t)b0 * A, T, B, A, BB, nb, tid);
  __syncthreads();
  for (int i = tid; i < rows; i += kLossThreads) {
    const int c = i % BB;
    if (c < nb) {
      const float* l = s_logits + (size_t)i * A;
      const float m = row_max<0>(l, A);
      float se, sel;
      row_sumexp_ent<0>(l, A, m, &se, &sel);
      const float lg = logf(se);
      int a = s_act[i];
      a = a < 0 ? 0 : (a >= A ? A - 1 : a);
      float la, lb;
      lse_pair(m, lg, A, &la, &lb);
      const float tl = (l[a] - la) - lb;                   // :95-96
      const float tls = (l[a] - m) - lg;                   // split form: the loss sums
      sum_kl += s_la[i] - tls;                             // :124
      s_la[i] = la;
      s_lb[i] = lb;
      s_tlp[i] = tls;
      s_blp[i] = tl - s_blp[i];                            // log rho
      s_ent[i] = lg - sel / se;                            // :119-120
    }
  }
  __syncthreads();

  // ---- phase C: reverse-time V-trace scan, one thread per column -----------
  float max_a = 0.f;
  if (tid < nb) {
    const int c = tid;
    const bool hcr = !isnan(p.cfg.clip_rho_threshold);
    const bool hcp = !isnan(p.cfg.clip_pg_rho_threshold);
    const bool has_ab = p.abandoned != nullptr;
    const float cs = TASKS ? s_cpop[c * 4] : pop_s;        // the column's PopArt s
    const float bootv = s_val[T * BB + c];                 // :82
    float acc = 0.f, vs_next = bootv, v_next = bootv;
    for (int t = T - 1; t >= 0; --t) {
      const int i = t * BB + c;
      const float tl = s_tlp[i];
      const float rho = expf(s_blp[i]);
      const float crho = hcr ? fminf(p.cfg.clip_rho_threshold, rho) : rho;
      const float cc = fminf(1.0f, rho) * p.cfg.lambda_;
      const float v = s_val[i], d = s_dis[i], r = s_rew[i];
      const bool masked = has_ab && s_ab[i];
      const float delta = masked ? 0.f : crho * (r + d * v_next - v);
      acc = delta + d * cc * acc;
      const float vs_t = acc + v;
      const float cpg = masked ? 0.f : (hcp ? fminf(p.cfg.clip_pg_rho_threshold, rho) : rho);
      const float pg = cpg * (r + d * vs_next - v);
      vs_next = vs_t;
      v_next = v;
      const float verr = vs_t - v;                         // :115
      if (POPART) {
        const float pgn = __fdiv_rn(pg, cs);               // generalized_onpolicy_loss.py:129-132
        sum_tp += tl * pgn;
        sum_vs += vs_t;
        sum_vs2 += (double)vs_t * vs_t;
        s_tlp[i] = pgn;
        s_blp[i] = __fdiv_rn(verr, cs);
      } else {
        sum_tp += tl * pg;                                 // :111-112
        sum_ve2 += verr * verr;                            // :116
        s_tlp[i] = pg;     // reuse: pg_adv
        s_blp[i] = verr;   // reuse: v_err
      }
      sum_h += s_ent[i];
      sum_v += v;
      max_a = fmaxf(max_a, fabsf((float)s_act[i]));
      const size_t g = (size_t)t * B + b0 + c;
      if (p.vs_out) p.vs_out[g] = vs_t;
      if (p.pg_out) p.pg_out[g] = pg;
    }
    if (TASKS) {   // one thread per column: its sums are the column's
      p.col_sums[2 * (size_t)(b0 + c)] = sum_vs;
      p.col_sums[2 * (size_t)(b0 + c) + 1] = sum_vs2;
    }
  }
  __syncthreads();

  // ---- phase D: gradients, thread-per-row in place, then a vectorised write-back -----
  const float invN = 1.0f / ((float)T * (float)B);
  const float kc = p.cfg.kl_cost;
  for (int i = tid; i < rows; i += kLossThreads) {
    const int c = i % BB;
    if (c < nb) {
      float* l = s_logits + (size_t)i * A;
      const float wpg = -(s_tlp[i] + kc) * invN, wec = ec * invN;
      int a = s_act[i];
      a = a < 0 ? 0 : (a >= A ? A - 1 : a);
      row_grad<0>(l, A, a, s_la[i], s_lb[i], s_ent[i], wpg, wec);
    }
  }
  __syncthreads();
  tile_copy<false>(s_logits, p.dlogits + (size_t)b0 * A, T, B, A, BB, nb, tid);
  {  // last row (bootstrap step): zero gradient
    float* dst = p.dlogits + ((size_t)T * B + b0) * A;
    for (int e = tid; e < nb * A; e += kLossThreads) dst[e] = 0.f;
  }
  for (int i = tid; i < (T + 1) * BB; i += kLossThreads) {
    const int t = i / BB, c = i - t * BB;
    if (c < nb) {
      if (POPART && t < T) {
        p.pop_td[(size_t)t * B + b0 + c] = s_blp[i];
      } else {
        // d(bc*0.5*mean((vs-V)^2))/dV = -bc*(vs-V)/N
        p.dbaseline[(size_t)t * B + b0 + c] = t < T ? -p.cfg.baseline_cost * s_blp[i] * invN : 0.f;
      }
    }
  }

  // ---- per-CTA partials, then last-CTA finalisation -------------------------
  double r;
  double* part = p.partials + (size_t)blockIdx.x * kLossPartials;
  r = block_reduce_sum_d(sum_tp);  if (tid == 0) part[0] = r;
  r = block_reduce_sum_d(sum_ve2); if (tid == 0) part[1] = r;
  r = block_reduce_sum_d(sum_h);   if (tid == 0) part[2] = r;
  r = block_reduce_sum_d(sum_kl);  if (tid == 0) part[3] = r;
  r = block_reduce_sum_d(sum_v);   if (tid == 0) part[4] = r;
  r = block_reduce_max(max_a, s_red);   if (tid == 0) part[5] = r;
  if (MODE == kPopArt) {
    r = block_reduce_sum_d(sum_vs);  if (tid == 0) part[6] = r;
    r = block_reduce_sum_d(sum_vs2); if (tid == 0) part[7] = r;
  }
  loss_finalize<MODE == kPopArt>(p, s_red, ec);
}

__global__ void __launch_bounds__(kLossThreads) vtrace_loss_kernel(const LossParams p) { loss_small_body<kPlain>(p); }
// min 2 CTAs/SM: without it ptxas caps this instantiation at 64 registers and spills in the scan
__global__ void __launch_bounds__(kLossThreads, 2) vtrace_popart_loss_kernel(const LossParams p) {
  loss_small_body<kPopArt>(p);
}
__global__ void __launch_bounds__(kLossThreads, 2) vtrace_popart_tasks_loss_kernel(const LossParams p) {
  loss_small_body<kPopArtTasks>(p);
}


// ---------------------------------------------------------------------------
// (a2, streaming form)  Same math, laid out for HBM throughput at large B.
//
// Persistent CTAs walk tiles of BB columns x T steps.  Each logits tile is ONE TMA tensor
// copy (cp.async.bulk.tensor.2d: box = [T] x [BB*A floats] of the [T+1, B*A] matrix) into a
// ring of three shared-memory buffers; the gradient tile is written in place and leaves
// through one TMA tensor store.  Load order is bl_0, ll_0, bl_1, ll_1, ... (load k ->
// buffer k % 3): both tiles of tile i+1 are requested right after phase A of tile i, so
// they stream in behind phases B..D while the dlogits store of tile i-1 drains -- HBM never
// idles behind the math.  The small per-row inputs (reward, done, action, baseline) of
// tile i+1 are prefetched into registers during tile i.
//   phase A   thread-per-row: behaviour log-prob                      (frees that buffer)
//   phase B   thread-per-row: lse, target log-prob, entropy, rho -> (delta_t, d_t*c_t, clipped pg rho)
//   scan      warp-per-column: acc_t = delta_t + (d_t c_t) acc_{t+1} as a suffix scan of affine
//             maps x -> Q + P x over lanes (each lane owns ceil(T/32) steps)
//   phase D   thread-per-row: pg advantage, loss sums, gradient in place, dbaseline
// Loss sums are kept per thread over all tiles of the CTA (fixed tile->CTA map =>
// deterministic), reduced once per CTA, finalised by the last CTA in index order.
constexpr int kStreamThreadsMax = 1024;
constexpr size_t kStreamSmemMax = 227 * 1024 - 2048;   // dynamic part; the kernel has ~1.2 KB static
constexpr int kStreamRounds = 4;    // register-prefetch rounds for the per-row inputs

__device__ __forceinline__ uint32_t sm_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_wait_or_trap(uint64_t* bar, uint32_t parity) {
  uint32_t done = 0;
  int spins = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}\n"
        : "=r"(done)
        : "r"(sm_u32(bar)), "r"(parity)
        : "memory");
    if (!done && ++spins > (1 << 24)) __trap();   // never hang the GPU
  }
}

struct SmallRegs {
  float rew[kStreamRounds], val[kStreamRounds];
  int act[kStreamRounds];
  uint8_t done[kStreamRounds], ab[kStreamRounds];
};

// POPART, TASKS: as in loss_small_body.  TASKS stages the state of every task in shared memory and
// takes each column's sums of vs in the scan.
template <int AS, int MODE>
__device__ __forceinline__ void loss_stream_body(const LossParams& p, const int ntiles, const int tile_stride_f,
                                                 const CUtensorMap& tm_bl, const CUtensorMap& tm_ll,
                                                 const CUtensorMap& tm_dl) {
  extern __shared__ __align__(128) float smem[];
  const int T = p.T, B = p.B, A = AS ? AS : p.A, BB = p.BB;
  const int rows = T * BB;
  const uint32_t tile_bytes = (uint32_t)(rows * A) * 4u;
  float* s_tiles = smem;                             // [3] x [T][BB][A], 128-byte aligned each
  float* s_tlp = s_tiles + (size_t)3 * tile_stride_f;   // [rows] target logp
  float* s_acc = s_tlp + rows;                       // [rows] behaviour logp -> delta -> vs - V
  float* s_la = s_acc + rows;                        // [rows] lse_pair a
  float* s_lb = s_la + rows;                         // [rows] lse_pair b
  float* s_ent = s_lb + rows;
  float* s_rew = s_ent + rows;
  float* s_dis = s_rew + rows;
  float* s_dc = s_dis + rows;                        // [rows] discount_t * c_t
  float* s_cpg = s_dc + rows;                        // [rows] clipped pg rho
  float* s_val = s_cpg + rows;                       // [(T+1)*BB]
  int* s_act = reinterpret_cast<int*>(s_val + (T + 1) * BB);
  float* s_red = reinterpret_cast<float*>(s_act + rows);   // [32]
  uint64_t* s_full = reinterpret_cast<uint64_t*>(s_red + 32);
  uint8_t* s_ab = reinterpret_cast<uint8_t*>(s_full + 3);   // [rows] abandoned[t+1], iff p.abandoned
  const int tid = threadIdx.x, nthreads = blockDim.x, warp = tid >> 5, lane = tid & 31;
  const float mul = p.cfg.entropy_cost_adjustment_speed;
  const float ec = expf(mul * __ldg(p.ecp));
  const bool hcr = !isnan(p.cfg.clip_rho_threshold);
  const bool hcp = !isnan(p.cfg.clip_pg_rho_threshold);
  const float invN = 1.0f / ((float)T * (float)B);
  const float kc = p.cfg.kl_cost;
  const int bb_sh = 31 - __clz(BB);                      // BB is a power of two
  int lpc = 32;                                          // lanes per column in the scan
  while (lpc > 1 && T <= lpc * 4) lpc >>= 1;
  constexpr bool POPART = MODE != kPlain, TASKS = MODE == kPopArtTasks;
  __shared__ float s_pop[4];                             // PopArt s, m, sigma, mu
  __shared__ float s_ptab[TASKS ? (kMaxTasks + 1) * 4 : 1];   // TASKS: (s, m, sigma, mu) by task, then identity

  if (TASKS && tid <= p.num_tasks) task_state(p, tid, s_ptab + tid * 4);
  if (tid == 0) {
    if (MODE == kPopArt) {
      s_pop[0] = popart_std(__ldg(p.pop_mom), __ldg(p.pop_mom + 1));
      s_pop[1] = __ldg(p.pop_mom);
      s_pop[2] = __ldg(p.pop_comp);
      s_pop[3] = __ldg(p.pop_comp + 1);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k)
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(sm_u32(s_full + k)));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_bl)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_ll)) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tm_dl)) : "memory");
  }
  __syncthreads();

  // per-thread sums stay fp32 (a thread adds one or a few rows per tile); the block and grid
  // reductions are float64
  float sum_tp = 0.f, sum_ve2 = 0.f, sum_h = 0.f, sum_kl = 0.f, sum_v = 0.f, max_a = 0.f;
  float sum_vs = 0.f, sum_vs2 = 0.f;
  // one thread, one instruction per tile
  auto issue_load = [&](int k, const CUtensorMap* tm, int tile) {
    uint64_t* bar = s_full + (k % 3);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(sm_u32(bar)),
                 "r"(tile_bytes)
                 : "memory");
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            sm_u32(s_tiles + (size_t)(k % 3) * tile_stride_f)),
        "l"(reinterpret_cast<uint64_t>(tm)), "r"(tile * BB * A), "r"(0), "r"(sm_u32(bar))
        : "memory");
  };
  auto load_small = [&](int tile, SmallRegs& r) {
#pragma unroll
    for (int k = 0; k < kStreamRounds; ++k) {
      const int i = tid + k * nthreads;
      if (i < (T + 1) * BB) {
        const int t = i >> bb_sh, c = i & (BB - 1);
        const size_t g = (size_t)t * B + (size_t)tile * BB + c;
        r.val[k] = __ldg(p.lb + g);
        if (t < T) {
          r.rew[k] = __ldg(p.rew + g + B);                 // env_outputs[1:], learner.py:87
          r.done[k] = p.done[g + B];
          if (p.abandoned) r.ab[k] = p.abandoned[g + B];
          r.act[k] = (int)p.act[g];                        // agent_outputs[:-1], :86
        }
        if (MODE == kPopArt && p.task_ids && t == 0 && __ldg(p.task_ids + tile * BB + c) != 0)
          atomicOr(p.task_error, 1);
      }
    }
  };
  auto store_small = [&](int tile, const SmallRegs& r) {
#pragma unroll
    for (int k = 0; k < kStreamRounds; ++k) {
      const int i = tid + k * nthreads;
      if (i < (T + 1) * BB) {
        if (TASKS) {
          const int c = i & (BB - 1);
          const float* q = s_ptab + task_slot(p.task_ids, p.num_tasks, p.task_error, tile * BB + c, i < BB) * 4;
          s_val[i] = popart_u(r.val[k], q[0], q[1], q[2], q[3]);
        } else {
          s_val[i] = POPART ? popart_u(r.val[k], s_pop[0], s_pop[1], s_pop[2], s_pop[3]) : r.val[k];
        }
        if (i < rows) {
          float rw = r.rew[k];
          if (p.cfg.max_abs_reward != 0.f)                 // :90-92
            rw = fminf(fmaxf(rw, -p.cfg.max_abs_reward), p.cfg.max_abs_reward);
          s_rew[i] = rw;
          s_dis[i] = r.done[k] ? 0.f : p.cfg.discounting;  // :93
          if (p.abandoned) s_ab[i] = r.ab[k];
          const int a = r.act[k];
          max_a = fmaxf(max_a, fabsf((float)a));
          s_act[i] = a < 0 ? 0 : (a >= A ? A - 1 : a);
        }
      }
    }
  };

  const int n_my = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;
  SmallRegs sm;
  if (n_my > 0) {
    if (tid == 0) {
      issue_load(0, &tm_bl, blockIdx.x);
      issue_load(1, &tm_ll, blockIdx.x);
    }
    load_small(blockIdx.x, sm);
    store_small(blockIdx.x, sm);
  }
  __syncthreads();

  for (int it = 0; it < n_my; ++it) {
    const int tile = blockIdx.x + it * gridDim.x;
    const int next = tile + gridDim.x;
    const bool has_next = it + 1 < n_my;
    const int k0 = 2 * it;
    if (has_next) load_small(next, sm);

    // ---- phase A: behaviour logits ----------------------------------------------------
    mbar_wait_or_trap(s_full + (k0 % 3), (uint32_t)((k0 / 3) & 1));
    {
      const float* tileA = s_tiles + (size_t)(k0 % 3) * tile_stride_f;
      for (int i = tid; i < rows; i += nthreads) {
        const float* l = tileA + (size_t)i * A;
        const float m = row_max<AS>(l, A);
        const float se = row_sumexp<AS>(l, A, m);
        const float lg = logf(se);
        float la, lb;
        lse_pair(m, lg, A, &la, &lb);
        s_acc[i] = (l[s_act[i]] - la) - lb;                // :97-98, for rho
        s_dc[i] = (l[s_act[i]] - m) - lse_residual_free(m, lg, A);   // split form, for the kl sum
      }
    }
    __syncthreads();
    if (tid == 0 && has_next) {
      // buffer (k0+2)%3 held the gradient tile of the previous iteration: its store has had
      // all of phase A to finish reading shared memory
      asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
      issue_load(k0 + 2, &tm_bl, next);
      issue_load(k0 + 3, &tm_ll, next);                    // into the buffer phase A just freed
    }

    // ---- phase B: learner logits, importance weights ----------------------------------
    mbar_wait_or_trap(s_full + ((k0 + 1) % 3), (uint32_t)(((k0 + 1) / 3) & 1));
    float* tileB = s_tiles + (size_t)((k0 + 1) % 3) * tile_stride_f;
    for (int i = tid; i < rows; i += nthreads) {
      const float* l = tileB + (size_t)i * A;
      const float m = row_max<AS>(l, A);
      float se, sel;
      row_sumexp_ent<AS>(l, A, m, &se, &sel);
      const float lg = logf(se);
      const int a = s_act[i];
      float la, lb;
      lse_pair(m, lg, A, &la, &lb);
      const float tl = (l[a] - la) - lb;                   // :95-96
      const float tls = (l[a] - m) - lg;                   // split form: the loss sums
      const float bp = s_acc[i];
      const float ent = lg - sel / se;                     // :119-120
      s_la[i] = la;
      s_lb[i] = lb;
      s_tlp[i] = tls;
      s_ent[i] = ent;
      sum_h += ent;
      sum_kl += s_dc[i] - tls;                             // :124
      const float rho = expf(tl - bp);                     // vtrace.py:84,110
      const float crho = hcr ? fminf(p.cfg.clip_rho_threshold, rho) : rho;
      const float cc = fminf(1.0f, rho) * p.cfg.lambda_;
      const float v = s_val[i], v_next = s_val[i + BB], d = s_dis[i];
      const bool masked = p.abandoned && s_ab[i];
      s_acc[i] = masked ? 0.f : crho * (s_rew[i] + d * v_next - v);   // delta_t, vtrace.py:122
      s_dc[i] = d * cc;
      s_cpg[i] = masked ? 0.f : (hcp ? fminf(p.cfg.clip_pg_rho_threshold, rho) : rho);
      sum_v += v;
    }
    __syncthreads();

    // ---- scan: acc_t = delta_t + d_t c_t acc_{t+1} (vtrace.py:128), in place -------------
    // LPC lanes share a column (32 / LPC columns per warp); a lane owns K = ceil(T / LPC)
    // consecutive steps, which compose to the affine map x -> Q + P x; a suffix scan of those
    // maps over the column's lanes gives every lane the accumulator entering its segment.
    {
      const int sub = lane & (lpc - 1);                    // lane within its column group
      const int K = (T + lpc - 1) / lpc;
      const int t_lo = sub * K, t_hi = min(t_lo + K, T);
      const int cols_per_warp = 32 / lpc;
      for (int c = warp * cols_per_warp + lane / lpc; c - lane / lpc < BB; c += (nthreads >> 5) * cols_per_warp) {
        const bool live = c < BB;
        float P = 1.f, Q = 0.f;
        if (live)
          for (int t = t_hi - 1; t >= t_lo; --t) {
            const float cf = s_dc[t * BB + c];
            Q = fmaf(cf, Q, s_acc[t * BB + c]);
            P *= cf;
          }
        for (int d = 1; d < lpc; d <<= 1) {
          const float Pd = __shfl_down_sync(0xffffffffu, P, d), Qd = __shfl_down_sync(0xffffffffu, Q, d);
          if (sub + d < lpc) {
            Q = fmaf(P, Qd, Q);
            P *= Pd;
          }
        }
        float acc = __shfl_down_sync(0xffffffffu, Q, 1);
        if (sub == lpc - 1) acc = 0.f;
        double cs1 = 0.0, cs2 = 0.0;                       // TASKS: this lane's sum of vs, vs^2
        if (live)
          for (int t = t_hi - 1; t >= t_lo; --t) {
            acc = fmaf(s_dc[t * BB + c], acc, s_acc[t * BB + c]);
            s_acc[t * BB + c] = acc;
            if (TASKS) {
              const float vs = acc + s_val[t * BB + c];      // phase D's vs, bit for bit
              cs1 += vs;
              cs2 += (double)vs * vs;
            }
          }
        if (TASKS) {   // the column's lanes, in a fixed tree
          for (int d = lpc >> 1; d > 0; d >>= 1) {
            cs1 += __shfl_down_sync(0xffffffffu, cs1, d);
            cs2 += __shfl_down_sync(0xffffffffu, cs2, d);
          }
          if (live && sub == 0) {
            p.col_sums[2 * ((size_t)tile * BB + c)] = cs1;
            p.col_sums[2 * ((size_t)tile * BB + c) + 1] = cs2;
          }
        }
      }
    }
    __syncthreads();

    // ---- phase D: advantages, loss sums, gradient in place -------------------------------
    for (int i = tid; i < rows; i += nthreads) {
      const int t = i >> bb_sh, c = i & (BB - 1);
      const float v = s_val[i], verr = s_acc[i];           // vs_t - V_t, :115
      const float vs_next = t + 1 < T ? s_acc[i + BB] + s_val[i + BB] : s_val[T * BB + c];
      const float pg = s_cpg[i] * (s_rew[i] + s_dis[i] * vs_next - v);   // vtrace.py:143-144
      const float tl = s_tlp[i];
      const size_t g = (size_t)t * B + (size_t)tile * BB + c;
      if (p.vs_out) p.vs_out[g] = verr + v;
      if (p.pg_out) p.pg_out[g] = pg;
      if (POPART) {
        const float s = TASKS ? s_ptab[task_slot(p.task_ids, p.num_tasks, nullptr, tile * BB + c, false) * 4]
                              : s_pop[0];
        const float pgn = __fdiv_rn(pg, s), vs = verr + v;   // generalized_onpolicy_loss.py:129-132
        sum_tp += tl * pgn;
        if (!TASKS) {
          sum_vs += vs;
          sum_vs2 += vs * vs;
        }
        p.pop_td[g] = __fdiv_rn(verr, s);
        row_grad<AS>(tileB + (size_t)i * A, A, s_act[i], s_la[i], s_lb[i], s_ent[i], -(pgn + kc) * invN, ec * invN);
      } else {
        sum_tp += tl * pg;                                 // :111-112
        sum_ve2 += verr * verr;                            // :116
        p.dbaseline[g] = -p.cfg.baseline_cost * verr * invN;
        row_grad<AS>(tileB + (size_t)i * A, A, s_act[i], s_la[i], s_lb[i], s_ent[i], -(pg + kc) * invN, ec * invN);
      }
    }
    // generic-proxy writes of the gradient tile -> visible to the TMA (async) proxy
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    if (tid == 0) {
      asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%1, %2}], [%3];" ::"l"(
                       reinterpret_cast<uint64_t>(&tm_dl)),
                   "r"(tile * BB * A), "r"(0), "r"(sm_u32(tileB))
                   : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    {  // bootstrap step: zero gradient
      float* dz = p.dlogits + ((size_t)T * B + (size_t)tile * BB) * A;
      for (int e = tid; e < BB * A; e += nthreads) dz[e] = 0.f;
      if (tid < BB) p.dbaseline[(size_t)T * B + (size_t)tile * BB + tid] = 0.f;
    }
    if (has_next) store_small(next, sm);   // every read of the per-row arrays is behind the barrier above
    __syncthreads();
  }
  if (tid == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");

  // ---- per-CTA partials, then last-CTA finalisation (same as vtrace_loss_kernel) ---------
  double r;
  double* part = p.partials + (size_t)blockIdx.x * kLossPartials;
  r = block_reduce_sum_d(sum_tp);  if (tid == 0) part[0] = r;
  r = block_reduce_sum_d(sum_ve2); if (tid == 0) part[1] = r;
  r = block_reduce_sum_d(sum_h);   if (tid == 0) part[2] = r;
  r = block_reduce_sum_d(sum_kl);  if (tid == 0) part[3] = r;
  r = block_reduce_sum_d(sum_v);   if (tid == 0) part[4] = r;
  r = block_reduce_max(max_a, s_red);   if (tid == 0) part[5] = r;
  if (MODE == kPopArt) {
    r = block_reduce_sum_d(sum_vs);  if (tid == 0) part[6] = r;
    r = block_reduce_sum_d(sum_vs2); if (tid == 0) part[7] = r;
  }
  loss_finalize<MODE == kPopArt>(p, s_red, ec);
}

template <int AS>
__global__ void __launch_bounds__(kStreamThreadsMax)
vtrace_loss_stream_kernel(const LossParams p, const int ntiles, const int tile_stride_f,
                          const __grid_constant__ CUtensorMap tm_bl, const __grid_constant__ CUtensorMap tm_ll,
                          const __grid_constant__ CUtensorMap tm_dl) {
  loss_stream_body<AS, kPlain>(p, ntiles, tile_stride_f, tm_bl, tm_ll, tm_dl);
}
template <int AS>
__global__ void __launch_bounds__(kStreamThreadsMax)
vtrace_popart_loss_stream_kernel(const LossParams p, const int ntiles, const int tile_stride_f,
                                 const __grid_constant__ CUtensorMap tm_bl, const __grid_constant__ CUtensorMap tm_ll,
                                 const __grid_constant__ CUtensorMap tm_dl) {
  loss_stream_body<AS, kPopArt>(p, ntiles, tile_stride_f, tm_bl, tm_ll, tm_dl);
}
template <int AS>
__global__ void __launch_bounds__(kStreamThreadsMax)
vtrace_popart_tasks_loss_stream_kernel(const LossParams p, const int ntiles, const int tile_stride_f,
                                       const __grid_constant__ CUtensorMap tm_bl,
                                       const __grid_constant__ CUtensorMap tm_ll,
                                       const __grid_constant__ CUtensorMap tm_dl) {
  loss_stream_body<AS, kPopArtTasks>(p, ntiles, tile_stride_f, tm_bl, tm_ll, tm_dl);
}

// ---------------------------------------------------------------------------
// (a2, PopArt phase 2)  After phase 1 (and the cross-replica sum of its two moment sums): the EMA
// and compensation update, the value loss and its gradients (steps 5-8 of the PopArt learner step,
// running_statistics.py:123-153, popart.py:163-183, generalized_onpolicy_loss.py:94-133).
// Grid-stride over the T x B value rows; every CTA derives the same new state from the same inputs,
// and the last CTA to arrive (ticket) reduces the per-CTA float64 partials in index order, writes
// the state and the loss terms.  No floating-point atomics: deterministic for a given shape.
//   e = n - (sigma+ V + mu+) = td + ((sigma V + mu) - (sigma+ V + mu+)),  td = (vs - u) / s
// (n = (vs - m)/s and u = s (sigma V + mu) + m).  The residual form is the kernels' own verr / s:
// with the state unchanged it gives phase 1's verr exactly, and it never subtracts two
// return-sized numbers.
constexpr int kPopThreads = 512;
constexpr int kPopPartials = 4;

struct PopArtUpdateParams {
  int T, B;
  float baseline_cost, beta;
  double count;            // elements behind pop_sums: world x T x B
  const float* lb;         // [T+1,B] learner baseline V
  const float* td;         // [T,B]
  const float* sums;       // [2]
  const double* sums_d;    // or [3] (sum vs, sum vs^2, rows), which then give the count
  float* mom;              // [2] mu1, mu2 (in/out)
  float* comp;             // [2] sigma, mu (in/out)
  float* dbaseline;        // rows [0,T)
  float* dcomp;            // [2] d sigma, d mu
  float* loss_terms;
  double* partials;        // [grid][4]
  unsigned int* ticket;
};

__global__ void __launch_bounds__(kPopThreads)
vtrace_popart_update_kernel(const PopArtUpdateParams p) {
  __shared__ bool s_last;
  const int tid = threadIdx.x;
  const float mu1 = p.mom[0], mu2 = p.mom[1], sigma = p.comp[0], mu = p.comp[1];
  // EMAMeanStd.update (running_statistics.py:123-147), in fp32 like the reference's variables
  const double count = p.sums_d ? p.sums_d[2] : p.count;
  const float sum1 = p.sums_d ? (float)p.sums_d[0] : p.sums[0], sum2 = p.sums_d ? (float)p.sums_d[1] : p.sums[1];
  const float bm1 = (float)((double)sum1 / count), bm2 = (float)((double)sum2 / count);
  const float mu1n = __fadd_rn(mu1, __fmul_rn(p.beta, __fsub_rn(bm1, mu1)));
  const float mu2n = __fadd_rn(mu2, __fmul_rn(p.beta, __fsub_rn(bm2, mu2)));
  const float s = popart_std(mu1, mu2), sn = popart_std(mu1n, mu2n);
  // popart.py:178-183
  const float sigma_n = __fmul_rn(__fdiv_rn(s, sn), sigma);
  const float mu_n = __fdiv_rn(__fadd_rn(__fsub_rn(mu1, mu1n), __fmul_rn(s, mu)), sn);

  const size_t n = (size_t)p.T * p.B;
  const float invN = 1.0f / ((float)p.T * (float)p.B);
  double se2 = 0.0, sev = 0.0, se = 0.0;
  for (size_t i = (size_t)blockIdx.x * kPopThreads + tid; i < n; i += (size_t)gridDim.x * kPopThreads) {
    const float V = __ldg(p.lb + i);
    const float e = __ldg(p.td + i) + (fmaf(sigma, V, mu) - fmaf(sigma_n, V, mu_n));
    // d(bc * 0.5 * mean(e^2)) / dV = -bc e sigma+ / N
    p.dbaseline[i] = (-p.baseline_cost * e * invN) * sigma_n;
    se2 += (double)e * e;
    sev += (double)e * V;
    se += e;
  }
  double r;
  double* part = p.partials + (size_t)blockIdx.x * kPopPartials;
  r = block_reduce_sum_d(se2); if (tid == 0) part[0] = r;
  r = block_reduce_sum_d(sev); if (tid == 0) part[1] = r;
  r = block_reduce_sum_d(se);  if (tid == 0) part[2] = r;
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  double a[3] = {0.0, 0.0, 0.0};
  for (unsigned int g = tid; g < gridDim.x; g += blockDim.x) {
    const volatile double* q = p.partials + (size_t)g * kPopPartials;
#pragma unroll
    for (int k = 0; k < 3; ++k) a[k] += q[k];
  }
  double tot[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) tot[k] = block_reduce_sum_d(a[k]);
  if (tid == 0) {
    const double nn = (double)n;
    const float mse = (float)(tot[0] / nn);
    const float v_loss = p.baseline_cost * 0.5f * mse;
    float* L = p.loss_terms;
    L[SEEDRL_LT_V] = v_loss;
    L[SEEDRL_LT_V_L2_ERROR] = sqrtf(mse);
    L[SEEDRL_LT_TOTAL] = L[SEEDRL_LT_POLICY] + v_loss + L[SEEDRL_LT_ENTROPY] + L[SEEDRL_LT_KL] +
                         L[SEEDRL_LT_ENTROPY_ADJ];
    L[SEEDRL_LT_POPART_MEAN] = mu1n;
    L[SEEDRL_LT_POPART_STD] = sn;
    p.dcomp[0] = (float)(-(double)p.baseline_cost * tot[1] / nn);
    p.dcomp[1] = (float)(-(double)p.baseline_cost * tot[2] / nn);
    p.mom[0] = mu1n;
    p.mom[1] = mu2n;
    p.comp[0] = sigma_n;
    p.comp[1] = mu_n;
    *p.ticket = 0u;
  }
}

// ---------------------------------------------------------------------------
// (a2, multi-task PopArt)  Phase 1 leaves each column's (sum_t vs, sum_t vs^2) in col_sums; this kernel
// reduces them by task into sums [K,3] = (sum vs, sum vs^2, rows), float64 throughout: the row counts
// stay exact to 2^53 (a float32 count stops at 2^24 = 8 replicas x T = 100 x B = 20 972), and the
// cross-replica SUM all-reduce adds them exactly.  Deterministic: a warp adds the columns of each task
// in lane order (warp_task_sums), each warp keeps its own per-task sums in shared memory in a fixed
// column order, a CTA adds its warps in order, and the last CTA adds the CTAs in index order.
constexpr int kTaskThreads = 256;
constexpr int kTaskPartials = 3 * kMaxTasks;   // doubles per CTA in the moments and update kernels

// Every lane gets the sum of `NV` values over the lanes of the warp whose slot equals its own, added in
// lane order; returns the mask of those lanes (the lowest one stores the group's sums).
template <int NV>
__device__ __forceinline__ unsigned warp_task_sums(int slot, const double* v, double* g) {
#pragma unroll
  for (int k = 0; k < NV; ++k) g[k] = 0.0;
  for (int j = 0; j < 32; ++j) {
    const int sj = __shfl_sync(0xffffffffu, slot, j);
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const double x = __shfl_sync(0xffffffffu, v[k], j);
      if (sj == slot) g[k] += x;
    }
  }
  return __match_any_sync(0xffffffffu, slot);
}

struct TaskMomentParams {
  int T, B, K;
  const int* task_ids;
  const double* col_sums;  // [B,2]
  double* sums;            // [K,3]
  double* partials;        // [grid][kTaskPartials]
  unsigned int* ticket;
};

__global__ void __launch_bounds__(kTaskThreads) vtrace_popart_task_moments_kernel(const TaskMomentParams p) {
  __shared__ double s_acc[kTaskThreads / 32][kMaxTasks][3];
  __shared__ bool s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int j = tid; j < (kTaskThreads / 32) * kMaxTasks * 3; j += kTaskThreads) (&s_acc[0][0][0])[j] = 0.0;
  __syncthreads();
  for (int base = blockIdx.x * kTaskThreads + warp * 32; base < p.B; base += gridDim.x * kTaskThreads) {
    const int b = base + lane;
    // ids were checked (and reported) by phase 1; a column outside [0, K) is left out here
    const int slot = b < p.B ? task_slot(p.task_ids, p.K, nullptr, b, false) : p.K;
    double v[2] = {0.0, 0.0}, g[2];
    if (slot < p.K) {
      v[0] = p.col_sums[2 * (size_t)b];
      v[1] = p.col_sums[2 * (size_t)b + 1];
    }
    const unsigned grp = warp_task_sums<2>(slot, v, g);
    if (lane == __ffs(grp) - 1 && slot < p.K) {
      s_acc[warp][slot][0] += g[0];
      s_acc[warp][slot][1] += g[1];
      s_acc[warp][slot][2] += (double)p.T * __popc(grp);
    }
  }
  __syncthreads();
  double* part = p.partials + (size_t)blockIdx.x * kTaskPartials;
  for (int j = tid; j < 3 * p.K; j += kTaskThreads) {
    double a = 0.0;
    for (int w = 0; w < kTaskThreads / 32; ++w) a += s_acc[w][j / 3][j % 3];
    part[j] = a;
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  for (int j = tid; j < 3 * p.K; j += kTaskThreads) {
    double a = 0.0;
    for (unsigned int g = 0; g < gridDim.x; ++g) a += __ldcg(p.partials + (size_t)g * kTaskPartials + j);
    p.sums[j] = a;
  }
  if (tid == 0) *p.ticket = 0u;
}

// Phase 2 with tasks: vtrace_popart_update_kernel with each task's own EMA and compensation update, and each
// row's value error taken with its column's task state.  A task without rows (count 0) keeps its state bit
// for bit and gets a zero gradient.  One thread per column (its T rows), so a thread's e V and e sums belong
// to one task; the per-task reduction is the moments kernel's.  Loss means run over all T x B rows.
struct PopArtTasksUpdateParams {
  int T, B, K;
  float baseline_cost, beta;
  const float* lb;         // [T+1,B]
  const float* td;         // [T,B]
  const int* task_ids;     // [B]
  const double* sums;      // [K,3]
  float* mom;              // [K,2] (in/out)
  float* comp;             // [K,2] (in/out)
  float* dbaseline;
  float* dcomp;            // [K,2]
  float* loss_terms;
  double* partials;        // [grid][kTaskPartials]
  unsigned int* ticket;
};

// task k's state after the update: (mu1', mu2', sigma+, mu+) and its (sigma, mu) before
__device__ __forceinline__ void task_update(const PopArtTasksUpdateParams& p, int k, float* o) {
  const float mu1 = p.mom[2 * k], mu2 = p.mom[2 * k + 1], sigma = p.comp[2 * k], mu = p.comp[2 * k + 1];
  const double count = p.sums[3 * k + 2];
  o[4] = sigma; o[5] = mu;
  if (count == 0.0) {
    o[0] = mu1; o[1] = mu2; o[2] = sigma; o[3] = mu;
    return;
  }
  const float bm1 = (float)(p.sums[3 * k] / count), bm2 = (float)(p.sums[3 * k + 1] / count);
  const float mu1n = __fadd_rn(mu1, __fmul_rn(p.beta, __fsub_rn(bm1, mu1)));
  const float mu2n = __fadd_rn(mu2, __fmul_rn(p.beta, __fsub_rn(bm2, mu2)));
  const float s = popart_std(mu1, mu2), sn = popart_std(mu1n, mu2n);
  o[0] = mu1n; o[1] = mu2n;
  o[2] = __fmul_rn(__fdiv_rn(s, sn), sigma);
  o[3] = __fdiv_rn(__fadd_rn(__fsub_rn(mu1, mu1n), __fmul_rn(s, mu)), sn);
}

__global__ void __launch_bounds__(kPopThreads) vtrace_popart_tasks_update_kernel(const PopArtTasksUpdateParams p) {
  __shared__ float s_st[kMaxTasks + 1][6];   // task_update's; entry K: identity
  __shared__ double s_acc[kPopThreads / 32][kMaxTasks][2];
  __shared__ bool s_last;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  if (tid < p.K) task_update(p, tid, s_st[tid]);
  if (tid == p.K) {
    s_st[tid][0] = 0.f; s_st[tid][1] = 1.f;
    s_st[tid][2] = s_st[tid][4] = 1.f;
    s_st[tid][3] = s_st[tid][5] = 0.f;
  }
  for (int j = tid; j < (kPopThreads / 32) * kMaxTasks * 2; j += kPopThreads) (&s_acc[0][0][0])[j] = 0.0;
  __syncthreads();
  const float invN = 1.0f / ((float)p.T * (float)p.B);
  double se2 = 0.0;
  for (int base = blockIdx.x * kPopThreads + warp * 32; base < p.B; base += gridDim.x * kPopThreads) {
    const int b = base + lane;
    const int slot = b < p.B ? task_slot(p.task_ids, p.K, nullptr, b, false) : p.K;
    double v[2] = {0.0, 0.0}, g[2];
    if (b < p.B) {
      const float sigma_n = s_st[slot][2], mu_n = s_st[slot][3], sigma = s_st[slot][4], mu = s_st[slot][5];
      for (int t = 0; t < p.T; ++t) {
        const size_t i = (size_t)t * p.B + b;
        const float V = __ldg(p.lb + i);
        const float e = __ldg(p.td + i) + (fmaf(sigma, V, mu) - fmaf(sigma_n, V, mu_n));
        p.dbaseline[i] = (-p.baseline_cost * e * invN) * sigma_n;
        se2 += (double)e * e;
        v[0] += (double)e * V;
        v[1] += e;
      }
    }
    const unsigned grp = warp_task_sums<2>(slot, v, g);
    if (lane == __ffs(grp) - 1 && slot < p.K) {
      s_acc[warp][slot][0] += g[0];
      s_acc[warp][slot][1] += g[1];
    }
  }
  double* part = p.partials + (size_t)blockIdx.x * kTaskPartials;
  const double r = block_reduce_sum_d(se2);
  if (tid == 0) part[2 * kMaxTasks] = r;
  __syncthreads();
  for (int j = tid; j < 2 * p.K; j += kPopThreads) {
    double a = 0.0;
    for (int w = 0; w < kPopThreads / 32; ++w) a += s_acc[w][j >> 1][j & 1];
    part[j] = a;
  }
  __syncthreads();
  if (tid == 0) {
    __threadfence();
    s_last = atomicAdd(p.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const double nn = (double)p.T * (double)p.B;
  for (int j = tid; j < 2 * p.K; j += kPopThreads) {
    double a = 0.0;
    for (unsigned int g = 0; g < gridDim.x; ++g) a += __ldcg(p.partials + (size_t)g * kTaskPartials + j);
    const int k = j >> 1;
    // d(bc * 0.5 * mean(e^2)) / d(sigma_k, mu_k) = -bc (sum_k e V, sum_k e) / N; exactly 0 without rows
    p.dcomp[j] = p.sums[3 * k + 2] == 0.0 ? 0.f : (float)(-(double)p.baseline_cost * a / nn);
  }
  double a2 = 0.0;
  for (unsigned int g = tid; g < gridDim.x; g += blockDim.x) a2 += __ldcg(p.partials + (size_t)g * kTaskPartials + 2 * kMaxTasks);
  const double tot2 = block_reduce_sum_d(a2);
  __syncthreads();   // every CTA read mom / comp before it took its ticket; the partial reads above are done
  if (tid < p.K) {
    const float* o = s_st[tid];
    p.mom[2 * tid] = o[0];
    p.mom[2 * tid + 1] = o[1];
    p.comp[2 * tid] = o[2];
    p.comp[2 * tid + 1] = o[3];
  }
  if (tid == 0) {
    const float mse = (float)(tot2 / nn);
    const float v_loss = p.baseline_cost * 0.5f * mse;
    float* L = p.loss_terms;
    L[SEEDRL_LT_V] = v_loss;
    L[SEEDRL_LT_V_L2_ERROR] = sqrtf(mse);
    L[SEEDRL_LT_TOTAL] = L[SEEDRL_LT_POLICY] + v_loss + L[SEEDRL_LT_ENTROPY] + L[SEEDRL_LT_KL] +
                         L[SEEDRL_LT_ENTROPY_ADJ];
    L[SEEDRL_LT_POPART_MEAN] = 0.f;   // unused with tasks: each task's state is in popart_moments
    L[SEEDRL_LT_POPART_STD] = 0.f;
    *p.ticket = 0u;
  }
}

// has_ab: room for the abandoned mask, rows bytes after the rest
static size_t loss_smem_bytes(int T, int A, int BB, bool has_ab) {
  const size_t rows = (size_t)T * BB;
  return (((rows * A + 3) & ~(size_t)3) + rows * 7 + (size_t)(T + 1) * BB + rows + 32) * 4 +
         (has_ab ? (rows + 3) & ~(size_t)3 : 0);
}

// Columns per CTA for vtrace_loss_kernel: the largest power of two <= 16 whose tile fits in
// shared memory, then halved while the grid would leave SMs idle (small B: latency matters,
// not bandwidth) as long as rows stay float4-copyable.
static int pick_bb(int T, int B, int A, bool has_ab, size_t* smem_bytes) {
  int BB = 16;
  while (BB >= 1 && loss_smem_bytes(T, A, BB, has_ab) > 200 * 1024) BB >>= 1;
  if (BB == 0) return 0;
  while (BB > 1 && ceil_div(B, BB) < kNumSMs && (((BB / 2) * A) & 3) == 0) BB >>= 1;
  *smem_bytes = loss_smem_bytes(T, A, BB, has_ab);
  return BB;
}

static int stream_tile_stride_f(int T, int A, int BB) {   // floats per ring buffer, 128-byte multiple
  return (T * BB * A + 31) & ~31;
}
static size_t stream_smem_bytes(int T, int A, int BB, bool has_ab) {
  const size_t rows = (size_t)T * BB;
  return (3 * (size_t)stream_tile_stride_f(T, A, BB) + 9 * rows + (size_t)(T + 1) * BB + rows + 32) * 4 + 3 * 8 + 128 +
         (has_ab ? rows : 0);
}

static int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = kNumSMs;
  }
  return n;
}

// [T1, B*A] fp32 matrix, box = T rows x BB*A floats (one tile), dense in shared memory.
static bool make_tile_map(CUtensorMap* tm, const float* base, int T1, int T, int B, int A, int BB) {
  const cuuint64_t gdim[2] = {(cuuint64_t)B * A, (cuuint64_t)T1};
  const cuuint64_t gstr[1] = {(cuuint64_t)B * A * sizeof(float)};
  const cuuint32_t box[2] = {(cuuint32_t)(BB * A), (cuuint32_t)T};
  const cuuint32_t estr[2] = {1, 1};
  return encode_tiled_fn()(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box,
                           estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// The streaming kernel applies when every tile is full, the TMA box is legal (inner extent
// BB*A <= 256 floats and a 16-byte multiple, T <= 256 rows, 16-byte aligned bases and row
// pitch), and there is at least one tile per SM.  Returns BB (0 = use vtrace_loss_kernel).
static int pick_stream(const LossParams& p, int forced_bb, int* threads, size_t* smem_bytes) {
  const int T = p.T, B = p.B, A = p.A;
  auto aligned16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!aligned16(p.ll) || !aligned16(p.bl) || !aligned16(p.dlogits)) return 0;
  if (T > 256 || (((size_t)B * A) & 3) != 0 || !encode_tiled_fn()) return 0;
  // two passes: first the largest BB that leaves room for two CTAs per SM (one CTA's
  // barriers and scan then hide behind the other's phases), else the largest that fits
  for (int pass = 0; pass < 2; ++pass)
  for (int BB = 16; BB >= 2; BB >>= 1) {
    if (forced_bb > 1 && BB != forced_bb) continue;
    if (B % BB != 0 || ((BB * A) & 3) != 0 || BB * A > 256) continue;
    if (B / BB < num_sms()) continue;
    const size_t bytes = stream_smem_bytes(T, A, BB, p.abandoned != nullptr);
    // the tasks kernel's static state table takes from the same 227 KB
    if (bytes > kStreamSmemMax - (p.task_ids && p.num_tasks > 0 ? (kMaxTasks + 1) * 16 : 0)) continue;
    if (pass == 0 && forced_bb <= 1 && 2 * (bytes + 2048 + 1024) > (size_t)228 * 1024) continue;
    const int rows = T * BB;
    const int rounds = ceil_div(rows, kStreamThreadsMax);
    int th = ceil_div(ceil_div(rows, rounds), 32) * 32;
    if (th < 128) th = 128;
    if ((T + 1) * BB > kStreamRounds * th) continue;
    *threads = th;
    *smem_bytes = bytes;
    return BB;
  }
  return 0;
}

template <int AS, int MODE>
static cudaError_t launch_stream(const LossParams& p, int ntiles, int threads, size_t smem, cudaStream_t stream,
                                 const CUtensorMap& tm_bl, const CUtensorMap& tm_ll, const CUtensorMap& tm_dl) {
  auto kernel = MODE == kPopArtTasks ? vtrace_popart_tasks_loss_stream_kernel<AS>
              : MODE == kPopArt      ? vtrace_popart_loss_stream_kernel<AS>
                                     : vtrace_loss_stream_kernel<AS>;
  const cudaError_t e = MODE == kPopArtTasks ? allow_smem<vtrace_popart_tasks_loss_stream_kernel<AS>>((int)kStreamSmemMax)
                      : MODE == kPopArt      ? allow_smem<vtrace_popart_loss_stream_kernel<AS>>((int)kStreamSmemMax)
                                             : allow_smem<vtrace_loss_stream_kernel<AS>>((int)kStreamSmemMax);
  if (e != cudaSuccess) return e;
  // persistent CTAs: as many per SM as shared memory and threads allow (small T: several,
  // so one CTA's barriers and scan hide behind another's copies)
  int per_sm = (int)((size_t)(228 * 1024) / (smem + 2048 + 1024));   // 228 KB/SM, 1 KB/CTA reserved
  if (per_sm > 2048 / threads) per_sm = 2048 / threads;
  if (per_sm > 6) per_sm = 6;
  if (per_sm < 1) per_sm = 1;
  int grid = num_sms() * per_sm;
  if (grid > ntiles) grid = ntiles;
  kernel<<<grid, threads, smem, stream>>>(
      p, ntiles, stream_tile_stride_f(p.T, p.A, p.BB), tm_bl, tm_ll, tm_dl);
  return cudaSuccess;
}

}  // namespace seedrl

using namespace seedrl;

static int g_loss_stream_enabled = 1;

// Test hook: 0 forces vtrace_loss_kernel for every shape, 1 (default) lets large aligned
// batches take vtrace_loss_stream_kernel, 2/4/8/16 additionally pins its columns per tile.
extern "C" int seedrl_debug_set_loss_stream(int enabled) {
  g_loss_stream_enabled = enabled < 0 ? 0 : enabled;
  return SEEDRL_OK;
}

extern "C" int seedrl_vtrace_from_importance_weights(
    int T, int B, const float* tlp, const float* blp, const float* disc, const float* rew,
    const float* val, const float* boot, float clip_rho, float clip_pg, float lambda_,
    float* vs, float* pg, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T >= 0 && B >= 0, "T and B must be non-negative");
  if (T == 0 || B == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(tlp && blp && disc && rew && val && boot && vs && pg, "null pointer");
  const int threads = 128;
  vtrace_kernel<5><<<ceil_div(B, threads), threads, 0, (cudaStream_t)stream>>>(
      T, B, tlp, blp, disc, rew, val, boot, clip_rho, clip_pg, lambda_, !isnan(clip_rho),
      !isnan(clip_pg), vs, pg);
  count_launch(PC_VTRACE, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_categorical_log_prob(int N, int A, const float* logits,
                                           const int64_t* actions, float* log_prob,
                                           seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 0 && A > 0, "bad N/A");
  if (N == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(logits && actions && log_prob, "null pointer");
  categorical_logprob_entropy_kernel<<<ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(
      N, A, logits, actions, log_prob, nullptr);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_categorical_entropy(int N, int A, const float* logits, float* entropy,
                                          seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 0 && A > 0, "bad N/A");
  if (N == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(logits && entropy, "null pointer");
  categorical_logprob_entropy_kernel<<<ceil_div(N, 8), 256, 0, (cudaStream_t)stream>>>(
      N, A, logits, nullptr, nullptr, entropy);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_categorical_sample(int N, int A, const float* logits,
                                         const float* gumbel_noise, uint64_t seed,
                                         uint64_t offset, int64_t* actions,
                                         seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 0 && A > 0, "bad N/A");
  if (N == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(logits && actions, "null pointer");
  categorical_sample_kernel<<<ceil_div(N, 128), 128, 0, (cudaStream_t)stream>>>(
      N, A, logits, gumbel_noise, seed, offset, nullptr, actions);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

__global__ void bump_counter_kernel(uint64_t* c) { *c += 1; }

// Same, with the Philox offset read from (and then incremented in) device memory: the call can be
// captured in a CUDA graph and still draw fresh noise on every replay.
extern "C" int seedrl_categorical_sample_counter(int N, int A, const float* logits, const float* gumbel_noise,
                                                 uint64_t seed, uint64_t* counter_dev, int64_t* actions,
                                                 seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(N >= 0 && A > 0, "bad N/A");
  if (N == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(logits && actions && counter_dev, "null pointer");
  categorical_sample_kernel<<<ceil_div(N, 128), 128, 0, (cudaStream_t)stream>>>(
      N, A, logits, gumbel_noise, seed, 0, counter_dev, actions);
  count_launch(PC_MISC, (cudaStream_t)stream);
  bump_counter_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(counter_dev);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" size_t seedrl_vtrace_loss_scratch_bytes(int T1, int B, int A) {
  (void)T1; (void)A;   // one partial slot per CTA; at most one CTA per column
  return 256 + (size_t)(B > kNumSMs ? B : kNumSMs) * kLossPartials * sizeof(double);
}

// Picks the kernel form (TMA-streamed at large aligned B, else vtrace_loss_kernel) and launches it;
// p has everything but BB.
template <int MODE>
static int launch_loss(LossParams p, cudaStream_t st) {
  const int T1 = p.T + 1, B = p.B, A = p.A;
  size_t smem = 0;
  auto small_kernel = MODE == kPopArtTasks ? vtrace_popart_tasks_loss_kernel
                    : MODE == kPopArt      ? vtrace_popart_loss_kernel
                                           : vtrace_loss_kernel;
  SEEDRL_CUDA(MODE == kPopArtTasks ? allow_smem<vtrace_popart_tasks_loss_kernel>(200 * 1024)
              : MODE == kPopArt    ? allow_smem<vtrace_popart_loss_kernel>(200 * 1024)
                                   : allow_smem<vtrace_loss_kernel>(200 * 1024));
  int threads = 0;
  p.BB = g_loss_stream_enabled ? pick_stream(p, g_loss_stream_enabled, &threads, &smem) : 0;
  alignas(64) CUtensorMap tm_bl, tm_ll, tm_dl;
  if (p.BB > 0 && !(make_tile_map(&tm_bl, p.bl, T1, p.T, B, A, p.BB) &&
                    make_tile_map(&tm_ll, p.ll, T1, p.T, B, A, p.BB) &&
                    make_tile_map(&tm_dl, p.dlogits, T1, p.T, B, A, p.BB)))
    p.BB = 0;
  if (p.BB > 0) {
    const int ntiles = B / p.BB;
    switch (A) {   // compile-time action counts of the reference's environments
      case 9:  SEEDRL_CUDA((launch_stream<9, MODE>(p, ntiles, threads, smem, st, tm_bl, tm_ll, tm_dl))); break;    // DMLab
      case 18: SEEDRL_CUDA((launch_stream<18, MODE>(p, ntiles, threads, smem, st, tm_bl, tm_ll, tm_dl))); break;   // Atari
      case 19: SEEDRL_CUDA((launch_stream<19, MODE>(p, ntiles, threads, smem, st, tm_bl, tm_ll, tm_dl))); break;   // football
      default: SEEDRL_CUDA((launch_stream<0, MODE>(p, ntiles, threads, smem, st, tm_bl, tm_ll, tm_dl))); break;
    }
  } else {
    p.BB = pick_bb(p.T, B, A, p.abandoned != nullptr, &smem);
    SEEDRL_CHECK_ARG(p.BB > 0, "unroll_length * num_actions too large for shared memory");
    small_kernel<<<ceil_div(B, p.BB), kLossThreads, smem, st>>>(p);
  }
  count_launch(PC_LOSS, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

static LossParams loss_params(int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
                              const float* behaviour_logits, const int64_t* actions, const float* rewards,
                              const uint8_t* done, const seedrl_loss_config* cfg, const float* entropy_cost_param,
                              float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
                              float* vs_out, float* pg_advantages_out, void* scratch) {
  LossParams p = {};
  p.T = T1 - 1; p.B = B; p.A = A;
  p.AP = A | 1;
  p.ll = learner_logits; p.lb = learner_baseline; p.bl = behaviour_logits;
  p.act = actions; p.rew = rewards; p.done = done; p.cfg = *cfg; p.ecp = entropy_cost_param;
  p.loss_terms = loss_terms; p.dlogits = dlogits; p.dbaseline = dbaseline;
  p.d_ecp = d_entropy_cost_param; p.vs_out = vs_out; p.pg_out = pg_advantages_out;
  p.ticket = reinterpret_cast<unsigned int*>(scratch);
  p.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
  return p;
}

extern "C" int seedrl_vtrace_loss_fwd_bwd_abandoned(
    int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
    const float* behaviour_logits, const int64_t* actions, const float* rewards,
    const uint8_t* done, const uint8_t* abandoned, const seedrl_loss_config* cfg, const float* entropy_cost_param,
    float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
    float* vs_out, float* pg_advantages_out, void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T1 >= 2 && B >= 1 && A >= 1, "need T1>=2, B>=1, A>=1");
  SEEDRL_CHECK_ARG(learner_logits && learner_baseline && behaviour_logits && actions &&
                       rewards && done && cfg && entropy_cost_param && loss_terms &&
                       dlogits && dbaseline && d_entropy_cost_param && scratch,
                   "null pointer");
  LossParams p = loss_params(T1, B, A, learner_logits, learner_baseline, behaviour_logits, actions, rewards, done,
                             cfg, entropy_cost_param, loss_terms, dlogits, dbaseline, d_entropy_cost_param,
                             vs_out, pg_advantages_out, scratch);
  p.abandoned = abandoned;
  return launch_loss<kPlain>(p, (cudaStream_t)stream);
}

extern "C" int seedrl_vtrace_loss_fwd_bwd(
    int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
    const float* behaviour_logits, const int64_t* actions, const float* rewards,
    const uint8_t* done, const seedrl_loss_config* cfg, const float* entropy_cost_param,
    float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
    float* vs_out, float* pg_advantages_out, void* scratch, seedrl_stream_t stream) {
  return seedrl_vtrace_loss_fwd_bwd_abandoned(T1, B, A, learner_logits, learner_baseline, behaviour_logits, actions,
                                              rewards, done, nullptr, cfg, entropy_cost_param, loss_terms, dlogits,
                                              dbaseline, d_entropy_cost_param, vs_out, pg_advantages_out, scratch,
                                              stream);
}

extern "C" int seedrl_vtrace_popart_loss_fwd_abandoned(
    int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
    const float* behaviour_logits, const int64_t* actions, const float* rewards,
    const uint8_t* done, const uint8_t* abandoned, const seedrl_loss_config* cfg, const float* entropy_cost_param,
    const float* popart_moments, const float* popart_compensation,
    float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
    float* vs_out, float* pg_advantages_out, float* td_out, float* moment_sums,
    void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T1 >= 2 && B >= 1 && A >= 1, "need T1>=2, B>=1, A>=1");
  SEEDRL_CHECK_ARG(learner_logits && learner_baseline && behaviour_logits && actions &&
                       rewards && done && cfg && entropy_cost_param && popart_moments &&
                       popart_compensation && loss_terms && dlogits && dbaseline &&
                       d_entropy_cost_param && td_out && moment_sums && scratch,
                   "null pointer");
  LossParams p = loss_params(T1, B, A, learner_logits, learner_baseline, behaviour_logits, actions, rewards, done,
                             cfg, entropy_cost_param, loss_terms, dlogits, dbaseline, d_entropy_cost_param,
                             vs_out, pg_advantages_out, scratch);
  p.pop_mom = popart_moments; p.pop_comp = popart_compensation;
  p.pop_td = td_out; p.pop_sums = moment_sums;
  p.abandoned = abandoned;
  return launch_loss<kPopArt>(p, (cudaStream_t)stream);
}

extern "C" int seedrl_vtrace_popart_loss_fwd(
    int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
    const float* behaviour_logits, const int64_t* actions, const float* rewards,
    const uint8_t* done, const seedrl_loss_config* cfg, const float* entropy_cost_param,
    const float* popart_moments, const float* popart_compensation,
    float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
    float* vs_out, float* pg_advantages_out, float* td_out, float* moment_sums,
    void* scratch, seedrl_stream_t stream) {
  return seedrl_vtrace_popart_loss_fwd_abandoned(
      T1, B, A, learner_logits, learner_baseline, behaviour_logits, actions, rewards, done, nullptr, cfg,
      entropy_cost_param, popart_moments, popart_compensation, loss_terms, dlogits, dbaseline, d_entropy_cost_param,
      vs_out, pg_advantages_out, td_out, moment_sums, scratch, stream);
}

// at most kNumSMs CTAs: their partials fit the kNumSMs x kLossPartials doubles that
// seedrl_vtrace_loss_scratch_bytes always provides
static int launch_popart_update(const PopArtUpdateParams& p, cudaStream_t st) {
  const size_t n = (size_t)p.T * p.B;
  const int grid = (int)std::min<size_t>(ceil_div_sz(n, (size_t)kPopThreads * 4), (size_t)kNumSMs);
  vtrace_popart_update_kernel<<<grid, kPopThreads, 0, st>>>(p);
  count_launch(PC_LOSS, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_vtrace_popart_update(
    int T1, int B, int world, float beta, float baseline_cost, const float* learner_baseline,
    const float* td, const float* moment_sums, float* popart_moments, float* popart_compensation,
    float* dbaseline, float* d_popart_compensation, float* loss_terms, void* scratch,
    seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T1 >= 2 && B >= 1 && world >= 1, "need T1>=2, B>=1, world>=1");
  SEEDRL_CHECK_ARG(beta >= 0.f && beta <= 1.f, "beta must be in [0, 1]");
  SEEDRL_CHECK_ARG(learner_baseline && td && moment_sums && popart_moments && popart_compensation &&
                       dbaseline && d_popart_compensation && loss_terms && scratch,
                   "null pointer");
  PopArtUpdateParams p = {};
  p.T = T1 - 1; p.B = B;
  p.baseline_cost = baseline_cost; p.beta = beta;
  p.count = (double)world * (double)p.T * (double)B;
  p.lb = learner_baseline; p.td = td; p.sums = moment_sums;
  p.mom = popart_moments; p.comp = popart_compensation;
  p.dbaseline = dbaseline; p.dcomp = d_popart_compensation; p.loss_terms = loss_terms;
  p.ticket = reinterpret_cast<unsigned int*>(scratch);
  p.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
  return launch_popart_update(p, (cudaStream_t)stream);
}

// ---- multi-task PopArt ----------------------------------------------------------------------------------
// Scratch: the loss scratch, then col_sums [B,2] doubles, then kNumSMs x kTaskPartials doubles for the
// moments and update kernels (at most kNumSMs CTAs each).
extern "C" size_t seedrl_vtrace_popart_tasks_scratch_bytes(int T1, int B, int A, int num_tasks) {
  (void)num_tasks;
  return seedrl_vtrace_loss_scratch_bytes(T1, B, A) + (size_t)B * 2 * sizeof(double) +
         (size_t)kNumSMs * kTaskPartials * sizeof(double);
}
static double* task_col_sums(void* scratch, int B) {   // the loss scratch depends on B alone
  return reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + seedrl_vtrace_loss_scratch_bytes(2, B, 1));
}

extern "C" int seedrl_vtrace_popart_tasks_loss_fwd(
    int T1, int B, int A, const float* learner_logits, const float* learner_baseline,
    const float* behaviour_logits, const int64_t* actions, const float* rewards,
    const uint8_t* done, const uint8_t* abandoned, const int32_t* task_ids, int num_tasks,
    const seedrl_loss_config* cfg, const float* entropy_cost_param,
    const float* popart_moments, const float* popart_compensation,
    float* loss_terms, float* dlogits, float* dbaseline, float* d_entropy_cost_param,
    float* vs_out, float* pg_advantages_out, float* td_out, double* moment_sums, int32_t* task_error,
    void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T1 >= 2 && B >= 1 && A >= 1, "need T1>=2, B>=1, A>=1");
  SEEDRL_CHECK_ARG(num_tasks >= 1 && num_tasks <= kMaxTasks, "num_tasks must be in [1, 64]");
  SEEDRL_CHECK_ARG(learner_logits && learner_baseline && behaviour_logits && actions &&
                       rewards && done && task_ids && cfg && entropy_cost_param && popart_moments &&
                       popart_compensation && loss_terms && dlogits && dbaseline &&
                       d_entropy_cost_param && td_out && moment_sums && task_error && scratch,
                   "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  LossParams p = loss_params(T1, B, A, learner_logits, learner_baseline, behaviour_logits, actions, rewards, done,
                             cfg, entropy_cost_param, loss_terms, dlogits, dbaseline, d_entropy_cost_param,
                             vs_out, pg_advantages_out, scratch);
  p.pop_mom = popart_moments; p.pop_comp = popart_compensation;
  p.pop_td = td_out;
  p.abandoned = abandoned;
  p.task_ids = task_ids; p.task_error = task_error;
  if (num_tasks == 1) {   // the single-task kernels: bit for bit seedrl_vtrace_popart_loss_fwd(_abandoned)
    p.pop_sums_d = moment_sums;
    return launch_loss<kPopArt>(p, st);
  }
  p.num_tasks = num_tasks;
  p.col_sums = task_col_sums(scratch, B);
  SEEDRL_TRY(launch_loss<kPopArtTasks>(p, st));
  TaskMomentParams q;
  q.T = p.T; q.B = B; q.K = num_tasks;
  q.task_ids = task_ids; q.col_sums = p.col_sums; q.sums = moment_sums;
  q.partials = p.col_sums + 2 * (size_t)B;
  q.ticket = p.ticket;
  vtrace_popart_task_moments_kernel<<<std::min(kNumSMs, ceil_div(B, kTaskThreads)), kTaskThreads, 0, st>>>(q);
  count_launch(PC_LOSS, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_vtrace_popart_tasks_update(
    int T1, int B, int num_tasks, float beta, float baseline_cost, const float* learner_baseline,
    const float* td, const int32_t* task_ids, const double* moment_sums, float* popart_moments,
    float* popart_compensation, float* dbaseline, float* d_popart_compensation, float* loss_terms,
    void* scratch, seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(T1 >= 2 && B >= 1, "need T1>=2, B>=1");
  SEEDRL_CHECK_ARG(num_tasks >= 1 && num_tasks <= kMaxTasks, "num_tasks must be in [1, 64]");
  SEEDRL_CHECK_ARG(beta >= 0.f && beta <= 1.f, "beta must be in [0, 1]");
  SEEDRL_CHECK_ARG(learner_baseline && td && task_ids && moment_sums && popart_moments && popart_compensation &&
                       dbaseline && d_popart_compensation && loss_terms && scratch,
                   "null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned int* ticket = reinterpret_cast<unsigned int*>(scratch);
  if (num_tasks == 1) {   // vtrace_popart_update_kernel, counting the rows from moment_sums
    PopArtUpdateParams p = {};
    p.T = T1 - 1; p.B = B;
    p.baseline_cost = baseline_cost; p.beta = beta;
    p.lb = learner_baseline; p.td = td; p.sums_d = moment_sums;
    p.mom = popart_moments; p.comp = popart_compensation;
    p.dbaseline = dbaseline; p.dcomp = d_popart_compensation; p.loss_terms = loss_terms;
    p.ticket = ticket;
    p.partials = reinterpret_cast<double*>(reinterpret_cast<char*>(scratch) + 256);
    return launch_popart_update(p, st);
  }
  PopArtTasksUpdateParams p;
  p.T = T1 - 1; p.B = B; p.K = num_tasks;
  p.baseline_cost = baseline_cost; p.beta = beta;
  p.lb = learner_baseline; p.td = td; p.task_ids = task_ids; p.sums = moment_sums;
  p.mom = popart_moments; p.comp = popart_compensation;
  p.dbaseline = dbaseline; p.dcomp = d_popart_compensation; p.loss_terms = loss_terms;
  p.partials = task_col_sums(scratch, B) + 2 * (size_t)B;
  p.ticket = ticket;
  vtrace_popart_tasks_update_kernel<<<std::min(kNumSMs, ceil_div(B, kPopThreads)), kPopThreads, 0, st>>>(p);
  count_launch(PC_LOSS, st);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}
