// (a7/a8) GPU-resident per-environment state: UnrollStore (common/utils.py:119-257) and
// the row scatter/gather behind Aggregator (common/utils.py:461-543).  Pure byte movement
// (HBM-bound): rows are copied with 16-byte vector accesses when row_bytes and the base
// pointers allow it, one CTA-row pair per (env, step) row otherwise byte-wise.
#include "common.cuh"

namespace seedrl {

__device__ __forceinline__ void copy_row(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                                         size_t bytes) {
  if (((uintptr_t)dst | (uintptr_t)src | bytes) % 16 == 0) {
    const int4* s = reinterpret_cast<const int4*>(src);
    int4* d = reinterpret_cast<int4*>(dst);
    for (size_t i = threadIdx.x; i < bytes / 16; i += blockDim.x) d[i] = s[i];
  } else if (((uintptr_t)dst | (uintptr_t)src | bytes) % 4 == 0) {
    const int* s = reinterpret_cast<const int*>(src);
    int* d = reinterpret_cast<int*>(dst);
    for (size_t i = threadIdx.x; i < bytes / 4; i += blockDim.x) d[i] = s[i];
  } else {
    for (size_t i = threadIdx.x; i < bytes; i += blockDim.x) dst[i] = src[i];
  }
}

// state[env_ids[j], index[env_ids[j]], :] = values[j, :]      utils.py:187-190
__global__ void store_append_kernel(uint8_t* state, const int32_t* __restrict__ index,
                                    const int32_t* __restrict__ env_ids, int full_length,
                                    size_t row_bytes, const uint8_t* __restrict__ values) {
  const int j = blockIdx.x;
  const int env = env_ids[j];
  const int t = index[env];
  if (t < 0 || t >= full_length) return;   // (the reference leaves OOB undefined)
  copy_row(state + ((size_t)env * full_length + t) * row_bytes, values + (size_t)j * row_bytes,
           row_bytes);
}

// index[env]++ ; completed ids compacted in env_ids order (utils.py:194,229-233).  Rows whose env id
// is >= id_limit (eval environments, which have no store rows) are skipped.
// Single CTA: n is an inference batch (<= a few thousand).
__global__ void store_advance_kernel(int32_t* index, const int32_t* __restrict__ env_ids, int n,
                                     int full_length, int32_t* __restrict__ completed_ids,
                                     int32_t* __restrict__ num_completed, int id_limit) {
  __shared__ int s_base;
  __shared__ int s_warp[32];
  if (threadIdx.x == 0) s_base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  for (int j0 = 0; j0 < n; j0 += blockDim.x) {
    const int j = j0 + threadIdx.x;
    int flag = 0, env = 0;
    if (j < n && (env = env_ids[j]) < id_limit) {
      const int v = index[env] + 1;
      index[env] = v;
      flag = (v == full_length);
    }
    const unsigned bal = __ballot_sync(0xffffffffu, flag);
    const int within = __popc(bal & ((1u << lane) - 1));
    if (lane == 0) s_warp[w] = __popc(bal);
    __syncthreads();
    int off = s_base;
    for (int k = 0; k < w; ++k) off += s_warp[k];
    if (flag) completed_ids[off + within] = env;
    __syncthreads();
    if (threadIdx.x == 0) {
      int tot = 0;
      for (int k = 0; k < nw; ++k) tot += s_warp[k];
      s_base += tot;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) *num_completed = s_base;
}

// unrolls <- state[completed] ; then state[env, :ov+1] = state[env, full-(ov+1):]   utils.py:234-252
// grid = (n_completed, full_length): block (i, t) copies row t of unroll i.
// time_major: destination is [full_length, ld, row] and unroll i lands in column col0 + i (ld =
// n_completed, col0 = 0 for a stand-alone output; ld = batch size when gathering straight into a
// column range of the learner's time-major minibatch).
__global__ void store_gather_kernel(const uint8_t* __restrict__ state,
                                    const int32_t* __restrict__ completed_ids, int ld, int col0,
                                    int full_length, size_t row_bytes, int time_major,
                                    uint8_t* __restrict__ unrolls) {
  const int i = blockIdx.x, t = blockIdx.y;
  const int env = completed_ids[i];
  const size_t dst_row = time_major ? ((size_t)t * ld + col0 + i) : ((size_t)i * full_length + t);
  copy_row(unrolls + dst_row * row_bytes, state + ((size_t)env * full_length + t) * row_bytes,
           row_bytes);
}
// state[env, r] = unroll_copy[i, full_length - j + r]: the carried rows are read from
// the gathered copy, so source and destination never alias (the reference's
// overlap >= unroll_length/2 case, tests/utils_test.py:191-271).
__global__ void store_carry_kernel(uint8_t* state, const int32_t* __restrict__ completed_ids,
                                   int ld, int col0, int full_length, size_t row_bytes, int j,
                                   int time_major, const uint8_t* __restrict__ unrolls) {
  const int i = blockIdx.x, r = blockIdx.y;   // r < j
  const int env = completed_ids[i];
  const int t = full_length - j + r;
  const size_t src_row = time_major ? ((size_t)t * ld + col0 + i) : ((size_t)i * full_length + t);
  copy_row(state + ((size_t)env * full_length + r) * row_bytes, unrolls + src_row * row_bytes,
           row_bytes);
}
__global__ void store_set_index_kernel(int32_t* index, const int32_t* __restrict__ ids, int n, int v) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) index[ids[i]] = v;
}
// state[env, :j] = 0
__global__ void store_zero_rows_kernel(uint8_t* state, const int32_t* __restrict__ ids,
                                       int full_length, size_t row_bytes) {
  const int i = blockIdx.x, r = blockIdx.y;
  uint8_t* p = state + ((size_t)ids[i] * full_length + r) * row_bytes;
  for (size_t k = threadIdx.x; k < row_bytes; k += blockDim.x) p[k] = 0;
}

// One launch for every per-environment row operation of an inference batch (a6, reference
// agents/vtrace/learner.py:381-403): block (j, f) moves row j of job f.
//   mode 0  gather   rows[j]  = table[env_ids[j]]                      (Aggregator.read, utils.py:504-516)
//   mode 1  scatter  table[env_ids[j]] = rows[j]                       (Aggregator.replace, :519-543)
//   mode 2  append   table[env_ids[j], index[env_ids[j]]] = rows[j]    (UnrollStore.append, :187-190),
//                    skipped for env ids >= id_limit
struct RowJobs { seedrl_row_job job[SEEDRL_MAX_ROW_JOBS]; };
__global__ void rows_multi_kernel(const __grid_constant__ RowJobs t, const int32_t* __restrict__ env_ids,
                                  const int32_t* __restrict__ index, int id_limit) {
  const seedrl_row_job jb = t.job[blockIdx.y];
  const int j = blockIdx.x;
  const int env = env_ids[j];
  uint8_t* table = reinterpret_cast<uint8_t*>(jb.table);
  uint8_t* rows = reinterpret_cast<uint8_t*>(jb.rows);
  if (jb.mode == 0) {
    copy_row(rows + (size_t)j * jb.row_bytes, table + (size_t)env * jb.row_bytes, jb.row_bytes);
  } else if (jb.mode == 1) {
    copy_row(table + (size_t)env * jb.row_bytes, rows + (size_t)j * jb.row_bytes, jb.row_bytes);
  } else {
    if (env >= id_limit) return;
    const int ti = index[env];
    if (ti < 0 || ti >= jb.full_length) return;
    copy_row(table + ((size_t)env * jb.full_length + ti) * jb.row_bytes, rows + (size_t)j * jb.row_bytes,
             jb.row_bytes);
  }
}

}  // namespace seedrl

using namespace seedrl;

extern "C" int seedrl_rows_multi_limit(const seedrl_row_job* jobs, int njobs, const int32_t* env_ids, int n,
                                       const int32_t* index, int32_t id_limit, seedrl_stream_t stream) {
  if (n == 0 || njobs == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(jobs && env_ids && n > 0 && njobs > 0 && njobs <= SEEDRL_MAX_ROW_JOBS, "bad argument");
  SEEDRL_CHECK_ARG(id_limit >= 0, "id_limit must be >= 0");
  RowJobs t;
  for (int i = 0; i < njobs; ++i) {
    SEEDRL_CHECK_ARG(jobs[i].table && jobs[i].rows && jobs[i].mode >= 0 && jobs[i].mode <= 2, "bad job");
    SEEDRL_CHECK_ARG(jobs[i].mode != 2 || (index && jobs[i].full_length > 0), "append job needs index");
    t.job[i] = jobs[i];
  }
  rows_multi_kernel<<<dim3(n, njobs), 128, 0, (cudaStream_t)stream>>>(t, env_ids, index, id_limit);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_rows_multi(const seedrl_row_job* jobs, int njobs, const int32_t* env_ids, int n,
                                 const int32_t* index, seedrl_stream_t stream) {
  return seedrl_rows_multi_limit(jobs, njobs, env_ids, n, index, INT32_MAX, stream);
}

extern "C" int seedrl_store_append_field(uint8_t* state, const int32_t* index, const int32_t* env_ids,
                                         int n, int full_length, size_t row_bytes,
                                         const uint8_t* values, seedrl_stream_t stream) {
  if (n == 0 || row_bytes == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(state && index && env_ids && values && n > 0 && full_length > 0, "bad argument");
  const int threads = row_bytes >= 4096 ? 256 : (row_bytes >= 512 ? 128 : 32);
  store_append_kernel<<<n, threads, 0, (cudaStream_t)stream>>>(state, index, env_ids, full_length,
                                                               row_bytes, values);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_store_advance_limit(int32_t* index, const int32_t* env_ids, int n, int full_length,
                                          int32_t* completed_ids, int32_t* num_completed, int32_t id_limit,
                                          seedrl_stream_t stream) {
  SEEDRL_CHECK_ARG(index && env_ids && completed_ids && num_completed && n >= 0, "bad argument");
  SEEDRL_CHECK_ARG(id_limit >= 0, "id_limit must be >= 0");
  store_advance_kernel<<<1, 256, 0, (cudaStream_t)stream>>>(index, env_ids, n, full_length,
                                                            completed_ids, num_completed, id_limit);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_store_advance(int32_t* index, const int32_t* env_ids, int n, int full_length,
                                    int32_t* completed_ids, int32_t* num_completed,
                                    seedrl_stream_t stream) {
  return seedrl_store_advance_limit(index, env_ids, n, full_length, completed_ids, num_completed, INT32_MAX,
                                    stream);
}

extern "C" int seedrl_store_gather_field(uint8_t* state, const int32_t* completed_ids,
                                         int n_completed, int full_length, size_t row_bytes,
                                         int overlap, int time_major, uint8_t* unrolls,
                                         seedrl_stream_t stream) {
  if (n_completed == 0 || row_bytes == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(state && completed_ids && unrolls && full_length > 0 && overlap >= 0, "bad argument");
  const int j = overlap + 1;
  SEEDRL_CHECK_ARG(full_length >= j, "num_overlapping_steps + 1 exceeds the unroll");
  const int threads = row_bytes >= 4096 ? 256 : (row_bytes >= 512 ? 128 : 32);
  store_gather_kernel<<<dim3(n_completed, full_length), threads, 0, (cudaStream_t)stream>>>(
      state, completed_ids, n_completed, 0, full_length, row_bytes, time_major, unrolls);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  store_carry_kernel<<<dim3(n_completed, j), threads, 0, (cudaStream_t)stream>>>(
      state, completed_ids, n_completed, 0, full_length, row_bytes, j, time_major, unrolls);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

// Zero-copy minibatch assembly (SURVEY 8(f) rank 2): the completed unrolls are gathered straight
// into columns [col0, col0 + n_completed) of the learner's time-major batch tensor
// [full_length, batch_cols, row_bytes] -- the reference's queue element copy, tf.stack and
// make_time_major transpose (agents/vtrace/learner.py:418-432, common/utils.py:735-761) collapse
// into this one gather.
extern "C" int seedrl_store_gather_field_into(uint8_t* state, const int32_t* completed_ids, int n_completed,
                                              int full_length, size_t row_bytes, int overlap, uint8_t* batch,
                                              int batch_cols, int col0, seedrl_stream_t stream) {
  if (n_completed == 0 || row_bytes == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(state && completed_ids && batch && full_length > 0 && overlap >= 0, "bad argument");
  SEEDRL_CHECK_ARG(col0 >= 0 && col0 + n_completed <= batch_cols, "columns out of range");
  const int j = overlap + 1;
  SEEDRL_CHECK_ARG(full_length >= j, "num_overlapping_steps + 1 exceeds the unroll");
  const int threads = row_bytes >= 4096 ? 256 : (row_bytes >= 512 ? 128 : 32);
  store_gather_kernel<<<dim3(n_completed, full_length), threads, 0, (cudaStream_t)stream>>>(
      state, completed_ids, batch_cols, col0, full_length, row_bytes, 1, batch);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  store_carry_kernel<<<dim3(n_completed, j), threads, 0, (cudaStream_t)stream>>>(
      state, completed_ids, batch_cols, col0, full_length, row_bytes, j, 1, batch);
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_store_finish(int32_t* index, const int32_t* completed_ids, int n_completed,
                                   int overlap, seedrl_stream_t stream) {
  if (n_completed == 0) return SEEDRL_OK;
  store_set_index_kernel<<<ceil_div(n_completed, 128), 128, 0, (cudaStream_t)stream>>>(
      index, completed_ids, n_completed, 1 + overlap);   // utils.py:254-255
  count_launch(PC_MISC, (cudaStream_t)stream);
  SEEDRL_CHECK_LAUNCH();
  return SEEDRL_OK;
}

extern "C" int seedrl_store_reset(uint8_t* state, int32_t* index, const int32_t* env_ids, int n,
                                  int full_length, size_t row_bytes, int overlap,
                                  seedrl_stream_t stream) {
  if (n == 0) return SEEDRL_OK;
  SEEDRL_CHECK_ARG(env_ids, "bad argument");
  if (index) {
    store_set_index_kernel<<<ceil_div(n, 128), 128, 0, (cudaStream_t)stream>>>(index, env_ids, n,
                                                                               overlap);  // :207-208
    count_launch(PC_MISC, (cudaStream_t)stream);
    SEEDRL_CHECK_LAUNCH();
  }
  if (state && overlap > 0 && row_bytes > 0) {                                            // :212-225
    store_zero_rows_kernel<<<dim3(n, overlap), 128, 0, (cudaStream_t)stream>>>(state, env_ids,
                                                                              full_length, row_bytes);
    count_launch(PC_MISC, (cudaStream_t)stream);
    SEEDRL_CHECK_LAUNCH();
  }
  return SEEDRL_OK;
}
