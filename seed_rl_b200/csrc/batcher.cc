// (a10) Host-side inference batcher.  Replaces the semantics of the reference's
// server-side dynamic batcher, grpc/ops/grpc.cc:591-861 (`DynamicFn::operator()`,
// `Computation`): many callers each contribute k rows of a fixed-size batch; when the
// batch is full one computation runs; outputs fan back out to the callers.
//
// H100-first differences (same observable behaviour, pinned by
// grpc/python/ops_test.py's batching tests):
//   * callers write their payload DIRECTLY into a pinned host slab at their claimed
//     row offset (no TensorProto -> tensor -> batch-tensor double copy,
//     grpc.cc:177-183,666-676); the slab is what the learner H2D-copies with one
//     cudaMemcpyAsync per field;
//   * slot claim is one short critical section; payload copies run outside the lock;
//   * `num_slabs` (>= 2) batches are in flight, like empty_computations_
//     (grpc.cc:656-661), so callers fill batch k+1 while batch k is on the GPU.
#include <cuda_runtime.h>
#include <stdlib.h>
#include <string.h>

#include <chrono>
#include <condition_variable>
#include <deque>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/seedrl_b200.h"

namespace seedrl {
extern thread_local std::string g_last_error;
}

namespace {

enum SlabState { FREE = 0, FILLING, FULL, COMPUTING, PUBLISHED };

struct Slab {
  std::vector<uint8_t*> in, out;
  SlabState state = FREE;
  int claimed = 0, committed = 0, refs = 0;
  int status = 0;
};

int fail(int code, const char* msg) {
  seedrl::g_last_error = msg;
  return code;
}

}  // namespace

struct seedrl_batcher {
  int batch_size, pinned;
  std::vector<size_t> in_row, out_row;
  std::vector<Slab> slabs;
  int cur = 0;                 // slab currently being filled
  std::deque<int> full_q;
  bool shutdown = false;
  std::mutex mu;
  std::condition_variable cv_free, cv_full, cv_pub;
};

static uint8_t* alloc_buf(size_t bytes, int pinned) {
  if (bytes == 0) bytes = 16;
  void* p = nullptr;
  if (pinned) {
    if (cudaHostAlloc(&p, bytes, cudaHostAllocPortable) != cudaSuccess) return nullptr;
  } else {
    if (posix_memalign(&p, 256, (bytes + 255) / 256 * 256) != 0) return nullptr;
  }
  memset(p, 0, bytes);
  return reinterpret_cast<uint8_t*>(p);
}
static void free_buf(uint8_t* p, int pinned) {
  if (!p) return;
  if (pinned) cudaFreeHost(p); else free(p);
}

extern "C" int seedrl_batcher_create(int batch_size, int num_slabs, int n_in,
                                     const size_t* in_row_bytes, int n_out,
                                     const size_t* out_row_bytes, int pinned,
                                     seedrl_batcher** out) {
  if (!out || batch_size <= 0 || num_slabs < 2 || n_in < 0 || n_out < 0)
    return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_create: bad argument (num_slabs >= 2)");
  seedrl_batcher* b = new seedrl_batcher();
  b->batch_size = batch_size;
  b->pinned = pinned;
  b->in_row.assign(in_row_bytes, in_row_bytes + n_in);
  b->out_row.assign(out_row_bytes, out_row_bytes + n_out);
  b->slabs.resize(num_slabs);
  for (Slab& s : b->slabs) {
    for (size_t rb : b->in_row) s.in.push_back(alloc_buf(rb * batch_size, pinned));
    for (size_t rb : b->out_row) s.out.push_back(alloc_buf(rb * batch_size, pinned));
    for (uint8_t* p : s.in) if (!p) { seedrl_batcher_destroy(b); return fail(SEEDRL_ERR_INTERNAL, "seedrl_batcher_create: slab allocation failed"); }
    for (uint8_t* p : s.out) if (!p) { seedrl_batcher_destroy(b); return fail(SEEDRL_ERR_INTERNAL, "seedrl_batcher_create: slab allocation failed"); }
  }
  b->slabs[0].state = FILLING;
  *out = b;
  return SEEDRL_OK;
}

extern "C" void seedrl_batcher_destroy(seedrl_batcher* b) {
  if (!b) return;
  for (Slab& s : b->slabs) {
    for (uint8_t* p : s.in) free_buf(p, b->pinned);
    for (uint8_t* p : s.out) free_buf(p, b->pinned);
  }
  delete b;
}

extern "C" int seedrl_batcher_claim(seedrl_batcher* b, int k, int* slab, int* row) {
  if (!b || !slab || !row || k <= 0) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_claim: bad argument");
  if (k > b->batch_size)
    return fail(SEEDRL_ERR_OUT_OF_RANGE, "seedrl_batcher_claim: more rows than the batch size");
  std::unique_lock<std::mutex> lk(b->mu);
  for (;;) {
    if (b->shutdown) return fail(SEEDRL_ERR_CANCELLED, "Server shutdown.");
    Slab& s = b->slabs[b->cur];
    // A slab whose rows are all claimed but not yet all committed (a caller was descheduled
    // between claim and commit) is still FILLING: when the other callers lap the ring and come
    // back to it, it is busy -- wait for it like for any slab in flight.
    if (s.state == FILLING && s.claimed < b->batch_size) {
      if (s.claimed + k > b->batch_size)   // grpc.cc:653 (CHECK-fails there)
        return fail(SEEDRL_ERR_OUT_OF_RANGE,
                    "seedrl_batcher_claim: call would straddle two batches (batch size must be a "
                    "multiple of the caller's row count)");
      *slab = b->cur;
      *row = s.claimed;
      s.claimed += k;
      s.refs += 1;
      if (s.claimed == b->batch_size) {    // swap to the next empty computation, grpc.cc:656-661
        const int nxt = (b->cur + 1) % (int)b->slabs.size();
        b->cur = nxt;
        if (b->slabs[nxt].state == FREE) b->slabs[nxt].state = FILLING;
      }
      return SEEDRL_OK;
    }
    if (s.state == FREE) { s.state = FILLING; continue; }
    b->cv_free.wait(lk);   // all slabs in flight: back-pressure
  }
}

extern "C" void* seedrl_batcher_input_ptr(seedrl_batcher* b, int slab, int field, int row) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size() || field < 0 || field >= (int)b->in_row.size()) return nullptr;
  return b->slabs[slab].in[field] + b->in_row[field] * (size_t)row;
}
extern "C" void* seedrl_batcher_output_ptr(seedrl_batcher* b, int slab, int field, int row) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size() || field < 0 || field >= (int)b->out_row.size()) return nullptr;
  return b->slabs[slab].out[field] + b->out_row[field] * (size_t)row;
}

extern "C" int seedrl_batcher_commit(seedrl_batcher* b, int slab, int k) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size() || k <= 0) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_commit: bad argument");
  std::lock_guard<std::mutex> lk(b->mu);
  Slab& s = b->slabs[slab];
  s.committed += k;                        // num_ready += n, grpc.cc:681
  if (s.committed == b->batch_size) {
    s.state = FULL;
    b->full_q.push_back(slab);
    b->cv_full.notify_one();
  }
  return SEEDRL_OK;
}

extern "C" int seedrl_batcher_wait_outputs(seedrl_batcher* b, int slab, int* status) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size()) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_wait_outputs: bad argument");
  std::unique_lock<std::mutex> lk(b->mu);
  Slab& s = b->slabs[slab];
  while (s.state != PUBLISHED && !b->shutdown) b->cv_pub.wait(lk);
  if (s.state != PUBLISHED) return fail(SEEDRL_ERR_CANCELLED, "Server shutdown.");   // grpc.cc:771-787
  if (status) *status = s.status;
  return SEEDRL_OK;
}

extern "C" int seedrl_batcher_release(seedrl_batcher* b, int slab) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size()) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_release: bad argument");
  std::lock_guard<std::mutex> lk(b->mu);
  Slab& s = b->slabs[slab];
  if (--s.refs == 0 && (s.state == PUBLISHED || b->shutdown)) {
    s.state = FREE; s.claimed = s.committed = 0; s.status = 0;
    b->cv_free.notify_all();
  }
  return SEEDRL_OK;
}

extern "C" int seedrl_batcher_next_full(seedrl_batcher* b, int timeout_ms, int* slab) {
  if (!b || !slab) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_next_full: bad argument");
  std::unique_lock<std::mutex> lk(b->mu);
  auto ready = [&] { return !b->full_q.empty() || b->shutdown; };
  if (timeout_ms < 0) b->cv_full.wait(lk, ready);
  else if (!b->cv_full.wait_for(lk, std::chrono::milliseconds(timeout_ms), ready))
    return fail(SEEDRL_ERR_UNAVAILABLE, "seedrl_batcher_next_full: timeout");
  if (b->full_q.empty()) return fail(SEEDRL_ERR_CANCELLED, "Server shutdown.");
  *slab = b->full_q.front();
  b->full_q.pop_front();
  b->slabs[*slab].state = COMPUTING;
  return SEEDRL_OK;
}

extern "C" int seedrl_batcher_publish(seedrl_batcher* b, int slab, int status) {
  if (!b || slab < 0 || slab >= (int)b->slabs.size()) return fail(SEEDRL_ERR_INVALID_ARGUMENT, "seedrl_batcher_publish: bad argument");
  std::lock_guard<std::mutex> lk(b->mu);
  Slab& s = b->slabs[slab];
  s.status = status;
  s.state = PUBLISHED;
  b->cv_pub.notify_all();
  return SEEDRL_OK;
}

extern "C" int seedrl_batcher_shutdown(seedrl_batcher* b) {
  if (!b) return SEEDRL_OK;
  std::lock_guard<std::mutex> lk(b->mu);
  b->shutdown = true;
  b->cv_free.notify_all();
  b->cv_full.notify_all();
  b->cv_pub.notify_all();
  return SEEDRL_OK;
}
