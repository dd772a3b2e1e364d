// Pieces shared by the network schedules (net.cu: ImpalaDeep / shallow IMPALA net, r2d2_net.cu:
// DuelingLSTMDQNNet): the parameter table, the workspace planner, the GEMM execution of one call, the
// recurrent core (lstm.cu) and the 'valid' strided convolution layer (strided_conv.cu).
#pragma once
#include <string.h>

#include <string>
#include <vector>

#include "kernels.h"

namespace seedrl {

// Parameters: one flat fp32 arena, tensors in the reference's tf.Module.trainable_variables order,
// Keras layouts, every tensor start aligned to 64 floats (256 B).
struct ParamInfo {
  std::string name;
  int rank;
  int64_t dims[4];
  size_t offset;   // floats
  size_t size;     // floats
};

struct ParamTable {
  std::vector<ParamInfo> list;
  size_t arena_floats = 0;

  int add(const std::string& name, std::initializer_list<int64_t> dims) {
    ParamInfo p;
    p.name = name;
    p.rank = (int)dims.size();
    size_t sz = 1;
    int i = 0;
    for (int64_t d : dims) { p.dims[i++] = d; sz *= (size_t)d; }
    for (; i < 4; ++i) p.dims[i] = 1;
    p.size = sz;
    p.offset = arena_floats;
    arena_floats += (sz + 63) / 64 * 64;
    list.push_back(p);
    return (int)list.size() - 1;
  }
  size_t offset(int idx) const { return list[idx].offset; }
  // The *_param_info copy-out (any output may be null); null if `index` is out of range.
  const ParamInfo* info(int index, char* name_buf, size_t name_buf_len, int64_t* dims, size_t* offset) const {
    if (index < 0 || index >= (int)list.size()) return nullptr;
    const ParamInfo& p = list[index];
    if (name_buf && name_buf_len) {
      strncpy(name_buf, p.name.c_str(), name_buf_len - 1);
      name_buf[name_buf_len - 1] = 0;
    }
    if (dims) for (int i = 0; i < 4; ++i) dims[i] = p.dims[i];
    if (offset) *offset = p.offset;
    return &p;
  }
};

// Workspace plan: buffers carved in order, each start aligned to 256 B.
struct Bump {
  size_t off = 0;
  size_t take(size_t bytes) {
    const size_t o = off;
    off += (bytes + 255) / 256 * 256;
    return o;
  }
};

template <typename T>
static inline T* W(void* ws, size_t off) {
  return reinterpret_cast<T*>(reinterpret_cast<char*>(ws) + off);
}

// The GEMMs of one forward / backward call.  mode 0: fp32 SIMT sgemm; 1: wgmma bf16; 2: wgmma bf16x3
// (fp32-faithful).  In modes 1 and 2 a shape gemm_tc does not take runs on sgemm.
struct GemmExec {
  int mode;
  bool gather;           // strided convolutions may gather their im2col operand inside gemm_tc
  float* ws;             // split-K partials / colsum row slabs
  size_t ws_bytes;
  int* err;              // bounded-wait error flag of the wgmma kernels
  cudaStream_t st;

  int gemm(bool ta, bool tb, int M, int N, int K, const float* A, int lda, const float* B, int ldb, float* C,
           int ldc, const GemmEpi& e) const {
    if (mode >= 1 && gemm_tc_supported(M, N, K))
      return gemm_tc(ta, tb, mode >= 2, M, N, K, A, lda, B, ldb, C, ldc, e, ws, ws_bytes, err, st);
    return sgemm(ta, tb, M, N, K, A, lda, B, ldb, C, ldc, e, st);
  }
  // op(A) = the im2col matrix described by cg (kernels.h ConvGather)
  int gemm_gather(bool ta, int M, int N, int K, const ConvGather& cg, const float* B, int ldb, float* C, int ldc,
                  const GemmEpi& e) const {
    return gemm_tc(ta, false, mode >= 2, M, N, K, nullptr, 0, B, ldb, C, ldc, e, ws, ws_bytes, err, st, &cg);
  }
  int colsum(int M, int N, const float* X, int ld, float* out) const {
    return seedrl::colsum(M, N, X, ld, out, st, ws, ws_bytes);
  }
};

// The LSTM recurrence of one call (lstm.cu), Keras LSTMCell(H) with done-resets over T1 steps, in lstm_mode
// `mode`: 2 tiled (lstm_tiled.cu), 3 tiled on wgmma bf16x3 (lstm_tc.cu); any other mode is refused.
//   forward   z [T1,B,4H]: x W + b in, activated gates out; hs, cs, hp [T1,B,H] (hp[t] = h[t-1] with step t's
//             resets applied)
//   backward  dz [T1,B,4H] from the forward's gates and cs and dhs [T1,B,H]
// counter: 64 barrier counters (256 B), reset by each launch; err: the bounded-wait error flag.
int lstm_recurrence_forward(int mode, int H, int T1, int B, const float* U, const uint8_t* done, float* z,
                            const float* h0, const float* c0, float* hs, float* cs, float* hp, unsigned int* counter,
                            int* err, cudaStream_t st);
int lstm_recurrence_backward(int mode, int H, int T1, int B, const float* U, const uint8_t* done, const float* gates,
                             const float* cs, const float* c0, const float* dhs, float* dz, unsigned int* counter,
                             int* err, cudaStream_t st);

// The recurrent core both nets share (lstm.cu): Dense(flat -> H) + ReLU, concat(that, reward,
// one_hot(prev_action, A)) = the core input [N, core_in], then Keras LSTMCell(H) with done-resets.
struct Core {
  int H, flat, A, core_in;              // core_in = H + 1 + A
  int dense_w, dense_b, w, u, b;        // parameter indices: Dense kernel / bias, core kernel / recurrent / bias
  bool clip_reward;                     // reward clipped to [-1, 1] (ImpalaDeep, dmlab/networks.py:111)
  bool flat_relu;                       // ReLU applied to the flat features as Dense reads them (ImpalaDeep)
  int lstm_mode = 2;
};
// Registers Dense (`dense` + "/kernel", "/bias"), then core/{kernel,recurrent_kernel,bias}.
Core core_create(ParamTable& t, const std::string& dense, int H, int flat, int A, bool clip_reward, bool flat_relu);

// The core's buffers in a workspace of T1 x B frames (N = T1 * B rows): core input, gates, h[t-1], c, h, the
// copy of c0, d h, d gates, d dense_out, the LSTM barrier counters.
struct CorePlan {
  int T1, B, N;
  size_t xc, z, hp, cs, hs, c0buf, dhs, dz, dd, counter;
};
CorePlan core_plan(const Core& k, Bump& b, int T1, int B);

// Forward up to hs (ws + p.hs, [T1, B, H]) from the flat features [N, flat].
int core_forward(const Core& k, const ParamTable& t, const CorePlan& p, const GemmExec& ex, void* ws, const float* prm,
                 const float* flat, const float* reward, const int64_t* prev_actions, const uint8_t* done,
                 const float* h0, const float* c0);
// The final h and c of the last core_forward (either may be null).
int core_final_state(const Core& k, const CorePlan& p, cudaStream_t st, void* ws, float* h_out, float* c_out);
// Backward from d hs (ws + p.dhs) to the core and Dense gradients and dflat [N, flat] (masked by flat > 0);
// head_ready (may be null) is recorded once every gradient but dflat is final.
int core_backward(const Core& k, const ParamTable& t, const CorePlan& p, const GemmExec& ex, void* ws,
                  const float* prm, float* grd, const uint8_t* done, const float* flat, float* dflat,
                  cudaEvent_t head_ready);

// Reads back the device-side error flag of the last forward/backward that used a workspace (set when
// a bounded mbarrier / grid-barrier wait of a wgmma or persistent kernel expired, i.e. the results are
// garbage).  Synchronises `st`.  `unit` names what the results belong to ("step", "unroll").
inline int read_error_flag(const int* flag_dev, cudaStream_t st, const char* unit) {
  int flag = 0;
  SEEDRL_CUDA(cudaMemcpyAsync(&flag, flag_dev, sizeof(int), cudaMemcpyDeviceToHost, st));
  SEEDRL_CUDA(cudaStreamSynchronize(st));
  if (flag != 0)
    return set_error(SEEDRL_ERR_INTERNAL, std::string("a tensor-core / persistent kernel timed out on a barrier: "
                                                      "results of this ") + unit + " are invalid");
  return SEEDRL_OK;
}

// One k x k / stride s 'valid' convolution on NHWC tensors (R2D2 body, shallow IMPALA net) as im2col + GEMM:
//   forward   col = im2col(x);  y = relu(col W + b)           (W is Keras HWIO = [k*k*cin, cout])
//   weights   dW = col^T dy (deterministic split-K), db = column sums of dy
//   data      dcol = dy W^T (written over col), dx = col2im(dcol) * (x > 0)   (gather form, no atomics)
// uint8 inputs are scaled by 1/255.  Where GemmExec allows it and the geometry gives aligned 8-element
// groups, gemm_tc gathers col straight from x while it stages its operand blocks; otherwise forward
// materialises col and wgrad reads the matrix the forward left there.
struct StridedConv {
  int k, s, cin, cout, hin, win, hout, wout;
  StridedConv() = default;
  StridedConv(int k_, int s_, int cin_, int cout_, int hin_, int win_)
      : k(k_), s(s_), cin(cin_), cout(cout_), hin(hin_), win(win_), hout((hin_ - k_) / s_ + 1),
        wout((win_ - k_) / s_ + 1) {}

  bool gathered(const GemmExec& ex, int N, bool u8, const void* x, ConvGather* cg) const;
  int im2col(int N, bool u8, const void* x, float* col, cudaStream_t st) const;
  // y[N*hout*wout, ldy] = relu(conv(x) + b)
  int forward(const GemmExec& ex, int N, bool u8, const void* x, const float* w, const float* b, float* col, float* y,
              int ldy) const;
  // dw[k*k*cin, lddw], db[cout] from dy[N*hout*wout, cout]
  int wgrad(const GemmExec& ex, int N, bool u8, const void* x, const float* col, const float* dy, float* dw, int lddw,
            float* db) const;
  // dx[N, hin, win, cin] masked by xmask > 0 (cin % 4 == 0, 16-byte aligned col / xmask / dx)
  int dgrad(const GemmExec& ex, int N, const float* dy, const float* w, float* col, const float* xmask,
            float* dx) const;
};

}  // namespace seedrl
