"""Timing of the learner's dense GEMM shapes (N = 1344 rows) on the wgmma GEMM:
back-to-back launches between CUDA events.   python tools/gemm_bench.py [split]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from seed_rl_b200 import _lib

L = _lib.lib()
split = int(sys.argv[1]) if len(sys.argv) > 1 else 0
R = 1344
SHAPES = [  # name, ta, tb, M, N, K, lda, ldb
    ('dense fwd', 0, 0, R, 256, 3872, 3872, 256), ('lstm proj', 0, 0, R, 1024, 275, 275, 1024),
    ('policy head', 0, 0, R, 18, 256, 256, 18), ('dW policy', 1, 0, 256, 18, R, 256, 18),
    ('dU (hp^T dz)', 1, 0, 256, 1024, R, 256, 1024), ('dWx (xc^T dz)', 1, 0, 275, 1024, R, 275, 1024),
    ('d dense_out', 0, 1, R, 256, 1024, 1024, 1024), ('dW dense', 1, 0, 3872, 256, R, 3872, 256),
    ('d flat', 0, 1, R, 3872, 256, 256, 256)]
ws = torch.empty(48 << 18, device='cuda'); err = torch.zeros(1, dtype=torch.int32, device='cuda')
tot = 0.0
for name, ta, tb, M, N, K, lda, ldb in SHAPES:
  A = torch.randn((K if ta else M), lda, device='cuda'); B = torch.randn((N if tb else K), ldb, device='cuda')
  C = torch.empty(M, N, device='cuda')
  fn = lambda: _lib.check(L.seedrl_debug_gemm_tc(ta, tb, split, M, N, K, _lib.ptr(A), lda, _lib.ptr(B), ldb, _lib.ptr(C), N,
                                                 None, None, 0, 0, 0, 0, _lib.ptr(ws), ws.numel() * 4, _lib.ptr(err),
                                                 _lib.stream_ptr()))
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(20):
    fn()
  e1.record(); torch.cuda.synchronize()
  us = e0.elapsed_time(e1) / 20 * 1e3
  tot += us
  mb = (M * K + K * N + M * N) * 4 / 1e6
  print('%-15s ta=%d tb=%d M=%4d N=%4d K=%4d  %7.1f us  %6.1f MB  %6.0f GB/s  %5.1f TFLOP/s' %
        (name, ta, tb, M, N, K, us, mb, mb / us * 1e3 / 1e3, 2.0 * M * N * K / us / 1e6), flush=True)
print('total %.1f us' % tot)
assert int(err.item()) == 0
