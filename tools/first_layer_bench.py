"""Times the fused first layer of ImpalaDeep (csrc/conv_first.cu) per channel count: the forward
(conv 3x3 C->16 on uint8 frames + bias + max-pool 3x3/2 SAME -> pooled plane tensors + arg-max
taps) and the weight gradient from the pooled gradient, at the learner's batch (T = 20, B = 64:
21 x 64 = 1 344 frames of 84x84).

Prints one line per (C, kernel): ms per call (CUDA events over --iters calls after --warmup),
algorithmic bytes (frames read once; pooled raw + ReLU planes and taps written / pooled gradient
planes and taps read) and their rate as a fraction of the H100 SXM data-sheet HBM bandwidth.

    python tools/first_layer_bench.py [--channels 1 4 8 12 16] [--iters 50]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from seed_rl_b200 import _lib  # noqa: E402

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


def _time(fn, warmup, iters):
  for _ in range(warmup):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(iters):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / iters


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--channels', type=int, nargs='+', default=[1, 4, 8, 12, 16])
  ap.add_argument('--T', type=int, default=20)
  ap.add_argument('--B', type=int, default=64)
  ap.add_argument('--H', type=int, default=84)
  ap.add_argument('--W', type=int, default=84)
  ap.add_argument('--warmup', type=int, default=10)
  ap.add_argument('--iters', type=int, default=50)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit('first_layer_bench needs a CUDA device')
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True)
  print('# device:', q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name())
  L = _lib.lib()
  st = _lib.stream_ptr()
  N, H, W = (args.T + 1) * args.B, args.H, args.W
  Ho, Wo = (H + 1) // 2, (W + 1) // 2
  pb = int(L.seedrl_debug_planes_bytes(N, Ho, Wo, 16))
  rng = np.random.default_rng(0)
  raw = torch.zeros(pb, dtype=torch.uint8, device='cuda'); relu = torch.zeros_like(raw)
  gp = torch.zeros_like(raw)
  idx = torch.zeros((N, Ho, Wo, 16), dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  bias = torch.zeros(16, device='cuda')
  db = torch.zeros(16, device='cuda')
  taps = N * Ho * Wo * 16
  for C in args.channels:
    frames = torch.as_tensor(rng.integers(0, 256, (N, H, W, C), dtype=np.uint8)).cuda()
    w = torch.as_tensor((rng.normal(size=(3, 3, C, 16)) * 0.1).astype(np.float32)).cuda()
    dw = torch.zeros_like(w)
    part = torch.empty(3 * 132 * (9 * C * 16 + 16), dtype=torch.float32, device='cuda')
    fwd = lambda: _lib.check(L.seedrl_debug_conv0pool_c(N, H, W, C, _lib.ptr(frames), _lib.ptr(w), _lib.ptr(bias),
                                                        _lib.ptr(raw), _lib.ptr(relu), _lib.ptr(idx), _lib.ptr(err), st))
    fwd()                                          # real arg-max taps for the weight gradient
    bwd = lambda: _lib.check(L.seedrl_debug_first_wgrad_pooled_c(N, H, W, C, _lib.ptr(frames), _lib.ptr(gp), _lib.ptr(idx),
                                                                 _lib.ptr(dw), _lib.ptr(db), _lib.ptr(part),
                                                                 part.numel() * 4, st))
    fb = frames.numel()
    for name, fn, nbytes in (('forward', fwd, fb + 2 * pb + taps), ('wgrad', bwd, fb + pb + taps)):
      ms = _time(fn, args.warmup, args.iters)
      rate = nbytes / (ms * 1e-3)
      print(json.dumps({'C': C, 'kernel': name, 'frames': N, 'ms': round(ms, 4), 'bytes': int(nbytes),
                        'GB_per_s': round(rate / 1e9, 1), 'frac_of_3.35TBps': round(rate / HBM_BYTES_PER_S, 3)}))
    assert int(err.item()) == 0


if __name__ == '__main__':
  main()
