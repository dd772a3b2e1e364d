#!/usr/bin/env python
"""Single-kernel timings of the plane-tensor conv path (csrc/conv_planes.cu) at the learner's
layer shapes: python tools/planes_bench.py  [SEEDRL_PLANES_CHUNK=16|32|64|128 in the env].

Every convp_kernel configuration the default ImpalaDeep step (net.cu torso_forward_planes /
torso_backward_planes) launches is timed with its real epilogue: shape x {bias, ReLU mask,
residual, raw / ReLU'd / fp32 NHWC output, flipped weights}.  Per configuration: ms per launch
(CUDA events over back-to-back launches after warm-up; each launch includes the debug entry
point's small weight-packing kernel), algorithmic HBM bytes (4 B per element of every plane
tensor read or written -- hi + lo bf16 --, 2 B for the mask's hi planes only, 4 B for fp32 NHWC;
padding positions not counted), GB/s and the fraction of the H100 SXM data-sheet HBM3 bandwidth."""
import os, subprocess, sys, json
import torch
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)) + '/..')
from seed_rl_b200 import _lib
L = _lib.lib()
N = int(os.environ.get('FRAMES', 1344))
NUM_SMS = 132
PEAK_GBPS = 3350.0          # H100 SXM data sheet, HBM3 (not a measured figure)
ITERS = 20


def ev(fn, k=ITERS):
  for _ in range(3): fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(k): fn()
  e1.record(); torch.cuda.synchronize()
  return e0.elapsed_time(e1) / k


def planes(H, C, relu=0):
  x = torch.randn(N, H, H, C, device='cuda')
  nb = int(L.seedrl_debug_planes_bytes(N, H, H, C))
  p = torch.empty(nb, dtype=torch.uint8, device='cuda')
  _lib.check(L.seedrl_debug_to_planes(N, H, H, C, relu, _lib.ptr(x), _lib.ptr(p), _lib.stream_ptr()))
  return p


def rate(alg, ms):
  return dict(ms=round(ms, 4), MB=round(alg / 1e6, 1), GBps=round(alg / ms / 1e6, 1),
              frac_datasheet=round(alg / ms / 1e6 / PEAK_GBPS, 3))


# (name, cin, cout, H, epilogue flags, launches per step).  cin/cout are the launched conv's: a data
# gradient ('flip') of a forward ci -> co conv runs co -> ci.
RES_FWD = [('r00', 'bias relu'), ('r01', 'bias res raw relu'), ('r10', 'bias relu')]
CONFIGS = []
for s, (C, H) in enumerate([(16, 42), (32, 21), (32, 11)]):
  if s == 1: CONFIGS.append(('s1_conv_fwd', 16, 32, 42, 'bias nhwc', 1))
  if s == 2: CONFIGS.append(('s2_conv_fwd', 32, 32, 21, 'bias nhwc', 1))
  CONFIGS.append(('s%d_r00_r10_fwd' % s, C, C, H, 'bias relu', 2))
  CONFIGS.append(('s%d_r01_fwd' % s, C, C, H, 'bias res raw relu', 1))
  CONFIGS.append(('s%d_r11_fwd' % s, C, C, H, 'bias res nhwc' if s == 2 else 'bias res raw', 1))
  CONFIGS.append(('s%d_r11_r01_dgrad' % s, C, C, H, 'flip mask raw', 2))
  CONFIGS.append(('s%d_r10_r00_dgrad' % s, C, C, H, 'flip mask res raw', 2))
  if s == 1: CONFIGS.append(('s1_conv_dgrad', 32, 16, 42, 'flip raw', 1))
  if s == 2: CONFIGS.append(('s2_conv_dgrad', 32, 32, 21, 'flip raw', 1))
assert sum(c[-1] for c in CONFIGS) == 28

smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip().splitlines()
out = {'device': torch.cuda.get_device_name(), 'nvidia_smi': smi[torch.cuda.current_device()] if smi else None,
       'chunk': os.environ.get('SEEDRL_PLANES_CHUNK', 'default'), 'frames': N,
       'peak_GBps_datasheet': PEAK_GBPS, 'convp': {}}
err = torch.zeros(1, dtype=torch.int32, device='cuda')
step_ms = step_bytes = 0.0
for (name, ci, co, H, flags, count) in CONFIGS:
  f = set(flags.split())
  xin = planes(H, ci, 1)
  w = torch.randn(3, 3, co, ci, device='cuda') * 0.1 if 'flip' in f else torch.randn(3, 3, ci, co, device='cuda') * 0.1
  b = torch.randn(co, device='cuda') if 'bias' in f else None
  mask = planes(H, co, 1) if 'mask' in f else None
  res = planes(H, co) if 'res' in f else None
  nbo = int(L.seedrl_debug_planes_bytes(N, H, H, co))
  raw = torch.empty(nbo, dtype=torch.uint8, device='cuda') if 'raw' in f else None
  relu = torch.empty(nbo, dtype=torch.uint8, device='cuda') if 'relu' in f else None
  nhwc = torch.empty(N, H, H, co, device='cuda') if 'nhwc' in f else None
  wq = torch.empty(2 * 9 * ci * co * 2, dtype=torch.uint8, device='cuda')
  def conv():
    _lib.check(L.seedrl_debug_convp(ci, co, N, H, H, _lib.ptr(xin), _lib.ptr(w), _lib.ptr(b), _lib.ptr(mask),
                                    _lib.ptr(res), int('flip' in f), _lib.ptr(raw), _lib.ptr(relu), _lib.ptr(nhwc),
                                    _lib.ptr(wq), _lib.ptr(err), _lib.stream_ptr()))
  ms = ev(conv)
  px = N * H * H
  alg = px * 4 * (ci + co * (('res' in f) + ('raw' in f) + ('relu' in f) + ('nhwc' in f))) + px * 2 * co * ('mask' in f)
  out['convp'][name] = dict(cin=ci, cout=co, H=H, epilogue=flags, per_step=count, **rate(alg, ms))
  step_ms += count * ms; step_bytes += count * alg
  del xin, mask, res, raw, relu, nhwc
out['convp_per_step'] = dict(launches=28, **rate(step_bytes, step_ms))

for (ci, co, H) in [(16, 16, 42), (32, 32, 21), (32, 32, 11)]:
  xin, dy = planes(H, ci, 1), planes(H, co)
  dw = torch.empty(3, 3, ci, co, device='cuda'); db = torch.empty(co, device='cuda')
  part = torch.empty(NUM_SMS * (9 * ci * co + co), device='cuda')
  def wg():
    _lib.check(L.seedrl_debug_wgradp(ci, co, N, H, H, _lib.ptr(xin), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db),
                                     _lib.ptr(part), part.numel() * 4, _lib.ptr(err), _lib.stream_ptr()))
  out['wgradp_%d_%d_%d' % (ci, co, H)] = rate(N * H * H * (ci + co) * 4, ev(wg))
  del xin, dy
# pools
for (C, H) in [(16, 84), (32, 42)]:
  x = torch.randn(N, H, H, C, device='cuda'); Ho = (H + 1) // 2
  nbp = int(L.seedrl_debug_planes_bytes(N, Ho, Ho, C))
  raw = torch.empty(nbp, dtype=torch.uint8, device='cuda'); rel = torch.empty(nbp, dtype=torch.uint8, device='cuda')
  idx = torch.empty(N, Ho, Ho, C, dtype=torch.uint8, device='cuda')
  f = lambda: _lib.check(L.seedrl_debug_poolp(0, N, H, H, C, _lib.ptr(x), _lib.ptr(raw), _lib.ptr(rel), None, _lib.ptr(idx), _lib.stream_ptr()))
  out['poolp_fwd_%d_%d' % (C, H)] = rate(N * H * H * C * 4 + 2 * N * Ho * Ho * C * 4 + N * Ho * Ho * C, ev(f))
  dxn = torch.empty(N, H, H, C, device='cuda')
  f = lambda: _lib.check(L.seedrl_debug_poolp(1, N, H, H, C, _lib.ptr(raw), None, None, _lib.ptr(dxn), _lib.ptr(idx), _lib.stream_ptr()))
  out['poolp_bwd_nhwc_%d_%d' % (C, H)] = rate(N * H * H * C * 4 + N * Ho * Ho * C * 5, ev(f))
  del x, raw, rel, dxn
assert int(err.item()) == 0
print(json.dumps(out))
