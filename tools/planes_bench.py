#!/usr/bin/env python
"""Single-kernel timings of the plane-tensor conv path (csrc/conv_planes.cu) at the learner's
layer shapes: python tools/planes_bench.py

Every convp_kernel configuration the default ImpalaDeep step (net.cu torso_forward /
torso_backward in conv mode tc3p) launches is timed with its real epilogue: shape x {bias, ReLU mask,
residual, raw / ReLU'd / fp32 NHWC output, flipped weights}.  Per configuration: ms per launch
(CUDA events over back-to-back launches after warm-up; each launch includes the debug entry
point's small weight-packing kernel), algorithmic HBM bytes (4 B per element of every plane
tensor read or written -- hi + lo bf16 --, 2 B for the mask's hi planes only, 4 B for fp32 NHWC;
padding positions not counted), GB/s and the fraction of the H100 SXM data-sheet HBM3 bandwidth.

The weight-gradient section times every launch of the step's conv3x3_wgrad category with its
count per step: the four wgradp_kernel shapes, first_wgrad_pooled_kernel at 84x84x4 and the one
batched reduce.  Each debug entry point runs its kernel and a reduce; torch.profiler splits the two.
tma_MB is what wgradp_kernel copies into shared memory, computed from the shapes by the launch
rules of conv_planes.cu launch_wgradp."""
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
       'frames': N, 'peak_GBps_datasheet': PEAK_GBPS, 'convp': {}}
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

def wgradp_tma_bytes(ci, co, H, W):
  """Bytes wgradp_kernel copies by TMA per launch: per K chunk of KC positions, the x hi + lo planes
  over KC + 8 positions and the dy hi + lo planes over KC + T (T = 2 * PW rounded up to 8)."""
  PW = W + 2
  Q = N * (H + 1) * PW
  T = (2 * PW + 7) // 8 * 8
  for KC in ((256, 128, 64) if co == 16 else (128, 64)):
    stage = 2 * (ci // 8) * (KC + 8) * 16 + 2 * (co // 8) * (KC + T) * 16
    nb = 6
    while nb > 1 and 128 + nb * stage > 227 * 1024: nb -= 1
    if nb >= 2:
      return dict(KC=KC, stages=nb, tma_MB=round((Q + PW + KC - 1) // KC * stage / 1e6, 1))
  raise ValueError('wgradp: does not fit')


def kernel_ms(fn, k=ITERS):
  """Device time per call of each kernel fn launches, from torch.profiler."""
  for _ in range(3): fn()
  torch.cuda.synchronize()
  with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(k): fn()
    torch.cuda.synchronize()
  out = {}
  for e in prof.key_averages():
    us = getattr(e, 'self_device_time_total', None)
    if us is None: us = e.self_cuda_time_total
    if us > 0:
      name = 'reduce' if 'reduce' in e.key else 'wgradp' if 'wgradp' in e.key else \
             'first_wgrad_pooled' if 'first_wgrad' in e.key else e.key[:40]
      out[name] = out.get(name, 0.0) + us / 1e3 / k
  return out


# (cin, cout, H, launches per step): net.cu torso_backward in conv mode tc3p
WGRAD = [(16, 16, 42, 4), (16, 32, 42, 1), (32, 32, 21, 5), (32, 32, 11, 4)]
wg = out['wgrad'] = {}
sums = dict(wgradp=0.0, reduce=0.0, first_wgrad_pooled=0.0, MB=0.0, tma_MB=0.0)
for (ci, co, H, count) in WGRAD:
  xin, dy = planes(H, ci, 1), planes(H, co)
  dw = torch.empty(3, 3, ci, co, device='cuda'); db = torch.empty(co, device='cuda')
  part = torch.empty(NUM_SMS * (9 * ci * co + co), device='cuda')
  def wg_call():
    _lib.check(L.seedrl_debug_wgradp(ci, co, N, H, H, _lib.ptr(xin), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db),
                                     _lib.ptr(part), part.numel() * 4, _lib.ptr(err), _lib.stream_ptr()))
  alg = N * H * H * (ci + co) * 4
  km = kernel_ms(wg_call)
  tma = wgradp_tma_bytes(ci, co, H, H)
  r = dict(cin=ci, cout=co, H=H, per_step=count, call_ms=round(ev(wg_call), 4), **tma,
           tma_over_alg=round(tma['tma_MB'] * 1e6 / alg, 2), reduce_ms=round(km.get('reduce', 0.0), 4),
           kernel=rate(alg, km.get('wgradp', 0.0)))
  wg['wgradp_%d_%d_%d' % (ci, co, H)] = r
  sums['wgradp'] += count * km.get('wgradp', 0.0); sums['MB'] += count * alg / 1e6
  sums['tma_MB'] += count * tma['tma_MB']
  del xin, dy
# the fused first layer's weight gradient (84x84x4 frames -> 16 channels, pooled to 42x42)
H0, C0 = 84, 4
Hp = (H0 + 1) // 2
pb = int(L.seedrl_debug_planes_bytes(N, Hp, Hp, 16))
frames = torch.randint(0, 256, (N, H0, H0, C0), dtype=torch.uint8, device='cuda')
w0 = torch.randn(3, 3, C0, 16, device='cuda') * 0.1
b0 = torch.zeros(16, device='cuda')
raw0, rel0, gp0 = (torch.zeros(pb, dtype=torch.uint8, device='cuda') for _ in range(3))
idx0 = torch.zeros(N, Hp, Hp, 16, dtype=torch.uint8, device='cuda')
_lib.check(L.seedrl_debug_conv0pool_c(N, H0, H0, C0, _lib.ptr(frames), _lib.ptr(w0), _lib.ptr(b0), _lib.ptr(raw0),
                                      _lib.ptr(rel0), _lib.ptr(idx0), _lib.ptr(err), _lib.stream_ptr()))
gp0.copy_(raw0)
dw0 = torch.empty_like(w0); db0 = torch.empty(16, device='cuda')
part0 = torch.empty(3 * NUM_SMS * (9 * C0 * 16 + 16), device='cuda')
def first_call():
  _lib.check(L.seedrl_debug_first_wgrad_pooled_c(N, H0, H0, C0, _lib.ptr(frames), _lib.ptr(gp0), _lib.ptr(idx0),
                                                 _lib.ptr(dw0), _lib.ptr(db0), _lib.ptr(part0), part0.numel() * 4,
                                                 _lib.stream_ptr()))
km = kernel_ms(first_call)
alg0 = frames.numel() + N * Hp * Hp * 16 * 5            # frames, gradient planes (hi + lo), argmax taps
wg['first_wgrad_pooled_4_16_84'] = dict(per_step=1, call_ms=round(ev(first_call), 4),
                                        kernel=rate(alg0, km.get('first_wgrad_pooled', 0.0)))
sums['first_wgrad_pooled'] = km.get('first_wgrad_pooled', 0.0); sums['MB'] += alg0 / 1e6
# the step runs ONE batched reduce for all 15 jobs: the largest single reduce bounds it from above
sums['reduce'] = max(v['reduce_ms'] for v in wg.values() if 'reduce_ms' in v)
out['wgrad_per_step'] = dict(
    wgradp_ms=round(sums['wgradp'], 4), first_wgrad_pooled_ms=round(sums['first_wgrad_pooled'], 4),
    reduce_ms_upper=round(sums['reduce'], 4),
    total_ms=round(sums['wgradp'] + sums['first_wgrad_pooled'] + sums['reduce'], 4),
    wgradp_tma_MB=round(sums['tma_MB'], 1),
    note='compare total_ms with kernel_time_ms_per_step.conv3x3_wgrad of a default bench.py run')
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
