"""Cost of the abandoned mask (--bootstrap_abandoned) in the loss kernels on one GPU; prints one JSON line.

Every measurement alternates three variants in one process: the existing entry point (abandoned NULL), the
_abandoned entry point with an all-zero mask, and with 1 % of the rows abandoned (each also done).
  vtrace_stream: the TMA-streamed V-trace loss kernel at B = 65 536, T1 = 21, A = 18, called through ctypes on
                 preallocated buffers; algorithmic bytes are bench.py's roofline_vtrace_loss count, plus
                 T1 x B bytes when the mask is passed.
  learner_step:  the ImpalaDeep V-trace learner step (conv_mode tc3p, lstm_mode tc3) at T = 20, B = 64, with
                 bootstrap_abandoned off, and on with the two masks.
  r2d2:          the R2D2 n-step (n = 5) and Retrace (lambda = 0.95) loss kernels at T = 101, B = 64, A = 18.
Kernel times are the mean of 20 back-to-back launches between one pair of CUDA events; each variant is timed
in `rounds` alternating rounds and the median is reported.  The card's name, power limit and maximum SM clock
are read in the same run.

  python tools/abandoned_bench.py [--steps 10] [--rounds 7]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from seed_rl_b200 import _lib  # noqa: E402
from seed_rl_b200.agents.r2d2 import learner as r2d2_learner  # noqa: E402
from seed_rl_b200.agents.vtrace import learner  # noqa: E402
from seed_rl_b200.common import optimizers, utils  # noqa: E402
from seed_rl_b200.dmlab import networks  # noqa: E402

T, A = 20, 18
VARIANTS = ('null', 'zero', 'one_percent')


def card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name(0) + ' (power limit not readable)'


def events_ms(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(n):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n


def masks(T1, B, g):
  """(done, abandoned) pairs of the three variants; the abandoned rows are also done."""
  dn = torch.rand(T1, B, device='cuda', generator=g) < 0.02
  ab = torch.rand(T1, B, device='cuda', generator=g) < 0.01
  return {'null': (dn, None), 'zero': (dn, torch.zeros_like(dn)), 'one_percent': (dn | ab, ab)}


def alternate(fns, rounds, n=20):
  for fn in fns.values():
    for _ in range(3):
      fn()
  times = {k: [] for k in fns}
  for _ in range(rounds):
    for k, fn in fns.items():
      times[k].append(events_ms(fn, n))
  return {k: float(np.median(v)) for k, v in times.items()}


def vtrace_stream(rounds):
  L = _lib.lib()
  B, T1 = 65536, T + 1
  g = torch.Generator(device='cuda').manual_seed(0)
  ll = torch.randn(T1, B, A, device='cuda', generator=g); lb = torch.randn(T1, B, device='cuda', generator=g)
  bl = torch.randn(T1, B, A, device='cuda', generator=g)
  act = torch.randint(0, A, (T1, B), device='cuda', generator=g)
  rew = torch.randn(T1, B, device='cuda', generator=g)
  ecp = torch.tensor(-0.8, device='cuda')
  cfg = learner._loss_config(learner.default_loss_settings())
  o = learner._loss_outputs(ll, lb, False)
  scratch = learner._loss_scratch(T1, B, A, ll.device)
  P = _lib.ptr
  fns = {}
  for name, (dn, ab) in masks(T1, B, g).items():
    def fn(dn=dn, ab=ab):
      head = (T1, B, A, P(ll), P(lb), P(bl), P(act), P(rew), P(dn))
      tail = (ctypes.byref(cfg), P(ecp), P(o['loss_terms']), P(o['dlogits']), P(o['dbaseline']),
              P(o['d_entropy_cost_param']), None, None, P(scratch), _lib.stream_ptr())
      if ab is None:
        _lib.check(L.seedrl_vtrace_loss_fwd_bwd(*head, *tail))
      else:
        _lib.check(L.seedrl_vtrace_loss_fwd_bwd_abandoned(*head, P(ab), *tail))
    fns[name] = fn
  med = alternate(fns, rounds)
  base = (161 + 76) * T * B + 4 * B + 32            # bench.py roofline_vtrace_loss
  out = {'B': B, 'T1': T1, 'A': A}
  for k, ms in med.items():
    nb = base + (0 if k == 'null' else T1 * B)
    out[k] = {'ms': ms, 'algorithmic_bytes': nb, 'GBps': nb / (ms * 1e-3) / 1e9}
  return out


def unroll(B, ab_p, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  T1 = T + 1
  ab = torch.rand(T1, B, device='cuda', generator=g) < ab_p
  env = utils.EnvOutput(torch.randn(T1, B, device='cuda', generator=g) * 300 + 500,
                        (torch.rand(T1, B, device='cuda', generator=g) < 0.02) | ab,
                        torch.randint(0, 256, (T1, B, 84, 84, 4), device='cuda', generator=g, dtype=torch.uint8),
                        ab, torch.zeros(T1, B, dtype=torch.int32, device='cuda'))
  ao = networks.AgentOutput(torch.randint(0, A, (T1, B), device='cuda', generator=g),
                            torch.randn(T1, B, A, device='cuda', generator=g), torch.zeros(T1, B, device='cuda'))
  state = (torch.zeros(B, 256, device='cuda'), torch.zeros(B, 256, device='cuda'))
  return learner.Unroll(state, torch.randint(0, A, (T1, B), device='cuda', generator=g), env, ao)


def learner_steps(steps, rounds):
  runs = {}
  for name, on, p in (('off', False, 0.0), ('on_zero', True, 0.0), ('on_one_percent', True, 0.01)):
    agent = networks.ImpalaDeep(A, seed=0, conv_mode='tc3p', lstm_mode='tc3')
    step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                               settings=learner.default_loss_settings(bootstrap_abandoned=on), check_errors_every=0)
    un = unroll(64, p)
    runs[name] = (lambda step=step, un=un: step.minimize(un))
  med = alternate(runs, rounds, n=steps)
  return {'ms_per_step': med}


def r2d2(rounds):
  L = _lib.lib()
  Tq, B = 101, 64
  g = torch.Generator(device='cuda').manual_seed(1)
  q = torch.randn(Tq, B, A, device='cuda', generator=g); qt = torch.randn(Tq, B, A, device='cuda', generator=g)
  act = torch.randint(0, A, (Tq, B), device='cuda', generator=g)
  rew = torch.randn(Tq, B, device='cuda', generator=g); w = torch.rand(B, device='cuda', generator=g)
  loss = torch.empty(B, device='cuda'); prio = torch.empty(B, device='cuda'); dq = torch.empty_like(q)
  scratch = torch.empty(int(L.seedrl_r2d2_loss_scratch_bytes(Tq, B, 5)), dtype=torch.uint8, device='cuda')
  P = _lib.ptr
  out = {'T': Tq, 'B': B, 'A': A}
  for rule in ('n_step', 'retrace'):
    fns = {}
    for name, (dn, ab) in masks(Tq, B, g).items():
      def fn(dn=dn, ab=ab, rule=rule):
        head = (Tq, B, A, P(q), P(qt), P(act), P(rew), P(dn))
        if rule == 'n_step':
          tail = (P(w), 0.997, 5, 0.9, 1e-3, P(loss), P(prio), P(dq), P(scratch), _lib.stream_ptr())
          f, fa = L.seedrl_r2d2_loss_fwd_bwd, L.seedrl_r2d2_loss_fwd_bwd_abandoned
        else:
          tail = (P(w), 0.997, 0.95, 0.9, 1e-3, P(loss), P(prio), P(dq), P(scratch), _lib.stream_ptr())
          f, fa = L.seedrl_r2d2_retrace_loss_fwd_bwd, L.seedrl_r2d2_retrace_loss_fwd_bwd_abandoned
        _lib.check(f(*head, *tail) if ab is None else fa(*head, P(ab), *tail))
      fns[name] = fn
    out[rule + '_ms'] = alternate(fns, rounds)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=7)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit('abandoned_bench.py needs a CUDA device')
  line = {'card': card(), 'vtrace_stream_kernel': vtrace_stream(args.rounds),
          'vtrace_learner_step_T20_B64': learner_steps(args.steps, args.rounds), 'r2d2_loss': r2d2(args.rounds)}
  print(json.dumps(line))


if __name__ == '__main__':
  main()
