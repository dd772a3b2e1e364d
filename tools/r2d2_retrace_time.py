#!/usr/bin/env python
"""Times the R2D2 loss under both Bellman target rules, n-step double-DQN (the reference's, default) and
Retrace(lambda) (--bellman_target=retrace), at the reference's default shapes, and prints one JSON line:

  * the two loss kernels alone at T = 101, B = 64, A = 18: device time per launch from CUDA events around
    back-to-back launches, and each kernel's own duration from torch.profiler in a separate pass;
  * the whole learner step (R2D2LearnerStep.minimize: burn-in 40 + unroll 100 + 1 rows, 84x84x1 frames
    stacked 4) under each rule, alternating the rules between timed windows;
  * the card's name and power limit, read in the same call.

  python tools/r2d2_retrace_time.py [--mode tc3|simt] [--steps 10] [--rounds 3]
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
from seed_rl_b200.agents.r2d2 import learner  # noqa: E402
from seed_rl_b200.atari import networks  # noqa: E402
from seed_rl_b200.common import optimizers, utils  # noqa: E402

A, OBS, S, BURN = 18, (84, 84, 1), 4, 40


def card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                     capture_output=True, text=True)
  return dict(torch_name=torch.cuda.get_device_name(0), nvidia_smi=q.stdout.strip() or q.stderr.strip())


def loss_kernels(T=101, B=64, launches=500):
  L = _lib.lib()
  g = torch.Generator(device='cuda').manual_seed(0)
  q = torch.randn(T, B, A, device='cuda', generator=g)
  qt = torch.randn(T, B, A, device='cuda', generator=g)
  act = torch.where(torch.rand(T, B, device='cuda', generator=g) < 0.7, q.argmax(-1),
                    torch.randint(0, A, (T, B), device='cuda', generator=g))
  rew = torch.randn(T, B, device='cuda', generator=g)
  done = (torch.rand(T, B, device='cuda', generator=g) < 0.01).to(torch.uint8)
  w = torch.rand(B, device='cuda', generator=g)
  loss, prio, dq = torch.empty(B, device='cuda'), torch.empty(B, device='cuda'), torch.empty_like(q)
  sn = torch.empty(int(L.seedrl_r2d2_loss_scratch_bytes(T, B, 5)), dtype=torch.uint8, device='cuda')
  sr = torch.empty(int(L.seedrl_r2d2_retrace_loss_scratch_bytes(T, B)), dtype=torch.uint8, device='cuda')
  p = _lib.ptr
  ins = (p(q), p(qt), p(act), p(rew), p(done), p(w))
  outs = (p(loss), p(prio), p(dq))
  st = _lib.stream_ptr()
  calls = {
      'n_step': lambda: L.seedrl_r2d2_loss_fwd_bwd(T, B, A, *ins, 0.997, 5, 0.9, 1e-3, *outs, p(sn), st),
      'retrace': lambda: L.seedrl_r2d2_retrace_loss_fwd_bwd(T, B, A, *ins, 0.997, 0.95, 0.9, 1e-3, *outs, p(sr), st)}
  for fn in calls.values():
    for _ in range(20):
      _lib.check(fn())
  torch.cuda.synchronize()
  per_launch = {k: [] for k in calls}
  for _ in range(3):                                      # alternate the two kernels
    for k, fn in calls.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(launches):
        fn()
      e1.record(); torch.cuda.synchronize()
      per_launch[k].append(e0.elapsed_time(e1) * 1e3 / launches)
  # each kernel's own duration, in a pass of its own
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(100):
      for fn in calls.values():
        fn()
    torch.cuda.synchronize()
  names = {'n_step': 'r2d2_loss_kernel', 'retrace': 'r2d2_retrace_loss_kernel'}
  kernel_us = {}
  for k, name in names.items():
    ev = [e for e in prof.key_averages() if name in e.key and ('retrace' in e.key) == (k == 'retrace')]
    kernel_us[k] = round(sum(e.device_time_total for e in ev) / max(1, sum(e.count for e in ev)), 2) if ev else None
  return dict(shape=[T, B, A], us_per_launch_events={k: [round(v, 2) for v in x] for k, x in per_launch.items()},
              kernel_us_profiler=kernel_us)


def learner_steps(mode, steps, rounds, B=64):
  T = BURN + 100 + 1
  g = torch.Generator(device='cuda').manual_seed(0)
  frames = torch.randint(0, 256, (T, B) + OBS, dtype=torch.uint8, device='cuda', generator=g)
  env = utils.EnvOutput(torch.randn(T, B, device='cuda', generator=g), torch.rand(T, B, device='cuda', generator=g) < 0.01,
                        frames, torch.zeros(T, B, dtype=torch.bool, device='cuda'),
                        torch.zeros(T, B, dtype=torch.int32, device='cuda'))
  agent = networks.DuelingLSTMDQNNet(A, OBS, S, seed=0, gemm_mode=mode)
  target = networks.DuelingLSTMDQNNet(A, OBS, S, seed=0, gemm_mode=mode)
  pa = torch.randint(0, A, (T, B), device='cuda', generator=g)
  act = torch.randint(0, A, (T, B), device='cuda', generator=g)
  unrolls = learner.Unroll(agent.initial_state(B), None, pa, env, learner.AgentOutput(act, None))
  sampled = learner.SampledUnrolls(unrolls, torch.arange(B, device='cuda'), torch.rand(B, device='cuda', generator=g))
  rules = {k: learner.R2D2LearnerStep(agent, target, optimizers.Adam(0.00048, epsilon=1e-3),
                                      settings=learner.default_settings(bellman_target=k))
           for k in learner.BELLMAN_TARGETS}
  for step in rules.values():
    for _ in range(2):
      step.minimize(sampled)
  torch.cuda.synchronize(); agent.check_errors()
  ms = {k: [] for k in rules}
  for _ in range(rounds):
    for k, step in rules.items():
      e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      e0.record()
      for _ in range(steps):
        step.minimize(sampled)
      e1.record(); torch.cuda.synchronize()
      ms[k].append(e0.elapsed_time(e1) / steps)
  agent.check_errors()
  return dict(mode=mode, T=T, B=B, steps_per_window=steps, ms_per_step={k: [round(v, 3) for v in x] for k, x in ms.items()},
              median_ms={k: round(float(np.median(x)), 3) for k, x in ms.items()})


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--mode', default='tc3', choices=['tc3', 'simt'])
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=3)
  a = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit('needs a CUDA device')
  out = dict(card=card(), loss_kernels=loss_kernels(), learner_step=learner_steps(a.mode, a.steps, a.rounds))
  print(json.dumps(out))


if __name__ == '__main__':
  main()
