"""Cost of the V-trace learner's PopArt (--popart) on one GPU; prints one JSON line.

  learner_step: the ImpalaDeep learner step (conv_mode tc3p, lstm_mode tc3) at T = 20, B = 64, with PopArt off
                and on: two learners in one process, timed in alternating rounds (CUDA events around `steps`
                minimize calls each), medians over the rounds.
  kernels:      over bench.py's roofline_vtrace_loss sweep (B = 64, 4096, 65536; T1 = 21, A = 18): the plain
                loss kernel (seedrl_vtrace_loss_fwd_bwd), PopArt phase 1 (seedrl_vtrace_popart_loss_fwd) and
                phase 2 (seedrl_vtrace_popart_update), each called through ctypes on preallocated buffers and
                timed as the mean of 20 back-to-back launches between one pair of events, after 3 warm-ups.
  multi-task:   the same learner step with --popart_tasks 30 (column b in task b % 30) in the same alternating
                rounds, and the multi-task phases (seedrl_vtrace_popart_tasks_loss_fwd, which includes the
                per-task moment reduction, and seedrl_vtrace_popart_tasks_update) at K = 30 over the same sweep,
                next to the single-task (K = 1) phases.
The card's name, power limit and maximum SM clock are read in the same run.

  python tools/popart_bench.py [--steps 10] [--rounds 5]
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
from seed_rl_b200.agents.vtrace import learner  # noqa: E402
from seed_rl_b200.common import optimizers, utils  # noqa: E402
from seed_rl_b200.dmlab import networks  # noqa: E402

T, A = 20, 18


def card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  except (OSError, subprocess.CalledProcessError):
    return torch.cuda.get_device_name(0) + ' (power limit not readable)'


def unroll(B, seed=0):
  g = torch.Generator(device='cuda').manual_seed(seed)
  T1 = T + 1
  env = utils.EnvOutput(torch.randn(T1, B, device='cuda', generator=g) * 300 + 500,
                        torch.rand(T1, B, device='cuda', generator=g) < 0.02,
                        torch.randint(0, 256, (T1, B, 84, 84, 4), device='cuda', generator=g, dtype=torch.uint8),
                        torch.zeros(T1, B, dtype=torch.bool, device='cuda'),
                        torch.zeros(T1, B, dtype=torch.int32, device='cuda'))
  ao = networks.AgentOutput(torch.randint(0, A, (T1, B), device='cuda', generator=g),
                            torch.randn(T1, B, A, device='cuda', generator=g), torch.zeros(T1, B, device='cuda'))
  state = (torch.zeros(B, 256, device='cuda'), torch.zeros(B, 256, device='cuda'))
  return learner.Unroll(state, torch.randint(0, A, (T1, B), device='cuda', generator=g), env, ao)


def events_ms(fn, n):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  torch.cuda.synchronize()
  e0.record()
  for _ in range(n):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / n


TASKS = 30


def learner_steps(steps, rounds):
  un = unroll(64)
  ids = (torch.arange(64, device='cuda') % TASKS).to(torch.int32)
  arms = {'off': dict(popart=False), 'on': dict(popart=True), 'tasks': dict(popart=True, popart_tasks=TASKS)}
  runs = {}
  for name, kw in arms.items():
    agent = networks.ImpalaDeep(A, seed=0, conv_mode='tc3p', lstm_mode='tc3')
    step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                               settings=learner.default_loss_settings(**kw), check_errors_every=0)
    for _ in range(3):
      step.minimize(un, task_ids=ids)
    runs[name] = step
  times = dict((k, []) for k in arms)
  for _ in range(rounds):
    for name in arms:
      times[name].append(events_ms(lambda: runs[name].minimize(un, task_ids=ids), steps))
  for s in runs.values():
    s.agent.check_errors()
  med = {k: float(np.median(v)) for k, v in times.items()}
  return {'ms_per_step_off': med['off'], 'ms_per_step_on': med['on'], 'rounds_off': times['off'],
          'rounds_on': times['on'], 'on_minus_off_ms': med['on'] - med['off'],
          'ms_per_step_tasks%d' % TASKS: med['tasks'], 'rounds_tasks%d' % TASKS: times['tasks'],
          'tasks_minus_on_ms': med['tasks'] - med['on']}


def kernels():
  L = _lib.lib()
  out = []
  st = learner.default_loss_settings(popart=True)
  cfg = learner._loss_config(st)
  for B in (64, 4096, 65536):
    T1 = T + 1
    g = torch.Generator(device='cuda').manual_seed(0)
    ll = torch.randn(T1, B, A, device='cuda', generator=g); lb = torch.randn(T1, B, device='cuda', generator=g)
    bl = torch.randn(T1, B, A, device='cuda', generator=g)
    act = torch.randint(0, A, (T1, B), device='cuda', generator=g)
    rew = torch.randn(T1, B, device='cuda', generator=g) * 300; dn = torch.rand(T1, B, device='cuda', generator=g) < 0.02
    ecp = torch.tensor(-0.8, device='cuda')
    o = learner._loss_outputs(ll, lb, False)
    mom = torch.tensor([0.0, 1.0], device='cuda'); comp = torch.tensor([1.0, 0.0], device='cuda')
    dcomp = torch.zeros(2, device='cuda')
    td = torch.empty(T1 - 1, B, device='cuda'); sums = torch.empty(2, device='cuda')
    scratch = learner._loss_scratch(T1, B, A, ll.device)
    P = _lib.ptr

    plain_cfg = learner._loss_config(learner.default_loss_settings())

    def plain():
      _lib.check(L.seedrl_vtrace_loss_fwd_bwd(
          T1, B, A, P(ll), P(lb), P(bl), P(act), P(rew), P(dn), ctypes.byref(plain_cfg), P(ecp),
          P(o['loss_terms']), P(o['dlogits']), P(o['dbaseline']), P(o['d_entropy_cost_param']), None, None,
          P(scratch), _lib.stream_ptr()))

    def phase1():
      _lib.check(L.seedrl_vtrace_popart_loss_fwd(
          T1, B, A, P(ll), P(lb), P(bl), P(act), P(rew), P(dn), ctypes.byref(cfg), P(ecp), P(mom), P(comp),
          P(o['loss_terms']), P(o['dlogits']), P(o['dbaseline']), P(o['d_entropy_cost_param']), None, None,
          P(td), P(sums), P(scratch), _lib.stream_ptr()))

    def phase2():
      _lib.check(L.seedrl_vtrace_popart_update(
          T1, B, 1, 1e-2, 0.5, P(lb), P(td), P(sums), P(mom), P(comp), P(o['dbaseline']), P(dcomp),
          P(o['loss_terms']), P(scratch), _lib.stream_ptr()))

    ids = (torch.arange(B, device='cuda') % TASKS).to(torch.int32)
    kmom = torch.tensor([[0.0, 1.0]] * TASKS, device='cuda'); kcomp = torch.tensor([[1.0, 0.0]] * TASKS, device='cuda')
    kdcomp = torch.zeros(TASKS, 2, device='cuda')
    ksums = torch.empty(TASKS, 3, dtype=torch.float64, device='cuda')
    kerr = torch.zeros(1, dtype=torch.int32, device='cuda')
    kscratch = learner._loss_scratch(T1, B, A, ll.device, TASKS)

    def tasks_phase1():
      _lib.check(L.seedrl_vtrace_popart_tasks_loss_fwd(
          T1, B, A, P(ll), P(lb), P(bl), P(act), P(rew), P(dn), None, P(ids), TASKS, ctypes.byref(cfg), P(ecp),
          P(kmom), P(kcomp), P(o['loss_terms']), P(o['dlogits']), P(o['dbaseline']), P(o['d_entropy_cost_param']),
          None, None, P(td), P(ksums), P(kerr), P(kscratch), _lib.stream_ptr()))

    def tasks_phase2():
      _lib.check(L.seedrl_vtrace_popart_tasks_update(
          T1, B, TASKS, 1e-2, 0.5, P(lb), P(td), P(ids), P(ksums), P(kmom), P(kcomp), P(o['dbaseline']), P(kdcomp),
          P(o['loss_terms']), P(kscratch), _lib.stream_ptr()))
    row = {'B': B}
    for name, fn in (('plain_loss_ms', plain), ('popart_phase1_ms', phase1), ('popart_phase2_ms', phase2),
                     ('tasks%d_phase1_ms' % TASKS, tasks_phase1), ('tasks%d_phase2_ms' % TASKS, tasks_phase2)):
      for _ in range(3):
        fn()
      row[name] = events_ms(fn, 20)
    assert int(kerr.item()) == 0
    out.append(row)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    sys.exit('popart_bench.py needs a CUDA device')
  line = {'card': card(), 'T': T, 'A': A, 'learner_step_B64': learner_steps(args.steps, args.rounds),
          'kernels': kernels()}
  print(json.dumps(line))


if __name__ == '__main__':
  main()
