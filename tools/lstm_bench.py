"""Device time of the LSTM recurrences, lstm_mode 'tiled' (fp32 CUDA cores) against 'tc3' (wgmma bf16x3),
and of the whole learner steps that contain them.

  python tools/lstm_bench.py [--runs 60] [--out FILE]

Recurrences alone: the forward and the BPTT kernel of each mode (one launch each per unroll), at
H = 256 (T1, B) = (21, 64), (21, 256), (1, 64) and H = 512 (141, 64).  Each run is one training forward and
its backward; the two kernels' device durations are read from torch.profiler's CUDA activity records (the
recurrence is one launch inside the library's forward / backward, so events recorded from Python around
it would also time its neighbours).  The modes alternate in rounds on the same inputs; after a warm-up the
median of all runs is reported.

Learner steps: the ImpalaDeep 'tc3p' step at T = 20, B = 64 and the R2D2 'tc3' step at the `bench.py
--agent r2d2` shape (B = 64, 141 rows of 84x84 frames stacked 4), with each LSTM mode: the median of
per-step CUDA-event times, and one step under the library's per-category kernel timing
(seedrl_profile_*; 'lstm_pointwise' holds the recurrences, including the 256-byte counter reset before
each).  Prints one JSON line per measurement, with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)

KERNELS = {'tiled': ('lstm2_fwd_kernel', 'lstm2_bwd_kernel'), 'tc3': ('lstm_tc_fwd_kernel', 'lstm_tc_bwd_kernel')}
MODES = ('tiled', 'tc3')


def card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True)
  return q.stdout.strip().splitlines()[torch.cuda.current_device()] if q.returncode == 0 else 'unknown'


def impala_case(T, B, mode):
  """ImpalaShallow (cheap torso, LSTM(256)): a closure running one training forward + backward."""
  from oracle import learner_oracle
  from seed_rl_b200.dmlab import networks
  A = 18
  agent = networks.ImpalaShallow(A, (84, 84, 4), seed=2, lstm_mode=mode)
  b = learner_oracle.synthetic_batch(T, B, A, seed=5)
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  env = (c(b['reward']), c(b['done']), c(b['observation']))
  state = (c(b['h0']), c(b['c0']))
  T1 = T + 1
  dl = torch.randn(T1, B, A, device='cuda')
  db = torch.randn(T1, B, device='cuda')
  prev = c(b['prev_actions'])

  def run():
    agent(prev, env, state, unroll=True, is_training=True)
    agent.backward(dl, db)
  return agent, run


def r2d2_case(T, B, mode, obs=(36, 36, 1), A=6):
  """DuelingLSTMDQNNet (LSTM(512)): one training forward + backward."""
  from oracle import r2d2_learner_oracle as RL
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import utils
  agent = networks.DuelingLSTMDQNNet(A, obs, 4, seed=11, lstm_mode=mode)
  b = RL.synthetic_replay_batch(T, B, A, obs, seed=3, done_p=0.01)
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']),
                        torch.zeros(T, B, dtype=torch.bool).cuda(), torch.zeros(T, B, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
  dq = torch.randn(T, B, A, device='cuda')
  x = (c(b['prev_actions']), env)

  def run():
    agent(x, state, unroll=True, is_training=True)
    agent.backward(dq)
  return agent, run


def kernel_times(run, names, n):
  """device durations (us) of the kernels whose names contain names[0] / names[1], over n runs"""
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(n):
      run()
    torch.cuda.synchronize()
  out = ([], [])
  for e in prof.events():
    for i, k in enumerate(names):
      if k in e.name:
        out[i].append(e.time_range.elapsed_us())
  assert len(out[0]) == n and len(out[1]) == n, (names, len(out[0]), len(out[1]))
  return out


def recurrences(args, hw):
  shapes = [('impala', 256, 20, 64), ('impala', 256, 20, 256), ('impala', 256, 0, 64), ('r2d2', 512, 141, 64)]
  for net, H, T, B in shapes:
    cases = {m: (impala_case(T, B, m) if net == 'impala' else r2d2_case(T, B, m)) for m in MODES}
    times = {m: ([], []) for m in MODES}
    for m in MODES:
      for _ in range(5):
        cases[m][1]()
    rounds = 3
    for _ in range(rounds):
      for m in MODES:
        f, b = kernel_times(cases[m][1], KERNELS[m], -(-args.runs // rounds))
        times[m][0].extend(f); times[m][1].extend(b)
    for m in MODES:
      cases[m][0].check_errors()
    T1 = T + 1 if net == 'impala' else T
    line = {'what': 'lstm recurrence device time', 'H': H, 'T1': T1, 'B': B, 'runs': len(times['tc3'][0]),
            'hardware': hw}
    for m in MODES:
      line['%s_fwd_us' % m] = float(np.median(times[m][0]))
      line['%s_bwd_us' % m] = float(np.median(times[m][1]))
    line['tc3_over_tiled_fwd'] = line['tc3_fwd_us'] / line['tiled_fwd_us']
    line['tc3_over_tiled_bwd'] = line['tc3_bwd_us'] / line['tiled_bwd_us']
    emit(args, line)
    del cases
    torch.cuda.empty_cache()


def profiled(step_fn):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  ncat = L.seedrl_profile_num_categories()
  ms_c = (ctypes.c_double * ncat)(); n_c = (ctypes.c_uint64 * ncat)()
  _lib.check(L.seedrl_profile_begin(_lib.stream_ptr()))
  step_fn()
  _lib.check(L.seedrl_profile_end(ms_c, n_c))
  return {L.seedrl_profile_category_name(i).decode(): round(ms_c[i], 4) for i in range(ncat)}


def step_times(fn, n):
  ts = []
  for _ in range(n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(); fn(); e1.record()
    ts.append((e0, e1))
  torch.cuda.synchronize()
  return [a.elapsed_time(b) for a, b in ts]


def learner_steps(args, hw):
  from oracle import learner_oracle
  from oracle import r2d2_learner_oracle as RL
  from seed_rl_b200.agents.r2d2 import learner as rlearner
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.atari import networks as anet
  from seed_rl_b200.common import optimizers, utils
  from seed_rl_b200.dmlab import networks
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  # ImpalaDeep, conv mode tc3p, T = 20, B = 64
  A, OBS = 18, (84, 84, 4)
  b = learner_oracle.synthetic_batch(20, 64, A, OBS, seed=1234)
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']),
                        torch.zeros(21, 64, dtype=torch.bool).cuda(), torch.zeros(21, 64, dtype=torch.int32).cuda())
  u = learner.Unroll((c(b['h0']), c(b['c0'])), c(b['prev_actions']), env,
                     networks.AgentOutput(c(b['action']), c(b['behaviour_logits']), c(b['behaviour_baseline'])))
  impala = {}
  for m in MODES:
    agent = networks.ImpalaDeep(A, OBS, seed=1, conv_mode='tc3p', lstm_mode=m)
    step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                               settings=learner.default_loss_settings())
    impala[m] = (agent, lambda step=step: step.minimize(u))
  # R2D2 at the bench.py --agent r2d2 shape
  st = rlearner.default_settings()
  T = st.burn_in + st.unroll_length + 1
  RA, ROBS = 18, (84, 84, 1)
  rb = RL.synthetic_replay_batch(T, 64, RA, ROBS, seed=21, done_p=0.01)
  renv = utils.EnvOutput(c(rb['reward']), c(rb['done']), c(rb['observation']),
                         torch.zeros(T, 64, dtype=torch.bool).cuda(), torch.zeros(T, 64, dtype=torch.int32).cuda())
  rstate = anet.AgentState((c(rb['h0']), c(rb['c0'])), c(rb['frame_state']))
  sampled = rlearner.SampledUnrolls(
      rlearner.Unroll(rstate, None, c(rb['prev_actions']), renv, rlearner.AgentOutput(c(rb['action']), None)),
      c(rb['indices']), c(rb['importance_weights']))
  r2d2 = {}
  for m in MODES:
    agent = anet.DuelingLSTMDQNNet(RA, ROBS, 4, seed=0, lstm_mode=m)
    target = anet.DuelingLSTMDQNNet(RA, ROBS, 4, seed=0, lstm_mode=m)
    step = rlearner.R2D2LearnerStep(agent, target, optimizers.Adam(0.00048, epsilon=1e-3), settings=st)
    r2d2[m] = (agent, lambda step=step: step.minimize(sampled))
  for name, cases, n in (('impala_deep tc3p T=20 B=64', impala, args.steps), ('r2d2 tc3 T=%d B=64' % T, r2d2,
                                                                              max(args.steps // 4, 5))):
    times = {m: [] for m in MODES}
    for m in MODES:
      step_times(cases[m][1], 5)
    for _ in range(3):
      for m in MODES:
        times[m].extend(step_times(cases[m][1], n))
    line = {'what': 'learner step', 'step': name, 'steps': 3 * n, 'hardware': hw}
    for m in MODES:
      cases[m][0].check_errors()
      line['%s_ms_per_step' % m] = float(np.median(times[m]))
      line['%s_kernel_time_ms' % m] = profiled(cases[m][1])
    emit(args, line)
    cases.clear()
    torch.cuda.empty_cache()


def emit(args, line):
  s = json.dumps(line)
  print(s, flush=True)
  if args.out:
    with open(args.out, 'a') as f:
      f.write(s + '\n')


def main():
  p = argparse.ArgumentParser()
  p.add_argument('--runs', type=int, default=60, help='recurrence runs per mode and shape (after 5 warm-up)')
  p.add_argument('--steps', type=int, default=20, help='learner steps per mode and round (3 rounds)')
  p.add_argument('--skip-steps', action='store_true', help='recurrences only')
  p.add_argument('--out', default=None, help='also append the JSON lines to this file')
  args = p.parse_args()
  if not torch.cuda.is_available():
    sys.exit('lstm_bench.py needs a CUDA device')
  torch.cuda.set_device(0)
  hw = card()
  recurrences(args, hw)
  if not args.skip_steps:
    learner_steps(args, hw)


if __name__ == '__main__':
  main()
