#!/usr/bin/env python
"""Bit-identity check of the central-inference hosts across two versions of the code.

`--out DIR` drives five host configurations through one seeded call sequence and writes one .npy file
per array: the returned actions, every Aggregator table, the unroll store (`_state`, `_index`, host
index), every unroll-queue item or assembled training batch, and the info items.  `--compare DIR_A
DIR_B` checks that two such dumps hold the same files with np.array_equal contents.  The driver uses
only the host constructors and `inference` (and reads their tables), so it runs unchanged on older
versions of the hosts.

Configurations: V-trace with the unroll queue (eager); V-trace with the assembler and the CUDA graph;
V-trace with the assembler and cuda_graph=False; R2D2 eager with a seeded generator; R2D2 with the CUDA
graph and a fixed epsilon_seed.  The call sequence has full and partial batches, done flags, run-id
resets and, for R2D2, eval environments.  Shapes: 'toy', and 'bench' (batch 64, 256 environments, the
networks and contraction modes of bench.py and tools/r2d2_inference_bench.py).
"""
import argparse
import json
import os
import sys
import threading

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {
    'toy': dict(vtrace=dict(A=18, obs=(84, 84, 4), N=3, num_envs=6, T=3, B=4, calls=40, conv_mode='simt'),
                r2d2=dict(A=6, obs=(36, 36, 1), N=4, num_envs=7, num_eval=2, unroll=4, burn_in=2, calls=60,
                          gemm_mode='tc3')),
    'bench': dict(vtrace=dict(A=18, obs=(84, 84, 4), N=64, num_envs=256, T=20, B=64, calls=120, conv_mode='tc3p'),
                  r2d2=dict(A=18, obs=(84, 84, 1), N=64, num_envs=256, num_eval=16, unroll=100, burn_in=40,
                            calls=440, gemm_mode='tc3')),
}


def call_sequence(obs, num_envs, N, calls, seed):
  """Random batches of N distinct env ids; every 7th call is a partial batch, two calls restart the
  actors of a quarter of their batch (new run ids)."""
  import numpy as np
  import torch
  from seed_rl_b200.common import utils
  rng = np.random.default_rng(seed)
  run_ids = rng.integers(1, 2**40, num_envs)
  seq = []
  for i in range(calls):
    ids = rng.permutation(num_envs)[:N].astype(np.int32)
    if i % 7 == 3:
      ids = ids[:N // 2 + 1]
    if i in (calls // 3, 2 * calls // 3):
      run_ids[ids[::4]] += 1
    n = len(ids)
    frames = torch.from_numpy(rng.integers(0, 256, (n,) + obs, dtype=np.uint8)).pin_memory().numpy()
    env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), rng.random(n) < 0.05, frames,
                          np.zeros(n, bool), np.full(n, i, np.int32))
    seq.append((ids, run_ids[ids].copy(), env, rng.normal(size=n).astype(np.float32)))
  return seq


def drain(queue):
  return [queue.dequeue() for _ in range(queue.size())]


def stacked(items):
  """Items (nests of tensors of one structure) -> one array per leaf, stacked over the items."""
  import numpy as np
  from seed_rl_b200.common import utils
  flat = [[np.asarray(t.cpu() if hasattr(t, 'cpu') else t) for t in utils.flatten(tuple(it))] for it in items]
  return {'%02d' % k: np.stack([f[k] for f in flat]) for k in range(len(flat[0]))} if flat else {}


def host_arrays(host, actions):
  import numpy as np
  out = {'actions': np.concatenate(actions), 'batch_sizes': np.array([len(a) for a in actions]),
         'env_run_ids': host.env_run_ids, 'store_index': host.store._index.cpu().numpy(),
         'store_host_index': np.asarray(host.store._host_index)}
  for k, t in enumerate(host.env_infos):
    out['env_infos_%d' % k] = t
  for agg in (host.first_agent_states, host.agent_states, host.actions):
    for k, t in enumerate(agg._state):
      out['%s_%d' % (agg.name, k)] = t.cpu().numpy()
  for k, t in enumerate(host.store._state):
    out['store_state_%02d' % k] = t.cpu().numpy()
  for k, v in stacked(drain(host.unroll_queue)).items():
    out['unrolls_' + k] = v
  for k, v in stacked(drain(host.info_queue)).items():
    out['infos_' + k] = v
  return out


def run_vtrace(c, mode):
  import torch
  from seed_rl_b200.agents.vtrace import learner_loop
  from seed_rl_b200.common import utils
  from seed_rl_b200.dmlab import networks
  agent = networks.ImpalaDeep(c['A'], c['obs'], seed=0, conv_mode=c['conv_mode'])
  TS = utils.TensorSpec
  info_queue = utils.StructuredFIFOQueue(-1, (TS([], 'int64', 'episode_num_frames'),
                                              TS([], 'float32', 'episode_returns'),
                                              TS([], 'float32', 'episode_raw_returns')))
  kw = {} if mode == 'queue' else dict(training_batch_size=c['B'], cuda_graph=(mode == 'graph'))
  host = learner_loop.InferenceHost(agent, c['num_envs'], c['T'], c['N'], c['obs'], info_queue=info_queue, **kw)
  host.unroll_queue = utils.StructuredFIFOQueue(-1, host.unroll_specs)      # nobody trains here
  batches = []

  def learner_thread():
    try:
      while True:
        slot, u = learner_loop.assembled_batch(host.assembler)
        batches.append([t.cpu().numpy() for t in utils.flatten(tuple(u))])
        host.assembler.release(slot)
    except utils.QueueClosedError:
      return
  if host.assembler is not None:
    th = threading.Thread(target=learner_thread)
    th.start()
  actions = [host.inference(*x) for x in call_sequence(c['obs'], c['num_envs'], c['N'], c['calls'], seed=1)]
  torch.cuda.synchronize()
  if host.assembler is not None:
    host.assembler.close()              # the learner thread drains the full batches, then stops
    th.join(300)
  out = host_arrays(host, actions)
  for k, v in stacked(batches).items():
    out['batches_' + k] = v
  agent.check_errors()
  return out


def run_r2d2(c, mode):
  import torch
  from seed_rl_b200.agents.r2d2 import learner, learner_loop
  from seed_rl_b200.atari import networks
  agent = networks.DuelingLSTMDQNNet(c['A'], c['obs'], 4, seed=1, gemm_mode=c['gemm_mode'])
  st = learner.default_settings(unroll_length=c['unroll'], burn_in=c['burn_in'])
  kw = dict(cuda_graph=True, epsilon_seed=7) if mode == 'graph' else {}
  host = learner_loop.R2D2InferenceHost(agent, c['num_envs'], c['num_eval'], c['N'], c['obs'], settings=st,
                                        unroll_queue_max_size=-1,
                                        generator=torch.Generator(device='cuda').manual_seed(2), **kw)
  actions = [host.inference(*x) for x in call_sequence(c['obs'], c['num_envs'], c['N'], c['calls'], seed=2)]
  torch.cuda.synchronize()
  out = host_arrays(host, actions)
  agent.check_errors()
  return out


def dump(out_dir, shapes):
  import numpy as np
  import torch
  torch.cuda.set_device(0)
  os.makedirs(out_dir, exist_ok=True)
  counts = {}
  for shape in shapes:
    c = SHAPES[shape]
    runs = [('vtrace_queue', run_vtrace, c['vtrace'], 'queue'), ('vtrace_graph', run_vtrace, c['vtrace'], 'graph'),
            ('vtrace_eager', run_vtrace, c['vtrace'], 'eager'), ('r2d2_eager', run_r2d2, c['r2d2'], 'eager'),
            ('r2d2_graph', run_r2d2, c['r2d2'], 'graph')]
    for name, fn, cfg, mode in runs:
      arrays = fn(cfg, mode)
      for k, v in arrays.items():
        np.save(os.path.join(out_dir, '%s_%s_%s.npy' % (shape, name, k)), v)
      counts['%s_%s' % (shape, name)] = {
          'arrays': len(arrays), 'unrolls': int(len(arrays['unrolls_00'])) if 'unrolls_00' in arrays else 0,
          'batches': int(len(arrays['batches_00'])) if 'batches_00' in arrays else 0,
          'infos': int(len(arrays['infos_00'])) if 'infos_00' in arrays else 0}
      torch.cuda.empty_cache()
  print(json.dumps({'dump': out_dir, 'configs': counts}))


def compare(a, b):
  import numpy as np
  fa, fb = sorted(os.listdir(a)), sorted(os.listdir(b))
  differ = [f for f in fa if f in fb and not np.array_equal(np.load(os.path.join(a, f)), np.load(os.path.join(b, f)))]
  only = sorted(set(fa) ^ set(fb))
  print(json.dumps({'files': len(fa), 'equal': not differ and not only, 'differ': differ, 'only_in_one': only}))
  return not differ and not only


def main():
  p = argparse.ArgumentParser(description=__doc__.split('\n')[0])
  p.add_argument('--out')
  p.add_argument('--shapes', default='toy,bench')
  p.add_argument('--compare', nargs=2, metavar=('DIR_A', 'DIR_B'))
  args = p.parse_args()
  sys.argv = sys.argv[:1]
  if args.compare:
    sys.exit(0 if compare(*args.compare) else 1)
  if not args.out:
    p.error('--out or --compare is required')
  dump(args.out, args.shapes.split(','))


if __name__ == '__main__':
  main()
