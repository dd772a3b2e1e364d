#!/usr/bin/env python
"""R2D2 central-inference throughput (agents/r2d2/learner.py:711-790 through the public
`R2D2InferenceHost.inference` call, no RPC transport): the eager host against the CUDA-graph host
(`cuda_graph=True`), alternating in one process, at N = 64 (256 envs) and N = 256 (1024 envs), and two
graph hosts sharing one agent on two threads.  bench.py's R2D2 arm: DuelingLSTMDQNNet(18, (84, 84, 1),
stack 4), gemm_mode 'tc3'.  A drain thread empties each host's unroll queue, as the learner's replay feed
would.  Wall clock per call (the call returns host actions: it is synchronous per batch).  One JSON line.

The learner needs about 184 k inferences/s per GPU to keep the replay ratio: at batch 64 and replay_ratio
1.5 each learner step inserts int(64 / 1.5) = 42 unrolls of 100 steps, and one step took 22.83 ms on an
H100 80GB HBM3 at 700 W (bench.py --agent r2d2)."""
import json
import os
import subprocess
import sys
import threading
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.argv = [sys.argv[0]]
import numpy as np
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.agents.r2d2 import learner_loop
from seed_rl_b200.atari import networks
from seed_rl_b200.common import utils

A, OBS, STACK = 18, (84, 84, 1), 4
TARGET = 42 * 100 / 22.83e-3


def gpu_info():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader',
                      '-i', str(torch.cuda.current_device())], capture_output=True, text=True, check=True)
  name, power, clock = (x.strip() for x in q.stdout.strip().split(','))
  return {'name': name, 'power_limit': power, 'max_sm_clock': clock}


class Driver(object):
  """One host with its env shard, its seeded inputs and a thread draining its unroll queue."""

  def __init__(self, agent, N, num_envs, cuda_graph, seed):
    self.host = learner_loop.R2D2InferenceHost(agent, num_envs, 0, N, OBS, cuda_graph=cuda_graph)
    self.N = N
    self.rng = np.random.default_rng(seed)
    self.run_ids = self.rng.integers(1, 2**40, num_envs)
    self.groups = [np.arange(g * N, (g + 1) * N, dtype=np.int32) for g in range(num_envs // N)]
    self.obs = [torch.from_numpy(self.rng.integers(0, 256, (N,) + OBS, dtype=np.uint8)).pin_memory().numpy()
                for _ in self.groups]
    self.zeros = np.zeros(N, np.float32)
    self.i = 0
    threading.Thread(target=self._drain, daemon=True).start()

  def _drain(self):
    try:
      while True:
        self.host.unroll_queue.dequeue()
    except utils.QueueClosedError:
      return

  def call(self):
    g = self.i % len(self.groups)
    ids = self.groups[g]
    env = utils.EnvOutput(self.rng.normal(size=self.N).astype(np.float32), self.rng.random(self.N) < 0.01,
                          self.obs[g], np.zeros(self.N, bool), np.full(self.N, self.i, np.int32))
    self.i += 1
    return self.host.inference(ids, self.run_ids[ids], env, self.zeros)

  def timed(self, iters):
    """-> (per-call seconds, library launches)."""
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    lat = []
    for _ in range(iters):
      t1 = time.perf_counter()
      self.call()
      lat.append(time.perf_counter() - t1)
    return lat, _lib.launch_count() - n0

  def close(self):
    self.host.unroll_queue.close()


def summary(N, lat, launches):
  lat = sorted(lat)
  return {'inferences_per_sec': N * len(lat) / sum(lat), 'us_per_batch_p50': lat[len(lat) // 2] * 1e6,
          'us_per_batch_p99': lat[int(len(lat) * 0.99)] * 1e6, 'library_launches_per_batch': launches / len(lat),
          'batches': len(lat)}


def eager_vs_graph(agent, N, num_envs, iters, rounds, warmup):
  drivers = {'eager': Driver(agent, N, num_envs, False, 1), 'graph': Driver(agent, N, num_envs, True, 1)}
  for d in drivers.values():
    for _ in range(warmup):     # the graph host captures on its first full batch
      d.call()
  lat = {k: [] for k in drivers}
  launches = dict.fromkeys(drivers, 0)
  for _ in range(rounds):       # alternate, so that both modes see the same machine state
    for k, d in drivers.items():
      l, n = d.timed(iters)
      lat[k] += l
      launches[k] += n
  for d in drivers.values():
    d.close()
  out = {'inference_batch_size': N, 'num_envs': num_envs}
  out.update({k: summary(N, lat[k], launches[k]) for k in drivers})
  return out


def two_lanes(agent, N, num_envs, iters, warmup):
  """Two graph hosts, each with its own env shard, store, graph, stream and thread, sharing the agent;
  the graphs are captured one at a time.  Aggregate wall-clock throughput."""
  dev = torch.cuda.current_device()
  capture_lock = threading.Lock()
  gate = threading.Barrier(3)
  lat, errors = [[], []], []

  def lane(k):
    d = None
    try:
      torch.cuda.set_device(dev)
      d = Driver(agent, N, num_envs, True, 100 + k)
      with capture_lock:
        for _ in range(warmup):
          d.call()
      gate.wait(300)
      lat[k] = d.timed(iters)[0]
      gate.wait(300)
    except Exception as exc:     # pylint: disable=broad-except
      errors.append(repr(exc)[:300])
      gate.abort()
    finally:
      if d is not None:
        d.close()
  threads = [threading.Thread(target=lane, args=(k,), daemon=True) for k in range(2)]
  for th in threads:
    th.start()
  try:
    gate.wait(300)
    t0 = time.perf_counter()
    gate.wait(300)
    wall = time.perf_counter() - t0
  except threading.BrokenBarrierError:
    raise RuntimeError('two_lanes failed: ' + ('; '.join(errors) or 'barrier broken'))
  for th in threads:
    th.join(30)
  allat = sorted(x for l in lat for x in l)
  return {'lanes': 2, 'inference_batch_size': N, 'envs_per_lane': num_envs, 'iters_per_lane': iters,
          'inferences_per_sec': 2 * N * iters / wall, 'us_per_batch_p50': allat[len(allat) // 2] * 1e6,
          'us_per_batch_p99': allat[int(len(allat) * 0.99)] * 1e6}


def main():
  if not torch.cuda.is_available():
    raise SystemExit('r2d2_inference_bench needs a CUDA device')
  torch.cuda.set_device(0)
  agent = networks.DuelingLSTMDQNNet(A, OBS, STACK, seed=0, gemm_mode='tc3')
  out = {'what': 'R2D2InferenceHost.inference: host batch -> H2D -> gather -> T=1 DuelingLSTMDQNNet (tc3) -> '
                 'epsilon-greedy -> store append -> scatter -> actions D2H; eager vs one CUDA-graph replay',
         'gpu': gpu_info(), 'target_inferences_per_sec': TARGET}
  out['batch_64'] = eager_vs_graph(agent, 64, 256, iters=200, rounds=4, warmup=30)
  out['batch_256'] = eager_vs_graph(agent, 256, 1024, iters=100, rounds=4, warmup=20)
  out['two_graph_hosts_batch_64'] = two_lanes(agent, 64, 256, iters=600, warmup=30)
  agent.check_errors()
  print(json.dumps(out))


if __name__ == '__main__':
  main()
