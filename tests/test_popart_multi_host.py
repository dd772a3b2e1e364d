"""CPU, world_size 2, gloo: PopArt across replicas.  Each replica reduces its own batch's moment sums, the
learner's moment exchange (LearnerStep._reduce_moment_sums, a SUM all-reduce) combines them, and the update
divides by world x T x B (seedrl_vtrace_popart_update's `world`).  Both replicas must end with the same state,
equal to one process's update on the concatenated batch (the reference's aggregation=MEAN for equal batches)."""
import json
import os
import sys
import types

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
T1, B, A = 11, 12, 6
STATE = np.array([30.0, 2500.0, 0.9, 0.1], np.float32)
BETA = 0.2


def _batch():
  g = np.random.default_rng(4)
  return (g.standard_normal((T1, 2 * B, A)).astype(np.float32), g.standard_normal((T1, 2 * B)).astype(np.float32),
          g.standard_normal((T1, 2 * B, A)).astype(np.float32), g.integers(0, A, (T1, 2 * B)),
          (g.standard_normal((T1, 2 * B)) * 300 + 400).astype(np.float32), g.random((T1, 2 * B)) < 0.1)


def _worker(rank, world, port, out):
  os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
  sys.path[:0] = [ROOT, HERE]
  import popart_reference as PR
  from seed_rl_b200.agents.vtrace import learner
  dist.init_process_group('gloo', rank=rank, world_size=world)
  cfg = learner.default_loss_settings(popart=True, popart_beta=BETA)
  mine = tuple(x[:, rank * B:(rank + 1) * B] for x in _batch())
  s1, s2 = PR.moment_sums(cfg, *mine, STATE)[:2]
  sums = torch.tensor([s1, s2], dtype=torch.float64)
  learner.LearnerStep._reduce_moment_sums(types.SimpleNamespace(pg=None), sums)
  n = world * (T1 - 1) * B
  r = PR.loss_and_grads(cfg, *mine, -1.0, STATE, BETA, global_means=(float(sums[0]) / n, float(sums[1]) / n))
  dist.barrier()
  dist.destroy_process_group()
  json.dump({'state': [float(x) for x in r['state']]}, open(os.path.join(out, 'r%d.json' % rank), 'w'))


def test_replicas_share_one_popart_update(tmp_path):
  world, port = 2, 29581
  mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
  r = [json.load(open(tmp_path / ('r%d.json' % i)))['state'] for i in range(world)]
  assert r[0] == r[1]
  import popart_reference as PR
  from seed_rl_b200.agents.vtrace import learner
  cfg = learner.default_loss_settings(popart=True, popart_beta=BETA)
  one = PR.loss_and_grads(cfg, *_batch(), -1.0, STATE, BETA)['state']
  np.testing.assert_allclose(r[0], one, rtol=1e-12)
  assert abs(one[0] - STATE[0]) > 1.0
