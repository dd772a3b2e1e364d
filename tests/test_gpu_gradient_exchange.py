"""The data-parallel gradient exchange of both learners, on one GPU, against an exact expectation.

A test-local stand-in for torch.distributed (is_initialized, get_world_size, all_reduce), installed with
monkeypatch, plays world = 2: all_reduce(t, SUM) adds, on the calling stream, the matching slice of the other
replica's precomputed gradient arena (or its PopArt moment sums); with async_op it returns a work object whose
wait() makes the caller's stream wait for the stream the reduction ran on, the ordering NCCL gives.

For two replicas the fp32 sum g_A + g_B does not depend on order, so the expectation is bit-exact: after
LearnerStep.minimize on batch A the parameters and Adam's m and v equal one process's Adam applied to g_A + g_B, with
g_A and g_B taken from runs of compute_gradients on the two batches (with PopArt, under the moment statistics of
both batches).  An element summed twice or never fails outright.

The overlapped exchange all-reduces bucket 1, floats [0, grad_split) = the heads, Dense and LSTM, on a side stream
once the library records head_ready_event, while the conv torso's backward still runs; bucket 2 follows on the
compute stream.  Besides the end result, the stand-in snapshots bucket 1 on the side stream right after the event;
it must equal the replica's final bucket 1.  That check only fails when a late write lands after the snapshot, so
test_head_event_follows_every_bucket_1_launch adds a timing-free one: in a torch.profiler trace of the backward,
taken in a child process, the library's cudaEventRecord comes right after the Dense bias colsum and before the
dflat GEMM.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)

A, OBS, T, B = 18, (84, 84, 4), 20, 64
WORLD = 2


class _Work(object):

  def __init__(self, event):
    self._event = event

  def wait(self):
    torch.cuda.current_stream().wait_event(self._event)


class _Exchange(object):
  """What torch.distributed does for one replica of WORLD, given the other replicas' gradient arenas and moment
  sums.  `grads` is this replica's gradient arena, to locate the slice an all_reduce is handed."""

  def __init__(self, others=(), other_sums=(), grads=None, snapshot_split=None):
    self.others, self.other_sums, self.grads = list(others), list(other_sums), grads
    self.snapshot_split = snapshot_split
    self.snapshot = None
    self.calls = []

  def install(self, monkeypatch):
    import torch.distributed as td
    monkeypatch.setattr(td, 'is_available', lambda: True)
    monkeypatch.setattr(td, 'is_initialized', lambda: True)
    monkeypatch.setattr(td, 'get_world_size', lambda group=None: WORLD)
    monkeypatch.setattr(td, 'all_reduce', self.all_reduce)

  def all_reduce(self, t, op=None, group=None, async_op=False):
    import torch.distributed as td
    assert op == td.ReduceOp.SUM
    base = self.grads.data_ptr() if self.grads is not None else None
    if base is not None and base <= t.data_ptr() < base + 4 * self.grads.numel():
      off = (t.data_ptr() - base) // 4
      self.calls.append(('grads', off, t.numel(), async_op))
      if async_op and off == 0 and t.numel() == self.snapshot_split:
        self.snapshot = t.clone()         # bucket 1 as the side stream sees it right after head_ready_event
      for o in self.others:
        t.add_(o[off:off + t.numel()])
    else:
      assert t.numel() == 2, 'only the gradient arena and the PopArt moment sums are exchanged'
      self.calls.append(('sums', 0, 2, async_op))
      for s in self.other_sums:
        t.add_(s)
    if async_op:
      ev = torch.cuda.Event()
      ev.record()
      return _Work(ev)
    return None


def _vtrace_batch(seed):
  from oracle import learner_oracle
  from test_gpu_parity import _batch_to_cuda
  return _batch_to_cuda(learner_oracle.synthetic_batch(T, B, A, OBS, seed=seed))


def _vtrace_step(net, conv_mode, popart, grad_reduce='sum', overlap=True):
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  agent = (networks.ImpalaDeep if net == 'deep' else networks.ImpalaShallow)(A, OBS, seed=1, conv_mode=conv_mode)
  opt = optimizers.Adam(optimizers.PolynomialDecay(4.8e-4, 10 ** 6, 0.0), beta_1=0.0, epsilon=3.125e-7)
  return learner.LearnerStep(agent, opt, settings=learner.default_loss_settings(popart=popart),
                             grad_reduce=grad_reduce, overlap_reduce=overlap)


def _bits(t):
  return t.detach().cpu().numpy().view(np.uint32)


def _gradients(monkeypatch, net, conv_mode, popart, batches):
  """-> per batch (its gradient arena after compute_gradients, the parameters then, its own moment sums), under the
  moment statistics of all batches.  compute_gradients exchanges no gradient without the overlap."""
  sums = []
  if popart:
    for u in batches:                    # the moment sums of each batch on its own
      ex = _Exchange()
      captured = []
      ex.all_reduce = lambda t, op=None, group=None, async_op=False: captured.append(t.clone())
      with monkeypatch.context() as mp:
        ex.install(mp)
        _vtrace_step(net, conv_mode, True, overlap=False).compute_gradients(u)
      sums.append(captured[0])
  out = []
  for i, u in enumerate(batches):
    ex = _Exchange(other_sums=[s for j, s in enumerate(sums) if j != i])
    with monkeypatch.context() as mp:
      ex.install(mp)
      step = _vtrace_step(net, conv_mode, popart, overlap=False)
      step.compute_gradients(u)
    torch.cuda.synchronize()
    assert [c[0] for c in ex.calls] == (['sums'] if popart else [])
    out.append((step.agent.grads.clone(), step.agent.params.clone(), sums[i] if popart else None))
  return out


def _expected(net, conv_mode, popart, params, g_sum, scale):
  """One process: Adam on g_A + g_B from the parameters replica A holds after compute_gradients."""
  step = _vtrace_step(net, conv_mode, popart)
  agent = step.agent
  agent.params.copy_(params)
  mul = step.settings.entropy_cost_adjustment_speed
  step.optimizer.apply_gradients(agent.params, g_sum.clone(), grad_scale=scale,
                                 clamp_index=agent.entropy_cost_param_index, clamp_lo=-20.0 / mul,
                                 clamp_hi=20.0 / mul)
  torch.cuda.synchronize()
  return agent.params, step.optimizer.m, step.optimizer.v


def _exchange_run(monkeypatch, net, conv_mode, popart, grad_reduce, overlap, u, other, other_sums):
  ex = _Exchange([other], [other_sums] if popart else [])
  with monkeypatch.context() as mp:
    ex.install(mp)
    step = _vtrace_step(net, conv_mode, popart, grad_reduce, overlap)
    assert step.world == WORLD
    ex.grads, ex.snapshot_split = step.agent.grads, step.agent.grad_split
    step.minimize(u)
  torch.cuda.synchronize()
  return step, ex


CASES = [('deep', 'tc3p', False, 'sum'), ('deep', 'tc3p', False, 'mean'), ('deep', 'tc3p', True, 'sum'),
         ('deep', 'tc3p', True, 'mean'), ('shallow', 'tc3', False, 'sum')]


@pytest.mark.parametrize('net,conv_mode,popart,grad_reduce', CASES)
def test_exchange_is_adam_of_the_sum(monkeypatch, net, conv_mode, popart, grad_reduce):
  ua, ub = _vtrace_batch(1234), _vtrace_batch(4321)
  (ga, pa, _), (gb, _, sb) = _gradients(monkeypatch, net, conv_mode, popart, [ua, ub])
  assert not torch.equal(ga, gb)
  scale = 0.5 if grad_reduce == 'mean' else 1.0
  want = _expected(net, conv_mode, popart, pa, ga + gb, scale)
  overlaps = (True, False) if net == 'deep' else (True,)
  for overlap in overlaps:
    step, ex = _exchange_run(monkeypatch, net, conv_mode, popart, grad_reduce, overlap, ua, gb, sb)
    split, n = step.agent.grad_split, step.agent.grads.numel()
    kinds = [c for c in ex.calls if c[0] == 'grads']
    assert kinds == ([('grads', 0, split, True), ('grads', split, n - split, False)] if overlap
                     else [('grads', 0, n, False)])
    assert [c for c in ex.calls if c[0] == 'sums'] == ([('sums', 0, 2, False)] if popart else [])
    what = '%s overlap=%s' % (grad_reduce, overlap)
    np.testing.assert_array_equal(_bits(step.agent.grads), _bits(ga + gb), err_msg='reduced gradient, ' + what)
    for got, exp, nm in zip((step.agent.params, step.optimizer.m, step.optimizer.v), want, ('params', 'm', 'v')):
      np.testing.assert_array_equal(_bits(got), _bits(exp), err_msg='%s, %s' % (nm, what))
    if overlap:
      np.testing.assert_array_equal(_bits(ex.snapshot), _bits(ga[:split]),
                                    err_msg='bucket 1 changed after head_ready_event')
  # the update is real: every tensor with a nonzero summed gradient moved
  assert (_bits(want[0]) != _bits(pa)).mean() > 0.5


def test_overlapped_backward_is_the_backward(monkeypatch):
  """seedrl_net_backward_overlap gives the gradients of seedrl_net_backward bit for bit."""
  for net, conv_mode in (('deep', 'tc3p'), ('shallow', 'tc3')):
    step = _vtrace_step(net, conv_mode, False)
    u = _vtrace_batch(99)
    step.compute_gradients(u)
    r = step.agent._loss_grads
    plain = step.agent.backward(r['dlogits'], r['dbaseline']).clone()
    ev = torch.cuda.Event()
    over = step.agent.backward(r['dlogits'], r['dbaseline'], head_ready_event=ev).clone()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_bits(over), _bits(plain), err_msg=net)


@pytest.mark.parametrize('net,conv_mode', [('deep', 'tc3p'), ('shallow', 'tc3')])
def test_grad_split_partitions_the_arena(net, conv_mode):
  """Every parameter tensor lies wholly in one bucket; bucket 1 is exactly the heads, Dense and LSTM tensors; the
  entropy_cost_param slot and the PopArt tail lie in bucket 2."""
  step = _vtrace_step(net, conv_mode, True)
  agent = step.agent
  split = agent.grad_split
  head = ('policy_logits/', 'baseline/', 'core/', 'conv_to_linear/')
  tensors = agent.param_info[:agent._n_tensors]
  bucket1 = set()
  for name, shape, off in tensors:
    end = off + int(np.prod(shape))
    assert end <= split or off >= split, '%s [%d, %d) straddles grad_split %d' % (name, off, end, split)
    if end <= split:
      bucket1.add(name)
  assert bucket1 == {name for name, _, _ in tensors if name.startswith(head)}
  assert bucket1 and len(bucket1) < len(tensors)
  # bucket 1 ends where its last tensor's 64-float slot ends: no gap floats of bucket 2's first tensor in it
  last = max(off + int(np.prod(shape)) for name, shape, off in tensors if name in bucket1)
  assert split == (last + 63) // 64 * 64
  assert split == min(off for name, _, off in tensors if name not in bucket1)
  assert agent.entropy_cost_param_index >= split
  assert agent.arena_floats >= split
  tail = [off for name, _, off in agent.param_info if name.startswith('popart/')]
  assert len(tail) == 2 and min(tail) >= agent.arena_floats


def _trace_launches(path):
  """-> [(kind, name)] in host call order: ('launch', kernel name) for each kernel launch, ('record', '') for each
  cudaEventRecord, ('memset', '') for each cudaMemsetAsync."""
  with open(path) as f:
    ev = json.load(f)['traceEvents']
  kernels = {e['args']['correlation']: e['name'] for e in ev
             if e.get('cat') == 'kernel' and 'correlation' in e.get('args', {})}
  api = sorted((e for e in ev if e.get('cat') in ('cuda_runtime', 'cuda_driver') and 'correlation' in e.get('args', {})),
               key=lambda e: e['args']['correlation'])
  out = []
  for e in api:
    c = e['args']['correlation']
    if c in kernels:
      out.append(('launch', kernels[c]))
    elif e['name'].startswith('cudaEventRecord'):
      out.append(('record', ''))
    elif e['name'].startswith('cudaMemsetAsync'):
      out.append(('memset', ''))
  return out


def _profile_backward(net, conv_mode, out_dir):
  """Writes out_dir/{plain,overlap}.json: torch.profiler traces of one backward without and with head_ready_event."""
  from torch.profiler import ProfilerActivity, profile
  step = _vtrace_step(net, conv_mode, False)
  step.compute_gradients(_vtrace_batch(7))
  r = step.agent._loss_grads
  torch.cuda.synchronize()
  ev = torch.cuda.Event()
  for name, kw in (('plain', {}), ('overlap', {'head_ready_event': ev})):
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
      step.agent.backward(r['dlogits'], r['dbaseline'], **kw)
      torch.cuda.synchronize()
    prof.export_chrome_trace(os.path.join(out_dir, '%s.json' % name))


@pytest.mark.parametrize('net,conv_mode', [('deep', 'tc3p'), ('shallow', 'tc3')])
def test_head_event_follows_every_bucket_1_launch(tmp_path, net, conv_mode):
  """In the host's call order, the library's cudaEventRecord (the second record of backward(head_ready_event=...),
  after networks.py's own) comes after the LSTM's BPTT and the Dense bias colsum, the last launches that write
  below grad_split, and right before the dflat GEMM, the first launch of the conv torso's backward.  The launch
  sequence is the plain backward's.  The profiling runs in a child process of its own, so this session's
  profiler state cannot reach the other tests of the suite, several of which read kernel names from
  torch.profiler."""
  code = ('import sys; sys.path[:0] = %r; import test_gpu_gradient_exchange as t; t._profile_backward(%r, %r, %r)'
          % ([ROOT, HERE], net, conv_mode, str(tmp_path)))
  p = subprocess.run([sys.executable, '-c', code], capture_output=True, text=True, timeout=300)
  assert p.returncode == 0, p.stdout[-2000:] + p.stderr[-4000:]
  plain, over = (_trace_launches(str(tmp_path / ('%s.json' % name))) for name in ('plain', 'overlap'))
  assert [x for x in over if x[0] == 'launch'] == [x for x in plain if x[0] == 'launch']
  start = [i for i, x in enumerate(over) if x[0] == 'memset']
  assert start, 'no cudaMemsetAsync of the gradient arena in the trace: %s' % over[:20]
  body = over[start[0]:]
  records = [i for i, x in enumerate(body) if x[0] == 'record']
  assert len(records) == 1, body
  k = records[0]
  before, after = [x[1].lower() for x in body[:k] if x[0] == 'launch'], [x[1].lower() for x in body[k:] if x[0] == 'launch']
  assert 'colsum' in before[-1], 'the last launch before the head event is %s, not the Dense bias colsum' % before[-1]
  assert 'gemm' in after[0], 'the first launch after the head event is %s, not the dflat GEMM' % after[0]
  assert any('lstm' in x for x in before) and not any('lstm' in x for x in after)
  assert sum('colsum' in x for x in before) >= 4      # policy and baseline biases, LSTM bias, Dense bias


def test_r2d2_replicas_clip_then_sum(monkeypatch):
  """R2D2LearnerStep with world = 2: each replica clips its gradient to global norm 40 on its own, then the SUM
  all-reduce, then Adam (scale 1, no clamp): parameters, m and v equal Adam(clip(g_A) + clip(g_B))."""
  from oracle import r2d2_learner_oracle as RL
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils
  ls = learner.default_settings()
  Tr, Br, S, obs = ls.burn_in + ls.unroll_length + 1, 64, 4, (84, 84, 1)
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()

  def sampled(seed):
    b = RL.synthetic_replay_batch(Tr, Br, A, obs, seed=seed, done_p=0.01)
    env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']), torch.zeros(Tr, Br, dtype=torch.bool).cuda(),
                          torch.zeros(Tr, Br, dtype=torch.int32).cuda())
    state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
    unrolls = learner.Unroll(state, None, c(b['prev_actions']), env, learner.AgentOutput(c(b['action']), None))
    return learner.SampledUnrolls(unrolls, c(b['indices']), c(b['importance_weights']))

  def make():
    agent, target = networks.DuelingLSTMDQNNet(A, obs, S, seed=5), networks.DuelingLSTMDQNNet(A, obs, S, seed=6)
    return learner.R2D2LearnerStep(agent, target, optimizers.Adam(4.8e-4, epsilon=1e-3), settings=ls)

  sa, sb = sampled(21), sampled(22)
  grads, norms = [], []
  for s in (sa, sb):
    step = make()
    step.update_target_agent()
    _, _, _, norm = step.compute_gradients(s)
    torch.cuda.synchronize()
    grads.append(step.agent.grads.clone())
    norms.append(float(norm))
    assert float(torch.linalg.vector_norm(step.agent.grads.double())) <= ls.clip_norm * (1 + 1e-5)
    if norms[-1] > ls.clip_norm:       # the clip bound: the arena now has norm 40
      assert abs(float(torch.linalg.vector_norm(step.agent.grads.double())) - ls.clip_norm) <= 1e-4 * ls.clip_norm
  ref = make()
  p0 = ref.agent.params.clone()
  ref.optimizer.apply_gradients(ref.agent.params, grads[0] + grads[1])
  torch.cuda.synchronize()
  ex = _Exchange([grads[1]])
  with monkeypatch.context() as mp:
    ex.install(mp)
    step = make()
    assert step.world == WORLD
    ex.grads = step.agent.grads
    step.minimize(sa)
  torch.cuda.synchronize()
  assert ex.calls == [('grads', 0, step.agent.grads.numel(), False)]
  for got, exp, nm in ((step.agent.params, ref.agent.params, 'params'), (step.optimizer.m, ref.optimizer.m, 'm'),
                       (step.optimizer.v, ref.optimizer.v, 'v')):
    np.testing.assert_array_equal(_bits(got), _bits(exp), err_msg=nm)
  assert (_bits(ref.agent.params) != _bits(p0)).mean() > 0.5
