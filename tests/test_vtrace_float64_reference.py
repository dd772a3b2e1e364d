"""CPU: tests/vtrace_float64_reference.py, the V-trace learner step in float32 / float64 that can be conditioned on
another implementation's ReLU masks and max-pool taps (tests/test_gpu_vtrace_float64.py holds the GPU step to it).

  * in float32 with its own decisions it is oracle/learner_oracle.py's step: logits, baseline, loss and logged
    terms, d loss / d outputs, every gradient and the parameters after one Adam step, for both nets;
  * conditioning on its own decisions changes nothing, bit for bit (the pool's backward is F.max_pool2d's kernel,
    so overlapping windows sum in the same order); a flipped mask or tap at frame (t, b) changes only the rows of
    column b from t up to the next done-reset;
  * float64 and float32 agree to fp32 rounding where they make the same decisions;
  * its `forward` (central inference's T1-step forward) in float32 is oracle/net_oracle.py's unroll, final state
    included; K chained one-step calls are one K-step call; conditioning on its own decisions changes nothing;
  * seedrl_debug_net_views names disjoint buffers of the sizes and formats the decisions need, inside the
    workspace, in every conv mode.
"""
import ctypes

import numpy as np
import pytest
import torch

import vtrace_float64_reference as RF
from oracle import learner_oracle, loss_oracle, net_oracle

A, OBS = 18, (84, 84, 4)
T, B = 5, 3
_cache = {}


def _problem(net):
  if net not in _cache:
    params = net_oracle.init_params(net, A, OBS, seed=1)
    b = learner_oracle.synthetic_batch(T, B, A, OBS, seed=1234)
    b['done'][:] = False
    b['done'][4, 1] = b['done'][2, 0] = b['done'][3, 2] = True      # a reset inside every column
    rng = np.random.default_rng(5)
    b['h0'] = rng.normal(size=b['h0'].shape).astype(np.float32)
    b['c0'] = rng.normal(size=b['c0'].shape).astype(np.float32)
    _cache[net] = (params, b, loss_oracle.default_config())
  return _cache[net]


def _run(net, dtype, **kw):
  params, b, cfg = _problem(net)
  key = (net, dtype)
  if not kw and key in _cache:
    return _cache[key]
  r = RF.step(net, params, b, cfg, dtype, **kw)
  if not kw:
    _cache[key] = r
  return r


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_float32_reference_is_the_oracle_step(net):
  params, b, cfg = _problem(net)
  cpu = learner_oracle.CpuLearner(net, A, OBS, cfg, params=params)
  total, logs, g, aux = cpu.grads(b)
  r = _run(net, torch.float32)
  np.testing.assert_array_equal(r['logits'], aux['logits'].detach().numpy())
  np.testing.assert_array_equal(r['baseline'], aux['baseline'].detach().numpy())
  assert r['total'] == float(total)
  assert list(r['logs']) == [k for k in logs if k != 'policy/max_action_abs(before_tanh)']
  for k, v in r['logs'].items():
    assert v == float(logs[k].detach()), k
  _, _, dl, db, dep, _ = loss_oracle.loss_and_grads(cfg, r['logits'], r['baseline'], b['behaviour_logits'],
                                                    b['action'], b['reward'], b['done'])
  np.testing.assert_array_equal(r['dlogits'], dl)
  np.testing.assert_array_equal(r['dbaseline'], db)
  assert list(r['grads']) == list(g) and len(g) == (40 if net == 'deep' else 14)
  for k in g:
    np.testing.assert_array_equal(r['grads'][k], g[k], err_msg=k)
  assert float(r['grads']['entropy_cost_param']) == dep == 0.0
  cpu.step(b)
  after = dict((k, v.detach().numpy()) for k, v in cpu.params.items())
  after['entropy_cost_param'] = cpu.entropy_cost_param.detach().numpy()
  for k, v in after.items():
    np.testing.assert_array_equal(r['params_after'][k], v, err_msg=k)
  # the recorded decisions, rows = the T+1 * B frames time-major
  N = (T + 1) * B
  if net == 'deep':
    shapes = {}
    for s, (hw, c) in enumerate(((42, 16), (21, 32), (11, 32))):
      shapes.update({'stack%d/%s' % (s, k): (N, hw, hw, c) for k in ('p', 'c0', 'o0', 'c1')})
      assert r['taps']['stack%d/pool' % s].shape == (N, hw, hw, c) and r['taps']['stack%d/pool' % s].max() <= 8
    shapes.update(o1=(N, 11, 11, 32), dense=(N, 256))
  else:
    shapes = dict(conv0=(N, 20, 20, 16), conv1=(N, 9, 9, 32), dense=(N, 256))
  assert {k: v.shape for k, v in r['masks'].items()} == shapes
  assert {k: v.shape for k, v in r['acts'].items()} == shapes
  for k in shapes:
    np.testing.assert_array_equal(r['masks'][k], r['acts'][k] > 0, err_msg=k)
  assert set(r['masks']) == set(RF.MASKS[net]) and set(r['taps']) == set(RF.POOLS[net])


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_conditioning_on_its_own_decisions_changes_nothing(net, dtype):
  r0 = _run(net, dtype)
  r1 = _run(net, dtype, masks=r0['masks'], taps=r0['taps'])
  for k in ('logits', 'baseline', 'dlogits', 'dbaseline'):
    np.testing.assert_array_equal(r1[k], r0[k], err_msg=k)
  assert r1['total'] == r0['total'] and r1['logs'] == r0['logs']
  for k in r0['grads']:
    np.testing.assert_array_equal(r1['grads'][k], r0['grads'][k], err_msg=k)
    np.testing.assert_array_equal(r1['params_after'][k], r0['params_after'][k], err_msg=k)
    np.testing.assert_array_equal(r1['update'][k], r0['update'][k], err_msg=k)
  for k in r0['acts']:
    np.testing.assert_array_equal(r1['acts'][k], r0['acts'][k], err_msg=k)
  # shared decisions that agree with its own are no near-ties to report
  assert all(v.size == 0 for v in r1['ties'].values()) and set(r1['ties']) == set(RF.MASKS[net] + RF.POOLS[net])


@pytest.mark.parametrize('net,name', [('deep', k) for k in RF.MASKS['deep'] + RF.POOLS['deep']] +
                         [('shallow', k) for k in RF.MASKS['shallow']])
def test_a_flipped_decision_changes_only_the_rows_that_depend_on_it(net, name):
  """One active ReLU unit switched off, or one pool tap moved inside its window, at frame (t, b): logits and
  baseline change at (t, b) and after it in column b until the next done-reset; the other columns, the earlier
  frames and the frames after the reset are unchanged, and so are d loss / d outputs of the other columns."""
  _, bt, _ = _problem(net)
  r0 = _run(net, torch.float64)
  t, b = 1, 1
  n = t * B + b
  masks = {k: v.copy() for k, v in r0['masks'].items()}
  taps = {k: v.copy() for k, v in r0['taps'].items()}
  if name in masks:
    row = masks[name][n].reshape(-1)
    on = np.flatnonzero(row)
    row[on[len(on) // 2]] = False
  else:
    tap = taps[name][n]
    c = tap.shape[0] // 2
    tap[c, c, :] = (tap[c, c, :] + 4) % 9          # a central window lies inside the image
  r1 = _run(net, torch.float64, masks=masks, taps=taps)
  assert r1['ties'][name].size == (1 if name in masks else taps[name].shape[-1])
  changed = np.any(r1['logits'] != r0['logits'], axis=-1) | (r1['baseline'] != r0['baseline'])
  reset = t + 1 + int(np.flatnonzero(bt['done'][t + 1:, b])[0])
  expect = np.zeros_like(changed)
  expect[t:reset, b] = True
  assert changed[t, b] and changed[t + 1, b]
  np.testing.assert_array_equal(changed & ~expect, False)
  for k in ('dlogits', 'dbaseline'):
    np.testing.assert_array_equal(np.delete(r1[k], b, axis=1), np.delete(r0[k], b, axis=1), err_msg=k)
  assert r1['total'] != r0['total']


def _inputs(b, t0=0, t1=None, h0=None, c0=None):
  """forward's inputs: rows t0..t1-1 of the batch, from state (h0, c0) (default the batch's)."""
  keys = ('prev_actions', 'reward', 'done', 'observation')
  return dict({k: b[k][t0:t1] for k in keys}, h0=b['h0'] if h0 is None else h0, c0=b['c0'] if c0 is None else c0)


@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_float32_forward_is_the_oracle_unroll(net):
  params, b, _ = _problem(net)
  logits, baseline, (h, c) = net_oracle.unroll(
      net, net_oracle.to_torch(params), torch.as_tensor(b['prev_actions']), torch.as_tensor(b['reward']),
      torch.as_tensor(b['done']), torch.as_tensor(b['observation']), (torch.as_tensor(b['h0']),
                                                                     torch.as_tensor(b['c0'])), A)
  r = RF.forward(net, params, _inputs(b), torch.float32)
  for k, v in (('logits', logits), ('baseline', baseline), ('h', h), ('c', c)):
    np.testing.assert_array_equal(r[k], v.detach().numpy(), err_msg=k)
  # the step's forward is this one
  np.testing.assert_array_equal(r['logits'], _run(net, torch.float32)['logits'])


@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_chained_one_step_forwards_are_one_unroll(net):
  """T+1 calls of one step, each from the state the previous one returned, across the done-resets of every
  column (rows 2, 3 and 4), equal one (T+1)-step call in float64; so do two calls of 2 and T-1 steps."""
  params, b, _ = _problem(net)
  whole = RF.forward(net, params, _inputs(b), torch.float64)
  for cuts in ([(t, t + 1) for t in range(T + 1)], [(0, 2), (2, T + 1)]):
    h, c, logits, baseline = b['h0'], b['c0'], [], []
    for t0, t1 in cuts:
      r = RF.forward(net, params, _inputs(b, t0, t1, h, c), torch.float64)
      h, c = r['h'], r['c']
      logits.append(r['logits']); baseline.append(r['baseline'])
    errs = {'logits': _relmax(np.concatenate(logits), whole['logits']),
            'baseline': _relmax(np.concatenate(baseline), whole['baseline']),
            'h': _relmax(h, whole['h']), 'c': _relmax(c, whole['c'])}
    assert max(errs.values()) < 1e-12, (cuts, errs)


@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_forward_conditioned_on_its_own_decisions_changes_nothing(net):
  params, b, _ = _problem(net)
  r0 = RF.forward(net, params, _inputs(b, 2, 3), torch.float64)
  r1 = RF.forward(net, params, _inputs(b, 2, 3), torch.float64, masks=r0['masks'], taps=r0['taps'])
  for k in ('logits', 'baseline', 'h', 'c'):
    np.testing.assert_array_equal(r1[k], r0[k], err_msg=k)
  for k in r0['acts']:
    np.testing.assert_array_equal(r1['acts'][k], r0['acts'][k], err_msg=k)
  assert all(v.size == 0 for v in r1['ties'].values()) and set(r1['ties']) == set(RF.MASKS[net] + RF.POOLS[net])
  assert r0['masks']['dense'].shape == (B, 256)


def test_a_tap_outside_the_image_is_an_error():
  params, b, cfg = _problem('deep')
  r0 = _run('deep', torch.float64)
  taps = {k: v.copy() for k, v in r0['taps'].items()}
  taps['stack2/pool'][0, 0, 0, 0] = 0              # 21 -> 11 pads one row above: window (0, 0) starts outside
  with pytest.raises(ValueError, match='outside the image'):
    RF.step('deep', params, b, cfg, torch.float64, masks=r0['masks'], taps=taps)


@pytest.mark.parametrize('net', ['deep', 'shallow'])
def test_float64_and_float32_agree_to_fp32_rounding(net):
  """Under the float64 step's decisions.  Where float32 on its own would decide otherwise, the unit or window is
  within fp32 rounding of its tie (the deep net has one such pool window at this shape)."""
  r64 = _run(net, torch.float64)
  r32 = _run(net, torch.float32, masks=r64['masks'], taps=r64['taps'])
  for k, v in r32['ties'].items():
    scale = np.abs(r64['acts'][k if k in r64['acts'] else k.replace('pool', 'p')]).max()
    assert v.size <= 2 and (v.size == 0 or v.max() < 1e-6 * scale), (k, v, scale)
  errs = {k: _relmax(r32[k], r64[k]) for k in ('logits', 'baseline', 'dlogits', 'dbaseline')}
  errs['total'] = abs(r32['total'] - r64['total']) / abs(r64['total'])
  errs.update({'act ' + k: _relmax(r32['acts'][k], r64['acts'][k]) for k in r64['acts']})
  errs.update({'grad ' + k: _relmax(r32['grads'][k], r64['grads'][k]) for k in r64['grads']
               if k != 'entropy_cost_param'})
  worst = max(errs, key=errs.get)
  print('float32 vs float64 (%s): worst %s %.2e' % (net, worst, errs[worst]))
  assert errs['logits'] < 2e-6 and errs['baseline'] < 2e-6, errs
  assert max(v for k, v in errs.items() if k.startswith('act ')) < 2e-6, errs
  assert errs[worst] < 1e-4, errs


# the shapes and settings of test_gpu_parity.py::test_vtrace_loss_fwd_bwd_vs_oracle
_LOSS_CASES = [(21, 64, 18, {}),
               (21, 64, 18, dict(kl_cost=0.3, entropy_cost=0.01, max_abs_reward=1.0, target_entropy=1.5, lambda_=0.9)),
               (2, 1, 1, {}), (6, 3, 5, dict(kl_cost=0.1)), (21, 70, 18, {}), (101, 33, 9, {}), (4, 257, 2, {})]


def _loss_inputs(T1, B, A, kw, seed=11):
  from test_gpu_parity import _loss_case
  c, _ = _loss_case(T1, B, A, seed)
  cfg = loss_oracle.default_config(**kw)
  ecp = np.float32(np.log(cfg.entropy_cost) / cfg.entropy_cost_adjustment_speed)
  return cfg, [c[k] for k in ('ll', 'lb', 'bl', 'act', 'rew', 'done')], ecp


@pytest.mark.parametrize('T1,B,A,kw', _LOSS_CASES)
def test_float32_loss_and_grads_is_the_oracle(T1, B, A, kw):
  """The loss-only reference in float32 is oracle/loss_oracle.loss_and_grads bit for bit: loss, the 11 logged
  terms, d loss / d logits and d baseline, d loss / d entropy_cost_param, vs and the pg advantages."""
  cfg, args, ecp = _loss_inputs(T1, B, A, kw)
  total, logs, dl, db, dep, aux = loss_oracle.loss_and_grads(cfg, *args)
  r = RF.loss_and_grads(cfg, *args, ecp, torch.float32)
  assert r[0] == float(total)
  assert list(r[1]) == list(logs) and len(logs) == 11
  for k, v in logs.items():
    assert r[1][k] == v, k
  np.testing.assert_array_equal(r[2], dl)
  np.testing.assert_array_equal(r[3], db)
  assert r[4] == dep
  np.testing.assert_array_equal(r[5], aux['vs'].numpy())
  np.testing.assert_array_equal(r[6], aux['pg_advantages'].numpy())
  assert r[2].dtype == r[3].dtype == r[5].dtype == np.float32
  if kw.get('target_entropy'):
    assert dep != 0.0


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_loss_and_grads_in_column_chunks_is_one_evaluation(dtype):
  """Column chunks of 16 and of 48 (a ragged last chunk) give the one-chunk result: vs and the pg advantages bit for
  bit, the gradients and the loss terms to the rounding of the means' divisors and of the float64 recombination."""
  kw = dict(kl_cost=0.3, entropy_cost=0.01, max_abs_reward=1.0, target_entropy=1.5, lambda_=0.9)
  cfg, args, ecp = _loss_inputs(21, 64, 18, kw)
  whole = RF.loss_and_grads(cfg, *args, ecp, dtype)
  tol = 1e-14 if dtype == torch.float64 else 1e-5
  for chunk in (16, 48):
    part = RF.loss_and_grads(cfg, *args, ecp, dtype, chunk=chunk)
    for i in (5, 6):
      np.testing.assert_array_equal(part[i], whole[i])
    for i in (2, 3):
      assert _relmax(part[i], whole[i]) < tol, (chunk, i, _relmax(part[i], whole[i]))
    assert abs(part[0] - whole[0]) <= tol * abs(whole[0])
    assert abs(part[4] - whole[4]) <= tol * abs(whole[4])
    assert list(part[1]) == list(whole[1])
    for k in whole[1]:
      assert abs(part[1][k] - whole[1][k]) <= tol * abs(whole[1][k]) + 1e-300, (chunk, k)


def _views(net, mode):
  """{index: (offset, bytes, format)} of seedrl_debug_net_views for a (21, 64) call, and the workspace size."""
  from seed_rl_b200 import _lib
  L = _lib.lib()
  h = ctypes.c_void_p()
  cfg = _lib.NetConfig(_lib.NET_DEEP if net == 'deep' else _lib.NET_SHALLOW, A, *OBS)
  _lib.check(L.seedrl_net_create(ctypes.byref(cfg), ctypes.byref(h)))
  try:
    _lib.check(L.seedrl_net_set_conv_mode(h, {'simt': 0, 'tc3': 2, 'tc3p': 3}[mode]))
    T1, Bw = 21, 64
    total = L.seedrl_net_workspace_bytes(h, T1, Bw)
    out = {}
    off, nb, fmt = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int()
    last = 16 if net == 'deep' else 2
    for i in range(last + 1):
      _lib.check(L.seedrl_debug_net_views(h, T1, Bw, i, ctypes.byref(off), ctypes.byref(nb), ctypes.byref(fmt)))
      out[i] = (off.value, nb.value, fmt.value)
    for bad in (-1, last + 1):
      assert L.seedrl_debug_net_views(h, T1, Bw, bad, ctypes.byref(off), ctypes.byref(nb), ctypes.byref(fmt)) == 3
    assert L.seedrl_debug_net_views(h, 0, Bw, 0, ctypes.byref(off), ctypes.byref(nb), ctypes.byref(fmt)) == 3
    assert L.seedrl_debug_net_views(h, T1, 0, 0, ctypes.byref(off), ctypes.byref(nb), ctypes.byref(fmt)) == 3
    return out, total, T1 * Bw
  finally:
    L.seedrl_net_destroy(h)


@pytest.mark.parametrize('net,mode', [('deep', 'simt'), ('deep', 'tc3'), ('deep', 'tc3p'), ('shallow', 'simt'),
                                      ('shallow', 'tc3')])
def test_debug_views_are_disjoint_buffers_of_the_decision_sizes(net, mode):
  from seed_rl_b200 import _lib
  views, total, N = _views(net, mode)
  want = {}
  if net == 'deep':
    for s, (hw, c) in enumerate(((42, 16), (21, 32), (11, 32))):
      for j in range(4):
        want[5 * s + j] = ((int(_lib.lib().seedrl_debug_planes_bytes(N, hw, hw, c)), 1) if mode == 'tc3p' else
                           (4 * N * hw * hw * c, 0))
      want[5 * s + 4] = (N * hw * hw * c, 2)
    want[15] = (4 * N * 11 * 11 * 32, 0)
  else:
    want[0] = (4 * N * 20 * 20 * 16, 0)
    want[1] = (4 * N * 9 * 9 * 32, 0)
  want[max(want) + 1] = (4 * N * (256 + 1 + A), 0)
  assert {i: v[1:] for i, v in views.items()} == want
  spans = sorted((o, o + nb) for o, nb, _ in views.values())
  assert all(o % 256 == 0 and e <= total for o, e in spans)
  assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
