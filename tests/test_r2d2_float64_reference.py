"""CPU: tests/r2d2_float64_reference.py, the R2D2 learner step in float32 / float64 that can be conditioned on
another implementation's ReLU masks and greedy actions (tests/test_gpu_r2d2_float64.py holds the GPU step to it).

  * in float32 with its own decisions it is oracle/r2d2_learner_oracle.py's step: q, loss, priorities, norm, every
    gradient and the parameters after one Adam step;
  * conditioning on its own decisions changes nothing, bit for bit; a flipped mask or greedy action changes only
    the rows that depend on it;
  * float64 and float32 agree to fp32 rounding where they make the same decisions;
  * its `forward` (central inference's T-step forward) in float32 is oracle/r2d2_net_oracle.py's unroll, final
    state included; K chained one-step calls are one K-step call; conditioning on its own masks changes nothing;
    `priorities` restates the step's;
  * seedrl_debug_r2d2_net_views names disjoint buffers of the sizes the masks need, inside the workspace.
"""
import ctypes

import numpy as np
import pytest
import torch

import r2d2_float64_reference as RF
from oracle import r2d2_learner_oracle as RL, r2d2_net_oracle as NO

A, OBS, S = 18, (84, 84, 1), 4
T, B, BURN_IN = 12, 3, 4
LR, ADAM_EPS = 0.00048, 1e-3
_cache = {}


def _settings():
  from seed_rl_b200.agents.r2d2 import learner
  return learner.default_settings(burn_in=BURN_IN)


def _problem():
  if 'problem' not in _cache:
    params = NO.init_params(A, OBS, S, seed=5)
    tparams = NO.init_params(A, OBS, S, seed=6)
    b = RL.synthetic_replay_batch(T, B, A, OBS, seed=21, done_p=0.15)
    _cache['problem'] = (params, tparams, b, RF.settings(A, S, _settings(), LR, ADAM_EPS))
  return _cache['problem']


def _run(dtype, **kw):
  params, tparams, b, st = _problem()
  return RF.step(params, tparams, b, st, dtype, **kw)


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def test_float32_reference_is_the_oracle_step():
  params, tparams, b, st = _problem()
  ls = _settings()
  assert b['done'][BURN_IN:].any() and b['done'][:BURN_IN].any()
  cpu = RL.CpuR2D2Learner(A, OBS, S, gamma=ls.discounting, burn_in=BURN_IN, n_steps=ls.n_steps,
                          clip_norm=ls.clip_norm, lr=LR, eps=ADAM_EPS, params=params, target_params=tparams)
  total, loss, prio, g, norm, aux = cpu.grads(b)
  r = _run(torch.float32)
  np.testing.assert_array_equal(r['q'], aux['q'].detach().numpy())
  np.testing.assert_array_equal(r['target_q'], aux['target_q'].numpy())
  assert r['total'] == total and r['norm'] == norm
  np.testing.assert_array_equal(r['loss_b'], loss)
  np.testing.assert_array_equal(r['priorities'], prio)
  assert list(r['grads']) == list(g)
  for k in g:
    np.testing.assert_array_equal(r['grads'][k], g[k], err_msg=k)
  cpu.step(b)
  for k, v in cpu.params.items():
    np.testing.assert_array_equal(r['params_after'][k], v.detach().numpy(), err_msg=k)
  assert r['scale'] < 1 or norm <= ls.clip_norm
  # the recorded decisions are the suffix unroll's, rows time-major
  N = (T - BURN_IN) * B
  shapes = dict(conv0=(N, 20, 20, 32), conv1=(N, 9, 9, 64), conv2=(N, 7, 7, 64), dense=(N, 512), value=(N, 512),
                advantage=(N, 512))
  assert {k: v.shape for k, v in r['masks'].items()} == shapes
  np.testing.assert_array_equal(r['greedy'], r['q'].argmax(-1))


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_conditioning_on_its_own_decisions_changes_nothing(dtype):
  r0 = _run(dtype)
  r1 = _run(dtype, masks=r0['masks'], greedy=r0['greedy'])
  for k in ('q', 'target_q', 'dq', 'loss_b', 'priorities'):
    np.testing.assert_array_equal(r1[k], r0[k], err_msg=k)
  assert (r1['total'], r1['norm'], r1['scale']) == (r0['total'], r0['norm'], r0['scale'])
  for k in r0['grads']:
    np.testing.assert_array_equal(r1['grads'][k], r0['grads'][k], err_msg=k)
    np.testing.assert_array_equal(r1['params_after'][k], r0['params_after'][k], err_msg=k)


@pytest.mark.parametrize('layer', RF.MASKS)
def test_a_flipped_mask_changes_only_the_rows_that_depend_on_it(layer):
  """One active unit switched off at frame (t, b): q changes at (t, b); the other batch columns and the earlier
  frames of column b are unchanged (the LSTM is causal), and so are the later frames for a head layer."""
  r0 = _run(torch.float64)
  t, b = 5, 1
  n = t * B + b
  masks = {k: v.copy() for k, v in r0['masks'].items()}
  row = masks[layer][n].reshape(-1)
  j = int(np.flatnonzero(row)[len(np.flatnonzero(row)) // 2])
  row[j] = False
  r1 = _run(torch.float64, masks=masks, greedy=r0['greedy'])
  changed = np.any(r1['q'] != r0['q'], axis=-1)
  expect = np.zeros_like(changed)
  if layer in ('value', 'advantage'):
    expect[t, b] = True
  else:
    expect[t:, b] = True
  assert changed[t, b]
  np.testing.assert_array_equal(changed & ~expect, False)
  np.testing.assert_array_equal(np.delete(r1['loss_b'], b), np.delete(r0['loss_b'], b))
  np.testing.assert_array_equal(np.delete(r1['priorities'], b), np.delete(r0['priorities'], b))
  assert r1['loss_b'][b] != r0['loss_b'][b]
  assert not np.array_equal(r1['grads']['body/conv0/kernel'], r0['grads']['body/conv0/kernel'])


def test_a_flipped_greedy_action_changes_only_its_column_target():
  r0 = _run(torch.float64)
  t, b = 6, 2
  greedy = r0['greedy'].copy()
  greedy[t, b] = (greedy[t, b] + 1) % A
  r1 = _run(torch.float64, masks=r0['masks'], greedy=greedy)
  np.testing.assert_array_equal(r1['q'], r0['q'])
  np.testing.assert_array_equal(np.delete(r1['loss_b'], b), np.delete(r0['loss_b'], b))
  assert r1['loss_b'][b] != r0['loss_b'][b]
  # the target value at row t enters the n-step targets of rows t - n_steps .. t - 1 of column b only
  diff = np.any(r1['dq'] != r0['dq'], axis=-1)
  expect = np.zeros_like(diff)
  expect[max(0, t - _settings().n_steps):t, b] = True
  assert diff.any()
  np.testing.assert_array_equal(diff & ~expect, False)


def test_float64_and_float32_agree_to_fp32_rounding():
  r64 = _run(torch.float64)
  r32 = _run(torch.float32)
  # no near-ties at this shape: both make the same decisions
  for k in RF.MASKS:
    np.testing.assert_array_equal(r32['masks'][k], r64['masks'][k], err_msg=k)
  np.testing.assert_array_equal(r32['greedy'], r64['greedy'])
  errs = {k: _relmax(r32[k], r64[k]) for k in ('q', 'target_q', 'dq', 'loss_b', 'priorities')}
  errs['norm'] = abs(r32['norm'] - r64['norm']) / r64['norm']
  errs.update({'grad ' + k: _relmax(r32['grads'][k], r64['grads'][k]) for k in r64['grads']})
  worst = max(errs, key=errs.get)
  print('float32 vs float64: worst %s %.2e' % (worst, errs[worst]))
  # the forward to a few fp32 roundings; the TD errors cancel (target - q) and carry that into the rest
  assert errs['q'] < 2e-6 and errs['target_q'] < 2e-6, errs
  assert errs[worst] < 1e-4, errs


def _inputs(b, t0=0, t1=None, h0=None, c0=None, frame_state=None):
  """forward's inputs: rows t0..t1-1 of the batch, from the given state (default the batch's)."""
  keys = ('prev_actions', 'reward', 'done', 'observation')
  return dict({k: b[k][t0:t1] for k in keys}, h0=b['h0'] if h0 is None else h0, c0=b['c0'] if c0 is None else c0,
              frame_state=b['frame_state'] if frame_state is None else frame_state)


def test_float32_forward_is_the_oracle_unroll():
  params, _, b, _ = _problem()
  state = NO.AgentState((torch.as_tensor(b['h0']), torch.as_tensor(b['c0'])), b['frame_state'])
  out, new_state = NO.unroll({k: torch.as_tensor(v) for k, v in params.items()}, b['prev_actions'], b['reward'],
                             b['done'], b['observation'], state, A, S)
  r = RF.forward(params, _inputs(b), A, S, torch.float32)
  np.testing.assert_array_equal(r['q'], out.q_values.numpy())
  np.testing.assert_array_equal(r['h'], new_state.core_state[0].numpy())
  np.testing.assert_array_equal(r['c'], new_state.core_state[1].numpy())
  np.testing.assert_array_equal(r['frame_state'], new_state.frame_stacking_state)
  np.testing.assert_array_equal(r['q'].argmax(-1), out.action.numpy())


def test_chained_one_step_forwards_are_one_unroll():
  """T calls of one step, each from the state (h, c and the frame-stacking state) the previous one returned,
  across the batch's done-resets, equal one T-step call in float64; so do two calls of 4 and T-4 steps."""
  params, _, b, _ = _problem()
  assert b['done'].any(axis=0).sum() >= 2
  whole = RF.forward(params, _inputs(b), A, S, torch.float64)
  for cuts in ([(t, t + 1) for t in range(T)], [(0, 4), (4, T)]):
    h, c, fs, q = b['h0'], b['c0'], b['frame_state'], []
    for t0, t1 in cuts:
      r = RF.forward(params, _inputs(b, t0, t1, h, c, fs), A, S, torch.float64)
      h, c, fs = r['h'], r['c'], r['frame_state']
      q.append(r['q'])
    errs = {'q': _relmax(np.concatenate(q), whole['q']), 'h': _relmax(h, whole['h']), 'c': _relmax(c, whole['c'])}
    assert max(errs.values()) < 1e-12, (cuts, errs)
    np.testing.assert_array_equal(fs, whole['frame_state'])


def test_forward_conditioned_on_its_own_masks_changes_nothing():
  params, _, b, _ = _problem()
  r0 = RF.forward(params, _inputs(b, 5, 6), A, S, torch.float64)
  r1 = RF.forward(params, _inputs(b, 5, 6), A, S, torch.float64, masks=r0['masks'])
  for k in ('q', 'h', 'c', 'frame_state'):
    np.testing.assert_array_equal(r1[k], r0[k], err_msg=k)
  for k in RF.MASKS:
    np.testing.assert_array_equal(r1['acts'][k], r0['acts'][k], err_msg=k)
    np.testing.assert_array_equal(r0['masks'][k], r0['acts'][k] > 0, err_msg=k)
  assert set(r1['ties']) == set(RF.MASKS) and all(v.size == 0 for v in r1['ties'].values())
  assert r0['masks']['dense'].shape == (B, 512)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_priorities_restate_the_step(dtype):
  _, _, b, st = _problem()
  r = _run(dtype)
  F = np.float64 if dtype == torch.float64 else np.float32
  got = RF.priorities(r['q'], r['target_q'], b['action'][BURN_IN:], b['reward'][BURN_IN:], b['done'][BURN_IN:],
                      r['greedy'], st, F)
  np.testing.assert_array_equal(got, r['priorities'])


def test_debug_views_are_disjoint_buffers_of_the_mask_sizes():
  from seed_rl_b200 import _lib
  L = _lib.lib()
  h = ctypes.c_void_p()
  _lib.check(L.seedrl_r2d2_net_create(A, OBS[0], OBS[1], S, ctypes.byref(h)))
  try:
    Tw, Bw = 101, 64
    N = Tw * Bw
    total = L.seedrl_r2d2_net_workspace_bytes(h, Tw, Bw)
    floats = [N * 20 * 20 * 32, N * 9 * 9 * 64, N * 7 * 7 * 64, N * (512 + 1 + A), N * 512, N * 512]
    spans = []
    for i, nf in enumerate(floats):
      off, nb = ctypes.c_size_t(), ctypes.c_size_t()
      _lib.check(L.seedrl_debug_r2d2_net_views(h, Tw, Bw, i, ctypes.byref(off), ctypes.byref(nb)))
      assert nb.value == 4 * nf and off.value % 256 == 0 and off.value + nb.value <= total, i
      spans.append((off.value, off.value + nb.value))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))
    off, nb = ctypes.c_size_t(), ctypes.c_size_t()
    assert L.seedrl_debug_r2d2_net_views(h, Tw, Bw, 6, ctypes.byref(off), ctypes.byref(nb)) == 3
    assert L.seedrl_debug_r2d2_net_views(h, 0, Bw, 0, ctypes.byref(off), ctypes.byref(nb)) == 3
  finally:
    L.seedrl_r2d2_net_destroy(h)
