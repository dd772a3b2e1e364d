"""CPU: multi-task PopArt (--popart_tasks).  The per-task composition of tests/popart_tasks_reference.py against
the unmodified reference modules run once per task on that task's columns (tests/golden/popart_tasks_golden.npz),
its reduction to tests/popart_reference.py at one task, the flag and settings defaults and validation, the
checkpoint check on the task count, and the column tasks the batch assembler records."""
import os

import numpy as np
import pytest
import torch

import abandoned_float64_reference as AR
import popart_reference as PR
import popart_tasks_reference as PT
from seed_rl_b200.agents.vtrace import learner
from seed_rl_b200.common import utils
from seed_rl_b200.dmlab import networks

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'popart_tasks_golden.npz')


def _close(name, x, ref, rtol):
  x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
  err = np.abs(x - ref).max() / max(np.abs(ref).max(), 1e-30)
  assert err <= rtol, '%s: %.3g > %.3g' % (name, err, rtol)


def _steps(d):
  k = 0
  while '%d_ll' % k in d:
    p = '%d_' % k
    yield p, tuple(d[p + x] for x in ('ll', 'lb', 'bl', 'act', 'rew', 'done')), d[p + 'task_ids']
    k += 1


@pytest.mark.parametrize('FT', [np.float32, np.float64])
def test_task_composition_against_golden(FT):
  """K reference PopArt modules, each fed its own task's columns, step by step from the state they held; the
  third step has no column of task 2, whose state must not move."""
  d = np.load(GOLDEN)
  discounting, lambda_, baseline_cost = (float(x) for x in d['cfg'])
  cfg = learner.default_loss_settings(popart=True, popart_tasks=int(d['K']), discounting=discounting,
                                      lambda_=lambda_, baseline_cost=baseline_cost)
  beta = float(d['beta'])
  rtol = 2e-5 if FT == np.float32 else 1e-4
  np.testing.assert_array_equal(d['0_state_before'], [[0, 1, 1, 0]] * int(d['K']))
  steps = 0
  for pre, batch, ids in _steps(d):
    r = PT.loss_and_grads(cfg, *batch, 0.0, d[pre + 'state_before'], ids, beta, FT)
    for key in ('vs', 'pg_adv', 'adv', 'e'):
      for k in range(int(d['K'])):   # each task on its own scale
        cols = ids == k
        if cols.any():
          _close(pre + key + str(k), r[key][:, cols], d[pre + key][:, cols], rtol)
    for k in range(int(d['K'])):
      _close(pre + 'state%d' % k, r['state'][k], d[pre + 'state_after'][k], rtol)
    _close(pre + 'policy', r['terms']['policy'], d[pre + 'policy_loss'], rtol)
    _close(pre + 'V', r['terms']['V'], d[pre + 'v_loss'], rtol)
    if not (ids == 2).any():
      np.testing.assert_array_equal(d[pre + 'state_after'][2], d[pre + 'state_before'][2])
      np.testing.assert_array_equal(r['state'][2], np.asarray(d[pre + 'state_before'][2], FT))
      assert np.all(r['dcomp'][2] == 0)
    steps += 1
  assert steps >= 4


def _batch(rng, T1=9, B=10, A=5, scale=300.0):
  return (rng.normal(size=(T1, B, A)).astype(np.float32), (rng.normal(size=(T1, B)) * 2).astype(np.float32),
          rng.normal(size=(T1, B, A)).astype(np.float32), rng.integers(0, A, (T1, B)),
          (rng.normal(size=(T1, B)) * scale).astype(np.float32), rng.random((T1, B)) < 0.1)


@pytest.mark.parametrize('FT', [np.float32, np.float64])
def test_one_task_is_the_single_task_composition(FT):
  rng = np.random.default_rng(5)
  batch = _batch(rng)
  cfg = learner.default_loss_settings(popart=True)
  state = np.array([3.0, 40.0, 1.2, -0.1], FT)
  ref = PR.loss_and_grads(cfg, *batch, -7.0, state, 0.05, FT)
  r = PT.loss_and_grads(cfg, *batch, -7.0, state[None], np.zeros(10, np.int32), 0.05, FT)
  for key in ('dlogits', 'dbaseline', 'vs', 'pg_adv', 'td'):
    np.testing.assert_array_equal(r[key], ref[key])
  np.testing.assert_array_equal(r['dcomp'][0], ref['dcomp'])
  np.testing.assert_array_equal(r['state'][0], ref['state'])
  for name in ('total', 'policy', 'V', 'entropy', 'kl', 'v_l2_error', 'v_mean', 'mean_entropy', 'mean_kl'):
    assert r['terms'][name] == ref['terms'][name], name


@pytest.mark.parametrize('FT', [np.float32, np.float64])
def test_one_task_with_a_mask_is_the_single_task_composition(FT):
  rng = np.random.default_rng(6)
  batch = _batch(rng)
  done, ab = AR.masks(9, 10, 7, p_done=0.0)
  batch = batch[:5] + (batch[5] | done,)
  cfg = learner.default_loss_settings(popart=True, lambda_=0.95)
  state = np.array([3.0, 40.0, 1.2, -0.1], FT)
  ref = PR.loss_and_grads(cfg, *batch, -7.0, state, 0.05, FT, abandoned=ab)
  r = PT.loss_and_grads(cfg, *batch, -7.0, state[None], np.zeros(10, np.int32), 0.05, FT, abandoned=ab)
  assert not np.array_equal(ref['vs'], PR.loss_and_grads(cfg, *batch, -7.0, state, 0.05, FT)['vs'])
  for key in ('dlogits', 'dbaseline', 'vs', 'pg_adv', 'td'):
    np.testing.assert_array_equal(r[key], ref[key])
  np.testing.assert_array_equal(r['dcomp'][0], ref['dcomp'])
  np.testing.assert_array_equal(r['state'][0], ref['state'])
  np.testing.assert_array_equal(r['sums'][0], ref['sums'])
  for name in ('total', 'policy', 'V', 'entropy', 'kl', 'v_l2_error', 'v_mean', 'mean_entropy', 'mean_kl'):
    assert r['terms'][name] == ref['terms'][name], name


def test_each_task_sees_its_own_columns_of_the_mask():
  """Two tasks with a mask: each task's outputs are the single-task composition on its columns of every input,
  the mask included; a task whose columns hold no abandoned transition is its unmasked composition."""
  rng = np.random.default_rng(8)
  batch = _batch(rng)
  ids = np.array([0, 0, 0, 1, 0, 1, 1, 1, 1, 1], np.int32)
  done, ab = AR.masks(9, 10, 9, p_done=0.0)
  ab[:, ids == 1] = False
  batch = batch[:5] + (batch[5] | done,)
  states = np.array([[3.0, 40.0, 1.2, -0.1], [30.0, 1000.0, 0.9, 0.2]])
  cfg = learner.default_loss_settings(popart=True, lambda_=0.95)
  r = PT.loss_and_grads(cfg, *batch, -7.0, states, ids, 0.05, abandoned=ab)
  for k, has_ab in ((0, True), (1, False)):
    cols = np.nonzero(ids == k)[0]
    sub = [np.ascontiguousarray(x[:, cols]) for x in batch + (ab,)]
    one = PR.loss_and_grads(cfg, *sub[:6], -7.0, states[k], 0.05, abandoned=sub[6] if has_ab else None)
    assert sub[6][1:].any() == has_ab
    for key in ('vs', 'pg_adv', 'td', 'e'):
      np.testing.assert_array_equal(r[key][:, cols], one[key], err_msg='%s %d' % (key, k))
    np.testing.assert_array_equal(r['state'][k], one['state'])
  masked = ab[1:]
  assert np.all(r['pg_adv'][masked] == 0)
  np.testing.assert_array_equal(r['vs'][masked], r['u'][:-1][masked])


def test_flag_and_settings_defaults():
  assert learner.default_loss_settings().popart_tasks == 1
  # positional construction of the eleven older fields is unaffected
  s = learner.LossSettings(.99, 1., .5, 2.5e-4, 0., 0., None, 10., True, 1e-2, False)
  assert s.popart_tasks == 1
  assert learner.FLAGS['popart_tasks'].default == 1
  learner.check_loss_settings(learner.default_loss_settings(popart=True, popart_tasks=64))
  learner.check_loss_settings(learner.default_loss_settings())


@pytest.mark.parametrize('kw', [dict(popart=True, popart_tasks=0), dict(popart=True, popart_tasks=65),
                                dict(popart=False, popart_tasks=2), dict(popart=True, popart_tasks=2.0)])
def test_settings_validation(kw):
  with pytest.raises(ValueError):
    learner.check_loss_settings(learner.default_loss_settings(**kw))


def test_checkpoint_task_count_mismatch_raises():
  one = {'popart_moments': torch.tensor([0.0, 1.0])}
  three = {'popart_moments': torch.tensor([[0.0, 1.0]] * 3)}
  networks.check_popart_state(one, True, 1)
  networks.check_popart_state(three, True, 3)
  networks.check_popart_state(three, True)            # no task count given: PopArt presence only
  with pytest.raises(ValueError, match='3 PopArt tasks'):
    networks.check_popart_state(three, True, 4)
  with pytest.raises(ValueError, match='1 PopArt tasks'):
    networks.check_popart_state(one, True, 30)
  with pytest.raises(ValueError, match='with PopArt'):
    networks.check_popart_state(three, False, None)


def test_assembler_records_env_id_mod_k():
  TS = utils.TensorSpec
  specs = (TS([], 'int64', 'a'),)
  state = (TS([5], 'float32', 'h'), TS([5], 'float32', 'c'))
  asm = utils.BatchAssembler(specs, state, full_length=4, batch_size=6, slots=2, device='cpu', num_tasks=4)
  placed = []
  for env_ids in ([13, 2, 7], [40, 9], [31, 6]):    # the last claim spills into the next slot
    start = 0
    while start < len(env_ids):
      slot, col0, n = asm.claim(len(env_ids) - start)
      ids = torch.tensor(env_ids[start:start + n], dtype=torch.int32)
      asm.place_task_ids(slot, col0, ids)
      asm.commit()
      placed.append((slot, col0, env_ids[start:start + n]))
      start += n
  slot, _, _ = asm.get(timeout=1.0)
  want = [e % 4 for s, _, ids in placed if s == slot for e in ids]
  assert asm.task_ids(slot).dtype == torch.int32
  assert asm.task_ids(slot).tolist() == want == [1, 2, 3, 0, 1, 3]
  one = utils.BatchAssembler(specs, state, full_length=4, batch_size=6, slots=2, device='cpu')
  assert one.task_ids(0) is None
