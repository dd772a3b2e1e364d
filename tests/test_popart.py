"""CPU: the PopArt restatement of tests/popart_reference.py against the reference's popart_test.py cases, the
float64 composition's own consistency (autograd, and the plain loss at beta = 0, with and without an abandoned
mask), the flags and their defaults, and the checkpoint check that keeps PopArt and non-PopArt learner states
apart."""
import os

import numpy as np
import pytest
import torch

import abandoned_float64_reference as AR
import popart_reference as PR
import vtrace_float64_reference as RF
from seed_rl_b200.agents.vtrace import learner
from seed_rl_b200.agents.vtrace import learner_loop
from seed_rl_b200.dmlab import networks


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'popart_golden.npz')
CASES = ('b1e-2', 'b3e-4', 'b1')


def _targets():
  return np.arange(20, dtype=np.float32)


# ---- reference popart_test.py, restated --------------------------------------------------------------------------
def test_normalization():
  p = PR.PopArt(1.0)
  p.update_normalization_statistics(_targets())
  n = p.normalize_target(_targets())
  np.testing.assert_allclose(n.mean(), 0.0, atol=1e-6)
  np.testing.assert_allclose(n.std(), 1.0, rtol=1e-6)


def test_variables():
  """Four variables, two trainable: the restatement's table against what the reference module created."""
  p = PR.PopArt(0.5)
  assert p.state.shape == (4,) and len(PR.PopArt.VARIABLES) == 4
  assert sum(PR.PopArt.TRAINABLE) == 2
  np.testing.assert_array_equal(np.load(GOLDEN)['trainable'], PR.PopArt.TRAINABLE)


def test_invariance():
  p = PR.PopArt(0.5)
  x = _targets()
  before = p.unnormalize_prediction(p.correct_prediction(x))
  p.update_normalization_statistics(x)
  after = p.unnormalize_prediction(p.correct_prediction(x))
  np.testing.assert_allclose(before, after, rtol=1e-6, atol=1e-5)


def test_invertible():
  p = PR.PopArt(0.5)
  x = _targets()
  p.update_normalization_statistics(x)
  np.testing.assert_allclose(p.unnormalize_prediction(p.normalize_target(x)), x, rtol=1e-6, atol=1e-5)


def test_advantage():
  p = PR.PopArt(0.5)
  x = _targets()
  p.update_normalization_statistics(x)
  adv = x - x[::-1]
  nt = p.normalize_target(x)
  np.testing.assert_allclose(p.normalize_advantage(adv), nt - nt[::-1], rtol=1e-6, atol=1e-6)


# ---- pinned to the unmodified reference (tests/golden/make_golden_popart.py) ----------------------------------
def _golden_steps(d, case):
  k = 0
  while '%s_%d_ll' % (case, k) in d:
    p = '%s_%d_' % (case, k)
    yield k, p, tuple(d[p + x] for x in ('ll', 'lb', 'bl', 'act', 'rew', 'done'))
    k += 1


def _close(name, x, ref, rtol):
  x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
  err = np.abs(x - ref).max() / max(np.abs(ref).max(), 1e-30)
  assert err <= rtol, '%s: %.3g > %.3g' % (name, err, rtol)


@pytest.mark.parametrize('case', CASES)
def test_popart_module_against_golden(case):
  """The restated PopArt module, fed the reference's own vs, makes the reference module's moves, step by step
  from the initial variables."""
  d = np.load(GOLDEN)
  p = PR.PopArt(float(d['%s_beta' % case]))
  steps = 0
  for k, pre, (ll, lb, bl, act, rew, done) in _golden_steps(d, case):
    np.testing.assert_allclose(p.state, d[pre + 'state_before'], rtol=1e-5)
    _close(pre + 'u', p.unnormalize_prediction(p.correct_prediction(lb)), d[pre + 'u'], 1e-6)
    _close(pre + 'n', p.normalize_target(d[pre + 'vs']), d[pre + 'n'], 1e-6)
    _close(pre + 'adv', p.normalize_advantage(d[pre + 'pg_adv']), d[pre + 'adv'], 1e-6)
    mean2, std2 = p.update_normalization_statistics(d[pre + 'vs'])
    _close(pre + 'mean', mean2, d[pre + 'PopArt__mean'], 1e-5)
    _close(pre + 'std', std2, d[pre + 'PopArt__std'], 1e-5)
    _close(pre + 'e', d[pre + 'n'] - p.correct_prediction(lb[:-1]), d[pre + 'e'], 1e-5)
    for i, v in enumerate(PR.PopArt.VARIABLES):
      _close(pre + v, p.state[i], d[pre + 'state_after'][i], 1e-5)
    steps += 1
  assert steps >= 3


@pytest.mark.parametrize('FT', [np.float32, np.float64])
@pytest.mark.parametrize('case', CASES)
def test_composition_against_golden(case, FT):
  """The composition the kernels implement (loss_and_grads, steps 1-9), step by step from the state the
  reference modules held before it, against the reference modules composed around the reference V-trace."""
  d = np.load(GOLDEN)
  discounting, lambda_, baseline_cost = (float(x) for x in d['cfg'])
  cfg = learner.default_loss_settings(popart=True, discounting=discounting, lambda_=lambda_,
                                      baseline_cost=baseline_cost)
  beta = float(d['%s_beta' % case])
  rtol = 2e-5 if FT == np.float32 else 1e-4     # float64 differs from the float32 reference by its rounding
  np.testing.assert_array_equal(d['%s_0_state_before' % case], [0, 1, 1, 0])
  for k, pre, b in _golden_steps(d, case):
    r = PR.loss_and_grads(cfg, *b, -1.0, d[pre + 'state_before'], beta, FT=FT)
    for key in ('u', 'vs', 'pg_adv', 'n', 'adv', 'e'):
      _close(pre + key, r[key], d[pre + key], rtol)
    _close(pre + 'policy', r['terms']['policy'], d[pre + 'policy_loss'], rtol)
    _close(pre + 'V', r['terms']['V'], d[pre + 'v_loss'], rtol)
    _close(pre + 'PopArt/mean', r['terms']['popart_mean'], d[pre + 'PopArt__mean'], rtol)
    _close(pre + 'PopArt/std', r['terms']['popart_std'], d[pre + 'PopArt__std'], rtol)
    for i in range(4):
      _close(pre + PR.PopArt.VARIABLES[i], r['state'][i], d[pre + 'state_after'][i], rtol)


# ---- the composition --------------------------------------------------------------------------------------------
def _batch(T1=9, B=6, A=5, seed=0):
  g = np.random.default_rng(seed)
  return (g.standard_normal((T1, B, A)).astype(np.float32), g.standard_normal((T1, B)).astype(np.float32),
          g.standard_normal((T1, B, A)).astype(np.float32), g.integers(0, A, (T1, B)),
          (g.standard_normal((T1, B)) * 200 + 300).astype(np.float32), g.random((T1, B)) < 0.1)


def test_composition_state_update_is_the_popart_module():
  cfg = learner.default_loss_settings(popart=True)
  b = _batch()
  state = np.array([40.0, 5000.0, 0.7, 0.2], np.float32)
  r = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3)
  p = PR.PopArt(0.3, FT=np.float64)
  p.first_moment, p.second_moment, p.compensation_std, p.compensation_mean = (np.float64(x) for x in state)
  mean2, std2 = p.update_normalization_statistics(r['vs'])
  np.testing.assert_allclose(r['state'], p.state, rtol=1e-12)
  assert np.isclose(r['terms']['popart_mean'], mean2) and np.isclose(r['terms']['popart_std'], std2)


def test_composition_gradients_match_autograd():
  cfg = learner.default_loss_settings(popart=True, baseline_cost=0.7)
  ll, lb, bl, act, rew, done = _batch()
  state = np.array([40.0, 5000.0, 0.7, 0.2], np.float32)
  r = PR.loss_and_grads(cfg, ll, lb, bl, act, rew, done, -1.0, state, 0.3)
  T = ll.shape[0] - 1
  s = np.sqrt(5000.0 - 1600.0)
  logits = torch.tensor(ll.astype(np.float64), requires_grad=True)
  V = torch.tensor(lb.astype(np.float64), requires_grad=True)
  sig = torch.tensor(float(r['state'][2]), dtype=torch.float64, requires_grad=True)
  mu = torch.tensor(float(r['state'][3]), dtype=torch.float64, requires_grad=True)
  a = torch.as_tensor(act[:-1])
  lsm = torch.log_softmax(logits[:-1], -1)
  tl = lsm.gather(-1, a[..., None])[..., 0]
  adv = torch.as_tensor(r['pg_adv']) / s
  n = (torch.as_tensor(r['vs']) - 40.0) / s
  e = n - (sig * V[:-1] + mu)
  ec = float(np.exp(10.0 * -1.0))
  ent = -(lsm.exp() * lsm).sum(-1).mean()
  total = -(tl * adv).mean() + 0.7 * 0.5 * (e ** 2).mean() - ec * ent
  total.backward()
  np.testing.assert_allclose(r['dlogits'], logits.grad.numpy(), rtol=1e-9, atol=1e-15)
  np.testing.assert_allclose(r['dbaseline'], V.grad.numpy(), rtol=1e-9, atol=1e-15)
  np.testing.assert_allclose(r['dcomp'], [float(sig.grad), float(mu.grad)], rtol=1e-9)
  np.testing.assert_allclose(r['terms']['total'], float(total.detach()), rtol=1e-12)
  assert T == 8


def test_composition_at_beta0_is_the_plain_loss():
  b = _batch(seed=3)
  r = PR.loss_and_grads(learner.default_loss_settings(popart=True), *b, -1.0, np.array([0, 1, 1, 0], np.float32), 0.0)
  total, logs, dl, db, dep, vs, pg = RF.loss_and_grads(learner.default_loss_settings(), *b, -1.0, torch.float64)
  np.testing.assert_allclose(r['dlogits'], dl, rtol=1e-12, atol=1e-18)
  np.testing.assert_allclose(r['dbaseline'], db, rtol=1e-12, atol=1e-18)
  np.testing.assert_allclose(r['terms']['total'], total, rtol=1e-12)
  np.testing.assert_array_equal(r['state'], [0, 1, 1, 0])


def _masked_batch(seed, T1=9, B=6):
  ll, lb, bl, act, rew, done = _batch(T1=T1, B=B, seed=seed)
  done_m, ab = AR.masks(T1, B, seed + 1, p_done=0.0)
  return (ll, lb, bl, act, rew, done | done_m), ab


@pytest.mark.parametrize('FT', [np.float32, np.float64])
def test_composition_without_abandonment_ignores_the_mask(FT):
  """abandoned=None and an all-false mask: the composition is the same bit for bit."""
  b, _ = _masked_batch(seed=4)
  cfg = learner.default_loss_settings(popart=True, lambda_=0.95)
  state = np.array([40.0, 5000.0, 0.7, 0.2], np.float32)
  r0 = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3, FT=FT)
  r1 = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3, FT=FT, abandoned=np.zeros(b[5].shape, bool))
  for key in ('dlogits', 'dbaseline', 'dcomp', 'state', 'vs', 'pg_adv', 'u', 'e', 'sums'):
    np.testing.assert_array_equal(r1[key], r0[key], err_msg=key)
  for name in r0['terms']:
    assert r1['terms'][name] == r0['terms'][name], name


def test_masked_composition_takes_the_masked_vtrace():
  """With abandoned transitions: vs = u and pg_adv = 0 exactly on the masked ones, every other output moves,
  and the moment sums are those of the masked vs."""
  b, ab = _masked_batch(seed=5)
  cfg = learner.default_loss_settings(popart=True, lambda_=0.95)
  state = np.array([40.0, 5000.0, 0.7, 0.2], np.float32)
  r = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3, abandoned=ab)
  plain = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3)
  m = ab[1:]
  assert m[0, 0] and m[-1, 1 % 6] and m.sum() >= 3
  np.testing.assert_array_equal(r['vs'][m], r['u'][:-1][m])
  assert np.all(r['pg_adv'][m] == 0) and not np.all(plain['pg_adv'][m] == 0)
  assert not np.array_equal(r['dbaseline'], plain['dbaseline']) and not np.array_equal(r['state'], plain['state'])
  np.testing.assert_allclose(r['sums'], [r['vs'].sum(), (r['vs'] ** 2).sum(), r['vs'].size], rtol=1e-12)


def test_masked_float32_composition_is_the_float64_one_rounded():
  """The float32 composition's masked recursion against the float64 definition: the same targets to float32
  rounding, masked transitions included."""
  b, ab = _masked_batch(seed=7)
  cfg = learner.default_loss_settings(popart=True, lambda_=0.95)
  state = np.array([40.0, 5000.0, 0.7, 0.2], np.float32)
  r32 = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3, FT=np.float32, abandoned=ab)
  r64 = PR.loss_and_grads(cfg, *b, -1.0, state, 0.3, abandoned=ab)
  for key in ('vs', 'pg_adv', 'dbaseline', 'state'):
    _close(key, r32[key], r64[key], 1e-5)
  assert np.all(r32['pg_adv'][ab[1:]] == 0)


def test_masked_composition_at_beta0_is_the_masked_plain_loss(monkeypatch):
  """beta = 0 from the initial state, with an abandoned mask: the plain loss of tests/test_gpu_abandoned.py (the
  float64 loss with its V-trace replaced by the masked one)."""
  b, ab = _masked_batch(seed=6)
  kw = dict(discounting=0.97, lambda_=0.95, kl_cost=0.01)
  r = PR.loss_and_grads(learner.default_loss_settings(popart=True, **kw), *b, -0.8,
                        np.array([0, 1, 1, 0], np.float32), 0.0, abandoned=ab)
  monkeypatch.setattr(RF, 'vtrace_from_importance_weights', AR.masked_vtrace(ab[1:]))
  total, logs, dl, db, dep, vs, pg = RF.loss_and_grads(learner.default_loss_settings(**kw), *b, -0.8, torch.float64)
  np.testing.assert_allclose(r['vs'], vs, rtol=1e-12, atol=1e-15)
  np.testing.assert_allclose(r['pg_adv'], pg, rtol=1e-12, atol=1e-15)
  np.testing.assert_allclose(r['dlogits'], dl, rtol=1e-12, atol=1e-18)
  np.testing.assert_allclose(r['dbaseline'], db, rtol=1e-12, atol=1e-18)
  np.testing.assert_allclose(r['terms']['total'], total, rtol=1e-12)
  for name, key in learner._LOG_NAMES:
    np.testing.assert_allclose(r['terms'][key], logs[name], rtol=1e-12, atol=1e-15, err_msg=name)
  np.testing.assert_array_equal(r['state'], [0, 1, 1, 0])
  assert np.all(db[:-1][ab[1:]] == 0)


# ---- flags and settings -----------------------------------------------------------------------------------------
def test_flag_and_setting_defaults():
  from absl import flags
  F = flags.FLAGS
  assert F['popart'].default is False
  assert F['popart_beta'].default == 1e-2
  d = learner.default_loss_settings()
  assert d.popart is False and d.popart_beta == 1e-2
  old = learner.LossSettings(.99, 1., .5, 0.00025, 0., 0., None, 10.)     # the eight fields of before
  assert old.popart is False and old.popart_beta == 1e-2


# ---- checkpoints ------------------------------------------------------------------------------------------------
class _FakeAgent(object):
  def __init__(self, popart):
    self.popart_moments = torch.zeros(2) if popart else None
    self.param_info = [('w', (2,), 0)]
    self.device = 'cpu'
    self.loaded = None

  def load_state_dict(self, d):
    self.loaded = d


class _FakeOpt(object):
  def load_state_dict(self, d, device=None):
    pass


@pytest.mark.parametrize('saved,running', [(True, False), (False, True)])
def test_checkpoint_popart_mismatch_raises(tmp_path, saved, running):
  agent_state = {'params': torch.zeros(2), 'param_info': [('w', (2,), 0)]}
  if saved:
    agent_state['popart_moments'] = torch.tensor([0.0, 1.0])
  path = str(tmp_path / 'ckpt.pt')
  torch.save({'agent': agent_state, 'optimizer': {}}, path)
  agent = _FakeAgent(running)
  with pytest.raises(ValueError, match='PopArt|popart'):
    learner_loop.restore_checkpoint(path, agent, _FakeOpt())
  assert agent.loaded is None
  learner_loop.restore_checkpoint(path, _FakeAgent(saved), _FakeOpt())    # the matching learner restores it
  with pytest.raises(ValueError):
    networks.check_popart_state(agent_state, running)
