"""CPU: the host half of the parameter update.  optimizers.Adam.apply_gradients computes Keras's bias-corrected step
size lr_t = lr(iterations) * sqrt(1 - b2^t) / (1 - b1^t), t = iterations + 1, in fp32 (Keras `_prepare_local`) and
passes it to seedrl_adam_apply; PolynomialDecay is tf.keras.optimizers.schedules.PolynomialDecay (cycle=False).

The library is replaced by a stub that records the arguments of seedrl_adam_apply, so no device is needed.  The
recorded lr_t is compared with the same formula evaluated in float64 from the fp32 constants (fp32 lr, b1, b2).  The
fp32 evaluation rounds b^t (numpy's powf, within one ulp, exact at t = 1) and then subtracts it from 1, which
magnifies that rounding by r = b^t / (1 - b^t); the bar is therefore
    |lr_t - lr_t64| <= u * lr_t64 * (6 + 2 r2 + 2 r1),   u = 2^-24, r = 0 at t = 1,
six roundings of the rest of the formula plus the conditioning of the two bias corrections.  At t = 1 it is 6 ulp-ish
(r = 0); at t = 10, b2 = 0.999 it is about 200 u, the size of one powf ulp after the cancellation.
"""
import types

import numpy as np
import pytest
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common import optimizers

U = 2.0 ** -24
ITERATIONS = (0, 1, 9, 999, 10 ** 6 - 1, 10 ** 6 + 5)
DECAY_STEPS = 10 ** 6
# (name, learning rate, beta_1, beta_2, epsilon): bench.py's two optimizers
SETTINGS = {
    'vtrace': (lambda: optimizers.PolynomialDecay(4.8e-4, DECAY_STEPS, 0.0), 0.0, 0.999, 3.125e-7),
    'r2d2': (lambda: 4.8e-4, 0.9, 0.999, 1e-3),
}


class _Recorder(object):
  """Stands in for the loaded library: records each seedrl_adam_apply call and returns SEEDRL_OK."""

  def __init__(self):
    self.calls = []

  def seedrl_adam_apply(self, *args):
    self.calls.append(args)
    return 0


@pytest.fixture
def recorder(monkeypatch):
  rec = _Recorder()
  monkeypatch.setattr(_lib, 'lib', lambda: rec)
  monkeypatch.setattr(_lib, 'stream_ptr', lambda: None)
  return rec


def _lr64(lr, b1, b2, iterations):
  f = np.float32
  t = iterations + 1
  b1, b2 = float(f(b1)), float(f(b2))
  return float(f(lr)) * np.sqrt(1.0 - b2 ** t) / (1.0 - b1 ** t)


def _bar(lr64, b1, b2, iterations):
  t = iterations + 1
  r = lambda b: 0.0 if t == 1 else float(np.float32(b)) ** t / (1.0 - float(np.float32(b)) ** t)
  return U * lr64 * (6.0 + 2.0 * r(b2) + 2.0 * r(b1))


@pytest.mark.parametrize('name', sorted(SETTINGS))
@pytest.mark.parametrize('iterations', ITERATIONS)
def test_lr_t_matches_float64(recorder, name, iterations):
  make_lr, b1, b2, eps = SETTINGS[name]
  lr = make_lr()
  opt = optimizers.Adam(lr, beta_1=b1, beta_2=b2, epsilon=eps)
  params, grads = torch.zeros(12), torch.zeros(12)
  opt.iterations = iterations
  opt.apply_gradients(params, grads, grad_scale=0.5, clamp_index=3, clamp_lo=-2.0, clamp_hi=2.0)
  assert opt.iterations == iterations + 1
  (n, _, _, _, _, lr_t, beta1, beta2, epsilon, scale, ci, lo, hi, _), = recorder.calls
  assert n == 12 and (beta1, beta2, epsilon, scale, ci, lo, hi) == (b1, b2, eps, 0.5, 3, -2.0, 2.0)
  assert float(np.float32(lr_t)) == lr_t, 'lr_t must be an fp32 value: the kernel takes a float'
  step_lr = lr(iterations) if callable(lr) else lr
  want = _lr64(step_lr, b1, b2, iterations)
  bar = _bar(want, b1, b2, iterations)
  assert abs(lr_t - want) <= bar, (lr_t, want, bar)
  if iterations >= DECAY_STEPS and name == 'vtrace':
    assert lr_t == 0.0                        # past decay_steps the schedule sits at its end rate, here 0
  else:
    assert lr_t > 0.0
    assert bar <= 5e-4 * want                 # the bar stays sharp at every tested step


def test_lr_t_bias_correction_at_the_first_step(recorder):
  """t = 1 with R2D2's b1 = 0.9: lr_t = lr * sqrt(1 - b2) / (1 - b1), about 0.316 lr; b^1 is exact, so only the
  final roundings separate it from float64."""
  opt = optimizers.Adam(4.8e-4, beta_1=0.9, beta_2=0.999, epsilon=1e-3)
  opt.apply_gradients(torch.zeros(4), torch.zeros(4))
  lr_t = recorder.calls[0][5]
  want = _lr64(4.8e-4, 0.9, 0.999, 0)
  assert abs(lr_t - want) <= 6 * U * want
  assert 0.315 < lr_t / 4.8e-4 < 0.317


def test_lr_t_follows_the_optimizer_iterations(recorder):
  """Three consecutive calls advance t: the recorded lr_t are those of iterations 0, 1, 2."""
  opt = optimizers.Adam(optimizers.PolynomialDecay(4.8e-4, DECAY_STEPS, 0.0), beta_1=0.0, epsilon=3.125e-7)
  p, g = torch.zeros(8), torch.zeros(8)
  for _ in range(3):
    opt.apply_gradients(p, g)
  for it, call in enumerate(recorder.calls):
    want = _lr64(opt.learning_rate(it), 0.0, 0.999, it)
    assert abs(call[5] - want) <= _bar(want, 0.0, 0.999, it)


@pytest.mark.parametrize('end_lr,power', [(0.0, 1.0), (0.0001, 1.0), (1e-5, 2.0)])
def test_polynomial_decay_before_at_and_past_decay_steps(end_lr, power):
  init, steps = 4.8e-4, 1000
  sched = optimizers.PolynomialDecay(init, steps, end_lr, power)
  for step in (0, 1, 9, 500, 999):
    want = (init - end_lr) * (1.0 - step / steps) ** power + end_lr
    assert abs(sched(step) - want) <= 1e-15 * init, step
  assert sched(0) == init
  for step in (steps, steps + 1, steps + 5, 10 * steps):
    assert sched(step) == end_lr, step               # cycle=False: held at the end rate
  vals = [sched(s) for s in range(0, steps + 1, 50)]
  assert all(a > b for a, b in zip(vals, vals[1:]))  # strictly decreasing up to decay_steps


def test_polynomial_decay_default_end_rate_is_keras():
  """tf.keras's default end_learning_rate is 1e-4."""
  assert optimizers.PolynomialDecay(1e-3, 10)(10) == 0.0001
