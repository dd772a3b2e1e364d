"""Generates tests/golden/popart_golden.npz.  Run ONLY in the build container (where
/root/reference exists):   python tests/golden/make_golden_popart.py

Executes the UNMODIFIED reference agents/policy_gradient/modules/popart.py (`PopArt`, compensation on) over
the UNMODIFIED running_statistics.py (`EMAMeanStd`), with the UNMODIFIED common/vtrace.py behind them, over
tf_numpy_shim: nothing is copied into this repo.  The only stand-ins are the ones the modules need to import
without TensorFlow: a `gin.configurable` no-op (tf_numpy_shim.install), a `logging_module.LoggingModule` whose
`log` records its scalars, a tf.Variable with assign / assign_add, and a `tf.function` no-op for the other
trackers the module file defines.

Each learner step composes them in the order generalized_onpolicy_loss.py:94-133 runs them, around the
V-trace compute_loss of agents/vtrace/learner.py:82-157 (values and bootstrap from the unnormalised corrected
baseline; reward clip off, the learner's discounts, rho-bar = 1, lambda):
  corrected = correct_prediction(V); u = unnormalize_prediction(corrected)      (all T+1 rows)
  vs, pg_adv = vtrace.from_importance_weights(..., values=u[:-1], bootstrap_value=u[-1])
  n = normalize_target(vs); adv = normalize_advantage(pg_adv); update_normalization_statistics(vs)
  e = n - correct_prediction(V[:-1])        (read after the update, as the reference's value loss does)
  policy loss = -mean(log pi(a) adv); value loss = baseline_cost 0.5 mean(e^2)
Several consecutive steps per case (the module's variables carry over), beta in {1e-2, 3e-4, 1}, rewards in
the hundreds, unclipped.  Every case stores its inputs and the state before and after each step, so machines
without /root/reference replay them (tests/test_popart.py)."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
sys.path.insert(0, HERE)
import tf_numpy_shim  # noqa: E402
from make_golden import _load  # noqa: E402

MODULES = os.path.join(REF, 'agents/policy_gradient/modules')


def _install():
  tf = tf_numpy_shim.install()
  T, raw = tf_numpy_shim.Tensor, tf_numpy_shim._raw
  f32 = np.float32
  T.__pow__ = lambda self, p: T(np.power(self.a, f32(p)).astype(self.a.dtype))

  class Variable(T):
    """tf.Variable: a mutable Tensor; records `trainable` for the variable count of popart_test.py."""

    def __init__(self, name=None, shape=None, trainable=True, dtype=None, initial_value=None, aggregation=None):
      super(Variable, self).__init__(np.asarray(raw(initial_value), f32).reshape(shape))
      self.name, self.trainable = name, trainable

    def assign(self, v):
      self.a = np.asarray(raw(v), f32).reshape(self.a.shape)

    def assign_add(self, v):
      self.a = (self.a + np.asarray(raw(v), f32)).astype(f32)

  tf.Variable = Variable
  tf.Module = type('Module', (object,), {})      # a class of its own: PopArt mixes it with LoggingModule
  tf.VariableAggregation = types.SimpleNamespace(MEAN='MEAN')
  tf.function = lambda f=None, **kw: f if f is not None else (lambda g: g)   # decorates unused trackers
  tf.zeros = lambda shape, dtype=f32: T(np.zeros(shape, dtype))
  tf.ones = lambda shape, dtype=f32: T(np.ones(shape, dtype))
  tf.sqrt = lambda x: T(np.sqrt(raw(x)))
  tf.clip_by_value = lambda x, lo, hi: T(np.clip(raw(x), f32(lo), f32(hi)).astype(f32))
  tf.squeeze = lambda x, axis=None: T(np.squeeze(raw(x), axis))
  tf.reduce_mean = lambda x, axis=None: T(np.mean(raw(x), axis=None if axis is None else tuple(axis), dtype=f32))

  logged = []

  class LoggingModule(object):
    def log(self, key, tensor):
      logged.append((key, np.asarray(raw(tensor), f32)))

  pkg = 'seed_rl.agents.policy_gradient.modules'
  for name in ('seed_rl', 'seed_rl.agents', 'seed_rl.agents.policy_gradient', pkg):
    sys.modules[name] = types.ModuleType(name)
  lm = types.ModuleType(pkg + '.logging_module')
  lm.LoggingModule = LoggingModule
  sys.modules[pkg + '.logging_module'] = lm
  sys.modules[pkg].logging_module = lm
  rs = _load(os.path.join(MODULES, 'running_statistics.py'), pkg + '.running_statistics')
  sys.modules[pkg + '.running_statistics'] = rs
  sys.modules[pkg].running_statistics = rs
  popart = _load(os.path.join(MODULES, 'popart.py'), pkg + '.popart')
  vtrace = _load(os.path.join(REF, 'common/vtrace.py'), 'ref_vtrace')
  return tf, popart, rs, vtrace, logged


def _log_softmax(x):
  m = x.max(-1, keepdims=True)
  return (x - m - np.log(np.exp(x - m).sum(-1, keepdims=True, dtype=np.float32))).astype(np.float32)


def main():
  tf, popart, rs, vtrace, logged = _install()
  T, raw = tf_numpy_shim.Tensor, tf_numpy_shim._raw
  f32 = np.float32
  out = {}
  rng = np.random.default_rng(23)
  T1, B, A, steps = 11, 8, 6, 4
  discounting, lambda_, baseline_cost = 0.99, 0.95, 0.5
  out['cfg'] = np.asarray([discounting, lambda_, baseline_cost], f32)
  for name, beta in (('b1e-2', 1e-2), ('b3e-4', 3e-4), ('b1', 1.0)):
    pa = popart.PopArt(rs.EMAMeanStd(beta))
    pa.init()
    tracker = pa.mean_std_tracker
    variables = (tracker.first_moment, tracker.second_moment, pa.compensation_std, pa.compensation_mean)
    out['trainable'] = np.asarray([v.trainable for v in variables])

    def state():
      return np.concatenate([np.asarray(raw(v), f32).reshape(-1) for v in variables])
    out['%s_beta' % name] = np.asarray(beta)
    for k in range(steps):
      ll = rng.normal(size=(T1, B, A)).astype(f32); bl = rng.normal(size=(T1, B, A)).astype(f32)
      lb = (rng.normal(size=(T1, B)) * 3).astype(f32); act = rng.integers(0, A, (T1, B))
      rew = (rng.normal(size=(T1, B)) * 200 + 300).astype(f32); done = rng.random((T1, B)) < 0.1
      p = '%s_%d_' % (name, k)
      out.update({p + 'll': ll, p + 'lb': lb, p + 'bl': bl, p + 'act': act, p + 'rew': rew, p + 'done': done,
                  p + 'state_before': state()})
      a = act[:-1]
      tlp = np.take_along_axis(_log_softmax(ll[:-1]), a[..., None], -1)[..., 0]
      blp = np.take_along_axis(_log_softmax(bl[:-1]), a[..., None], -1)[..., 0]
      disc = ((~done[1:]).astype(f32) * f32(discounting)).astype(f32)
      u = pa.unnormalize_prediction(pa.correct_prediction(T(lb)))
      ret = vtrace.from_importance_weights(T(tlp), T(blp), T(disc), T(rew[1:]), u[:-1], u[-1], lambda_=lambda_)
      n = pa.normalize_target(ret.vs)
      adv = pa.normalize_advantage(ret.pg_advantages)
      del logged[:]
      pa.update_normalization_statistics(ret.vs)
      e = raw(n) - raw(pa.correct_prediction(T(lb[:-1])))
      out.update({p + 'u': raw(u), p + 'vs': raw(ret.vs), p + 'pg_adv': raw(ret.pg_advantages), p + 'n': raw(n),
                  p + 'adv': raw(adv), p + 'e': e, p + 'state_after': state(),
                  p + 'policy_loss': -np.mean(tlp * raw(adv), dtype=f32),
                  p + 'v_loss': f32(baseline_cost) * f32(0.5) * np.mean(e * e, dtype=f32)})
      for key, v in logged:
        out[p + key.replace('/', '__')] = v
  np.savez_compressed(os.path.join(HERE, 'popart_golden.npz'), **out)
  print('wrote popart_golden.npz:', len(out), 'arrays; trainable', out['trainable'])


if __name__ == '__main__':
  main()
