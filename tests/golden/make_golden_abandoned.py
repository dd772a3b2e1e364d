"""Generates tests/golden/abandoned_golden.npz.  Run ONLY in the build container (where
/root/reference exists):   python tests/golden/make_golden_abandoned.py

Executes the UNMODIFIED reference agents/policy_gradient/modules/advantages.py (`vtrace` and `NStep`) over
tf_numpy_shim: nothing is copied into this repo.  The stand-ins added here after install() are the ones NStep
needs: tf.zeros, tf.ones and a tf.Module whose __init__ takes a name.

The cases have terminated and abandoned rows at the first, interior and last transitions of the unroll, next
to each other and alone.  In the learner's indexing (row t+1 of reward / done / abandoned belongs to
transition t), the reference gets rewards = reward[1:], done_terminated = (done & ~abandoned)[1:] and
done_abandoned = abandoned[1:].

V-trace.  advantages.vtrace computes, with rho_t = min(exp(log_rho_t), 1), nt = not terminated and
na = not abandoned,
  delta_t = na_t (r_t + gamma nt_t V_{t+1} - V_t),   acc_t = rho_t (delta_t + na_t nt_t gamma lambda acc_{t+1}),
  target_t = V_t + acc_t.
common/vtrace.py with rho-bar = c-bar = 1 computes, with d_t = gamma (1 - done_t) and c_t = lambda min(1, rho_t),
  acc_t = min(1, rho_t) delta'_t + d_t c_t acc_{t+1},   vs_t = V_t + acc_t.
With the abandoned transitions' delta' set to 0 and done = terminated | abandoned, d_t = gamma nt_t na_t and
delta'_t = delta_t (an unmasked row has na_t = 1), so acc_t = rho_t (delta_t + gamma lambda nt_t na_t acc_{t+1}):
the two recursions are the same and target = vs.  That is what the fixture pins (`vtrace_*_targets`).  The
reference's advantages are defined differently from common/vtrace.py's pg_advantages (no bootstrap on vs_{t+1},
no clipped pg rho), so they are not pinned.

R2D2.  NStep(n) with values = q*_0 .. q*_{T-1} (the rescaled-back target Q at the online argmax) gives the
n-step targets before h of rows 1..T-1 (`nstep_*_targets`), the padding at the unroll's end included: its
padded rows are abandoned and so bootstrap from q*_{T-1}."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
sys.path.insert(0, HERE)
import tf_numpy_shim  # noqa: E402
from make_golden import _load  # noqa: E402


def _install():
  tf = tf_numpy_shim.install()
  T = tf_numpy_shim.Tensor
  tf.zeros = lambda shape, dtype=np.float32: T(np.zeros(shape, dtype))
  tf.ones = lambda shape, dtype=np.float32: T(np.ones(shape, dtype))

  class Module(object):
    def __init__(self, name=None):
      self.name = name
  tf.Module = Module
  return _load(os.path.join(REF, 'agents/policy_gradient/modules/advantages.py'), 'ref_advantages')


def _masks(T1, B, rng):
  """done, abandoned [T1,B]: columns with abandonment at the first, an interior and the last transition,
  next to terminations, several per column, and none."""
  done = np.zeros((T1, B), bool)
  ab = np.zeros((T1, B), bool)
  ab[1, 0] = True                          # first transition
  ab[T1 // 2, 1] = True                    # interior
  ab[T1 - 1, 2] = True                     # last transition
  ab[3, 3] = True; done[2, 3] = True; done[4, 3] = True    # between two terminations
  ab[2, 4] = True; ab[5, 4] = True; done[T1 - 2, 4] = True
  done[1, 5] = True; done[T1 - 1, 5] = True               # terminations only
  extra = rng.random((T1, B)) < 0.15
  done[:, 6:] |= extra[:, 6:]
  ab[:, 6:] |= (rng.random((T1, B)) < 0.15)[:, 6:]
  done |= ab
  return done, ab


def main():
  adv = _install()
  T = tf_numpy_shim.Tensor
  raw = tf_numpy_shim._raw
  f32 = np.float32
  rng = np.random.default_rng(41)
  out = {}
  T1, B = 12, 9
  gamma = 0.97
  out['gamma'] = np.asarray(gamma)
  for case in range(2):
    p = 'c%d_' % case
    done, ab = _masks(T1, B, rng)
    values = rng.normal(size=(T1, B)).astype(f32)
    rew = (rng.normal(size=(T1, B)) * 2).astype(f32)
    log_rhos = (rng.normal(size=(T1 - 1, B)) * 0.5).astype(f32)
    q_star = rng.normal(size=(T1, B)).astype(f32) * 3
    out.update({p + 'done': done, p + 'abandoned': ab, p + 'values': values, p + 'reward': rew,
                p + 'log_rhos': log_rhos, p + 'q_star': q_star})
    term, aband = T((done & ~ab)[1:]), T(ab[1:])
    for lam in (0.95, 1.0):
      tgt, _ = adv.vtrace(T(values), T(rew[1:]), term, aband, gamma, T(log_rhos), T(np.zeros_like(log_rhos)),
                          lambda_=lam, max_importance_weight=1.)
      out[p + 'vtrace_l%g_targets' % lam] = raw(tgt)
    for n in (1, 3, 5):
      tgt, _ = adv.NStep(n)(T(q_star), T(rew[1:]), term, aband, gamma, None, None)
      out[p + 'nstep_n%d_targets' % n] = raw(tgt)
  np.savez_compressed(os.path.join(HERE, 'abandoned_golden.npz'), **out)
  print('wrote abandoned_golden.npz:', len(out), 'arrays')


if __name__ == '__main__':
  main()
