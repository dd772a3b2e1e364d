"""Generates tests/golden/r2d2_retrace_golden.npz.  Run ONLY in the build container (where
/root/reference exists):   python tests/golden/make_golden_r2d2_retrace.py

The reference has no Retrace.  Two reductions pin the Retrace targets to its own n-step function,
executed UNMODIFIED (agents/r2d2/learner.py `n_step_bellman_target`, pulled out by AST) over
tf_numpy_shim; nothing is copied into this repo:
  * lambda = 0 gives n_step_bellman_target with n_steps = 1           ('l0_*' cases);
  * lambda = 1 with every replayed action greedy gives it with n_steps >= T - 1, whose padded tail
    bootstraps from the last q_target, as Retrace does        ('l1_*' cases).
Each case stores its inputs (rewards, done, q = h^-1(Q_target(x, a*))) next to the output, so
machines without /root/reference can replay them."""
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = '/root/reference'
sys.path.insert(0, HERE)
import tf_numpy_shim  # noqa: E402
from make_golden import _extract_function  # noqa: E402
from make_golden_r2d2 import extend  # noqa: E402


def main():
  tf = extend(tf_numpy_shim.install())
  ns = {'tf': tf, 'FLAGS': types.SimpleNamespace(value_function_rescaling_epsilon=1e-3, n_steps=5), 'np': np}
  nstep = _extract_function(os.path.join(REF, 'agents/r2d2/learner.py'), 'n_step_bellman_target', ns)
  T = tf_numpy_shim.Tensor
  rng = np.random.default_rng(11)
  f32 = np.float32
  out = {}
  # (T, B, gamma, n_steps); done_p 0.2 puts episode ends inside most sequences
  cases = {'l0_a': (2, 3, 0.997, 1), 'l0_b': (4, 3, 0.9, 1), 'l0_c': (20, 4, 0.997, 1), 'l0_d': (101, 5, 0.997, 1),
           'l1_a': (2, 3, 0.997, 1), 'l1_b': (4, 3, 0.9, 3), 'l1_c': (20, 4, 0.997, 22), 'l1_d': (101, 5, 0.997, 100),
           'l1_e': (101, 5, 0.99, 104)}
  for name, (Tn, B, gamma, n) in cases.items():
    r = rng.normal(size=(Tn, B)).astype(f32)
    d = rng.random((Tn, B)) < 0.2
    q = (rng.normal(size=(Tn, B)) * 10).astype(f32)
    out['%s_in' % name] = np.stack([r, d.astype(f32), q])
    out['%s_cfg' % name] = np.asarray([n, gamma])
    out['%s_out' % name] = nstep(T(r), T(d), T(q), gamma, n).a
  np.savez_compressed(os.path.join(HERE, 'r2d2_retrace_golden.npz'), **out)
  print('wrote r2d2_retrace_golden.npz:', sorted(out))


if __name__ == '__main__':
  main()
