"""CPU ORACLE (test infrastructure, NOT product code) -- numpy restatement of the
optimizer on the hot path.

The reference applies `tf.keras.optimizers.Adam` (TF 2.4.1, NOT vendored under
/root/reference; pinned by docker/Dockerfile.atari:14) built at
dmlab/vtrace_main.py:46-51 and applied at agents/vtrace/learner.py:272-273.
Its dense update rule (`_resource_apply_dense`, non-amsgrad), as published:

    t      = iterations + 1
    lr_t   = lr(iterations) * sqrt(1 - beta2^t) / (1 - beta1^t)
    m      = beta1*m + (1-beta1)*g
    v      = beta2*v + (1-beta2)*g^2
    theta -= lr_t * m / (sqrt(v) + eps)          # eps OUTSIDE the bias correction

No reference test exercises Adam on this path => PARITY UNPINNED (SURVEY 8c);
the only pinned optimizer-side semantic is cross-replica SUM of gradients
(tests/utils_test.py:609-650).
"""
import numpy as np


def polynomial_decay(initial_lr, step, decay_steps, end_lr=0.0, power=1.0):
  """tf.keras.optimizers.schedules.PolynomialDecay (cycle=False), used at
  dmlab/vtrace_main.py:47-48."""
  step = min(float(step), float(decay_steps))
  return (initial_lr - end_lr) * (1.0 - step / float(decay_steps)) ** power + end_lr


def keras_adam_step(p, g, m, v, iterations, lr, beta1=0.9, beta2=0.999, eps=1e-7):
  """One dense Adam step, fp32 throughout like TF's kernels.  `iterations` =
  optimizer.iterations BEFORE the step (0 for the first step).  Returns new (p, m, v).

  Restates Keras `Adam._prepare_local` (fp32 tensors: beta powers, `1 - beta`,
  lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t)) followed by the fused
  `training_ops.resource_apply_adam` update in the form its Eigen kernel uses:
      m += (g - m) * (1 - beta1);  v += (g*g - v) * (1 - beta2)
      var -= (m * lr_t) / (sqrt(v) + eps)
  Note `1 - beta2` is an fp32 subtraction, exact for beta2 in [0.5, 1]: 1 - fp32(0.999) = 0.000999987125, not the
  decimal 0.001."""
  f = np.float32
  t = f(iterations + 1)
  b1, b2 = f(beta1), f(beta2)
  b1p, b2p = np.power(b1, t, dtype=f), np.power(b2, t, dtype=f)
  lr_t = f(lr) * (np.sqrt(f(1) - b2p, dtype=f) / (f(1) - b1p))
  p, g, m, v = (np.asarray(x, f) for x in (p, g, m, v))
  m2 = m + (g - m) * (f(1) - b1)
  v2 = v + (g * g - v) * (f(1) - b2)
  p2 = p - (m2 * lr_t) / (np.sqrt(v2) + f(eps))
  return p2.astype(f), m2.astype(f), v2.astype(f)


def keras_adam_lr_t(iterations, lr, beta1, beta2):
  """fp32 lr_t exactly as keras_adam_step computes it (shared with nobody: the product
  recomputes it in seed_rl_b200/common/optimizers.py)."""
  f = np.float32
  t = f(iterations + 1)
  return f(lr) * (np.sqrt(f(1) - np.power(f(beta2), t, dtype=f), dtype=f) /
                  (f(1) - np.power(f(beta1), t, dtype=f)))
