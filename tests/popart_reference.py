"""PopArt value normalisation restated in numpy, for the tests of the V-trace learner's --popart.

`PopArt` restates the reference's agents/policy_gradient/modules/popart.py (compensation on) over
running_statistics.py `EMAMeanStd`, in a numpy dtype: float32 is the reference's own arithmetic.

`loss_and_grads` is the learner step's loss with PopArt, steps 1-9 of the composition the kernels implement
(generalized_onpolicy_loss.py:94-133,169-199 around a V-trace advantage estimator), with its analytic
gradients, in a numpy dtype (float64: the yardstick of the GPU tests; float32: the rounding bar):

  1. m = mu1, s = clip(sqrt(mu2 - mu1^2), 1e-6, 1e6)
  2. u = s (sigma V + mu) + m over all T+1 rows
  3. V-trace on values u[:-1], bootstrap u[-1] -> vs, pg_adv; with an abandoned mask [T+1,B], the masked V-trace
     of tests/abandoned_float64_reference.py on abandoned[1:] (transition t masked iff row t+1 is abandoned), in
     float32 the same recursion with those transitions masked
  4. n = (vs - m) / s, a = pg_adv / s
  5. mu1' = mu1 + beta (mean vs - mu1), mu2' = mu2 + beta (mean vs^2 - mu2), over all replicas
  6. sigma+ = (s / s') sigma, mu+ = (m - m' + s mu) / s'
  7. losses: policy -mean(log pi(a) a); value bc 0.5 mean(e^2), e = n - (sigma+ V + mu+) on rows [:-1]
  8. dlogits with a for pg_adv; dV = -bc e sigma+ / N (last row 0); d sigma = -bc mean(e V), d mu = -bc mean(e)
"""
import numpy as np

import abandoned_float64_reference as AR
import vtrace_float64_reference as RF


class PopArt(object):
  """popart.PopArt(running_statistics.EMAMeanStd(beta)) in numpy dtype FT; variables as attributes."""

  # the module's variables (popart_test.py test_variables: four, of which the compensation pair is trained)
  VARIABLES = ('first_moment', 'second_moment', 'compensation_std', 'compensation_mean')
  TRAINABLE = (False, False, True, True)

  def __init__(self, beta=1e-2, FT=np.float32, std_min_value=1e-6, std_max_value=1e6):
    self.FT = FT
    self.beta = FT(beta)
    self.std_min_value, self.std_max_value = std_min_value, std_max_value
    self.first_moment = FT(0)
    self.second_moment = FT(1)
    self.compensation_std = FT(1)
    self.compensation_mean = FT(0)

  def get_mean_std(self):                                       # running_statistics.py:149-153
    std = np.sqrt(self.FT(self.second_moment - self.first_moment ** 2))
    return self.first_moment, self.FT(np.clip(std, self.std_min_value, self.std_max_value))

  def normalize_target(self, x):
    m, s = self.get_mean_std()
    return ((np.asarray(x, self.FT) - m) / s).astype(self.FT)

  def normalize_advantage(self, x):
    return (np.asarray(x, self.FT) / self.get_mean_std()[1]).astype(self.FT)

  def correct_prediction(self, x):
    return (self.compensation_std * np.asarray(x, self.FT) + self.compensation_mean).astype(self.FT)

  def unnormalize_prediction(self, x):
    m, s = self.get_mean_std()
    return (s * np.asarray(x, self.FT) + m).astype(self.FT)

  def update_from_means(self, batch_first_moment, batch_second_moment):
    """update_normalization_statistics given the global batch means of data and data^2."""
    mean1, std1 = self.get_mean_std()
    FT = self.FT
    self.first_moment = FT(self.first_moment + self.beta * (FT(batch_first_moment) - self.first_moment))
    self.second_moment = FT(self.second_moment + self.beta * (FT(batch_second_moment) - self.second_moment))
    mean2, std2 = self.get_mean_std()
    self.compensation_std = FT(std1 / std2 * self.compensation_std)
    self.compensation_mean = FT((mean1 - mean2 + std1 * self.compensation_mean) / std2)
    return mean2, std2

  def update_normalization_statistics(self, data):
    data = np.asarray(data, self.FT)
    return self.update_from_means(np.mean(data, dtype=self.FT), np.mean(data * data, dtype=self.FT))

  @property
  def state(self):
    return np.array([self.first_moment, self.second_moment, self.compensation_std, self.compensation_mean],
                    self.FT)


def _log_softmax(x):
  m = x.max(-1, keepdims=True)
  z = x - m
  return z - np.log(np.exp(z).sum(-1, keepdims=True))


def _masked_recursion(masked):
  """vtrace_float64_reference's recursion in dtype FT with no delta and no policy gradient at the transitions
  `masked` [T,B]: the rounding of the masked V-trace in float32."""
  def f(target_action_log_probs, behaviour_action_log_probs, discounts, rewards, values, bootstrap_value, FT,
        lambda_=1.0):
    rhos = np.exp(np.asarray(target_action_log_probs, FT) - np.asarray(behaviour_action_log_probs, FT))
    discounts, rewards, values = (np.asarray(a, FT) for a in (discounts, rewards, values))
    boot = np.asarray(bootstrap_value, FT)
    keep = (~masked).astype(FT)
    clipped = np.minimum(FT(1.0), rhos) * keep
    cs = np.minimum(FT(1.0), rhos) * FT(lambda_)
    deltas = clipped * (rewards + discounts * np.concatenate([values[1:], boot[None]], 0) - values)
    acc = np.zeros_like(boot)
    out = [None] * len(deltas)
    for i in range(len(deltas) - 1, -1, -1):
      acc = deltas[i] + discounts[i] * cs[i] * acc
      out[i] = acc
    vs = np.stack(out, 0) + values
    pg = clipped * (rewards + discounts * np.concatenate([vs[1:], boot[None]], 0) - values)
    return vs.astype(FT), pg.astype(FT)
  return f


def _vtrace(abandoned, FT):
  """Step 3's V-trace: vtrace_float64_reference's recursion; with a mask that has an abandoned transition, in
  float64 the masked definition of abandoned_float64_reference, in any other dtype the recursion with those
  transitions masked.  A mask without one is no mask, so that an all-false mask gives the unmasked composition
  bit for bit."""
  if abandoned is None or not np.asarray(abandoned, bool)[1:].any():
    return RF.vtrace_from_importance_weights
  masked = np.asarray(abandoned, bool)[1:]
  return AR.masked_vtrace(masked) if FT == np.float64 else _masked_recursion(masked)


def moment_sums(cfg, ll, lb, bl, act, rew, done, state, FT=np.float64, abandoned=None):
  """Steps 1-3 on one replica's batch: -> (sum vs, sum vs^2, vs, pg_adv, u).  abandoned: bool [T+1,B] or None."""
  mu1, mu2, sigma, mu = (FT(x) for x in state)
  s = FT(np.clip(np.sqrt(FT(mu2 - mu1 * mu1)), 1e-6, 1e6))
  m = mu1
  lb = np.asarray(lb, FT)
  u = s * (sigma * lb + mu) + m
  ll, bl = np.asarray(ll, FT), np.asarray(bl, FT)
  a = np.asarray(act)[:-1].astype(np.int64)
  r = np.asarray(rew, FT)[1:]
  if cfg.max_abs_reward:
    r = np.clip(r, -cfg.max_abs_reward, cfg.max_abs_reward).astype(FT)
  disc = (~np.asarray(done, bool)[1:]).astype(FT) * FT(cfg.discounting)
  tl = np.take_along_axis(_log_softmax(ll[:-1]), a[..., None], -1)[..., 0]
  blp = np.take_along_axis(_log_softmax(bl[:-1]), a[..., None], -1)[..., 0]
  vs, pg = _vtrace(abandoned, FT)(tl, blp, disc, r, u[:-1], u[-1], FT, lambda_=cfg.lambda_)
  return vs.sum(dtype=np.float64), (vs.astype(np.float64) ** 2).sum(), vs, pg, u


def loss_and_grads(cfg, ll, lb, bl, act, rew, done, ecp, state, beta, FT=np.float64, global_means=None,
                   abandoned=None):
  """Steps 1-9 in dtype FT.  state = (mu1, mu2, sigma, mu) before the step; global_means = (mean vs,
  mean vs^2) over every replica's batch (default: this batch alone); abandoned = bool [T+1,B] or None.
  Returns a dict: loss terms by their learner names, dlogits, dbaseline, dcomp = (d sigma, d mu), state
  (after the step), vs, pg_adv, and sums = (sum vs, sum vs^2, rows) of this batch."""
  mu1, mu2, sigma, mu = (FT(x) for x in state)
  ll, lb = np.asarray(ll, FT), np.asarray(lb, FT)
  T1, B, A = ll.shape
  T = T1 - 1
  N = T * B
  s1, s2, vs, pg, u = moment_sums(cfg, ll, lb, bl, act, rew, done, state, FT, abandoned)
  if global_means is None:
    global_means = (s1 / N, s2 / N)
  s = FT(np.clip(np.sqrt(FT(mu2 - mu1 * mu1)), 1e-6, 1e6))
  m = mu1
  n = (vs - m) / s
  adv = pg / s
  beta = FT(beta)
  mu1n = FT(mu1 + beta * (FT(global_means[0]) - mu1))
  mu2n = FT(mu2 + beta * (FT(global_means[1]) - mu2))
  sn = FT(np.clip(np.sqrt(FT(mu2n - mu1n * mu1n)), 1e-6, 1e6))
  sigma_n = FT(s / sn * sigma)
  mu_n = FT((m - mu1n + s * mu) / sn)
  V = lb[:-1]
  e = n - (sigma_n * V + mu_n)
  bc = FT(cfg.baseline_cost)
  # the policy, entropy and KL terms, as vtrace_float64_reference computes them
  a = np.asarray(act)[:-1].astype(np.int64)
  lsm = _log_softmax(ll[:-1])
  p = np.exp(lsm)
  tl = np.take_along_axis(lsm, a[..., None], -1)[..., 0]
  blp = np.take_along_axis(_log_softmax(np.asarray(bl, FT)[:-1]), a[..., None], -1)[..., 0]
  H = -(p * lsm).sum(-1)
  mul = FT(cfg.entropy_cost_adjustment_speed)
  ec = FT(np.exp(mul * FT(ecp)))
  policy = -np.mean(tl * adv, dtype=FT)
  mse = np.mean(e * e, dtype=FT)
  v_loss = bc * FT(0.5) * mse
  mean_h = np.mean(H, dtype=FT)
  entropy_loss = -ec * mean_h
  kl = blp - tl
  kl_loss = FT(cfg.kl_cost) * np.mean(kl, dtype=FT)
  adj = ec * (mean_h - FT(cfg.target_entropy)) if cfg.target_entropy else FT(0)
  dep = mul * ec * (mean_h - FT(cfg.target_entropy)) if cfg.target_entropy else FT(0)
  total = policy + v_loss + entropy_loss + kl_loss + adj
  onehot = np.zeros_like(p)
  np.put_along_axis(onehot, a[..., None], 1.0, -1)
  kc = FT(cfg.kl_cost)
  dl = np.zeros_like(ll)
  dl[:-1] = (-(adv + kc) / FT(N))[..., None] * (onehot - p) + (ec / FT(N)) * p * (lsm + H[..., None])
  db = np.zeros_like(lb)
  db[:-1] = -bc * e * sigma_n / FT(N)
  dcomp = np.array([-bc * np.mean(e * V, dtype=FT), -bc * np.mean(e, dtype=FT)], FT)
  terms = {'total': total, 'policy': policy, 'V': v_loss, 'entropy': entropy_loss, 'kl': kl_loss,
           'entropy_adj': adj, 'v_mean': np.mean(u[:-1], dtype=FT), 'v_l2_error': np.sqrt(mse),
           'mean_entropy': mean_h, 'entropy_cost': ec, 'mean_kl': np.mean(kl, dtype=FT),
           'max_action_abs': float(np.abs(a).max()), 'popart_mean': mu1n, 'popart_std': sn}
  return dict(terms=terms, dlogits=dl, dbaseline=db, dcomp=dcomp, d_entropy_cost_param=dep,
              state=np.array([mu1n, mu2n, sigma_n, mu_n], FT), vs=vs, pg_adv=pg, td=(vs - u[:-1]) / s,
              u=u, n=n, adv=adv, e=e, sums=np.array([s1, s2, N], np.float64))
