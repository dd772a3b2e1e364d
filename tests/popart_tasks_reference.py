"""Multi-task PopArt restated from tests/popart_reference.py, for the tests of --popart_tasks.

A multi-task step is K single-task PopArt steps, task k fed only the columns whose task id is k, with the loss
terms and gradients weighted by each task's share N_k / N of the T x B rows (every mean of the learner runs
over all rows).  Each task's moments move by the sums of its own rows over every replica (`global_sums`); a
task without rows anywhere keeps its state and has a zero compensation gradient.  In a numpy dtype: float64 is
the GPU tests' yardstick, float32 the rounding bar.
"""
import numpy as np

import popart_reference as PR

_MEAN_TERMS = ('total', 'policy', 'entropy', 'kl', 'entropy_adj', 'v_mean', 'mean_entropy', 'mean_kl')


def _columns(arrays, cols):
  """The columns `cols` of each [T1,B,...] array, C-contiguous: numpy's pairwise sums then run in the order
  they run on a whole batch, so one task reduces to popart_reference bit for bit."""
  return [np.ascontiguousarray(np.asarray(x)[:, cols]) for x in arrays]


def task_sums(cfg, ll, lb, bl, act, rew, done, states, task_ids, FT=np.float64, abandoned=None):
  """[K,3] float64 (sum vs, sum vs^2, rows) of one replica's batch, each task over its own columns (and its
  columns of the abandoned mask [T+1,B], if any)."""
  states = np.asarray(states)
  out = np.zeros((len(states), 3))
  T = np.asarray(ll).shape[0] - 1
  for k in range(len(states)):
    cols = np.nonzero(np.asarray(task_ids) == k)[0]
    if cols.size:
      sub = _columns((ll, lb, bl, act, rew, done) + (() if abandoned is None else (abandoned,)), cols)
      s1, s2 = PR.moment_sums(cfg, *sub[:6], states[k], FT, *sub[6:])[:2]
      out[k] = (s1, s2, T * cols.size)
  return out


def _updated(state, means, beta, FT):
  pa = PR.PopArt(beta, FT)
  pa.first_moment, pa.second_moment, pa.compensation_std, pa.compensation_mean = (FT(x) for x in state)
  pa.update_from_means(*means)
  return pa.state


def loss_and_grads(cfg, ll, lb, bl, act, rew, done, ecp, states, task_ids, beta, FT=np.float64, global_sums=None,
                   abandoned=None):
  """states [K,4] = (mu1, mu2, sigma, mu) per task before the step; task_ids [B]; global_sums [K,3] over every
  replica (default: this batch's task_sums); abandoned = bool [T+1,B] or None.  Returns what
  popart_reference.loss_and_grads returns, with dcomp [K,2], state [K,4] and sums [K,3] (this batch's)."""
  states = np.asarray(states, FT)
  K = len(states)
  task_ids = np.asarray(task_ids)
  ll = np.asarray(ll, FT)
  T1, B, A = ll.shape
  N = (T1 - 1) * B
  sums = task_sums(cfg, ll, lb, bl, act, rew, done, states, task_ids, FT, abandoned)
  if global_sums is None:
    global_sums = sums
  dl, db = np.zeros_like(ll), np.zeros((T1, B), FT)
  vs, pg, td, e, adv = (np.zeros((T1 - 1, B), FT) for _ in range(5))
  u = np.zeros((T1, B), FT)
  dcomp = np.zeros((K, 2), FT)
  new = states.copy()
  terms = dict((k, FT(0)) for k in _MEAN_TERMS)
  dep = FT(0)
  max_a = 0.0
  for k in range(K):
    cols = np.nonzero(task_ids == k)[0]
    n = global_sums[k, 2]
    means = (global_sums[k, 0] / n, global_sums[k, 1] / n) if n else None
    if cols.size == 0:
      if means is not None:
        new[k] = _updated(states[k], means, beta, FT)
      continue
    sub = _columns((ll, lb, bl, act, rew, done) + (() if abandoned is None else (abandoned,)), cols)
    r = PR.loss_and_grads(cfg, *sub[:6], ecp, states[k], beta, FT, global_means=means,
                          abandoned=sub[6] if abandoned is not None else None)
    w = FT(cols.size * (T1 - 1)) / FT(N)       # the task's share of the rows
    dl[:, cols] = r['dlogits'] * w
    db[:, cols] = r['dbaseline'] * w
    dcomp[k] = r['dcomp'] * w
    new[k] = r['state']
    for name in _MEAN_TERMS:
      terms[name] = terms[name] + w * FT(r['terms'][name])
    dep = dep + w * FT(r['d_entropy_cost_param'])
    max_a = max(max_a, r['terms']['max_action_abs'])
    terms['entropy_cost'] = r['terms']['entropy_cost']
    vs[:, cols], pg[:, cols], td[:, cols], e[:, cols], adv[:, cols] = r['vs'], r['pg_adv'], r['td'], r['e'], r['adv']
    u[:, cols] = r['u']
  mse = np.mean(e * e, dtype=FT)
  v_loss = FT(cfg.baseline_cost) * FT(0.5) * mse
  terms.update(V=v_loss, v_l2_error=np.sqrt(mse), max_action_abs=max_a)
  return dict(terms=terms, dlogits=dl, dbaseline=db, dcomp=dcomp, d_entropy_cost_param=dep, state=new,
              vs=vs, pg_adv=pg, td=td, e=e, adv=adv, u=u, sums=sums)
