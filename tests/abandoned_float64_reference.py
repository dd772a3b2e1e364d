"""Float64 reference of the abandoned-episode semantics of the V-trace and R2D2 losses
(seedrl_vtrace_loss_fwd_bwd_abandoned, seedrl_r2d2_loss_fwd_bwd_abandoned,
seedrl_r2d2_retrace_loss_fwd_bwd_abandoned in include/seedrl_b200.h).

An abandoned row marks the transition into it as not real: a time limit ended the episode and the row holds
the reset observation (its `done` is set too).  Transition t is masked iff row t+1 is abandoned.

Written from the definitions, not from the kernels' recursions: the V-trace targets as the explicit sum
vs_t = V_t + sum_{s>=t} (prod_{t<=k<s} d_k c_k) delta_s, the n-step targets as a forward walk over the window,
Retrace as its backward recursion.  Pinned to the reference's own advantages.vtrace and advantages.NStep by
tests/golden/abandoned_golden.npz (tests/test_abandoned.py)."""
import numpy as np

F = np.float64


def vtrace(log_rhos, discounts, rewards, values, bootstrap_value, abandoned, clip_rho_threshold=1.0,
           clip_pg_rho_threshold=1.0, lambda_=1.0):
  """V-trace on [T,B] inputs in the indexing of common/vtrace.py (rewards / discounts of transition t),
  with abandoned [T,B] = abandoned[t+1] of the learner's [T+1,B] column: -> (vs, pg_advantages)."""
  log_rhos, discounts, rewards, values = (np.asarray(a, F) for a in (log_rhos, discounts, rewards, values))
  boot = np.asarray(bootstrap_value, F)
  masked = np.asarray(abandoned, bool)
  T = log_rhos.shape[0]
  rhos = np.exp(log_rhos)
  crho = np.minimum(clip_rho_threshold, rhos) if clip_rho_threshold is not None else rhos
  cpg = np.minimum(clip_pg_rho_threshold, rhos) if clip_pg_rho_threshold is not None else rhos
  cs = np.minimum(1.0, rhos) * lambda_
  v_next = np.concatenate([values[1:], boot[None]], 0)
  delta = np.where(masked, 0.0, crho * (rewards + discounts * v_next - values))
  vs = values.copy()
  for t in range(T):
    w = np.ones_like(boot)
    for s in range(t, T):
      vs[t] += w * delta[s]
      w = w * discounts[s] * cs[s]
  vs_next = np.concatenate([vs[1:], boot[None]], 0)
  pg = np.where(masked, 0.0, cpg * (rewards + discounts * vs_next - values))
  return vs, pg


def masked_vtrace(abandoned_next):
  """A stand-in for vtrace_float64_reference.vtrace_from_importance_weights (same signature) that applies
  the mask abandoned_next [T,B]: lets that module's loss and learner step run with abandoned rows."""
  def f(target_action_log_probs, behaviour_action_log_probs, discounts, rewards, values, bootstrap_value, FT,
        clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0, lambda_=1.0):
    lr = np.asarray(target_action_log_probs, F) - np.asarray(behaviour_action_log_probs, F)
    vs, pg = vtrace(lr, discounts, rewards, values, bootstrap_value, abandoned_next, clip_rho_threshold,
                    clip_pg_rho_threshold, lambda_)
    return vs.astype(FT), pg.astype(FT)
  return f


def h(x, eps):
  x = np.asarray(x, F)
  return np.sign(x) * (np.sqrt(np.abs(x) + 1.0) - 1.0) + eps * x


def h_inv(x, eps):
  x = np.asarray(x, F)
  return np.sign(x) * (np.square((np.sqrt(1.0 + 4.0 * eps * (np.abs(x) + 1.0 + eps)) - 1.0) / (2.0 * eps)) - 1.0)


def n_step_targets(q_star, reward, done, abandoned, gamma, n):
  """Targets of rows 1..T-1 (the target of transition t is row t+1), before h: q_star, reward, done,
  abandoned [T,B] with row i = the transition into x_i.  Walk i = t+1 .. t+n: an abandoned row stops with
  G + gamma^(i-1-t) q*_{i-1}; else G += gamma^(i-1-t) r_i, and a terminated row stops with G; past the
  window, G + gamma^n q*_{t+n}, where rows past the unroll's end have reward 0, no done, and q*_{T-1}
  discounted by their distance (the reference's padding)."""
  q_star, reward = np.asarray(q_star, F), np.asarray(reward, F)
  done, ab = np.asarray(done, bool), np.asarray(abandoned, bool)
  T, B = q_star.shape
  out = np.zeros((T - 1, B), F)
  for b in range(B):
    for t in range(T - 1):
      G, disc, tgt = 0.0, 1.0, None
      for i in range(t + 1, t + n + 1):
        if i < T:
          if ab[i, b]:
            tgt = G + disc * q_star[i - 1, b]
            break
          G += disc * reward[i, b]
          if done[i, b]:
            tgt = G
            break
        disc *= gamma
      if tgt is None:
        j = t + n
        tgt = G + (disc * q_star[j, b] if j < T else gamma ** (T - 1 - t) * q_star[T - 1, b])
      out[t, b] = tgt
  return out


def retrace_targets(q_star, q_act, greedy_taken, reward, done, abandoned, gamma, lam):
  """Retrace targets Y of rows 1..T-1 (target policy greedy in the online network, c_i = lam 1[a_i = a*_i]):
  Y[T-1] = r + g q*_{T-1}; Y[i] = r_i + g_i (q*_i + c_i (Y[i+1] - qa_i)), or r_i + g_i q*_i when row i+1 is
  abandoned; g_i = gamma (1 - done_i)."""
  q_star, q_act, reward = (np.asarray(a, F) for a in (q_star, q_act, reward))
  done, ab = np.asarray(done, bool), np.asarray(abandoned, bool)
  T, B = q_star.shape
  Y = np.zeros((T, B), F)
  for i in range(T - 1, 0, -1):
    v = q_star[i].copy()
    if i + 1 < T:
      c = lam * np.asarray(greedy_taken[i], F)
      v = np.where(ab[i + 1], v, v + c * (Y[i + 1] - q_act[i]))
    Y[i] = reward[i] + gamma * (1.0 - done[i]) * v
  return Y[1:]


def r2d2_loss(q_train, q_target, action, reward, done, abandoned, gamma, rule, param, eta=0.9, eps=1e-3,
              weights=None):
  """-> dict(targets [T-1,B] (rescaled), td, loss [B], priorities [B], dq [T,B,A]) of the R2D2 loss with
  the n-step (param = n) or Retrace (param = lambda) targets; greedy a* = argmax q_train (first maximum)."""
  q_train, q_target = np.asarray(q_train, F), np.asarray(q_target, F)
  action = np.asarray(action, np.int64)
  T, B, A = q_train.shape
  ab = np.asarray(abandoned, bool) if abandoned is not None else np.zeros((T, B), bool)
  greedy = np.asarray(q_train, np.float32).argmax(-1)
  q_star = h_inv(np.take_along_axis(q_target, greedy[..., None], -1)[..., 0], eps)
  if rule == 'n_step':
    y = n_step_targets(q_star, reward, done, ab, gamma, int(param))
  else:
    q_act = h_inv(np.take_along_axis(q_target, action[..., None], -1)[..., 0], eps)
    y = retrace_targets(q_star, q_act, greedy == action, reward, done, ab, gamma, float(param))
  tgt = h(y, eps)
  rq = np.take_along_axis(q_train, action[..., None], -1)[..., 0][:-1]
  td = np.where(ab[1:], 0.0, tgt - rq)
  w = np.ones(B, F) if weights is None else np.asarray(weights, F)
  dq = np.zeros((T, B, A), F)
  tt, bb = np.meshgrid(np.arange(T - 1), np.arange(B), indexing='ij')
  dq[tt, bb, action[:-1]] = -(w / B)[None] * td
  a = np.abs(td)
  return dict(targets=tgt, td=td, loss=0.5 * (td * td).sum(0), priorities=eta * a.max(0) + (1 - eta) * a.mean(0),
              dq=dq)


# ---- test inputs ------------------------------------------------------------------------------------------------
def masks(T1, B, seed, p_done=0.1, p_abandoned=0.05):
  """done, abandoned bool [T1,B]: random rows, plus abandoned rows at the first, an interior and the last
  transition, next to terminated rows; every abandoned row is done (the inference host guarantees it)."""
  rng = np.random.default_rng(seed)
  done = rng.random((T1, B)) < p_done
  ab = rng.random((T1, B)) < p_abandoned
  ab[1, 0] = True
  ab[T1 - 1, 1 % B] = True
  k = min(max(T1 // 2, 1), T1 - 1)
  ab[k, 2 % B] = True
  done[k - 1, 2 % B] = True
  if k + 1 < T1:
    done[k + 1, 2 % B] = True
  return done | ab, ab


def r2d2_inputs(T, B, A, seed, p_greedy=0.7):
  """q_train, q_target [T,B,A], action int64 [T,B] (greedy in q_train with probability p_greedy), reward,
  done, abandoned [T,B], importance weights [B] (float32 / bool)."""
  rng = np.random.default_rng(seed)
  q = rng.normal(size=(T, B, A)).astype(np.float32)
  qt = (q + 0.3 * rng.normal(size=(T, B, A))).astype(np.float32)
  act = np.where(rng.random((T, B)) < p_greedy, q.argmax(-1), rng.integers(0, A, (T, B))).astype(np.int64)
  rew = rng.normal(size=(T, B)).astype(np.float32)
  done, ab = masks(T, B, seed + 1)
  w = rng.uniform(0.2, 1.0, B).astype(np.float32)
  return q, qt, act, rew, done, ab, w
