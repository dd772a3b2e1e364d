"""CPU ORACLE (test infrastructure, NOT product code) of the opt-in Retrace(lambda) targets of the R2D2
learner: the targets, h and the loss in float64.

Retrace (Munos et al. 2016) is not in the reference.  The target policy is greedy in the online network
(a* = argmax_a Q_online, first maximum, as the double-DQN argmax of learner.py:298-305), so the trace is
c_i = lambda 1[a_i = a*_i].  Everything else -- value rescaling, the indexing of the targets against
replay_q, priorities, loss -- is the reference's compute_loss_and_priorities_from_agent_outputs
(agents/r2d2/learner.py:258-330).  The targets are written as the explicit sum, not the recursion the
kernel runs, and are pinned (tests/test_r2d2_retrace.py) to the unmodified reference
n_step_bellman_target in its two reductions (tests/golden/make_golden_r2d2_retrace.py) and to a
hand-computed case.  `CpuR2D2Learner` extends oracle.r2d2_learner_oracle's learner to either rule.
"""
import collections

import numpy as np
import torch

from oracle import r2d2_learner_oracle as RL, r2d2_oracle as R

F64 = np.float64


def value_function_rescaling(x, eps=1e-3):
  x = np.asarray(x, F64)
  return np.sign(x) * (np.sqrt(np.abs(x) + 1.) - 1.) + eps * x


def retrace_targets(reward, done, q_star, q_act, greedy, gamma, lam):
  """[T,B] inputs, row i of reward / done being the transition into x_i.  Returns Y [T,B]:
      Y[i] = sum_{j>=i} (prod_{k=i}^{j-1} g_k c_k) (r_j + g_j (q*_j - c_j qa_j)),
  g_k = gamma (1 - done_k), c_k = lam 1[greedy_k], c_{T-1} = 0 (nothing is known past the last row)."""
  r = np.asarray(reward, F64)
  g = gamma * (1. - np.asarray(done, F64))
  c = lam * np.asarray(greedy, F64)
  c[-1] = 0.
  qs, qa = np.asarray(q_star, F64), np.asarray(q_act, F64)
  T = r.shape[0]
  y = np.zeros_like(r)
  for i in range(T):
    for j in range(i, T):
      y[i] += np.prod(g[i:j] * c[i:j], axis=0) * (r[j] + g[j] * (qs[j] - c[j] * qa[j]))
  return y


def rescaled_targets(train_q, target_q, replay_action, reward, done, gamma, lam, eps=1e-3):
  """h(Y[1:]) [T-1,B]: the targets matched against replay_q[:-1] (learner.py:316-322)."""
  train_q = np.asarray(train_q)
  T, B, A = train_q.shape
  tt, bb = np.meshgrid(np.arange(T), np.arange(B), indexing='ij')
  a_star = train_q.argmax(-1)
  a = np.clip(np.asarray(replay_action), 0, A - 1)
  # h^-1 of the target network's values as the reference evaluates it, in fp32 (the pinned restatement):
  # (sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps) cancels, so its fp32 rounding is part of the definition
  gq = np.asarray(target_q, np.float32)
  y = retrace_targets(reward, done, R.inverse_value_function_rescaling(gq[tt, bb, a_star], eps),
                      R.inverse_value_function_rescaling(gq[tt, bb, a], eps), a == a_star, gamma, lam)
  return value_function_rescaling(y[1:], eps)


def loss_and_priorities(train_q, target_q, replay_action, reward, done, gamma, lam, eta=0.9, eps=1e-3,
                        importance_weights=None):
  """Returns (loss [B], priorities [B], td [T-1,B], dq [T,B,A]) in float64; dq is the gradient of
  mean_b(w_b loss_b) w.r.t. train_q."""
  tq = np.asarray(train_q, F64)
  T, B, A = tq.shape
  a = np.clip(np.asarray(replay_action), 0, A - 1)
  tt, bb = np.meshgrid(np.arange(T - 1), np.arange(B), indexing='ij')
  td = rescaled_targets(train_q, target_q, a, reward, done, gamma, lam, eps) - tq[tt, bb, a[:-1]]
  abs_td = np.abs(td)
  priorities = eta * abs_td.max(axis=0) + (1. - eta) * abs_td.mean(axis=0)
  loss = 0.5 * np.square(td).sum(axis=0)
  w = np.ones(B) if importance_weights is None else np.asarray(importance_weights, F64)
  dq = np.zeros((T, B, A))
  dq[tt, bb, a[:-1]] = -(w[None] / B) * td
  return loss, priorities, td, dq


def compute_loss_and_priorities(p_train, p_target, batch, A, stack_size, gamma, burn_in, n_steps=5, eps=1e-3,
                                bellman_target='n_step', retrace_lambda=0.95):
  """oracle.r2d2_learner_oracle.compute_loss_and_priorities with the target rule selectable."""
  if bellman_target == 'n_step':
    return RL.compute_loss_and_priorities(p_train, p_target, batch, A, stack_size, gamma, burn_in, n_steps, eps)
  if bellman_target != 'retrace':
    raise ValueError(bellman_target)
  fs = batch['frame_state'] if stack_size > 1 else ()
  state = RL.N.AgentState((torch.as_tensor(batch['h0']), torch.as_tensor(batch['c0'])), fs)
  if burn_in:
    pre, suf = RL._split(batch, burn_in)
    with torch.no_grad():
      _, train_state = RL._unroll(p_train, pre, state, A, stack_size)
      _, target_state = RL._unroll(p_target, pre, state, A, stack_size)
  else:
    suf = batch
    train_state = target_state = state
  train_out, _ = RL._unroll(p_train, suf, train_state, A, stack_size)
  with torch.no_grad():
    target_out, _ = RL._unroll(p_target, suf, target_state, A, stack_size)
  q = train_out.q_values
  tq, gq = q.detach().numpy(), target_out.q_values.numpy()
  loss_np, prio, td, _ = loss_and_priorities(tq, gq, suf['action'], suf['reward'], suf['done'], gamma,
                                             retrace_lambda, eps=eps)
  target = rescaled_targets(tq, gq, suf['action'], suf['reward'], suf['done'], gamma, retrace_lambda, eps)
  replay_q = torch.gather(q, 2, torch.as_tensor(np.asarray(suf['action'])).long()[..., None])[..., 0][:-1]
  td_t = torch.as_tensor(target.astype(np.float32)) - replay_q
  loss = 0.5 * (td_t * td_t).sum(dim=0)
  return loss, prio.astype(np.float32), dict(q=q, target_q=target_out.q_values, loss_np=loss_np, abs_td=np.abs(td))


class CpuR2D2Learner(RL.CpuR2D2Learner):
  """oracle.r2d2_learner_oracle.CpuR2D2Learner with `bellman_target` 'n_step' or 'retrace'."""

  def __init__(self, *args, bellman_target='n_step', retrace_lambda=0.95, **kw):
    super(CpuR2D2Learner, self).__init__(*args, **kw)
    self.bellman_target, self.retrace_lambda = bellman_target, retrace_lambda

  def grads(self, batch):
    for t in self.params.values():
      t.grad = None
    loss, prio, aux = compute_loss_and_priorities(self.params, self.target, batch, self.A, self.stack, self.gamma,
                                                  self.burn_in, self.n_steps, bellman_target=self.bellman_target,
                                                  retrace_lambda=self.retrace_lambda)
    total = (loss * torch.as_tensor(batch['importance_weights'])).mean()
    total.backward()
    g = collections.OrderedDict((k, v.grad.numpy().copy()) for k, v in self.params.items())
    norm = float(np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g.values())))
    return float(total.detach()), loss.detach().numpy(), prio, g, norm, aux
