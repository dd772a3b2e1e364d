"""CPU reference (test infrastructure, not product code) of one whole R2D2 learner step in float32 or float64,
optionally conditioned on the discrete decisions of another implementation.

It is oracle/r2d2_learner_oracle.py's step -- burn-in prefix unrolled by both networks without gradient, suffix
by both, n-step double-DQN loss on the suffix, importance-weighted mean, global-norm clip, one Keras Adam step --
composed from the same pieces (oracle/r2d2_net_oracle.py's layer list and LSTM cell, net_oracle._conv_nhwc,
r2d2_oracle.stack_frames, optim_oracle.keras_adam_step), with two differences:

  * the network, the value rescaling h and h^-1, the n-step target, the loss, the priorities and the clip scale
    are evaluated in `dtype` (float32 or float64); tests/test_r2d2_float64_reference.py pins the float32 form to
    the oracle.  h and h^-1 take the oracle's literal formulas in float32 and a form without cancellation in
    float64 (see value_function_rescaling below);
  * the step is piecewise smooth, and its pieces can be chosen from outside.  Every ReLU of the gradient-carrying
    suffix unroll of the online network is evaluated as z * mask, with mask = z > 0 by default or the given
    `masks[name]` (MASKS: the three convolutions, the body Dense, the value and advantage hidden layers), and the
    double-DQN target takes the given `greedy` action [T, B] instead of the argmax of the online q.  Given the
    decisions a GPU step made (its ReLU outputs > 0, the first maximum of its q), the reference is a smooth
    function of the parameters and the inputs, so its distance to that step measures arithmetic alone.

`forward` is the network part alone over T >= 1 steps (central inference: T = 1), conditioned the same way, and
`priorities` the initial priorities central inference computes from a completed unroll's behaviour q.

The forward values of a ReLU are continuous through its kink, so the burn-in unrolls and the target network need
no conditioning: they always use their own masks.
"""
import collections

import numpy as np
import torch

from oracle import net_oracle, optim_oracle, r2d2_net_oracle as N, r2d2_oracle as R

MASKS = ('conv0', 'conv1', 'conv2', 'dense', 'value', 'advantage')


class _Relu(object):
  """z * mask, mask = z > 0 or the given one; records the masks it used ([rows, ...] bool numpy), the
  pre-activations (`acts`) and, where a given mask differs from z > 0, |z| there (`ties`)."""

  def __init__(self, given=None):
    self.given, self.used, self.acts, self.ties = given, {}, {}, {}

  def __call__(self, name, z):
    own = z.detach() > 0
    if self.given is None:
      m = own
    else:
      m = torch.as_tensor(np.asarray(self.given[name], bool))
      if tuple(m.shape) != tuple(z.shape):
        raise ValueError('mask %s has shape %s, the layer %s' % (name, tuple(m.shape), tuple(z.shape)))
      self.ties[name] = z.detach()[m != own].abs().numpy()
    self.used[name] = m.numpy()
    self.acts[name] = z.detach().numpy()
    return z * m.to(z.dtype)


def _plain_relu(_, z):
  return torch.relu(z)


# _torso and _head restate r2d2_net_oracle.torso / head with the ReLU made pluggable (the masks need it): a change
# to the oracle's layers must be mirrored here.  test_float32_reference_is_the_oracle_step pins them bit for bit.
def _torso(p, prev_action, reward, frames01, A, relu):
  x = frames01
  for i, (_, _, s) in enumerate(N.CONVS):
    x = relu('conv%d' % i, net_oracle._conv_nhwc(x, p['body/conv%d/kernel' % i], p['body/conv%d/bias' % i], s, False))
  x = x.reshape(x.shape[0], -1)
  x = relu('dense', x @ p['body/dense/kernel'] + p['body/dense/bias'])
  one_hot = torch.nn.functional.one_hot(prev_action.long(), A).to(x.dtype)
  return torch.cat([x, reward[:, None], one_hot], dim=1)


def _head(p, core, relu):
  value = relu('value', core @ p['value/hidden/kernel'] + p['value/hidden/bias']) @ p['value/head/kernel'] + \
      p['value/head/bias']
  adv = relu('advantage', core @ p['advantage/hidden/kernel'] + p['advantage/hidden/bias']) @ \
      p['advantage/head/kernel']
  return value + (adv - adv.mean(dim=-1, keepdim=True))


def _unroll(p, part, state, A, stack_size, dtype, relu):
  """r2d2_net_oracle.unroll in `dtype` with the ReLUs of `relu`: -> (q [T,B,A], (h, c, frame_state))."""
  T, B = part['prev_actions'].shape
  stacked, frame_state = R.stack_frames(np.asarray(part['observation']).astype(np.float32), state[2],
                                        np.asarray(part['done'], bool), stack_size)
  x = torch.as_tensor(stacked).to(dtype) / 255
  tor = _torso(p, torch.as_tensor(np.asarray(part['prev_actions'])).reshape(T * B),
               torch.as_tensor(np.asarray(part['reward'])).to(dtype).reshape(T * B),
               x.reshape((T * B,) + tuple(x.shape[2:])), A, relu).reshape(T, B, -1)
  h, c = state[0], state[1]
  d_all = torch.as_tensor(np.asarray(part['done'], bool))
  outs = []
  for t in range(T):
    d = d_all[t][:, None]
    h = torch.where(d, torch.zeros_like(h), h)
    c = torch.where(d, torch.zeros_like(c), c)
    h, c = N.lstm_cell(p, tor[t], h, c)
    outs.append(h)
  q = _head(p, torch.stack(outs).reshape(T * B, -1), relu)
  return q.reshape(T, B, A), (h, c, frame_state)


# ---- the post-network arithmetic of r2d2_oracle, in a given numpy dtype ------------------------------------------
# h and h^-1 in two algebraically equal forms.  The literal one is the reference's text (r2d2_oracle's): in float32
# both of its subtractions cancel, sqrt(|x| + 1) - 1 for small |x| and, with eps = 1e-3, first sqrt(...) - 1 ~ 2e-3
# and then inner^2 - 1, so h^-1 keeps ~11 good bits near 0.  The stable one has no subtraction of nearly equal
# numbers; it is what seed_rl_b200/csrc/r2d2_thread.inl computes, in the same order of operations.  In float32 the
# module's step is the oracle's, so it uses the literal form; in float64 it is the function itself, the stable form.
def literal_value_function_rescaling(x, eps, F):
  """h(x) = sign(x) (sqrt(|x| + 1) - 1) + eps x."""
  x = np.asarray(x, F)
  return (np.sign(x) * (np.sqrt(np.abs(x) + F(1.)) - F(1.)) + F(eps) * x).astype(F)


def literal_inverse_value_function_rescaling(x, eps, F):
  """h^-1(x) = sign(x) (((sqrt(1 + 4 eps (|x| + 1 + eps)) - 1) / (2 eps))^2 - 1)."""
  x = np.asarray(x, F)
  e = F(eps)
  inner = (np.sqrt(F(1.) + F(4.) * e * (np.abs(x) + F(1.) + e)) - F(1.)) / (F(2.) * e)
  return (np.sign(x) * (np.square(inner) - F(1.))).astype(F)


def stable_value_function_rescaling(x, eps, F):
  """h(x) = sign(x) |x| / (sqrt(|x| + 1) + 1) + eps x; +-inf map to themselves."""
  x = np.asarray(x, F)
  a = np.abs(x)
  with np.errstate(invalid='ignore'):
    m = np.where(a < F(np.inf), a / (np.sqrt(a + F(1.)) + F(1.)), a).astype(F)
  return (np.sign(x) * m + F(eps) * x).astype(F)


def stable_inverse_value_function_rescaling(x, eps, F):
  """h^-1(x) = sign(x) d (2 + d), d = 2 |x| / (s + 1 + 2 eps), s = sqrt(1 + 4 eps (|x| + 1 + eps)): since
  s^2 = (1 + 2 eps)^2 + 4 eps |x|, s - 1 - 2 eps = 4 eps |x| / (s + 1 + 2 eps), so the literal inner - 1 is d and
  inner^2 - 1 = d (2 + d).  +-inf map to themselves."""
  x = np.asarray(x, F)
  e = F(eps)
  a = np.abs(x)
  s = np.sqrt(F(1.) + F(4.) * e * (a + F(1.) + e))
  with np.errstate(invalid='ignore', over='ignore'):
    d = np.where(a < F(np.inf), F(2.) * a / (s + F(1.) + F(2.) * e), a).astype(F)
    return (np.sign(x) * (d * (F(2.) + d))).astype(F)


def value_function_rescaling(x, eps, F):
  f = literal_value_function_rescaling if F == np.float32 else stable_value_function_rescaling
  return f(x, eps, F)


def inverse_value_function_rescaling(x, eps, F):
  f = literal_inverse_value_function_rescaling if F == np.float32 else stable_inverse_value_function_rescaling
  return f(x, eps, F)


def n_step_bellman_target(rewards, done, q_target, gamma, n_steps, F):
  rewards = np.asarray(rewards, F); q_target = np.asarray(q_target, F)
  done = np.asarray(done, bool)
  g = F(gamma)
  target = np.concatenate([np.zeros_like(q_target[0:1]), q_target] +
                          [q_target[-1:] / F(gamma ** k) for k in range(1, n_steps)], axis=0)
  done = np.concatenate([done] + [np.zeros_like(done[0:1])] * n_steps, axis=0)
  rewards = np.concatenate([rewards] + [np.zeros_like(rewards[0:1])] * n_steps, axis=0)
  for _ in range(n_steps):
    rewards = rewards[:-1]
    done = done[:-1]
    target = (rewards + g * (F(1.) - done.astype(F)) * target[1:]).astype(F)
  return target


def n_step_targets(target_q, greedy, reward, done, st, F):
  """The rescaled n-step double-DQN targets of rows 0..T-2: target_q [T,B,A] at the greedy actions [T,B]."""
  T, B = np.shape(greedy)
  tt, bb = np.meshgrid(np.arange(T), np.arange(B), indexing='ij')
  qtarget_max = inverse_value_function_rescaling(np.asarray(target_q)[tt, bb, greedy], st.eps, F)
  return value_function_rescaling(n_step_bellman_target(reward, done, qtarget_max, st.gamma, st.n_steps, F)[1:],
                                  st.eps, F)


def priorities(q, target_q, action, reward, done, greedy, st, F):
  """The step's priorities [B] from given q-values alone (numpy, in F): the initial priorities of a completed
  unroll, which central inference computes with q = target_q = the behaviour q of the suffix."""
  q = np.asarray(q, F)
  T, B = np.shape(greedy)
  td = n_step_targets(target_q, greedy, reward, done, st, F) - np.take_along_axis(
      q, np.asarray(action).astype(np.int64)[..., None], axis=2)[:-1, :, 0]
  abs_td = np.abs(td).astype(F)
  return (F(st.eta) * abs_td.max(axis=0) + F(1 - st.eta) * abs_td.mean(axis=0, dtype=F)).astype(F)


def forward(params, inputs, num_actions, stack_size, dtype=torch.float64, masks=None):
  """The network's forward over T >= 1 steps (central inference: T = 1), without gradients.  inputs:
  prev_actions, reward, done [T,B], observation uint8 [T,B,H,W,1], h0 / c0 [B,512] (any float dtype) and, when
  stack_size > 1, frame_state int32 [B, H*W]; masks as in `step` (rows = the T * B frames, time-major).
  Returns a dict: q [T,B,A], h, c, frame_state (the state after the last step), acts (the ReLU inputs), masks
  and ties (see _Relu)."""
  p = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in params.items()}
  state = (torch.as_tensor(np.asarray(inputs['h0'])).to(dtype), torch.as_tensor(np.asarray(inputs['c0'])).to(dtype),
           inputs['frame_state'] if stack_size > 1 else ())
  relu = _Relu(masks)
  with torch.no_grad():
    q, (h, c, fs) = _unroll(p, inputs, state, num_actions, stack_size, dtype, relu)
  return dict(q=q.numpy(), h=h.numpy(), c=c.numpy(), frame_state=fs, acts=relu.acts, masks=relu.used,
              ties=relu.ties)


# ---- the step ----------------------------------------------------------------------------------------------------
Settings = collections.namedtuple('Settings', 'num_actions stack_size gamma burn_in n_steps eps clip_norm lr '
                                              'adam_eps eta')


def settings(num_actions, stack_size, learner_settings, lr, adam_eps):
  """From seed_rl_b200.agents.r2d2.learner.R2D2Settings and the optimizer's lr / epsilon."""
  s = learner_settings
  return Settings(num_actions, stack_size, s.discounting, s.burn_in, s.n_steps, s.value_function_rescaling_epsilon,
                  s.clip_norm, lr, adam_eps, 0.9)


def step(params, target_params, batch, st, dtype=torch.float64, masks=None, greedy=None):
  """One learner step.  params / target_params: {name: array} (any float dtype; evaluated in `dtype`);
  batch: r2d2_learner_oracle.synthetic_replay_batch's fields (h0 / c0 of any float dtype); st: Settings.
  masks: None or {MASKS name: bool [T*B, ...] (rows time-major) of the suffix unroll}; greedy: None or int [T, B].
  Returns a dict: q, target_q [T,B,A], dq [T,B,A] (d total / d q), loss_b [B], total, priorities [B], grads
  {name: array} (before the clip), norm (before the clip), scale (the clip's factor), params_after {name: fp32}
  (one Keras Adam step from zero slots with the clipped gradients), update {name: float64} (params - params_after
  before the fp32 rounding of the subtraction), masks and greedy (the decisions used)."""
  F = np.float64 if dtype == torch.float64 else np.float32
  A = st.num_actions
  p = collections.OrderedDict((k, torch.as_tensor(np.asarray(v)).to(dtype).requires_grad_(True))
                              for k, v in params.items())
  tp = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in target_params.items()}
  keys = ('observation', 'reward', 'done', 'prev_actions', 'action')
  pre = {k: batch[k][:st.burn_in] for k in keys}
  suf = {k: batch[k][st.burn_in:] for k in keys}
  fs = batch['frame_state'] if st.stack_size > 1 else ()
  state = (torch.as_tensor(np.asarray(batch['h0'])).to(dtype), torch.as_tensor(np.asarray(batch['c0'])).to(dtype), fs)
  with torch.no_grad():
    _, train_state = _unroll(p, pre, state, A, st.stack_size, dtype, _plain_relu)
    _, target_state = _unroll(tp, pre, state, A, st.stack_size, dtype, _plain_relu)
  relu = _Relu(masks)
  q, _ = _unroll(p, suf, train_state, A, st.stack_size, dtype, relu)
  q.retain_grad()
  with torch.no_grad():
    qt, _ = _unroll(tp, suf, target_state, A, st.stack_size, dtype, _plain_relu)
  T, B = q.shape[0], q.shape[1]
  qn, qtn = q.detach().numpy(), qt.numpy()
  a_star = qn.argmax(-1) if greedy is None else np.asarray(greedy)
  if a_star.shape != (T, B):
    raise ValueError('greedy must be [%d, %d]' % (T, B))
  target = n_step_targets(qtn, a_star, suf['reward'], suf['done'], st, F)
  replay_q = torch.gather(q, 2, torch.as_tensor(np.asarray(suf['action'])).long()[..., None])[..., 0][:-1]
  td = torch.as_tensor(target) - replay_q
  loss = 0.5 * (td * td).sum(dim=0)
  total = (loss * torch.as_tensor(np.asarray(batch['importance_weights'])).to(dtype)).mean()
  total.backward()
  abs_td = np.abs(td.detach().numpy()).astype(F)
  prio = (F(st.eta) * abs_td.max(axis=0) + F(1 - st.eta) * abs_td.mean(axis=0, dtype=F)).astype(F)
  g = collections.OrderedDict((k, v.grad.numpy().copy()) for k, v in p.items())
  norm = float(np.sqrt(sum(float((x.astype(np.float64) ** 2).sum()) for x in g.values())))
  scale = F(st.clip_norm / max(norm, st.clip_norm)) if st.clip_norm else F(1)
  after, update = collections.OrderedDict(), collections.OrderedDict()
  for k, v in p.items():
    z = np.zeros(tuple(v.shape), np.float32)
    after[k] = optim_oracle.keras_adam_step(v.detach().numpy(), g[k] * scale, z, z, 0, st.lr, eps=st.adam_eps)[0]
    # the step itself, without the rounding of storing p - step in fp32
    update[k] = -optim_oracle.keras_adam_step(z, g[k] * scale, z, z, 0, st.lr, eps=st.adam_eps)[0].astype(np.float64)
  return dict(q=qn, target_q=qtn, dq=q.grad.numpy().copy(), loss_b=loss.detach().numpy(), total=float(total.detach()),
              priorities=prio, grads=g, norm=norm, scale=float(scale), params_after=after, update=update,
              masks=relu.used, greedy=a_star)


def perturbed(params, target_params, batch, delta, seed=0):
  """Every parameter of both networks, h0 and c0 multiplied by 1 + delta N(0, 1) (float64)."""
  rng = np.random.default_rng(seed)
  f = lambda v: np.asarray(v, np.float64) * (1. + delta * rng.normal(size=np.shape(v)))
  p = collections.OrderedDict((k, f(v)) for k, v in params.items())
  tp = collections.OrderedDict((k, f(v)) for k, v in target_params.items())
  b = dict(batch, h0=f(batch['h0']), c0=f(batch['c0']))
  return p, tp, b
