"""CPU reference (test infrastructure, not product code) of one whole V-trace learner step in float32 or float64,
optionally conditioned on the discrete decisions of another implementation.

It is oracle/learner_oracle.py's step -- ImpalaDeep or ImpalaShallow unrolled over T+1 rows with done-resets,
compute_loss (log-softmax, V-trace, the five loss terms and the logged scalars), the gradient, one Keras Adam step
(beta_1 = 0) with the entropy_cost_param clamp -- composed from the same pieces (net_oracle._conv_nhwc and
lstm_cell, optim_oracle.keras_adam_step), with two differences:

  * the network, log-softmax, V-trace and the loss are evaluated in `dtype` (float32 or float64);
    tests/test_vtrace_float64_reference.py pins the float32 form to the oracle bit for bit;
  * the step is piecewise smooth, and its pieces can be chosen from outside.  Every ReLU is evaluated as z * mask,
    with mask = z > 0 by default or the given `masks[name]`, and every max-pool as a gather at a tap per pooled
    element and channel, the first maximum of its window by default or the given `taps[name]`.  The pool's
    backward scatters there with the same aten kernel F.max_pool2d's backward runs, so a reference conditioned on
    its own decisions is bit-equal to the unconditioned one.  Given the decisions a GPU step made, the reference
    is a smooth function of the parameters and inputs, and its distance to that step measures arithmetic alone.

Decision names (masks over the T+1 * B frames, time-major, NHWC or [rows, units]):
  ImpalaDeep     'stack<s>/p', 'stack<s>/c0', 'stack<s>/o0', 'stack<s>/c1' for s = 0..2 (the ReLUs of
                 dmlab/networks.py's _Stack: relu(p) and relu(o0) open res blocks 0 and 1, relu(c0) / relu(c1) sit
                 between their convolutions), 'o1' (the last stack's output, ReLU'd as Dense reads it), 'dense';
                 pools 'stack<s>/pool': uint8 taps [N, Ho, Wo, C], kh * 3 + kw from the TF-'SAME' window start.
  ImpalaShallow  'conv0', 'conv1', 'dense'; no pools.
`forward` is the network part alone over T1 >= 1 steps (central inference: T1 = 1), returning the final state too.
Nothing else needs sharing: the V-trace clips enter the loss as stop-gradient values that are continuous in the
logits, log-softmax, entropy and the LSTM are smooth, and done-resets and the reward clip act on inputs.
"""
import collections

import numpy as np
import torch
import torch.nn.functional as F

from oracle import net_oracle, optim_oracle

MASKS = {'deep': tuple('stack%d/%s' % (s, k) for s in range(3) for k in ('p', 'c0', 'o0', 'c1')) + ('o1', 'dense'),
         'shallow': ('conv0', 'conv1', 'dense')}
POOLS = {'deep': tuple('stack%d/pool' % s for s in range(3)), 'shallow': ()}
LR, BETA1, BETA2, ADAM_EPS = 0.00048, 0.0, 0.999, 3.125e-7      # optim_oracle / CpuLearner defaults


class _TapPool(torch.autograd.Function):
  """Max-pool 3x3 / 2 of a -inf padded NCHW tensor as a gather at flat indices into each padded plane; the
  backward is F.max_pool2d's own (max_pool2d_with_indices_backward), summing overlapping windows in its order."""

  @staticmethod
  def forward(ctx, xp, ind, like):
    ctx.save_for_backward(xp, ind)
    y = torch.empty_like(like)
    y.copy_(xp.flatten(2).gather(2, ind.flatten(2)).view(ind.shape))
    return y

  @staticmethod
  def backward(ctx, gy):
    xp, ind = ctx.saved_tensors
    return torch.ops.aten.max_pool2d_with_indices_backward(gy, xp, [3, 3], [2, 2], [0, 0], [1, 1], False,
                                                           ind), None, None


class _Decisions(object):
  """The ReLUs and pools of one unroll: given decisions or their own.  Records the decisions used, the
  pre-activation of every ReLU (`acts`) and, where a given decision differs from the one the reference would
  make itself, how far from a tie it is (`ties`: |z| for a ReLU, max - x[tap] for a pool)."""

  def __init__(self, masks=None, taps=None):
    self.masks_in, self.taps_in = masks, taps
    self.masks, self.taps, self.acts, self.ties = {}, {}, {}, {}

  def relu(self, name, z):
    own = z.detach() > 0
    if self.masks_in is None:
      m = own
    else:
      m = torch.as_tensor(np.asarray(self.masks_in[name], bool))
      if tuple(m.shape) != tuple(z.shape):
        raise ValueError('mask %s has shape %s, the layer %s' % (name, tuple(m.shape), tuple(z.shape)))
      self.ties[name] = z.detach()[m != own].abs().numpy()
    self.masks[name] = m.numpy()
    self.acts[name] = z.detach().numpy()
    return z * m.to(z.dtype)

  def pool(self, name, x):
    """Keras MaxPool2D(3, 2, 'same') of NHWC x (net_oracle._maxpool_same_nhwc's padding and layout)."""
    N, H, W, C = x.shape
    pt, pb = net_oracle._tf_same_pad(H, 3, 2)
    pl, pr = net_oracle._tf_same_pad(W, 3, 2)
    xp = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb), value=float('-inf'))
    Wp = xp.shape[3]
    y_own, ind_own = F.max_pool2d(xp.detach(), 3, 2, return_indices=True)
    Ho, Wo = y_own.shape[2:]
    oh = torch.arange(Ho).view(1, 1, Ho, 1)
    ow = torch.arange(Wo).view(1, 1, 1, Wo)
    own = ((ind_own // Wp - 2 * oh) * 3 + ind_own % Wp - 2 * ow).permute(0, 2, 3, 1)
    if self.taps_in is None:
      t = own
      ind = ind_own
    else:
      t = torch.as_tensor(np.asarray(self.taps_in[name]).astype(np.int64))
      if tuple(t.shape) != (N, Ho, Wo, C):
        raise ValueError('taps %s have shape %s, the pool %s' % (name, tuple(t.shape), (N, Ho, Wo, C)))
      tc = t.permute(0, 3, 1, 2)
      r, c = 2 * oh + tc // 3, 2 * ow + tc % 3
      if bool(((tc < 0) | (tc > 8) | (r < pt) | (r >= pt + H) | (c < pl) | (c >= pl + W)).any()):
        raise ValueError('taps %s: a tap outside the image' % name)
      ind = torch.empty_like(ind_own)
      ind.copy_(r * Wp + c)
    y = _TapPool.apply(xp, ind, y_own)
    if self.taps_in is not None:
      self.ties[name] = (y_own - y.detach()).permute(0, 2, 3, 1)[t != own].numpy()
    self.taps[name] = t.numpy().astype(np.uint8)
    return y.permute(0, 2, 3, 1)


# _torso restates net_oracle.torso with the ReLU and the pool made pluggable: a change to the oracle's layers must be
# mirrored here.  test_float32_reference_is_the_oracle_step pins it bit for bit.
def _torso(net, p, prev_action, reward, frame, A, dtype, dec):
  x = frame.to(dtype) / 255.0
  if net == 'deep':
    for si in range(3):
      s = 'stack%d/' % si
      x = net_oracle._conv_nhwc(x, p[s + 'conv/kernel'], p[s + 'conv/bias'], 1, True)
      x = dec.pool(s + 'pool', x)
      for bi in (0, 1):
        blk = x
        x = dec.relu(s + ('p', 'o0')[bi], x)
        x = net_oracle._conv_nhwc(x, p[s + 'res_%d/conv2d_0/kernel' % bi], p[s + 'res_%d/conv2d_0/bias' % bi], 1,
                                  True)
        x = dec.relu(s + ('c0', 'c1')[bi], x)
        x = net_oracle._conv_nhwc(x, p[s + 'res_%d/conv2d_1/kernel' % bi], p[s + 'res_%d/conv2d_1/bias' % bi], 1,
                                  True)
        x = x + blk
    x = dec.relu('o1', x)
  else:
    x = dec.relu('conv0', net_oracle._conv_nhwc(x, p['conv0/kernel'], p['conv0/bias'], 4, False))
    x = dec.relu('conv1', net_oracle._conv_nhwc(x, p['conv1/kernel'], p['conv1/bias'], 2, False))
  x = x.reshape(x.shape[0], -1)
  x = dec.relu('dense', x @ p['conv_to_linear/kernel'] + p['conv_to_linear/bias'])
  clipped_reward = torch.clamp(reward, -1, 1)[:, None]
  one_hot = F.one_hot(prev_action.long(), A).to(dtype)
  return torch.cat([x, clipped_reward, one_hot], dim=1)


def _unroll(net, p, batch, A, dtype, dec):
  """net_oracle.unroll in `dtype`: -> logits [T1,B,A], baseline [T1,B], the final (h, c) [B,256]."""
  prev_actions = torch.as_tensor(np.asarray(batch['prev_actions']))
  T1, B = prev_actions.shape
  frame = torch.as_tensor(np.asarray(batch['observation']))
  tor = _torso(net, p, prev_actions.reshape(T1 * B), torch.as_tensor(np.asarray(batch['reward'])).to(dtype).reshape(
      T1 * B), frame.reshape((T1 * B,) + tuple(frame.shape[2:])), A, dtype, dec).reshape(T1, B, -1)
  h = torch.as_tensor(np.asarray(batch['h0'])).to(dtype)
  c = torch.as_tensor(np.asarray(batch['c0'])).to(dtype)
  done = torch.as_tensor(np.asarray(batch['done']))
  outs = []
  for t in range(T1):
    d = done[t].bool()[:, None]
    h = torch.where(d, torch.zeros_like(h), h)
    c = torch.where(d, torch.zeros_like(c), c)
    h, c = net_oracle.lstm_cell(p, tor[t], h, c)
    outs.append(h)
  core = torch.stack(outs)
  logits = core @ p['policy_logits/kernel'] + p['policy_logits/bias']
  baseline = (core @ p['baseline/kernel'] + p['baseline/bias'])[..., 0]
  return logits, baseline, (h, c)


# ---- compute_loss after the unroll: loss_oracle / vtrace_oracle restated in `dtype` -------------------------------
def vtrace_from_importance_weights(target_action_log_probs, behaviour_action_log_probs, discounts, rewards, values,
                                   bootstrap_value, FT, clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0,
                                   lambda_=1.0):
  """vtrace_oracle.from_importance_weights in numpy dtype FT: -> (vs, pg_advantages)."""
  log_rhos = np.asarray(target_action_log_probs, FT) - np.asarray(behaviour_action_log_probs, FT)
  discounts, rewards, values = (np.asarray(a, FT) for a in (discounts, rewards, values))
  bootstrap_value = np.asarray(bootstrap_value, FT)
  rhos = np.exp(log_rhos)
  clipped_rhos = np.minimum(FT(clip_rho_threshold), rhos)
  cs = np.minimum(FT(1.0), rhos) * FT(lambda_)
  values_t_plus_1 = np.concatenate([values[1:], bootstrap_value[None]], axis=0)
  deltas = clipped_rhos * (rewards + discounts * values_t_plus_1 - values)
  acc = np.zeros_like(bootstrap_value)
  out = [None] * discounts.shape[0]
  for i in range(discounts.shape[0] - 1, -1, -1):
    acc = deltas[i] + discounts[i] * cs[i] * acc
    out[i] = acc
  vs = np.stack(out, axis=0) + values
  vs_t_plus_1 = np.concatenate([vs[1:], bootstrap_value[None]], axis=0)
  clipped_pg_rhos = np.minimum(FT(clip_pg_rho_threshold), rhos)
  pg_advantages = clipped_pg_rhos * (rewards + discounts * vs_t_plus_1 - values)
  return vs.astype(FT), pg_advantages.astype(FT)


def compute_loss(cfg, logits, baseline, batch, entropy_cost_param, dtype):
  """loss_oracle.compute_loss_from_outputs in `dtype`: -> (total, logs {name: tensor})."""
  return _compute_loss(cfg, logits, baseline, batch, entropy_cost_param, dtype)[:2]


def _compute_loss(cfg, logits, baseline, batch, entropy_cost_param, dtype):
  """compute_loss, and the stop-gradient V-trace targets: -> (total, logs, vs, pg_advantages)."""
  FT = np.float64 if dtype == torch.float64 else np.float32
  behaviour_logits = torch.as_tensor(np.asarray(batch['behaviour_logits'])).to(dtype)
  actions = torch.as_tensor(np.asarray(batch['action'])).long()
  rewards = torch.as_tensor(np.asarray(batch['reward'])).to(dtype)
  done = torch.as_tensor(np.asarray(batch['done'])).bool()
  bootstrap_value = baseline[-1]
  a = actions[:-1]
  beh_logits = behaviour_logits[:-1]
  rewards = rewards[1:]
  done = done[1:]
  tgt_logits = logits[:-1]
  values = baseline[:-1]
  if cfg.max_abs_reward:
    rewards = torch.clamp(rewards, -cfg.max_abs_reward, cfg.max_abs_reward)
  discounts = (~done).to(dtype) * cfg.discounting
  tgt_lsm = torch.log_softmax(tgt_logits, -1)
  beh_lsm = torch.log_softmax(beh_logits, -1)
  tgt_logp = tgt_lsm.gather(-1, a[..., None])[..., 0]
  beh_logp = beh_lsm.gather(-1, a[..., None])[..., 0]
  vs, pg_adv = vtrace_from_importance_weights(
      tgt_logp.detach().numpy(), beh_logp.detach().numpy(), discounts.numpy(), rewards.numpy(),
      values.detach().numpy(), bootstrap_value.detach().numpy(), FT, lambda_=cfg.lambda_)
  vs, pg_adv = torch.from_numpy(vs), torch.from_numpy(pg_adv)
  policy_loss = -torch.mean(tgt_logp * pg_adv)
  v_error = vs - values
  v_loss = cfg.baseline_cost * 0.5 * torch.mean(v_error ** 2)
  entropy = torch.mean(-(tgt_lsm.exp() * tgt_lsm).sum(-1))
  mul = cfg.entropy_cost_adjustment_speed
  entropy_cost = torch.exp(mul * entropy_cost_param)
  entropy_loss = entropy_cost.detach() * -entropy
  kl = beh_logp - tgt_logp
  kl_loss = cfg.kl_cost * torch.mean(kl)
  if cfg.target_entropy:
    adj = entropy_cost * (entropy.detach() - cfg.target_entropy)
  else:
    adj = 0. * entropy_cost
  total = policy_loss + v_loss + entropy_loss + kl_loss + adj
  logs = collections.OrderedDict([
      ('V/value function', values.mean()),
      ('V/L2 error', torch.sqrt(torch.mean(v_error ** 2))),
      ('losses/policy', policy_loss),
      ('losses/V', v_loss),
      ('losses/entropy', entropy_loss),
      ('losses/kl', kl_loss),
      ('losses/total', total),
      ('policy/max_action_abs(before_tanh)', a.abs().max()),
      ('policy/entropy', entropy),
      ('policy/entropy_cost', entropy_cost),
      ('policy/kl(old|new)', kl.mean()),
  ])
  return total, logs, vs, pg_adv


# Logged terms that are means over the T x B rows, and may be averaged over column chunks with weights Bc / B.
_MEAN_LOGS = ('V/value function', 'losses/policy', 'losses/V', 'losses/entropy', 'losses/kl', 'losses/total',
              'policy/entropy', 'policy/entropy_cost', 'policy/kl(old|new)')


def loss_and_grads(cfg, ll, lb, bl, act, rew, done, ecp, dtype, chunk=None):
  """loss_oracle.loss_and_grads in `dtype`, on the network outputs alone (inputs time-major with T+1 rows:
  ll, bl [T1,B,A], lb, act, rew, done [T1,B]; ecp the entropy cost parameter as the GPU holds it).
  Returns (total, logs {name: float}, dlogits [T1,B,A], dbaseline [T1,B], d_entropy_cost_param, vs [T,B],
  pg_advantages [T,B]); vs and pg_advantages are stop-gradient, as in compute_loss.

  `chunk` columns at a time keep the autograd graph of a large B within host memory.  Every output but the
  loss terms is per column; the loss terms are means over all T x B rows, so a chunk of Bc columns contributes
  its own means with weight Bc / B (and its gradients scaled by the same weight), summed in float64.  The one
  term that is not a mean, V/L2 error = sqrt(mean (vs - V)^2), is rebuilt from the weighted mean of its square.
  With a single chunk (the default) this is compute_loss and autograd, unchanged."""
  ll, lb, bl = (np.asarray(x) for x in (ll, lb, bl))
  B = ll.shape[1]
  chunk = B if chunk is None else min(int(chunk), B)
  dl = np.empty(ll.shape, np.float64 if dtype == torch.float64 else np.float32)
  db = np.empty(lb.shape, dl.dtype)
  vs = np.empty((lb.shape[0] - 1, B), dl.dtype)
  pg = np.empty_like(vs)
  sums = collections.OrderedDict()
  total = dep = 0.0
  for b0 in range(0, B, chunk):
    cols = slice(b0, min(b0 + chunk, B))
    w = (cols.stop - cols.start) / B
    logits = torch.tensor(ll[:, cols], dtype=dtype, requires_grad=True)
    baseline = torch.tensor(lb[:, cols], dtype=dtype, requires_grad=True)
    ep = torch.tensor(float(ecp), dtype=dtype, requires_grad=True)
    batch = dict(behaviour_logits=bl[:, cols], action=np.asarray(act)[:, cols], reward=np.asarray(rew)[:, cols],
                 done=np.asarray(done)[:, cols])
    t, logs, vs_c, pg_c = _compute_loss(cfg, logits, baseline, batch, ep, dtype)
    t.backward()
    if w == 1.0:
      dl[:], db[:] = logits.grad.numpy(), baseline.grad.numpy()
    else:
      dl[:, cols], db[:, cols] = logits.grad.numpy() * w, baseline.grad.numpy() * w
    vs[:, cols], pg[:, cols] = vs_c.numpy(), pg_c.numpy()
    total += w * float(t.detach())
    dep += w * (float(ep.grad) if ep.grad is not None else 0.0)
    for k, v in logs.items():
      v = float(v.detach())
      if k == 'policy/max_action_abs(before_tanh)':
        sums[k] = max(sums.get(k, 0.0), v)
      elif k == 'V/L2 error':
        sums[k] = sums.get(k, 0.0) + w * v * v
      else:
        assert k in _MEAN_LOGS, k
        sums[k] = sums.get(k, 0.0) + w * v
  if chunk == B:
    sums['V/L2 error'] = float(logs['V/L2 error'].detach())
  else:
    sums['V/L2 error'] = float(np.sqrt(sums['V/L2 error']))
  return total, sums, dl, db, dep, vs, pg


# ---- the step ------------------------------------------------------------------------------------------------------
def step(net, params, batch, cfg, dtype=torch.float64, masks=None, taps=None):
  """One learner step.  net: 'deep' | 'shallow'; params: {name: array} (any float dtype; evaluated in `dtype`);
  batch: learner_oracle.synthetic_batch's fields (h0 / c0 of any float dtype); cfg: loss_oracle.LossConfig.
  masks: None or {MASKS[net] name: bool array}; taps: None or {POOLS[net] name: uint8 [N, Ho, Wo, C]}.
  Returns a dict: logits [T1,B,A], baseline [T1,B], total, logs {name: float} (the continuous logged terms),
  dlogits, dbaseline (d total / d outputs), acts {MASKS name: the ReLU's input}, grads {name: array} (the 39
  tensors, then entropy_cost_param), params_after {name: fp32} (one Keras Adam step from zero slots, the clamp
  on entropy_cost_param), update {name: float64} (params - params_after before the fp32 rounding of the
  subtraction), masks, taps (the decisions used) and ties (see _Decisions)."""
  A = np.asarray(batch['behaviour_logits']).shape[-1]
  p = collections.OrderedDict((k, torch.as_tensor(np.asarray(v)).to(dtype).requires_grad_(True))
                              for k, v in params.items())
  mul = cfg.entropy_cost_adjustment_speed
  ecp_value = np.float32(np.log(cfg.entropy_cost) / mul)            # the fp32 parameter both sides hold
  ecp = torch.tensor(float(ecp_value), dtype=dtype, requires_grad=True)
  dec = _Decisions(masks, taps)
  logits, baseline, _ = _unroll(net, p, batch, A, dtype, dec)
  logits.retain_grad()
  baseline.retain_grad()
  total, logs = compute_loss(cfg, logits, baseline, batch, ecp, dtype)
  total.backward()
  g = collections.OrderedDict((k, v.grad.numpy().copy()) for k, v in p.items())
  g['entropy_cost_param'] = ecp.grad.numpy().copy() if ecp.grad is not None else np.zeros((), ecp.detach().numpy().dtype)
  values = collections.OrderedDict((k, v.detach().numpy()) for k, v in p.items())
  values['entropy_cost_param'] = np.asarray(ecp_value)
  after, update = collections.OrderedDict(), collections.OrderedDict()
  for k in g:
    z = np.zeros(np.shape(g[k]), np.float32)
    p2 = optim_oracle.keras_adam_step(values[k], g[k] * np.float32(1.0), z, z, 0, LR, BETA1, BETA2, ADAM_EPS)[0]
    if k == 'entropy_cost_param':       # constraint, learner.py:231
      p2 = np.clip(p2, -20.0 / mul, 20.0 / mul).astype(np.float32)
    after[k] = p2
    # the step itself, without the rounding of storing p - step in fp32
    update[k] = -optim_oracle.keras_adam_step(z, g[k], z, z, 0, LR, BETA1, BETA2, ADAM_EPS)[0].astype(np.float64)
  skip = ('policy/max_action_abs(before_tanh)',)
  return dict(logits=logits.detach().numpy(), baseline=baseline.detach().numpy(), total=float(total.detach()),
              logs=collections.OrderedDict((k, float(v.detach())) for k, v in logs.items() if k not in skip),
              dlogits=logits.grad.numpy().copy(), dbaseline=baseline.grad.numpy().copy(), acts=dec.acts, grads=g,
              params_after=after, update=update, masks=dec.masks, taps=dec.taps, ties=dec.ties)


def forward(net, params, inputs, dtype=torch.float64, masks=None, taps=None):
  """The network's forward over T1 >= 1 steps (central inference: T1 = 1), without gradients.  inputs:
  prev_actions [T1,B], reward, done [T1,B], observation [T1,B,H,W,C] uint8, h0 / c0 [B,256] (any float dtype);
  params, masks and taps as in `step` (rows = the T1 * B frames, time-major).  Returns a dict: logits [T1,B,A],
  baseline [T1,B], h, c (the state after the last step), acts, masks, taps and ties (see _Decisions)."""
  A = np.shape(params['policy_logits/bias'])[0]
  p = {k: torch.as_tensor(np.asarray(v)).to(dtype) for k, v in params.items()}
  dec = _Decisions(masks, taps)
  with torch.no_grad():
    logits, baseline, (h, c) = _unroll(net, p, inputs, A, dtype, dec)
  return dict(logits=logits.numpy(), baseline=baseline.numpy(), h=h.numpy(), c=c.numpy(), acts=dec.acts,
              masks=dec.masks, taps=dec.taps, ties=dec.ties)


def perturbed(params, batch, delta, seed=0):
  """Every parameter, h0 and c0 multiplied by 1 + delta N(0, 1) (float64)."""
  rng = np.random.default_rng(seed)
  f = lambda v: np.asarray(v, np.float64) * (1. + delta * rng.normal(size=np.shape(v)))
  p = collections.OrderedDict((k, f(v)) for k, v in params.items())
  return p, dict(batch, h0=f(batch['h0']), c0=f(batch['c0']))
