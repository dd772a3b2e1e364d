"""CPU ORACLE (test infrastructure, NOT product code) -- torch-CPU fp32 restatement of
the policy networks on the hot path:

  ImpalaDeep     /root/reference/dmlab/networks.py:26-171  (the reference's net)
  ImpalaShallow  NOT in the reference (SURVEY 0): defined from the IMPALA paper
                 (conv 8x8/4 ->16, conv 4x4/2 ->32, FC 256, LSTM 256), VALID
                 padding, same torso->LSTM->heads protocol as ImpalaDeep.

Keras layer arithmetic (TF 2.4.1 Conv2D / MaxPool2D(padding='same') / Dense /
LSTMCell, not vendored under /root/reference) is restated from its published
semantics; the reference's tests pin only shapes/variable counts
(tests/agents_test.py:45 -> 39 trainable tensors) => the layer NUMERICS are parity-unpinned
(cross-checked against an independent numpy-loop restatement,
tests/test_oracle_layers_independent.py).  The WIRING of ImpalaDeep is pinned: the unmodified
reference classes run over a Keras-layer shim (tests/golden/make_golden_net.py) reproduce
this file's outputs for the same weights (tests/test_oracle_golden.py).

Weights use the Keras layouts: conv kernel HWIO [kh,kw,cin,cout], dense
[in,out], LSTM kernel [in,4H] / recurrent [H,4H] with gate order i,f,c,o.
Activations are NHWC like the reference.
"""
import collections
import math

import numpy as np
import torch
import torch.nn.functional as F

AgentOutput = collections.namedtuple('AgentOutput', 'action policy_logits baseline')

LSTM_UNITS = 256
DENSE_UNITS = 256


def _tf_same_pad(n, k, s):
  """TF 'SAME' padding (before, after) for input size n, window k, stride s."""
  out = -(-n // s)
  total = max((out - 1) * s + k - n, 0)
  return total // 2, total - total // 2


def conv_out_hw(h, w, k, s, same):
  if same:
    return -(-h // s), -(-w // s)
  return (h - k) // s + 1, (w - k) // s + 1


def param_specs(net, num_actions, obs_shape):
  """[(name, shape)] in tf.Module.trainable_variables order (attributes sorted
  by name: _baseline, _conv_to_linear, _core, _policy_logits, _stacks)."""
  H, W, C = obs_shape
  specs = [('baseline/kernel', (LSTM_UNITS, 1)), ('baseline/bias', (1,))]
  if net == 'deep':
    h, w, c = H, W, C
    conv = []
    for si, ch in enumerate((16, 32, 32)):
      conv += [('stack%d/conv/kernel' % si, (3, 3, c, ch)),
               ('stack%d/conv/bias' % si, (ch,))]
      for j in (0, 1):
        for bi in (0, 1):
          conv += [('stack%d/res_%d/conv2d_%d/kernel' % (si, bi, j), (3, 3, ch, ch)),
                   ('stack%d/res_%d/conv2d_%d/bias' % (si, bi, j), (ch,))]
      c = ch
      h, w = -(-h // 2), -(-w // 2)
    flat = h * w * c
  elif net == 'shallow':
    h, w = conv_out_hw(H, W, 8, 4, False)
    h, w = conv_out_hw(h, w, 4, 2, False)
    conv = [('conv0/kernel', (8, 8, C, 16)), ('conv0/bias', (16,)),
            ('conv1/kernel', (4, 4, 16, 32)), ('conv1/bias', (32,))]
    flat = h * w * 32
  else:
    raise ValueError(net)
  core_in = DENSE_UNITS + 1 + num_actions
  specs += [('conv_to_linear/kernel', (flat, DENSE_UNITS)),
            ('conv_to_linear/bias', (DENSE_UNITS,)),
            ('core/kernel', (core_in, 4 * LSTM_UNITS)),
            ('core/recurrent_kernel', (LSTM_UNITS, 4 * LSTM_UNITS)),
            ('core/bias', (4 * LSTM_UNITS,)),
            ('policy_logits/kernel', (LSTM_UNITS, num_actions)),
            ('policy_logits/bias', (num_actions,))]
  return specs + conv


# When set to torch.bfloat16, the 3x3 convolutions with >= 16 input channels round their
# OPERANDS (activations, weights, and -- in the backward -- the incoming gradient) to bf16
# and accumulate in fp32: the arithmetic contract of the wgmma tensor-core path
# (seed_rl_b200 conv_mode='tc').  The fp32 reference semantics are CONV_OPERAND_DTYPE=None.
CONV_OPERAND_DTYPE = None


class _RoundedOperandConv(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, w, b, pads, dt):
    q = lambda t: t.to(dt).to(torch.float32)
    xq, wq = q(x), q(w)
    ctx.save_for_backward(xq, wq)
    ctx.pads, ctx.dt = pads, dt
    y = F.conv2d(F.pad(xq.permute(0, 3, 1, 2), pads), wq.permute(3, 2, 0, 1), b)
    return y.permute(0, 2, 3, 1)

  @staticmethod
  def backward(ctx, gy):
    xq, wq = ctx.saved_tensors
    gq = gy.to(ctx.dt).to(torch.float32)
    with torch.enable_grad():
      x2 = xq.detach().requires_grad_(True)
      w2 = wq.detach().requires_grad_(True)
      y = F.conv2d(F.pad(x2.permute(0, 3, 1, 2), ctx.pads), w2.permute(3, 2, 0, 1)).permute(0, 2, 3, 1)
      gx, gw = torch.autograd.grad(y, (x2, w2), gq)
    return gx, gw, gy.sum((0, 1, 2)), None, None     # bias gradient stays fp32


def _conv_nhwc(x, w_hwio, b, stride, same):
  """x [N,H,W,C] -> [N,H',W',O].  Keras Conv2D(padding='same'|'valid')."""
  if (CONV_OPERAND_DTYPE is not None and same and stride == 1 and tuple(w_hwio.shape[:2]) == (3, 3)
      and w_hwio.shape[2] >= 16):
    return _RoundedOperandConv.apply(x, w_hwio, b, (1, 1, 1, 1), CONV_OPERAND_DTYPE)
  N, H, W, C = x.shape
  kh, kw = w_hwio.shape[:2]
  xc = x.permute(0, 3, 1, 2)
  if same:
    pt, pb = _tf_same_pad(H, kh, stride)
    pl, pr = _tf_same_pad(W, kw, stride)
    xc = F.pad(xc, (pl, pr, pt, pb))
  y = F.conv2d(xc, w_hwio.permute(3, 2, 0, 1), b, stride=stride)
  return y.permute(0, 2, 3, 1)


def _maxpool_same_nhwc(x, k=3, s=2):
  """Keras MaxPool2D(pool_size=3, strides=2, padding='same') -- TF pads
  asymmetrically: (0,1) for 84->42 and 42->21, (1,1) for 21->11."""
  N, H, W, C = x.shape
  pt, pb = _tf_same_pad(H, k, s)
  pl, pr = _tf_same_pad(W, k, s)
  xc = F.pad(x.permute(0, 3, 1, 2), (pl, pr, pt, pb), value=float('-inf'))
  return F.max_pool2d(xc, k, s).permute(0, 2, 3, 1)


def torso(net, p, prev_action, reward, frame, num_actions):
  """dmlab/networks.py:94-114 (_torso) on a folded batch [N, ...]."""
  x = frame.to(torch.float32) / 255.0                          # :98-100
  if net == 'deep':
    for si in range(3):                                        # _Stack.__call__ :46-60
      x = _conv_nhwc(x, p['stack%d/conv/kernel' % si], p['stack%d/conv/bias' % si], 1, True)
      x = _maxpool_same_nhwc(x)
      for bi in (0, 1):
        blk = x
        x = F.relu(x)
        x = _conv_nhwc(x, p['stack%d/res_%d/conv2d_0/kernel' % (si, bi)],
                       p['stack%d/res_%d/conv2d_0/bias' % (si, bi)], 1, True)
        x = F.relu(x)
        x = _conv_nhwc(x, p['stack%d/res_%d/conv2d_1/kernel' % (si, bi)],
                       p['stack%d/res_%d/conv2d_1/bias' % (si, bi)], 1, True)
        x = x + blk
    x = F.relu(x)                                              # :105
  else:
    x = F.relu(_conv_nhwc(x, p['conv0/kernel'], p['conv0/bias'], 4, False))
    x = F.relu(_conv_nhwc(x, p['conv1/kernel'], p['conv1/bias'], 2, False))
  x = x.reshape(x.shape[0], -1)                                # Flatten (h,w,c)
  x = F.relu(x @ p['conv_to_linear/kernel'] + p['conv_to_linear/bias'])  # :108-109
  clipped_reward = torch.clamp(reward, -1, 1)[:, None]         # :112
  one_hot = F.one_hot(prev_action.long(), num_actions).to(torch.float32)  # :113
  return torch.cat([x, clipped_reward, one_hot], dim=1)        # :114


def lstm_cell(p, x, h, c):
  """Keras LSTMCell(256): z = xW + hU + b; gates i,f,c,o; sigmoid/tanh."""
  z = x @ p['core/kernel'] + h @ p['core/recurrent_kernel'] + p['core/bias']
  i, f, g, o = z.chunk(4, dim=1)
  c2 = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
  h2 = torch.sigmoid(o) * torch.tanh(c2)
  return h2, c2


def unroll(net, p, prev_actions, reward, done, frame, core_state, num_actions):
  """dmlab/networks.py:153-171 (_unroll).  Inputs time-major [T, B, ...].
  core_state = (h, c) each [B,256].  Returns (logits [T,B,A], baseline [T,B],
  (h, c))."""
  T, B = prev_actions.shape
  tor = torso(net, p, prev_actions.reshape(T * B), reward.reshape(T * B),
              frame.reshape((T * B,) + tuple(frame.shape[2:])), num_actions)
  tor = tor.reshape(T, B, -1)                                  # batch_apply
  h, c = core_state
  outs = []
  for t in range(T):                                           # :160-168
    d = done[t].bool()[:, None]
    h = torch.where(d, torch.zeros_like(h), h)
    c = torch.where(d, torch.zeros_like(c), c)
    h, c = lstm_cell(p, tor[t], h, c)
    outs.append(h)
  core = torch.stack(outs)                                     # [T,B,256]
  logits = core @ p['policy_logits/kernel'] + p['policy_logits/bias']   # :116
  baseline = (core @ p['baseline/kernel'] + p['baseline/bias'])[..., 0]  # :117
  return logits, baseline, (h, c)


# ---------------------------------------------------------------------------
# Keras default initialisers (TF 2.4.1): glorot_uniform kernels, zero biases,
# orthogonal recurrent kernel, unit_forget_bias.
def init_params(net, num_actions, obs_shape, seed=0):
  rng = np.random.default_rng(seed)
  out = collections.OrderedDict()
  for name, shape in param_specs(net, num_actions, obs_shape):
    if name.endswith('bias'):
      a = np.zeros(shape, np.float32)
      if name == 'core/bias':
        a[LSTM_UNITS:2 * LSTM_UNITS] = 1.0
    elif name == 'core/recurrent_kernel':
      m = rng.normal(size=(shape[1], shape[0]))
      q, r = np.linalg.qr(m)
      q = q * np.sign(np.diag(r))
      a = q.T.astype(np.float32)
    else:
      rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
      fan_in, fan_out = shape[-2] * rf, shape[-1] * rf
      lim = math.sqrt(6.0 / (fan_in + fan_out))
      a = rng.uniform(-lim, lim, shape).astype(np.float32)
    out[name] = a
  return out


def to_torch(params, requires_grad=False):
  return collections.OrderedDict(
      (k, torch.tensor(np.asarray(v), dtype=torch.float32, requires_grad=requires_grad))
      for k, v in params.items())
