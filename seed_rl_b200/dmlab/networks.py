"""Policy networks on the hot path -- mirror of the reference's `dmlab/networks.py`
(`ImpalaDeep`, AgentOutput; reference dmlab/networks.py:22-171) with the same agent
protocol:

    agent.initial_state(batch_size) -> (h, c)
    agent(prev_actions, env_outputs, core_state, unroll=False, is_training=False)
        -> (AgentOutput(action, policy_logits, baseline), core_state)
    agent.get_action(...)  == agent(...)
    agent.trainable_variables  (39 tensors for ImpalaDeep, reference tests/agents_test.py:45)

All math runs in libseedrl_b200 (seedrl_net_forward / seedrl_net_backward); parameters
live in ONE flat fp32 HBM arena (Keras layouts, tf.Module variable order), which is what
the fused Adam kernel and the NCCL all-reduce operate on.  `ImpalaShallow` is the
IMPALA-paper shallow net (not in the reference, SURVEY 0), same protocol.
"""
import collections
import ctypes
import math

import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common.cuda_net import CudaNet

AgentOutput = collections.namedtuple('AgentOutput', 'action policy_logits baseline')

LSTM_UNITS = 256


class _CudaAgent(CudaNet):
  _NET = None
  _LIB = 'seedrl_net'
  _EXTRA_PARAMS = 1        # entropy_cost_param (learner.py:225-234)

  def __init__(self, num_actions, obs_shape=(84, 84, 4), seed=0, device=None, conv_mode='simt',
               lstm_mode='tiled'):
    """conv_mode selects the arithmetic of every contraction (3x3 convs, Dense, LSTM input
    projection, policy head): 'simt' = fp32 CUDA cores (the 2e-3 parity path), 'tc' = wgmma
    tensor cores with bf16 operands and fp32 accumulation, 'tc3' = wgmma with bf16x3 split
    operands (fp32-faithful).  lstm_mode selects how the recurrent products of the LSTM core are
    computed: 'tiled' = one persistent kernel each way on fp32 CUDA cores, 'tc3' = the same
    recurrence on wgmma with bf16x3 operands."""
    self._num_actions = int(num_actions)
    self._obs_shape = tuple(int(x) for x in obs_shape)
    if self._NET == _lib.NET_DEEP and (len(self._obs_shape) != 3 or not 1 <= self._obs_shape[2] <= 16):
      raise ValueError('ImpalaDeep takes (H, W, C) uint8 frames with 1 to 16 channels, got %s'
                       % (self._obs_shape,))
    L = _lib.lib()
    cfg = _lib.NetConfig(self._NET, self._num_actions, *self._obs_shape)
    h = ctypes.c_void_p()
    _lib.check(L.seedrl_net_create(ctypes.byref(cfg), ctypes.byref(h)))
    self._h = h
    modes = {'simt': 0, 'tc': 1, 'tc3': 2, 'tc3p': 3}
    if conv_mode not in modes:
      raise ValueError("conv_mode must be 'simt', 'tc' (bf16), 'tc3' (bf16x3, fp32-faithful) or "
                       "'tc3p' (bf16x3 on HBM-resident operand planes, TMA-fed)")
    if conv_mode == 'tc3p' and self._NET != _lib.NET_DEEP:
      raise ValueError("conv_mode 'tc3p' is built for the deep net")
    self.conv_mode = conv_mode
    _lib.check(L.seedrl_net_set_conv_mode(h, modes[conv_mode]))
    lstm_modes = {'tiled': 2, 'tc3': 3}
    if lstm_mode not in lstm_modes:
      raise ValueError("lstm_mode must be 'tiled' or 'tc3' (the tiled recurrence on wgmma bf16x3)")
    self.lstm_mode = lstm_mode
    _lib.check(L.seedrl_net_set_lstm_mode(h, lstm_modes[lstm_mode]))
    self._setup(seed, device)
    self._rng_offset = 0
    self._seed = seed

  def _param_rank(self, index, name_buf, dims, offset):
    return _lib.lib().seedrl_net_param_info(self._h, index, name_buf, len(name_buf), dims, ctypes.byref(offset))

  @property
  def entropy_cost_param(self):
    return self._view(self.params, self._n_tensors)

  @property
  def entropy_cost_param_index(self):
    return self.param_info[self._n_tensors][2]

  # ---- protocol ---------------------------------------------------------------
  def initial_state(self, batch_size):
    z = torch.zeros([batch_size, LSTM_UNITS], dtype=torch.float32, device=self.device)
    return (z, z.clone())

  def _next_rng_offset(self):
    with self._lock:
      o = self._rng_offset
      self._rng_offset += 1
    return o

  def get_action(self, *args, **kwargs):
    return self.__call__(*args, **kwargs)

  def __call__(self, prev_actions, env_outputs, core_state, unroll=False,
               is_training=False, gumbel_noise=None, rng_counter=None):
    """rng_counter: optional int64 CUDA scalar tensor holding the Philox offset of the sampling
    kernel; it is read and incremented ON THE DEVICE, which makes the whole call capturable in a
    CUDA graph (InferenceHost replays one graph per inference batch)."""
    reward, done, frame = env_outputs[0], env_outputs[1], env_outputs[2]
    prev_actions = _lib.require_cuda(prev_actions, torch.int64, 'prev_actions')
    reward = _lib.require_cuda(reward, torch.float32, 'reward')
    done = _lib.require_cuda(done, torch.bool, 'done')
    frame = _lib.require_cuda(frame, torch.uint8, 'observation')
    if not unroll:   # add the time dimension (networks.py:141-144)
      prev_actions, reward, done, frame = (t.unsqueeze(0) for t in (prev_actions, reward, done, frame))
    T1, B = int(prev_actions.shape[0]), int(prev_actions.shape[1])
    if tuple(frame.shape[2:]) != self._obs_shape:
      raise ValueError('observation shape %s, expected %s' % (tuple(frame.shape[2:]), self._obs_shape))
    h0 = _lib.require_cuda(core_state[0], torch.float32, 'core_state.h')
    c0 = _lib.require_cuda(core_state[1], torch.float32, 'core_state.c')
    A = self._num_actions
    logits = torch.empty([T1, B, A], dtype=torch.float32, device=self.device)
    baseline = torch.empty([T1, B], dtype=torch.float32, device=self.device)
    h = torch.empty_like(h0)
    c = torch.empty_like(c0)
    ws = self.workspace(T1, B)
    L = _lib.lib()
    st = _lib.stream_ptr()
    _lib.check(L.seedrl_net_forward(
        self._h, _lib.ptr(self.params), T1, B, _lib.ptr(prev_actions), _lib.ptr(reward),
        _lib.ptr(done), _lib.ptr(frame), _lib.ptr(h0), _lib.ptr(c0), _lib.ptr(logits),
        _lib.ptr(baseline), _lib.ptr(h), _lib.ptr(c), _lib.ptr(ws), ws.numel(), st))
    # sample a new action (networks.py:121-122)
    action = torch.empty([T1 * B], dtype=torch.int64, device=self.device)
    noise = None
    if gumbel_noise is not None:
      noise = _lib.require_cuda(gumbel_noise, torch.float32, 'gumbel_noise')
    if rng_counter is not None:
      _lib.check(L.seedrl_categorical_sample_counter(
          T1 * B, A, _lib.ptr(logits), _lib.ptr(noise), int(self._seed), _lib.ptr(rng_counter), _lib.ptr(action), st))
    else:
      _lib.check(L.seedrl_categorical_sample(
          T1 * B, A, _lib.ptr(logits), _lib.ptr(noise), int(self._seed), int(self._next_rng_offset()),
          _lib.ptr(action), st))
    action = action.view(T1, B)
    if is_training:
      self._saved = (T1, B, ws, prev_actions, reward, done, frame)
    out = AgentOutput(action, logits, baseline)
    if not unroll:
      out = AgentOutput(*(t.squeeze(0) for t in out))
    return out, (h, c)

  def backward(self, dlogits, dbaseline, head_ready_event=None):
    """d loss / d parameters for the last is_training unroll -> self.grads (overwritten).
    head_ready_event: a torch.cuda.Event recorded once grads[:self.grad_split] (heads, Dense,
    LSTM) are final -- before the convolution torso's backward -- for an overlapped all-reduce."""
    if self._saved is None:
      raise RuntimeError('backward() needs a preceding __call__(..., unroll=True, is_training=True)')
    T1, B, ws, prev_actions, reward, done, frame = self._saved
    L = _lib.lib()
    if head_ready_event is None:
      _lib.check(L.seedrl_net_backward(
          self._h, _lib.ptr(self.params), T1, B, _lib.ptr(prev_actions), _lib.ptr(reward),
          _lib.ptr(done), _lib.ptr(frame), _lib.ptr(dlogits), _lib.ptr(dbaseline),
          _lib.ptr(self.grads), _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    else:
      head_ready_event.record()        # creates the underlying cudaEvent_t; re-recorded by the library
      _lib.check(L.seedrl_net_backward_overlap(
          self._h, _lib.ptr(self.params), T1, B, _lib.ptr(prev_actions), _lib.ptr(reward),
          _lib.ptr(done), _lib.ptr(frame), _lib.ptr(dlogits), _lib.ptr(dbaseline),
          _lib.ptr(self.grads), _lib.ptr(ws), ws.numel(), ctypes.c_void_p(head_ready_event.cuda_event),
          _lib.stream_ptr()))
    return self.grads

  @property
  def grad_split(self):
    return int(_lib.lib().seedrl_net_grad_split(self._h))

  # learner.py:225-234 adds these to the agent when it has no entropy_cost()
  def init_entropy_cost(self, entropy_cost, adjustment_speed):
    self._entropy_mul = float(adjustment_speed)
    self.entropy_cost_param.fill_(math.log(entropy_cost) / adjustment_speed)

  def entropy_cost(self):
    return torch.exp(self._entropy_mul * self.entropy_cost_param)

  # ---- PopArt (popart.py; the V-trace learner's --popart) ---------------------------
  popart_moments = None    # [2] EMA moments (mu1, mu2), [K,2] with K tasks: a device buffer of their own, not trained
  popart_tasks = 0         # K once enable_popart() ran
  popart_task_error = None  # K > 1: device int32 flag, set by the loss kernel for a task id outside [0, K)

  def enable_popart(self, num_tasks=1):
    """Appends the trained compensation (sigma, mu) = (1, 0) after entropy_cost_param, in a tail of
    the parameter and gradient arenas (so Adam and the gradient all-reduce take them with everything
    else), and creates the moments (0, 1).  With num_tasks = K > 1 every task has its own pair of each:
    the compensation is a [K,2] view of the tail and the moments are [K,2].  The tail holds 2K floats
    rounded up to 64.  The network's own arena, its offsets and grad_split are unchanged.  Call before an
    optimizer creates its slots and before anything keeps a pointer to `params` (inference hosts, CUDA
    graphs): both arenas are reallocated."""
    K = int(num_tasks)
    if not 1 <= K <= MAX_POPART_TASKS:
      raise ValueError('num_tasks must be in [1, %d], got %r' % (MAX_POPART_TASKS, num_tasks))
    if self.popart_moments is not None:
      if K != self.popart_tasks:
        raise ValueError('PopArt is enabled with %d tasks, not %d' % (self.popart_tasks, K))
      return
    off = self.arena_floats
    params = torch.zeros(off + -(-2 * K // 64) * 64, dtype=torch.float32, device=self.device)
    params[:off].copy_(self.params)
    params[off:off + 2 * K:2] = 1.0
    self.params, self.grads = params, torch.zeros_like(params)
    if K == 1:
      self.param_info = self.param_info + [('popart/compensation_std', (), off),
                                           ('popart/compensation_mean', (), off + 1)]
      self.popart_moments = torch.tensor([0.0, 1.0], dtype=torch.float32, device=self.device)
    else:
      for k in range(K):
        self.param_info = self.param_info + [('popart/compensation_std/%d' % k, (), off + 2 * k),
                                             ('popart/compensation_mean/%d' % k, (), off + 2 * k + 1)]
      self.popart_moments = torch.tensor([[0.0, 1.0]] * K, dtype=torch.float32, device=self.device)
      self.popart_task_error = torch.zeros(1, dtype=torch.int32, device=self.device)
    self.popart_tasks = K

  @property
  def popart_compensation(self):
    """(sigma, mu), [K,2] with K > 1 tasks: a view of the parameter arena."""
    return self._popart_tail(self.params)

  @property
  def popart_compensation_grad(self):
    return self._popart_tail(self.grads)

  def _popart_tail(self, arena):
    off, K = self.arena_floats, self.popart_tasks
    return arena[off:off + 2] if K == 1 else arena[off:off + 2 * K].view(K, 2)

  def check_errors(self):
    """CudaNet.check_errors, and with K > 1 PopArt tasks, whether a task id outside [0, K) reached the
    loss since the agent was created."""
    super(_CudaAgent, self).check_errors()
    if self.popart_task_error is not None and int(self.popart_task_error.item()) != 0:
      raise RuntimeError('a task id outside [0, %d) reached the multi-task PopArt loss' % self.popart_tasks)

  def state_dict(self):
    d = super(_CudaAgent, self).state_dict()
    if self.popart_moments is not None:
      d['popart_moments'] = self.popart_moments.detach().cpu()
    return d

  def load_state_dict(self, d):
    check_popart_state(d, self.popart_moments is not None, self.popart_tasks)
    super(_CudaAgent, self).load_state_dict(d)
    if self.popart_moments is not None:
      self.popart_moments.copy_(d['popart_moments'].to(self.device))


MAX_POPART_TASKS = 64


def popart_tasks_of(agent_state):
  """The PopArt task count of a checkpoint's agent state (0: written without PopArt)."""
  m = agent_state.get('popart_moments')
  if m is None:
    return 0
  return 1 if m.dim() == 1 else int(m.shape[0])


def check_popart_state(agent_state, popart, num_tasks=None):
  """Raises ValueError when a checkpoint's agent state and a learner disagree on PopArt, or, given the
  learner's num_tasks, on its task count."""
  has = 'popart_moments' in agent_state
  if has and not popart:
    raise ValueError('the checkpoint was written with PopArt (--popart); this learner runs without it')
  if popart and not has:
    raise ValueError('the checkpoint was written without PopArt; this learner runs with --popart')
  if has and num_tasks is not None and popart_tasks_of(agent_state) != num_tasks:
    raise ValueError('the checkpoint was written with %d PopArt tasks (--popart_tasks); this learner runs with %d'
                     % (popart_tasks_of(agent_state), num_tasks))


class ImpalaDeep(_CudaAgent):
  """reference dmlab/networks.py:63-171."""
  _NET = _lib.NET_DEEP


class ImpalaShallow(_CudaAgent):
  """IMPALA-paper shallow net: conv 8x8/4 ->16, conv 4x4/2 ->32, FC 256, LSTM 256."""
  _NET = _lib.NET_SHALLOW
