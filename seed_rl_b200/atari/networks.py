"""reference atari/networks.py: the bit-packed frame stacking (`stack_frames`,
`initial_frame_stacking_state`, :33-173) and the R2D2 agent network `DuelingLSTMDQNNet`
(:221-340, with `_unroll_cell` :176-218), same agent protocol as the reference:

    agent.initial_state(batch_size) -> AgentState(core_state=(h, c), frame_stacking_state)
    agent((prev_actions, env_outputs), agent_state, unroll=False)
        -> (AgentOutput(action int32, q_values float32), AgentState)
    agent.trainable_variables     (18 tensors, tf.Module order: _advantage, _body, _core, _value)

All math runs in libseedrl_b200 (seedrl_r2d2_stack_frames, seedrl_r2d2_net_forward /
_backward: csrc/r2d2_kernels.cu, csrc/r2d2_net.cu)."""
import collections
import ctypes

import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common.cuda_net import CudaNet

AgentOutput = collections.namedtuple('AgentOutput', 'action q_values')
AgentState = collections.namedtuple('AgentState', 'core_state frame_stacking_state')
LSTM_UNITS = 512

STACKING_STATE_DTYPE = torch.int32


def initial_frame_stacking_state(stack_size, batch_size, observation_shape, device='cuda'):
  """reference :33-54: () when stack_size == 1, else zeros int32 [batch_size, prod(obs_shape)]."""
  if stack_size == 1:
    return ()
  n = 1
  for d in observation_shape:
    n *= int(d)
  return torch.zeros([batch_size, n], dtype=STACKING_STATE_DTYPE, device=device)


def stack_frames(frames, frame_stacking_state, done, stack_size):
  """reference :57-173.  frames: uint8 [time, batch, *obs, 1] (un-normalised); state int32
  [batch, prod(obs)] bit-packed; done bool [time, batch].  Returns (stacked uint8
  [time, batch, *obs, stack_size], newest first, frames across an episode boundary zeroed;
  new int32 state).  The reference returns float32 with the same values; here the stack stays
  uint8 and the /255 lives in the first convolution."""
  if tuple(frames.shape[0:2]) != tuple(done.shape[0:2]):
    raise ValueError('Expected same first 2 dims for frames and dones. Got {} vs {}.'.format(
        tuple(frames.shape[0:2]), tuple(done.shape[0:2])))
  if stack_size > 4:
    raise ValueError('Only up to stack size 4 is supported due to bit-packing.')
  if stack_size > 1 and frames.shape[-1] != 1:
    raise ValueError('Due to frame stacking, we require last observation dimension to be 1. Got {}'.format(
        frames.shape[-1]))
  if stack_size == 1:
    return frames, ()
  if frame_stacking_state.dtype != STACKING_STATE_DTYPE:
    raise ValueError('Expected dtype {} got {}'.format(STACKING_STATE_DTYPE, frame_stacking_state.dtype))
  fr = _lib.require_cuda(frames, torch.uint8, 'frames')
  st = _lib.require_cuda(frame_stacking_state, torch.int32, 'frame_stacking_state')
  dn = _lib.require_cuda(done, torch.bool, 'done')
  T, B = int(fr.shape[0]), int(fr.shape[1])
  obs = tuple(int(x) for x in fr.shape[2:-1])
  P = 1
  for d in obs:
    P *= d
  out = torch.empty((T, B) + obs + (stack_size,), dtype=torch.uint8, device=fr.device)
  new_state = torch.empty_like(st)
  _lib.check(_lib.lib().seedrl_r2d2_stack_frames(T, B, P, stack_size, _lib.ptr(fr), _lib.ptr(st), _lib.ptr(dn),
                                                 _lib.ptr(out), _lib.ptr(new_state), _lib.stream_ptr()))
  return out, new_state


class DuelingLSTMDQNNet(CudaNet):
  """reference atari/networks.py:221-340.  Conv 8x8/4 -> 32, 4x4/2 -> 64, 3x3/1 -> 64 ('valid',
  ReLU), Dense(512, ReLU), concat(reward, one_hot(prev_action)), LSTMCell(512) with done-resets,
  dueling value / advantage heads, greedy action.  Parameters live in one flat fp32 HBM arena
  (Keras layouts, tf.Module variable order)."""
  _LIB = 'seedrl_r2d2_net'

  def __init__(self, num_actions, observation_shape, stack_size=1, seed=0, device=None, gemm_mode='tc3',
               lstm_mode='tiled'):
    """gemm_mode: 'tc3' = wgmma bf16x3 (fp32-faithful) for every contraction (convolutions as
    im2col GEMMs, Dense, LSTM projection, heads); 'simt' = fp32 CUDA cores.  lstm_mode: how the
    recurrent products of the LSTM core are computed: 'tiled' = one persistent kernel each way on
    fp32 CUDA cores, 'tc3' = the same recurrence on wgmma with bf16x3 operands."""
    L = _lib.lib()
    self._num_actions = int(num_actions)
    self._observation_shape = tuple(int(x) for x in observation_shape)
    self._stack_size = int(stack_size)
    if len(self._observation_shape) != 3:
      raise ValueError('observation_shape must be [height, width, channels]')
    if self._stack_size > 1 and self._observation_shape[-1] != 1:
      raise ValueError('Due to frame stacking, we require last observation dimension to be 1. Got {}'.format(
          self._observation_shape[-1]))
    self._channels = self._stack_size if self._stack_size > 1 else self._observation_shape[-1]
    h = ctypes.c_void_p()
    _lib.check(L.seedrl_r2d2_net_create(self._num_actions, self._observation_shape[0], self._observation_shape[1],
                                        self._channels, ctypes.byref(h)))
    self._h = h
    modes = {'simt': 0, 'tc3': 2}
    if gemm_mode not in modes:
      raise ValueError("gemm_mode must be 'simt' or 'tc3'")
    self.gemm_mode = gemm_mode
    _lib.check(L.seedrl_r2d2_net_set_mode(h, modes[gemm_mode]))
    lstm_modes = {'tiled': 2, 'tc3': 3}
    if lstm_mode not in lstm_modes:
      raise ValueError("lstm_mode must be 'tiled' or 'tc3' (the tiled recurrence on wgmma bf16x3)")
    self.lstm_mode = lstm_mode
    _lib.check(L.seedrl_r2d2_net_set_lstm_mode(h, lstm_modes[lstm_mode]))
    self._setup(seed, device)

  def _param_rank(self, index, name_buf, dims, offset):
    rank = ctypes.c_int()
    _lib.check(_lib.lib().seedrl_r2d2_net_param_info(self._h, index, name_buf, len(name_buf), dims,
                                                     ctypes.byref(rank), ctypes.byref(offset)))
    return rank.value

  def assign_from(self, other):
    """update_target_agent (agents/r2d2/learner.py:535-544): target_var.assign(source_var)."""
    if other.arena_floats != self.arena_floats:
      raise ValueError('Mismatch in number of net tensors')
    self.params.copy_(other.params)

  # ---- protocol ---------------------------------------------------------------
  def initial_state(self, batch_size):
    z = torch.zeros([batch_size, LSTM_UNITS], dtype=torch.float32, device=self.device)
    return AgentState(core_state=(z, z.clone()),
                      frame_stacking_state=initial_frame_stacking_state(
                          self._stack_size, batch_size, self._observation_shape, device=self.device))

  def __call__(self, input_, agent_state, unroll=False, is_training=False):
    prev_actions, env_outputs = input_
    reward, done, observation = env_outputs[0], env_outputs[1], env_outputs[2]
    prev_actions = _lib.require_cuda(prev_actions.to(torch.int64), torch.int64, 'prev_actions')
    reward = _lib.require_cuda(reward, torch.float32, 'reward')
    done = _lib.require_cuda(done, torch.bool, 'done')
    observation = _lib.require_cuda(observation, torch.uint8, 'observation')
    if not unroll:    # add the time dimension (networks.py:309-312)
      prev_actions, reward, done, observation = (t.unsqueeze(0) for t in (prev_actions, reward, done, observation))
    T, B = int(prev_actions.shape[0]), int(prev_actions.shape[1])
    if tuple(observation.shape[2:]) != self._observation_shape:
      raise ValueError('observation shape %s, expected %s' % (tuple(observation.shape[2:]), self._observation_shape))
    stacked, frame_state = stack_frames(observation, agent_state.frame_stacking_state, done, self._stack_size)
    h0 = _lib.require_cuda(agent_state.core_state[0], torch.float32, 'core_state.h')
    c0 = _lib.require_cuda(agent_state.core_state[1], torch.float32, 'core_state.c')
    A = self._num_actions
    q = torch.empty([T, B, A], dtype=torch.float32, device=self.device)
    action = torch.empty([T, B], dtype=torch.int32, device=self.device)
    h = torch.empty_like(h0)
    c = torch.empty_like(c0)
    ws = self.workspace(T, B)
    _lib.check(_lib.lib().seedrl_r2d2_net_forward(
        self._h, _lib.ptr(self.params), T, B, _lib.ptr(prev_actions), _lib.ptr(reward), _lib.ptr(done),
        _lib.ptr(stacked), _lib.ptr(h0), _lib.ptr(c0), _lib.ptr(q), _lib.ptr(action), _lib.ptr(h), _lib.ptr(c),
        _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    if is_training:
      self._saved = (T, B, ws, done, stacked)
    out = AgentOutput(action, q)
    if not unroll:
      out = AgentOutput(*(t.squeeze(0) for t in out))
    return out, AgentState((h, c), frame_state)

  def backward(self, dq):
    """d loss / d parameters of the last is_training unroll -> self.grads (overwritten)."""
    if self._saved is None:
      raise RuntimeError('backward() needs a preceding __call__(..., unroll=True, is_training=True)')
    T, B, ws, done, stacked = self._saved
    dq = _lib.require_cuda(dq, torch.float32, 'dq')
    if tuple(dq.shape) != (T, B, self._num_actions):
      raise ValueError('dq must be [T, B, num_actions] of the training unroll')
    _lib.check(_lib.lib().seedrl_r2d2_net_backward(
        self._h, _lib.ptr(self.params), T, B, _lib.ptr(stacked), _lib.ptr(done), _lib.ptr(dq), _lib.ptr(self.grads),
        _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))
    return self.grads
