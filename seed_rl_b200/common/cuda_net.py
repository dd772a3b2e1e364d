"""What the agent networks of libseedrl_b200 share on the Python side (dmlab/networks.py: ImpalaDeep and
ImpalaShallow; atari/networks.py: DuelingLSTMDQNNet): the network handle, the parameter table, the flat
parameter and gradient arenas with their named views, the Keras initialisation, the per-thread workspace
cache, the error check of the last training call and the checkpoint format."""
import collections
import ctypes
import math
import threading

import numpy as np
import torch

from seed_rl_b200 import _lib


class CudaNet(object):
  """Subclasses create the handle (`self._h`), set their modes and call `_setup`.  They provide `_LIB`, the
  prefix of their C-ABI entry points, and `_param_rank`, their readout of one parameter-table entry."""

  _LIB = None
  _EXTRA_PARAMS = 0        # table entries after the network's tensors (ImpalaDeep: entropy_cost_param)

  def _fn(self, name):
    return getattr(_lib.lib(), self._LIB + '_' + name)

  def _param_rank(self, index, name_buf, dims, offset):
    """Fills the name, dims and offset of table entry `index`; -> its rank."""
    raise NotImplementedError

  def _setup(self, seed, device):
    self._n_tensors = int(self._fn('num_param_tensors')(self._h))
    self.arena_floats = int(self._fn('arena_floats')(self._h))
    self.num_params = int(self._fn('num_params')(self._h))
    self.param_info = []       # (name, shape, offset in floats), the whole table
    for i in range(self._n_tensors + self._EXTRA_PARAMS):
      name, dims, off = ctypes.create_string_buffer(128), (ctypes.c_int64 * 4)(), ctypes.c_size_t()
      rank = self._param_rank(i, name, dims, off)
      self.param_info.append((name.value.decode(), tuple(int(dims[k]) for k in range(rank)), int(off.value)))
    self.device = torch.device(device if device is not None else ('cuda:%d' % torch.cuda.current_device()))
    # flat arenas: params / grads (Adam slots live in the optimizer)
    self.params = torch.zeros(self.arena_floats, dtype=torch.float32, device=self.device)
    self.grads = torch.zeros_like(self.params)
    self._init_parameters(seed)
    self._workspaces = {}      # thread id -> OrderedDict((T1, B) -> workspace), least recently used first
    self._lock = threading.Lock()
    self._saved = None         # the last is_training call: (T1, B, workspace, what backward() needs)

  def __del__(self):
    try:
      if getattr(self, '_h', None):
        self._fn('destroy')(self._h)
        self._h = None
    except Exception:   # interpreter shutdown
      pass

  # ---- parameters ---------------------------------------------------------------
  def _view(self, arena, i):
    _, shape, off = self.param_info[i]
    n = int(np.prod(shape)) if shape else 1
    return arena[off:off + n].view(shape if shape else ())

  @property
  def trainable_variables(self):
    return [self._view(self.params, i) for i in range(self._n_tensors)]

  @property
  def variable_names(self):
    return [p[0] for p in self.param_info[:self._n_tensors]]

  def named_parameters(self):
    return collections.OrderedDict((self.param_info[i][0], self._view(self.params, i)) for i in range(self._n_tensors))

  def named_gradients(self):
    return collections.OrderedDict((p[0], self._view(self.grads, i)) for i, p in enumerate(self.param_info))

  def load_named_parameters(self, named):
    """Copies {name: array} (Keras layouts, any entry of the table) into the arena."""
    mine = collections.OrderedDict((p[0], self._view(self.params, i)) for i, p in enumerate(self.param_info))
    for k, v in named.items():
      t = torch.as_tensor(np.asarray(v, np.float32))
      if tuple(t.shape) != tuple(mine[k].shape):
        raise ValueError('shape mismatch for %s: %s vs %s' % (k, tuple(t.shape), tuple(mine[k].shape)))
      mine[k].copy_(t)

  def _init_parameters(self, seed):
    """Keras defaults (TF 2.4.1): glorot_uniform kernels, zero biases, orthogonal recurrent kernel,
    unit_forget_bias.  One-time host-side work."""
    rng = np.random.default_rng(seed)
    units = dict((p[0], p[1]) for p in self.param_info)['core/recurrent_kernel'][0]
    for i in range(self._n_tensors):
      name, shape, _ = self.param_info[i]
      if name.endswith('bias'):
        a = np.zeros(shape, np.float32)
        if name == 'core/bias':
          a[units:2 * units] = 1.0
      elif name == 'core/recurrent_kernel':
        q, r = np.linalg.qr(rng.normal(size=(shape[1], shape[0])))
        a = (q * np.sign(np.diag(r))).T.astype(np.float32)
      else:
        rf = int(np.prod(shape[:-2])) if len(shape) > 2 else 1
        lim = math.sqrt(6.0 / (shape[-2] * rf + shape[-1] * rf))
        a = rng.uniform(-lim, lim, shape).astype(np.float32)
      self._view(self.params, i).copy_(torch.from_numpy(a))

  # ---- workspaces ---------------------------------------------------------------
  def workspace(self, T1, B):
    """The activation workspace of a (T1, B) call on the calling thread.  Threads never share one: the
    inference thread and the learner thread use this agent's parameters at once.  Each thread keeps its
    two most recently used shapes (the learner's one, or R2D2's burn-in and suffix; a full and a partial
    inference batch); a miss evicts the older one.  Whoever needs a workspace past that holds a reference:
    backward() the one of its training forward, a CUDA graph the one it captured."""
    key = (int(T1), int(B))
    with self._lock:
      mine = self._workspaces.setdefault(threading.get_ident(), collections.OrderedDict())
      ws = mine.get(key)
      if ws is None:
        if len(mine) >= 2:
          mine.popitem(last=False)      # freed before the new one is allocated
        ws = torch.empty(int(self._fn('workspace_bytes')(self._h, *key)), dtype=torch.uint8, device=self.device)
        mine[key] = ws
      else:
        mine.move_to_end(key)
    return ws

  def check_errors(self):
    """Raises if a kernel of the last training forward/backward hit a bounded-wait timeout
    (synchronises the current stream; call where the loss is read anyway)."""
    if self._saved is None:
      return
    T1, B, ws = self._saved[:3]
    _lib.check(self._fn('check_error')(self._h, T1, B, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()))

  def state_dict(self):
    return {'params': self.params.detach().cpu(), 'param_info': self.param_info}

  def load_state_dict(self, d):
    self.params.copy_(d['params'].to(self.device))
