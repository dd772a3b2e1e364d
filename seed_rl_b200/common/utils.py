"""Runtime utilities on the hot path -- mirror of the reference's `common/utils.py`
for the pieces the V-trace learner uses:

  EnvOutput                     utils.py:41-42
  UnrollStore                   utils.py:119-257   (GPU-resident, scatter/gather kernels)
  Aggregator                    utils.py:461-543   (GPU-resident tables)
  StructuredFIFOQueue           utils.py:680-711   (host queue of GPU-resident nests)
  batch_apply / make_time_major utils.py:714-761   (views; no data movement)
  validate_learner_config       utils.py:989-1002

  PrioritizedReplay             utils.py:260-370   (GPU-resident; sampling = seedrl_replay_sample)
  ProgressLogger                utils.py:546-677   (periodic scalar export; JSON-lines writer)

HER / TPU encode are out of scope (SURVEY 2 row 4).
"""
import collections
import threading

import numpy as np
import torch

from seed_rl_b200 import _lib

EnvOutput = collections.namedtuple(
    'EnvOutput', 'reward done observation abandoned episode_step')

TensorSpec = collections.namedtuple('TensorSpec', 'shape dtype name')
TensorSpec.__new__.__defaults__ = (None,)


# ---- a minimal tf.nest -----------------------------------------------------------
def _is_leaf(x):
  return isinstance(x, TensorSpec) or not isinstance(x, (tuple, list))


def flatten(nest):
  if _is_leaf(nest):
    return [nest]
  out = []
  for e in nest:
    out.extend(flatten(e))
  return out


def pack_sequence_as(structure, flat):
  it = iter(flat)

  def rec(s):
    if _is_leaf(s):
      return next(it)
    vals = [rec(e) for e in s]
    if hasattr(s, '_fields'):
      return type(s)(*vals)
    return type(s)(vals)

  out = rec(structure)
  return out


def map_structure(fn, *nests):
  flats = [flatten(n) for n in nests]
  for f in flats[1:]:
    if len(f) != len(flats[0]):
      raise ValueError("The two structures don't have the same nested structure.")
  return pack_sequence_as(nests[0], [fn(*xs) for xs in zip(*flats)])


def assert_same_structure(a, b):
  if len(flatten(a)) != len(flatten(b)):
    raise ValueError("The two structures don't have the same nested structure.")


_TORCH_DTYPES = {
    'float32': torch.float32, 'float64': torch.float64, 'int32': torch.int32,
    'int64': torch.int64, 'uint8': torch.uint8, 'bool': torch.bool, 'int8': torch.int8,
}


def as_torch_dtype(d):
  if isinstance(d, torch.dtype):
    return d
  return _TORCH_DTYPES[np.dtype(d).name]


def _ids_to_device(env_ids, device):
  """Returns (int32 cuda tensor, host numpy copy or None)."""
  host = None
  if isinstance(env_ids, torch.Tensor):
    if env_ids.device.type != 'cuda':
      host = env_ids.numpy()
  else:
    host = np.asarray(env_ids)
  if host is not None:
    dev = torch.as_tensor(host.astype(np.int32)).to(device, non_blocking=True)
  else:
    dev = env_ids.to(torch.int32)
  return dev.contiguous(), host


def _check_no_duplicates(env_ids_dev, env_ids_host, what):
  if env_ids_host is not None:
    dup = len(np.unique(env_ids_host)) != len(env_ids_host)
  else:
    dup = torch.unique(env_ids_dev).numel() != env_ids_dev.numel()
  if dup:
    # tf.debugging.assert_equal(..., message=...), utils.py:173-176 / 533-540
    raise ValueError('Duplicate environment ids in %s' % what)


class UnrollStore(object):
  """Combines individual environment steps into unrolls (reference utils.py:119-257),
  with the per-env ring buffers resident in HBM."""

  def __init__(self, num_envs, unroll_length, timestep_specs,
               num_overlapping_steps=0, name='UnrollStore', device='cuda',
               time_major=False):
    self.name = name
    self._specs = timestep_specs
    self._flat_specs = flatten(timestep_specs)
    self._full_length = num_overlapping_steps + unroll_length + 1     # :129
    self._unroll_length = unroll_length
    self._num_overlapping_steps = num_overlapping_steps
    self._num_envs = num_envs
    self._time_major = time_major
    self._device = torch.device(device)
    self._state = [
        torch.zeros([num_envs, self._full_length] + list(s.shape),
                    dtype=as_torch_dtype(s.dtype), device=self._device)
        for s in self._flat_specs]                                    # :131-139
    self._index = torch.full([num_envs], num_overlapping_steps, dtype=torch.int32,
                             device=self._device)                     # :142-145
    self._completed = torch.empty([num_envs], dtype=torch.int32, device=self._device)
    self._ncomp = torch.zeros([1], dtype=torch.int32, device=self._device)
    # host mirror of `_index`: which unrolls complete is a pure function of the ids appended so
    # far, so the host never has to read the device counter back (no sync per inference batch)
    self._host_index = np.full([num_envs], num_overlapping_steps, np.int32)

  @property
  def unroll_specs(self):
    return map_structure(
        lambda s: TensorSpec([self._full_length] + list(s.shape), s.dtype, s.name),
        self._specs)

  def _row_bytes(self, i):
    s = self._state[i]
    return int(s[0, 0].numel()) * s.element_size()

  def append(self, env_ids, values, check_duplicates=True):
    """Appends values; returns (completed env ids int64 [n], completed unrolls)."""
    ids, host = _ids_to_device(env_ids, self._device)
    if check_duplicates:
      _check_no_duplicates(ids, host, 'store %s' % self.name)
    assert_same_structure(values, self._specs)
    self.device_append(ids, flatten(values))
    nc = None
    if host is not None and self._host_index is not None:
      nc = int(self.host_advance(host)[0].size)
    else:
      self._host_index = None          # ids live on the device only: fall back to reading the counter
    return self.complete(nc)

  def device_append(self, ids_i32, flat_values, id_limit=None):
    """The device half of `append` (:187-194): every field of the step into its ring row (ONE
    launch) + the index advance / completed-id compaction.  No host work: capturable in a CUDA graph.
    id_limit: rows whose env id is >= id_limit are skipped (a fixed-size batch that also carries
    environments the store has no rows for); feed `host_advance` only the ids below it."""
    L = _lib.lib()
    n = int(ids_i32.numel())
    st = _lib.stream_ptr()
    keep = []
    for i, (s, v) in enumerate(zip(self._state, flat_values)):
      v = _lib.require_cuda(v, s.dtype, 'values')
      if v.shape[0] != n:                                             # :178-184
        raise ValueError('Batch dimension must equal the number of environments in store %s.'
                         % self.name)
      keep.append(v)
    if id_limit is not None and len(keep) > 16:
      raise ValueError('device_append with id_limit takes at most 16 fields (store %s has %d)'
                       % (self.name, len(keep)))
    if n and len(keep) <= 16:
      _lib.rows_multi([(s, v, _lib.ROW_APPEND) for s, v in zip(self._state, keep)], ids_i32, index=self._index,
                      id_limit=id_limit)
    else:
      for i, (s, v) in enumerate(zip(self._state, keep)):
        _lib.check(L.seedrl_store_append_field(
            _lib.ptr(s), _lib.ptr(self._index), _lib.ptr(ids_i32), n, self._full_length,
            self._row_bytes(i), _lib.ptr(v), st))
    if id_limit is None:
      _lib.check(L.seedrl_store_advance(
          _lib.ptr(self._index), _lib.ptr(ids_i32), n, self._full_length,
          _lib.ptr(self._completed), _lib.ptr(self._ncomp), st))      # :194
    else:
      _lib.check(L.seedrl_store_advance_limit(
          _lib.ptr(self._index), _lib.ptr(ids_i32), n, self._full_length,
          _lib.ptr(self._completed), _lib.ptr(self._ncomp), int(id_limit), st))

  def host_advance(self, host_ids):
    """The host half: which of these environments complete an unroll with this step (a pure
    function of the ids appended so far).  Returns (completed env ids, their positions in the
    batch), in batch order -- the order the device kernel compacts them in."""
    hid = np.asarray(host_ids).astype(np.int64).reshape(-1)
    self._host_index[hid] += 1
    pos = np.nonzero(self._host_index[hid] == self._full_length)[0]
    done_host = hid[pos]
    self._host_index[done_host] = 1 + self._num_overlapping_steps     # :254-255
    return done_host, pos

  def complete(self, nc=None):
    """Gathers the `nc` unrolls completed by the last device_append: (completed env ids, unrolls)."""
    L = _lib.lib()
    st = _lib.stream_ptr()
    if nc is None:
      nc = int(self._ncomp.item())      # device-resident ids: the one host sync that sizes the outputs
    done_ids = self._completed[:nc]
    unrolls = []
    for i, s in enumerate(self._state):
      tail = list(s.shape[2:])
      shape = ([self._full_length, nc] if self._time_major else [nc, self._full_length]) + tail
      u = torch.empty(shape, dtype=s.dtype, device=self._device)
      _lib.check(L.seedrl_store_gather_field(
          _lib.ptr(s), _lib.ptr(done_ids), nc, self._full_length, self._row_bytes(i),
          self._num_overlapping_steps, 1 if self._time_major else 0, _lib.ptr(u), st))
      unrolls.append(u)
    _lib.check(L.seedrl_store_finish(_lib.ptr(self._index), _lib.ptr(done_ids), nc,
                                     self._num_overlapping_steps, st))
    return done_ids.to(torch.int64), pack_sequence_as(self._specs, unrolls)

  def complete_into(self, nc, into, on_placed=None):
    """Gathers the `nc` unrolls completed by the last device_append straight into free columns of
    `into` (a BatchAssembler): no per-unroll tensors, no stack, no transpose.  Returns (completed
    env ids, [(slot, col0, n)])."""
    L = _lib.lib()
    st = _lib.stream_ptr()
    done_ids = self._completed[:nc]
    placed, start = [], 0
    while start < nc:
      slot, col0, room = into.claim(nc - start)
      ids = done_ids[start:start + room]
      for i, s in enumerate(self._state):
        dst = into.field(slot, i)
        _lib.check(L.seedrl_store_gather_field_into(
            _lib.ptr(s), _lib.ptr(ids), room, self._full_length, self._row_bytes(i),
            self._num_overlapping_steps, _lib.ptr(dst), into.batch_size, col0, st))
      if on_placed is not None:
        on_placed(slot, col0, ids)       # e.g. the first agent states of these unrolls
      into.commit()                      # publishes the slot if this filled it
      placed.append((slot, col0, room))
      start += room
    _lib.check(L.seedrl_store_finish(_lib.ptr(self._index), _lib.ptr(done_ids), nc,
                                     self._num_overlapping_steps, st))
    return done_ids.to(torch.int64), placed

  def reset(self, env_ids):
    """Reset after actor preemption (reference utils.py:198-225)."""
    L = _lib.lib()
    ids, host = _ids_to_device(env_ids, self._device)
    n = int(ids.numel())
    if n == 0:
      return
    if host is not None and self._host_index is not None:
      self._host_index[np.asarray(host).astype(np.int64).reshape(-1)] = self._num_overlapping_steps
    else:
      self._host_index = None
    st = _lib.stream_ptr()
    _lib.check(L.seedrl_store_reset(None, _lib.ptr(self._index), _lib.ptr(ids), n,
                                    self._full_length, 0, self._num_overlapping_steps, st))
    for i, s in enumerate(self._state):
      _lib.check(L.seedrl_store_reset(_lib.ptr(s), None, _lib.ptr(ids), n, self._full_length,
                                      self._row_bytes(i), self._num_overlapping_steps, st))


class BatchAssembler(object):
  """Zero-copy minibatch assembly (SURVEY 8(f) rank 2).  Holds `slots` preallocated time-major
  training batches ([T+1, B, ...] per field of the unroll specs, plus the [B, ...] first agent
  states); the inference thread's UnrollStore.complete_into(nc, self) gathers every completed
  unroll straight into the next free column.  A full slot is handed to the learner (`get`), which
  returns it with `release(slot)` once its step is enqueued.  Replaces the reference's
  capacity-1 queue of single unrolls + tf.stack + make_time_major (agents/vtrace/learner.py:336,
  418-432); the back-pressure is the same: with every slot full or in use, `claim` blocks the
  inference thread.

  num_tasks = K > 1 (multi-task PopArt) also keeps, per slot, the int32 [B] task of every column: the
  filling thread records env_id % K for the columns it placed (`place_task_ids`), and `task_ids(slot)`
  hands them to the learner next to the batch."""

  def __init__(self, timestep_specs, state_specs, full_length, batch_size, slots=2, device='cuda', num_tasks=1):
    self._specs = timestep_specs
    self.batch_size = int(batch_size)
    self.full_length = int(full_length)
    dev = torch.device(device)
    flat = flatten(timestep_specs)
    self._fields = [[torch.zeros([full_length, batch_size] + list(s.shape), dtype=as_torch_dtype(s.dtype),
                                 device=dev) for s in flat] for _ in range(slots)]
    self._states = [[torch.zeros([batch_size] + list(s.shape), dtype=as_torch_dtype(s.dtype), device=dev)
                     for s in flatten(state_specs)] for _ in range(slots)]
    self._state_specs = state_specs
    self.num_tasks = int(num_tasks)
    self._task_ids = ([torch.zeros([batch_size], dtype=torch.int32, device=dev) for _ in range(slots)]
                      if self.num_tasks > 1 else None)
    self._fill = [0] * slots
    self._free = collections.deque(range(slots))     # slots the inference thread may fill
    self._cur = None
    self._ready = collections.deque()                # full slots, with the event that completes them
    self._released = {}                              # slot -> event after which it may be rewritten
    self._cv = threading.Condition()
    self._closed = False

  def field(self, slot, i):
    return self._fields[slot][i]

  def state(self, slot):
    return pack_sequence_as(self._state_specs, self._states[slot])

  def place_task_ids(self, slot, col0, env_ids):
    """Records env_id % num_tasks, on the device, as the task of columns col0.. of `slot`."""
    if self._task_ids is not None:
      n = int(env_ids.numel())
      self._task_ids[slot][col0:col0 + n].copy_(torch.remainder(env_ids, self.num_tasks).to(torch.int32))

  def task_ids(self, slot):
    """The int32 [B] column tasks of `slot` (None with one task)."""
    return None if self._task_ids is None else self._task_ids[slot]

  def claim(self, want):
    """-> (slot, first free column, columns granted <= want).  Blocks while no slot is free."""
    with self._cv:
      while self._cur is None:
        if self._closed:
          raise QueueClosedError('assembler closed')
        if self._free:
          self._cur = self._free.popleft()
          self._fill[self._cur] = 0
          ev = self._released.pop(self._cur, None)
          if ev is not None and torch.cuda.is_available():
            torch.cuda.current_stream().wait_event(ev)   # the step that read this slot has finished
        else:
          self._cv.wait(0.05)
      slot, col0 = self._cur, self._fill[self._cur]
      n = min(int(want), self.batch_size - col0)
      self._fill[slot] += n
      return slot, col0, n

  def commit(self):
    """Called by the filling thread after the gathers of a claim are enqueued: publishes the slot
    if it is full."""
    with self._cv:
      if self._cur is not None and self._fill[self._cur] == self.batch_size:
        ev = None
        if torch.cuda.is_available():
          ev = torch.cuda.Event()
          ev.record(torch.cuda.current_stream())
        self._ready.append((self._cur, ev))
        self._cur = None
        self._cv.notify_all()

  def get(self, timeout=None):
    """-> (slot, first agent states, time-major nest of the unroll specs); the caller's current
    stream waits for the gathers that filled it."""
    with self._cv:
      while not self._ready:
        if self._closed:
          raise QueueClosedError('assembler closed')
        if not self._cv.wait(timeout if timeout is not None else 0.05) and timeout is not None:
          raise TimeoutError('no full batch')
      slot, ev = self._ready.popleft()
    if ev is not None:
      torch.cuda.current_stream().wait_event(ev)
    return slot, self.state(slot), pack_sequence_as(self._specs, self._fields[slot])

  def release(self, slot):
    ev = None
    if torch.cuda.is_available():
      ev = torch.cuda.Event()
      ev.record(torch.cuda.current_stream())
    with self._cv:
      self._released[slot] = ev
      self._free.append(slot)
      self._cv.notify_all()

  def close(self):
    with self._cv:
      self._closed = True
      self._cv.notify_all()


class Aggregator(object):
  """Per-environment state tables (reference utils.py:461-543), kept as HBM-resident
  tensors; reset/add/read/replace are single indexed row operations."""

  def __init__(self, num_envs, specs, name='Aggregator', device='cuda'):
    self.name = name
    self._specs = specs
    self._device = torch.device(device)
    self._state = [
        torch.zeros([num_envs] + list(s.shape), dtype=as_torch_dtype(s.dtype),
                    device=self._device) for s in flatten(specs)]

  def _ids(self, env_ids):
    if isinstance(env_ids, torch.Tensor):
      return env_ids.to(self._device).long()
    return torch.as_tensor(np.asarray(env_ids, np.int64)).to(self._device)

  def reset(self, env_ids):                                           # :481-485
    ids = self._ids(env_ids)
    for s in self._state:
      s[ids] = 0

  def add(self, env_ids, values):                                     # :488-501
    assert_same_structure(values, self._specs)
    ids = self._ids(env_ids)
    for s, v in zip(self._state, flatten(values)):
      v = torch.as_tensor(v, device=self._device).to(s.dtype)
      if v.dim() < s.dim():
        v = v.expand([ids.numel()] + list(s.shape[1:]))
      s.index_add_(0, ids, v.contiguous())

  def read(self, env_ids):                                            # :504-516
    ids = self._ids(env_ids)
    return pack_sequence_as(self._specs, [s.index_select(0, ids) for s in self._state])

  def replace(self, env_ids, values, debug_op_name='', debug_tensors=None, check_unique=True):  # :519-543
    """check_unique=False skips the duplicate-id assertion (a device sort + a host read-back) for
    callers whose ids are unique by construction (ids the unroll store just reported complete)."""
    ids = self._ids(env_ids)
    if ids.dim() != 1:
      raise ValueError('Invalid rank for aggregator %s' % self.name)
    if check_unique and torch.unique(ids).numel() != ids.numel():
      raise ValueError('Duplicate environment ids in Aggregator: %s with op name "%s"' %
                       (self.name, debug_op_name))
    assert_same_structure(values, self._specs)
    for s, v in zip(self._state, flatten(values)):
      v = torch.as_tensor(v, device=self._device).to(s.dtype)
      if v.dim() < s.dim():
        v = v.expand([ids.numel()] + list(s.shape[1:]))
      s[ids] = v


class PrioritizedReplay(object):
  """Prioritized replay buffer (reference utils.py:260-370) with storage, priorities and the
  sampling arithmetic resident in HBM.  Not thread-safe, like the reference's: call insert()
  and sample() from a single thread.

  Sampling (:327-352) for priority_exp != 0 is ONE kernel (seedrl_replay_sample: p_i =
  prio_i^alpha / sum, inverse-CDF draw, importance weights normalised by their max); the
  reference draws the indices with tf.random.categorical -- same distribution, different random
  stream (its own test is statistical, tests/utils_test.py:353-365)."""

  def __init__(self, size, specs, importance_sampling_exponent, name='PrioritizedReplay', device='cuda'):
    self._size = int(size)
    self._specs = specs
    self._device = torch.device(device)
    self._priorities = torch.zeros([self._size], dtype=torch.float32, device=self._device)
    self._buffer = map_structure(
        lambda ts: torch.zeros([self._size] + list(ts.shape), dtype=as_torch_dtype(ts.dtype), device=self._device),
        specs)
    self.num_inserted = 0
    self._importance_sampling_exponent = float(importance_sampling_exponent)

  def insert(self, values, priorities):
    """FIFO insertion/removal with wrap-around (:277-309).  Returns the inserted indices."""
    assert_same_structure(values, self._buffer)
    flat_v = [_lib.require_cuda(v, b.dtype, 'values') for v, b in zip(flatten(values), flatten(self._buffer))]
    append_size = int(flat_v[0].shape[0])
    start = self.num_inserted
    insert_indices = (torch.arange(start, start + append_size, device=self._device) % self._size)
    for b, v in zip(flatten(self._buffer), flat_v):
      if tuple(v.shape[1:]) != tuple(b.shape[1:]):
        raise ValueError('value of shape %s does not match the spec %s' % (tuple(v.shape[1:]), tuple(b.shape[1:])))
      b.index_copy_(0, insert_indices, v)
    self.num_inserted += append_size
    self._priorities.index_copy_(0, insert_indices, _lib.require_cuda(priorities, torch.float32, 'priorities'))
    return insert_indices

  def sample(self, num_samples, priority_exp, generator=None, uniforms=None):
    """(:311-357) -> (indices int64 [num_samples], weights float32 [num_samples], sampled values
    with an added front batch dimension)."""
    if self.num_inserted <= 0:
      raise ValueError('Cannot sample if replay buffer is empty')
    limit = min(self._size, self.num_inserted)
    if priority_exp == 0:
      indices = torch.randint(0, limit, [num_samples], dtype=torch.int64, device=self._device, generator=generator)
      weights = torch.ones([num_samples], dtype=torch.float32, device=self._device)
    else:
      if uniforms is None:
        uniforms = torch.rand(num_samples, device=self._device, generator=generator)
      u = _lib.require_cuda(uniforms, torch.float32, 'uniforms')
      indices = torch.empty(num_samples, dtype=torch.int64, device=self._device)
      weights = torch.empty(num_samples, dtype=torch.float32, device=self._device)
      _lib.check(_lib.lib().seedrl_replay_sample(
          limit, _lib.ptr(self._priorities), float(priority_exp), self._importance_sampling_exponent,
          int(num_samples), _lib.ptr(u), _lib.ptr(indices), _lib.ptr(weights), None, _lib.stream_ptr()))
    sampled_values = map_structure(lambda b: b.index_select(0, indices), self._buffer)
    return indices, weights, sampled_values

  def update_priorities(self, indices, priorities):
    """(:359-370) duplicate indices: which priority wins is unspecified, as in the reference."""
    self._priorities.index_copy_(0, _lib.require_cuda(indices, torch.int64, 'indices'),
                                 _lib.require_cuda(priorities, torch.float32, 'priorities'))


class SummaryWriter(object):
  """Stand-in for tf.summary.create_file_writer (TensorFlow is not part of this stack): scalars
  go to `<logdir>/summaries.jsonl`, one {"step", "tag", "value", "wall_time"} object per line --
  the same (step, tag, value) triples TensorBoard event files hold."""

  def __init__(self, logdir, filename='summaries.jsonl'):
    import os
    os.makedirs(logdir, exist_ok=True)
    self.path = os.path.join(logdir, filename)
    self._f = open(self.path, 'a')
    self._lock = threading.Lock()
    self.step = 0

  def set_step(self, step):
    self.step = int(step)

  def scalar(self, tag, value, step=None):
    import json, time
    with self._lock:
      self._f.write(json.dumps({'step': int(self.step if step is None else step), 'tag': tag,
                                'value': float(value), 'wall_time': time.time()}) + '\n')

  def flush(self):
    with self._lock:
      self._f.flush()

  def close(self):
    with self._lock:
      self._f.close()


class ProgressLogger(object):
  """Periodic logging of the training progress (reference utils.py:546-677): the learner
  thread hands the step's scalars over with `step_end` (device tensors: no host sync on the hot
  path); a logger thread exports the latest values with exponential back-off of the period
  (initial_period * period_factor^k, capped at max_period) plus `speed/steps_per_sec`."""

  def __init__(self, summary_writer=None, initial_period=0.1, period_factor=1.01, max_period=10.0,
               starting_step=0):
    self.summary_writer = None
    self.last_log_time = None
    self.last_log_step = 0
    self.period = initial_period
    self.period_factor = period_factor
    self.max_period = max_period
    self.log_keys = []
    self.log_keys_set = set()
    self.step_cnt = -1
    self.ready_values = None
    self.logger_thread = None
    self.logging_callback = None
    self.terminator = None
    self._lock = threading.Lock()
    self.reset(summary_writer, starting_step)

  def reset(self, summary_writer=None, starting_step=0):
    import timeit
    with self._lock:
      self.summary_writer = summary_writer
      self.step_cnt = int(starting_step)
      self.ready_values = None
      self.last_log_time = timeit.default_timer()
      self.last_log_step = int(starting_step)

  def start(self, logging_callback=None):
    assert self.logger_thread is None
    self.logging_callback = logging_callback
    self.terminator = threading.Event()
    self.logger_thread = threading.Thread(target=self._logging_loop, daemon=True)
    self.logger_thread.start()

  def shutdown(self):
    assert self.logger_thread
    self.terminator.set()
    self.logger_thread.join()
    self.logger_thread = None

  def log_session(self):
    return []

  def log(self, session, name, value):
    if name not in self.log_keys_set:
      self.log_keys.append(name)
      self.log_keys_set.add(name)
    session.append(value)

  def log_session_from_dict(self, dic):
    session = self.log_session()
    for key in dic:
      self.log(session, key, dic[key])
    return session

  def step_end(self, session, strategy=None, step_increment=1):
    """`strategy` is accepted for signature compatibility (one replica per process here; the
    reference logs replica 0's value, utils.py:631-635)."""
    with self._lock:
      self.ready_values = list(session)
      self.step_cnt += int(step_increment)

  def _log(self):
    import timeit
    logging_time = timeit.default_timer()
    with self._lock:
      step_cnt, values = self.step_cnt, self.ready_values
    if step_cnt == self.last_log_step or values is None:
      return
    assert len(values) == len(self.log_keys), (
        'Mismatch between number of keys and values to log: %r vs %r' % (values, self.log_keys))
    values = [float(v) for v in values]      # device -> host here, on the logger thread
    w = self.summary_writer
    if w:
      w.set_step(step_cnt)
    if self.logging_callback:
      self.logging_callback()
    dt = logging_time - self.last_log_time
    df = float(step_cnt - self.last_log_step)
    if w:
      for key, value in zip(self.log_keys, values):
        w.scalar(key, value)
      w.scalar('speed/steps_per_sec', df / dt)
      w.flush()
    self.last_values = dict(zip(self.log_keys, values), **{'speed/steps_per_sec': df / dt})
    self.last_log_time, self.last_log_step = logging_time, step_cnt

  def _logging_loop(self):
    import timeit
    last_log_try = timeit.default_timer()
    while not self.terminator.is_set():
      try:
        self._log()
      except Exception:                       # pylint: disable=broad-except
        import logging as _logging
        _logging.getLogger(__name__).critical('Logging failed.', exc_info=True)
      now = timeit.default_timer()
      elapsed = now - last_log_try
      last_log_try = now
      self.period = min(self.period_factor * self.period, self.max_period)
      self.terminator.wait(timeout=max(0, self.period - elapsed))


class QueueClosedError(RuntimeError):
  """tf.errors.CancelledError analogue for a closed queue."""


class StructuredFIFOQueue(object):
  """FIFO of nests (reference utils.py:680-711 over tf.queue.FIFOQueue).  Elements
  stay wherever their tensors live (HBM); capacity gives the same back-pressure as
  the reference's capacity-1 unroll queue (learner.py:336).  capacity -1 = unbounded."""

  def __init__(self, capacity, specs, shared_name=None, name='structured_fifo_queue'):
    self._specs = specs
    self._capacity = capacity
    self._q = collections.deque()
    self._cv = threading.Condition()
    self._closed = False

  def size(self):
    with self._cv:
      return len(self._q)

  def close(self, cancel_pending_enqueues=True):
    with self._cv:
      self._closed = True
      self._cv.notify_all()

  def enqueue(self, vals, name=None):
    assert_same_structure(vals, self._specs)
    with self._cv:
      while self._capacity > 0 and len(self._q) >= self._capacity and not self._closed:
        self._cv.wait()
      if self._closed:
        raise QueueClosedError('Queue is closed.')
      self._q.append(vals)
      self._cv.notify_all()

  def enqueue_many(self, vals, name=None):
    assert_same_structure(vals, self._specs)
    flat = flatten(vals)
    n = int(flat[0].shape[0]) if flat else 0
    for i in range(n):
      self.enqueue(pack_sequence_as(self._specs, [f[i] for f in flat]))

  def dequeue(self, name=None):
    with self._cv:
      while not self._q and not self._closed:
        self._cv.wait()
      if not self._q:
        raise QueueClosedError('Queue is closed and empty.')
      v = self._q.popleft()
      self._cv.notify_all()
      return v

  def dequeue_many(self, batch_size, name=None):
    items = [self.dequeue() for _ in range(batch_size)]
    return map_structure(lambda *xs: torch.stack([torch.as_tensor(x) for x in xs]), *items)


def batch_apply(fn, inputs):
  """Folds time into batch, runs fn, unfolds (reference utils.py:714-732)."""
  flat = flatten(inputs)
  T = int(flat[0].shape[0])
  batched = map_structure(lambda t: t.reshape([-1] + list(t.shape[2:])), inputs)
  output = fn(*batched)
  return map_structure(lambda t: t.reshape([T, -1] + list(t.shape[1:])), output)


def make_time_major(x):
  """Transposes batch and time (reference utils.py:735-761); rank<2 passes through."""
  def transpose(t):
    if t.dim() < 2:
      return t
    return t.transpose(0, 1).contiguous()
  return map_structure(transpose, x)


def validate_learner_config(config, num_hosts=1):
  """reference utils.py:989-1002."""
  assert config.num_envs > 0
  assert config.env_batch_size > 0
  if config.inference_batch_size == -1:
    config.inference_batch_size = max(config.env_batch_size,
                                      config.num_envs // (2 * num_hosts))
  assert config.inference_batch_size > 0
  assert config.inference_batch_size % config.env_batch_size == 0, (
      'Learner-side batch size (=%d) must be exact multiple of the '
      'actor-side batch size (=%d).' %
      (config.inference_batch_size, config.env_batch_size))
  assert config.num_envs >= config.inference_batch_size * num_hosts, (
      'Inference batch size is bigger than the number of environments.')
