"""Central inference on one GPU, shared by the V-trace and the R2D2 learner: the `inference` closure
the reference builds around its unroll store (agents/vtrace/learner.py:349-407,
agents/r2d2/learner.py:711-790).

Per batch: run-id resets and episode statistics on the host -> H2D -> ONE gather launch (previous
action + agent state) -> T=1 forward + action selection -> ONE store append -> ONE scatter launch ->
actions D2H.  The device part is `_device_step`, run eagerly or, for a batch of exactly
`inference_batch_size` rows with `use_graph`, as one CUDA-graph replay; everything around it is the
same code for both.  The agents subclass `InferenceHostBase` for their specs, their policy and what
happens to completed unrolls.
"""
from absl import logging
import numpy as np
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common import utils
from seed_rl_b200.grpc import ops as grpc


class InferenceHostBase(object):
  """Per-environment tables, the unroll store and the bound `inference` function.  Subclasses
  provide `_policy` and `_completed_unrolls`, and set `unroll_specs` and `unroll_queue`."""

  algorithm = None        # the agent's name in error messages

  def __init__(self, agent, num_envs, inference_batch_size, observation_shape, action_dtype,
               agent_state_specs, agent_output_specs, unroll_length, num_overlapping_steps=0,
               time_major=False, id_limit=None, num_action_repeats=1, device='cuda', info_queue=None,
               use_graph=False, allow_abandoned=False):
    """id_limit: environments with ids >= id_limit have no store rows (None: every environment has).
    use_graph: replay the device side of every batch of exactly `inference_batch_size` rows as one
    CUDA graph; other batch sizes run it eagerly.  allow_abandoned: accept rows with
    `abandoned` set (each must also have `done`: the reset observation after a time limit), for a
    learner that bootstraps from them; otherwise they raise, as in the reference."""
    self.agent = agent
    self.allow_abandoned = bool(allow_abandoned)
    self.device = torch.device(device)
    self.N = N = int(inference_batch_size)
    self.num_action_repeats = num_action_repeats
    TS = utils.TensorSpec
    self.env_output_specs = utils.EnvOutput(
        TS([], 'float32', 'reward'), TS([], 'bool', 'done'), TS(list(observation_shape), 'uint8', 'observation'),
        TS([], 'bool', 'abandoned'), TS([], 'int32', 'episode_step'))
    action_specs = TS([], action_dtype, 'action')
    self.agent_state_specs = agent_state_specs
    self._id_limit = id_limit
    self._num_store_envs = num_envs if id_limit is None else id_limit
    self.store = utils.UnrollStore(self._num_store_envs, unroll_length,
                                   (action_specs, self.env_output_specs, agent_output_specs),
                                   num_overlapping_steps=num_overlapping_steps, device=device, time_major=time_major)
    # run ids / episode stats feed host-side logging only -> host tables
    self.env_run_ids = np.zeros([num_envs], np.int64)
    self.env_infos = [np.zeros([num_envs], np.int64), np.zeros([num_envs], np.float32),
                      np.zeros([num_envs], np.float32)]
    self.first_agent_states = utils.Aggregator(num_envs, agent_state_specs, 'first_agent_states', device)
    self.agent_states = utils.Aggregator(num_envs, agent_state_specs, 'agent_states', device)
    self.actions = utils.Aggregator(num_envs, action_specs, 'actions', device)
    self.info_queue = info_queue
    self.inference_specs = (
        TS([N], 'int32', 'env_id'), TS([N], 'int64', 'run_id'),
        utils.map_structure(lambda s: TS([N] + list(s.shape), s.dtype, s.name), self.env_output_specs),
        TS([N], 'float32', 'raw_reward'))
    self.output_specs = TS([N], action_dtype, 'action')
    self.stream = torch.cuda.Stream(device=self.device)
    self.use_graph = bool(use_graph)
    if self.use_graph and not 1 <= N <= num_envs:     # the capture runs on env ids 0..N-1
      raise ValueError('cuda_graph needs 1 <= inference_batch_size <= num_envs, got %d and %d' % (N, num_envs))
    self._graph = None
    self._actions_pin = torch.zeros([N], dtype=utils.as_torch_dtype(action_dtype)).pin_memory()

    @grpc.function(self.inference_specs, self.output_specs)
    def inference(env_ids, run_ids, env_outputs, raw_rewards):
      return self._inference(env_ids, run_ids, env_outputs, raw_rewards)
    self.inference = inference

  def _policy(self, ids32, prev_actions, env_outputs, prev_states, counter):
    """T=1 forward and action selection -> (agent outputs, new agent states).  `counter` is the
    graph's int64 device scalar of Philox offsets, or None on the eager path."""
    raise NotImplementedError

  def _completed_unrolls(self, nc):
    """Takes the `nc` unrolls the last append completed out of the store, with their first agent
    states -> (completed env ids, a batch of unroll-queue items or None)."""
    raise NotImplementedError

  def _episode_infos(self, done_ids):
    """The info-queue items of the environments whose episode ended."""
    return tuple(torch.as_tensor(t[done_ids]) for t in self.env_infos)

  def _begin_batch(self, env_ids, run_ids, env_outputs, raw_rewards):
    """Validation, run-id resets and episode statistics (host tables, plus the rare device resets on
    the current stream).  Invalid batches raise before any table is touched."""
    abandoned = np.asarray(env_outputs.abandoned, bool)
    if abandoned.any():
      if not self.allow_abandoned:
        raise ValueError('Abandoned done states are not supported in %s.' % self.algorithm)
      if (abandoned & ~np.asarray(env_outputs.done, bool)).any():
        raise ValueError('An abandoned step must also be done (env ids %s).' %
                         np.asarray(env_ids)[abandoned & ~np.asarray(env_outputs.done, bool)])
    utils._check_no_duplicates(None, env_ids, 'inference batch')
    # Reset the environments that had their first run or crashed.
    previous = self.env_run_ids[env_ids]
    self.env_run_ids[env_ids] = run_ids
    reset_ids = env_ids[previous != run_ids]
    if reset_ids.size:
      logging.info('Environment ids needing reset: %s', reset_ids)
      for t in self.env_infos:
        t[reset_ids] = 0
      self.store.reset(reset_ids[reset_ids < self._num_store_envs])
      init = self.agent.initial_state(len(reset_ids))
      self.first_agent_states.replace(reset_ids, init)
      self.agent_states.replace(reset_ids, init)
      self.actions.reset(reset_ids)
    self.env_infos[1][env_ids] += np.asarray(env_outputs.reward)
    self.env_infos[2][env_ids] += np.asarray(raw_rewards)
    done_ids = env_ids[np.asarray(env_outputs.done)]
    if self.info_queue is not None and done_ids.size:
      self.info_queue.enqueue_many(self._episode_infos(done_ids))
    for t in self.env_infos:
      t[done_ids] = 0
    self.env_infos[0][env_ids] += self.num_action_repeats

  def _device_step(self, ids32, env_dev, counter):
    """Everything of one inference batch that runs on the device.  Host-free: on the graph's
    static buffers it is captured once and replayed per batch.  -> (flat previous agent states,
    agent outputs)."""
    n = int(ids32.numel())
    tables = self.agent_states._state
    prev_actions = torch.empty([n], dtype=self.actions._state[0].dtype, device=self.device)
    prev_states = [torch.empty([n] + list(t.shape[1:]), dtype=t.dtype, device=self.device) for t in tables]
    _lib.rows_multi([(self.actions._state[0], prev_actions, _lib.ROW_GATHER)] +
                    [(t, r, _lib.ROW_GATHER) for t, r in zip(tables, prev_states)], ids32)
    agent_outputs, curr_states = self._policy(
        ids32, prev_actions, env_dev, utils.pack_sequence_as(self.agent_state_specs, prev_states), counter)
    self.store.device_append(ids32, utils.flatten((prev_actions, env_dev, agent_outputs)), id_limit=self._id_limit)
    _lib.rows_multi([(t, r.contiguous(), _lib.ROW_SCATTER) for t, r in zip(tables, utils.flatten(curr_states))] +
                    [(self.actions._state[0], agent_outputs.action.contiguous(), _lib.ROW_SCATTER)], ids32)
    return prev_states, agent_outputs

  def _build_graph(self):
    N, dev = self.N, self.device
    self._g_ids = torch.arange(N, dtype=torch.int32, device=dev)     # distinct ids for the warm-up / capture
    self._g_env = utils.EnvOutput(*(torch.zeros([N] + list(s.shape), dtype=utils.as_torch_dtype(s.dtype), device=dev)
                                    for s in self.env_output_specs))
    self._g_pin = [torch.zeros_like(t, device='cpu').pin_memory() for t in (self._g_ids,) + tuple(self._g_env)]
    self._g_counter = torch.zeros([], dtype=torch.int64, device=dev)
    # one eager warm-up (lazy initialisation: workspaces, kernel attributes), then every table it
    # touched is restored; the capture itself executes nothing
    touched = (self.actions._state + self.agent_states._state + self.store._state +
               [self.store._index, self._g_counter])
    saved = [t.clone() for t in touched]
    self._device_step(self._g_ids, self._g_env, self._g_counter)
    for t, sv in zip(touched, saved):
      t.copy_(sv)
    self.stream.synchronize()
    g = torch.cuda.CUDAGraph()
    # thread_local: other threads (the learner, other hosts) may launch on their streams meanwhile
    with torch.cuda.graph(g, stream=self.stream, capture_error_mode='thread_local'):
      self._g_prev_states, self._g_out = self._device_step(self._g_ids, self._g_env, self._g_counter)
    # the agent's (1, N) workspace the graph captured: eager batches of other sizes may evict it from the
    # agent's cache, and every replay still writes into it
    self._g_workspace = self.agent.workspace(1, N)
    self._graph = g

  def _inference(self, env_ids, run_ids, env_outputs, raw_rewards):
    env_ids, run_ids = np.asarray(env_ids), np.asarray(run_ids)
    n = len(env_ids)
    with torch.cuda.stream(self.stream):
      self._begin_batch(env_ids, run_ids, env_outputs, raw_rewards)
      if self.use_graph and n == self.N:
        if self._graph is None:
          self._build_graph()
        # inputs: host arrays -> pinned staging -> the graph's static device buffers
        srcs = (env_ids.astype(np.int32),) + tuple(np.asarray(x) for x in env_outputs)
        for pin, dst, src in zip(self._g_pin, (self._g_ids,) + tuple(self._g_env), srcs):
          t = torch.from_numpy(np.ascontiguousarray(src))
          if t.numel() >= 65536 and t.is_pinned():
            dst.copy_(t, non_blocking=True)        # the batcher's slabs are pinned: DMA straight from them
          else:
            pin.numpy()[...] = src                 # small fields / pageable memory: own pinned staging
            dst.copy_(pin, non_blocking=True)
        self._graph.replay()
        prev_states, agent_outputs = self._g_prev_states, self._g_out
      else:
        ids32 = torch.as_tensor(env_ids.astype(np.int32)).to(self.device, non_blocking=True)
        env_dev = utils.EnvOutput(*(torch.as_tensor(np.asarray(x)).to(self.device, non_blocking=True)
                                    for x in env_outputs))
        prev_states, agent_outputs = self._device_step(ids32, env_dev, None)
      # completed unrolls, known on the host from the ids appended so far; positions in the batch
      store_pos = np.nonzero(env_ids < self._num_store_envs)[0]
      done_ids, pos = self.store.host_advance(env_ids[store_pos])
      pending = None
      if done_ids.size:
        completed_ids, pending = self._completed_unrolls(int(done_ids.size))
        # the state the next unroll starts from = the state this step started from
        pos_dev = torch.as_tensor(store_pos[pos].astype(np.int64)).to(self.device, non_blocking=True)
        self.first_agent_states.replace(completed_ids, [t.index_select(0, pos_dev) for t in prev_states],
                                        check_unique=False)
      actions = self._actions_pin[:n]
      actions.copy_(agent_outputs.action, non_blocking=True)
      self.stream.synchronize()
    # The unrolls were produced on self.stream, which is drained now: only now are they handed to
    # the learner thread (which consumes them on another stream).
    if pending is not None:
      self.unroll_queue.enqueue_many(pending)
    return actions.numpy().copy()
