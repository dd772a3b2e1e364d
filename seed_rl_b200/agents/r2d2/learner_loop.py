"""`learner_loop` of the R2D2 agent -- mirror of reference agents/r2d2/learner.py:478-900: the
central inference closure bound on the RPC server (:686-790: run-id resets, epsilon-greedy, unroll
store with `burn_in` overlapping steps, initial priorities from the behaviour Q values, unroll
queue), the replay-feeding dataset (`create_dataset`, :389-467) and the training loop (:805-900:
target sync every `update_target_every_n_step`, minimize, priority write-back, checkpoints), for one
replica (= one GPU / process).

Everything per-environment lives in HBM (previous action, LSTM state, bit-packed frame-stacking
state, unroll store); the inference batch does: H2D -> one gather launch -> T=1
`seedrl_r2d2_net_forward` (frame stacking + DuelingLSTMDQNNet) -> epsilon-greedy -> one append
launch into the store -> one scatter launch -> actions D2H.  With `cuda_graph=True` the device part
of a full batch is one CUDA-graph replay and epsilon-greedy is drawn on the device.
"""
import math
import os
import time

from absl import flags
from absl import logging
import numpy as np
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.agents.r2d2 import learner
from seed_rl_b200.atari import networks
from seed_rl_b200.common import utils
from seed_rl_b200.grpc import ops as grpc

FLAGS = flags.FLAGS


class R2D2InferenceHost(object):
  """What the reference builds around `inference` (learner.py:656-793) for one GPU."""

  def __init__(self, agent, num_envs, num_eval_envs, inference_batch_size, observation_shape, settings=None,
               num_action_repeats=1, device='cuda', unroll_queue_max_size=100, generator=None, cuda_graph=False,
               epsilon_seed=0):
    """generator: the torch generator epsilon-greedy draws from on the eager path.  cuda_graph: replay
    the device side of every batch of exactly `inference_batch_size` rows as one CUDA graph, with
    epsilon-greedy drawn on the device from Philox keyed by `epsilon_seed` (a different random stream
    than `generator`'s, so the explored actions differ; the distribution is the same).  Other batch
    sizes take the eager path."""
    self.agent = agent
    self.settings = s = settings or learner.default_settings()
    self.device = torch.device(device)
    self.N = int(inference_batch_size)
    self.num_envs, self.num_eval_envs = int(num_envs), int(num_eval_envs)
    self.num_training_envs = self.num_envs - self.num_eval_envs                      # :122-123
    if self.num_training_envs <= 0:
      raise ValueError('Total number of environments ({}) should be greater than number of environments '
                       'reserved to eval ({})'.format(num_envs, num_eval_envs))            # :473-476
    self.num_action_repeats = num_action_repeats
    self.generator = generator
    TS = utils.TensorSpec
    A = agent._num_actions
    self.env_output_specs = utils.EnvOutput(
        TS([], 'float32', 'reward'), TS([], 'bool', 'done'), TS(list(observation_shape), 'uint8', 'observation'),
        TS([], 'bool', 'abandoned'), TS([], 'int32', 'episode_step'))
    action_specs = TS([], 'int32', 'action')
    agent_output_specs = networks.AgentOutput(TS([], 'int32', 'action'), TS([A], 'float32', 'q_values'))
    npix = int(np.prod(observation_shape))
    self.agent_state_specs = networks.AgentState(
        (TS([networks.LSTM_UNITS], 'float32', 'h'), TS([networks.LSTM_UNITS], 'float32', 'c')),
        TS([npix], 'int32', 'frame_stacking_state') if agent._stack_size > 1 else ())
    # Buffer of incomplete unrolls: training environments only, burn_in overlapping steps (:659-662)
    self.store = utils.UnrollStore(self.num_training_envs, s.unroll_length,
                                   (action_specs, self.env_output_specs, agent_output_specs),
                                   num_overlapping_steps=s.burn_in, device=device, time_major=False)
    self.env_run_ids = np.zeros([num_envs], np.int64)
    self.env_infos = [np.zeros([num_envs], np.int64), np.zeros([num_envs], np.float32),
                      np.zeros([num_envs], np.float32)]
    self.first_agent_states = utils.Aggregator(num_envs, self.agent_state_specs, 'first_agent_states', device)
    self.agent_states = utils.Aggregator(num_envs, self.agent_state_specs, 'agent_states', device)
    self.actions = utils.Aggregator(num_envs, action_specs, 'actions', device)
    self.unroll_specs = learner.Unroll(self.agent_state_specs, TS([], 'float32', 'priority'),
                                       *self.store.unroll_specs)
    self.unroll_queue = utils.StructuredFIFOQueue(unroll_queue_max_size, self.unroll_specs)   # :686-687
    self.info_queue = utils.StructuredFIFOQueue(-1, (TS([], 'int64', 'episode_num_frames'),
                                                     TS([], 'float32', 'episode_returns'),
                                                     TS([], 'float32', 'episode_raw_returns'),
                                                     TS([], 'int32', 'env_ids')))
    N = self.N
    self.inference_specs = (
        TS([N], 'int32', 'env_id'), TS([N], 'int64', 'run_id'),
        utils.map_structure(lambda t: TS([N] + list(t.shape), t.dtype, t.name), self.env_output_specs),
        TS([N], 'float32', 'raw_reward'))
    self.output_specs = TS([N], 'int32', 'action')
    self.stream = torch.cuda.Stream(device=self.device)
    self.use_graph = bool(cuda_graph)
    if self.use_graph and not 1 <= N <= self.num_envs:
      raise ValueError('cuda_graph needs 1 <= inference_batch_size <= num_envs, got %d and %d' % (N, self.num_envs))
    self.epsilon_seed = int(epsilon_seed)
    # the eager path's per-env epsilons (:129-152), built once; the graph's Philox offset
    self.envs_epsilon = learner.get_envs_epsilon(torch.arange(self.num_envs, device=self.device),
                                                 self.num_training_envs, self.num_eval_envs,
                                                 s.eval_epsilon).contiguous()
    self.epsilon_counter = torch.zeros([], dtype=torch.int64, device=self.device)
    self._graph = None

    @grpc.function(self.inference_specs, self.output_specs)
    def inference(env_ids, run_ids, env_outputs, raw_rewards):
      return self._inference(env_ids, run_ids, env_outputs, raw_rewards)
    self.inference = inference

  def _state_tables(self, agg):
    return list(agg._state)

  def _begin_batch(self, env_ids, run_ids, env_outputs, raw_rewards):
    """reference learner.py:731-757: run-id resets and episode statistics (host work, plus the rare
    device resets on the current stream)."""
    reward, done = np.asarray(env_outputs.reward), np.asarray(env_outputs.done)
    previous = self.env_run_ids[env_ids]                                       # :731-733
    self.env_run_ids[env_ids] = run_ids
    reset_ids = env_ids[previous != run_ids]
    if np.asarray(env_outputs.abandoned).any():                                # :746-748
      raise ValueError('Abandoned done states are not supported in R2D2.')
    utils._check_no_duplicates(None, env_ids, 'inference batch')
    if reset_ids.size:                                                         # :734-744
      logging.info('Environments needing reset: %s', reset_ids)
      for t in self.env_infos:
        t[reset_ids] = 0
      tr = reset_ids[reset_ids < self.num_training_envs]
      if tr.size:
        self.store.reset(tr)
      init = self.agent.initial_state(len(reset_ids))
      self.first_agent_states.replace(reset_ids, init)
      self.agent_states.replace(reset_ids, init)
      self.actions.reset(reset_ids)
    # episode statistics (:751-757), host tables: they only feed logging
    self.env_infos[1][env_ids] += reward
    self.env_infos[2][env_ids] += np.asarray(raw_rewards)
    done_ids = env_ids[done]
    if done_ids.size:
      self.info_queue.enqueue_many(tuple(torch.as_tensor(t[done_ids]) for t in self.env_infos) +
                                   (torch.as_tensor(done_ids.astype(np.int32)),))
    for t in self.env_infos:
      t[done_ids] = 0
    self.env_infos[0][env_ids] += self.num_action_repeats

  def _completed_unrolls(self, completed_ids, unrolls):
    """(:805-821) the queue elements of the unrolls the store just completed: their first agent
    states and initial priorities from the behaviour Q values of the suffix."""
    s = self.settings
    _, unrolled_env, unrolled_agent = unrolls
    first = self.first_agent_states.read(completed_ids)                      # :805
    _, ao_suf = learner.split_structure(tuple(utils.make_time_major(unrolled_agent)), s.burn_in)
    _, env_suf = learner.split_structure(tuple(utils.make_time_major(unrolled_env)), s.burn_in)
    ao = learner.AgentOutput(*ao_suf)
    _, priorities, _ = learner.compute_loss_and_priorities_from_agent_outputs(
        ao, ao, utils.EnvOutput(*env_suf), ao, s.discounting, n_steps=s.n_steps,
        value_function_rescaling_epsilon=s.value_function_rescaling_epsilon)
    return learner.Unroll(first, priorities, *unrolls)

  # ---- CUDA-graph path ---------------------------------------------------------------------------
  def _device_step(self, ids32, env_dev, counter):
    """Everything of one inference batch that runs on the device (:760-803,829-830), on static
    buffers: captured once, replayed per batch."""
    n = int(ids32.numel())
    tables = self._state_tables(self.agent_states)
    prev_actions = torch.empty([n], dtype=torch.int32, device=self.device)
    prev_flat = [torch.empty([n] + list(t.shape[1:]), dtype=t.dtype, device=self.device) for t in tables]
    _lib.rows_multi([(self.actions._state[0], prev_actions, _lib.ROW_GATHER)] +
                    [(t, r, _lib.ROW_GATHER) for t, r in zip(tables, prev_flat)], ids32)
    agent_outputs, curr_states = self.agent((prev_actions, env_dev),
                                            utils.pack_sequence_as(self.agent_state_specs, prev_flat))
    learner.device_epsilon_greedy(agent_outputs.action, ids32, self.envs_epsilon, self.agent._num_actions,
                                  self.epsilon_seed, counter)
    # eval environments (ids >= num_training_envs) are skipped by the append (:792-803)
    self.store.device_append(ids32, utils.flatten((prev_actions, env_dev, agent_outputs)),
                             id_limit=self.num_training_envs)
    curr_flat = [t.contiguous() for t in utils.flatten(curr_states)]
    _lib.rows_multi([(t, r, _lib.ROW_SCATTER) for t, r in zip(tables, curr_flat)] +
                    [(self.actions._state[0], agent_outputs.action, _lib.ROW_SCATTER)], ids32)
    return prev_flat, agent_outputs

  def _build_graph(self):
    N, dev = self.N, self.device
    dt = utils.as_torch_dtype
    self._g_ids = torch.zeros([N], dtype=torch.int32, device=dev)
    self._g_env = utils.EnvOutput(*(torch.zeros([N] + list(s.shape), dtype=dt(s.dtype), device=dev)
                                    for s in self.env_output_specs))
    self._g_pin = [torch.zeros_like(t, device='cpu').pin_memory() for t in (self._g_ids,) + tuple(self._g_env)]
    with torch.cuda.stream(self.stream):
      self._g_ids.copy_(torch.arange(N, dtype=torch.int32))       # distinct ids for the warm-up / capture
      # one eager warm-up (lazy initialisation: workspaces, kernel attributes), then every table it
      # touched is restored; the capture itself executes nothing
      touched = (self.actions._state + self.agent_states._state + self.store._state +
                 [self.store._index, self.epsilon_counter])
      saved = [t.clone() for t in touched]
      self._device_step(self._g_ids, self._g_env, self.epsilon_counter)
      for t, sv in zip(touched, saved):
        t.copy_(sv)
      self.stream.synchronize()
      g = torch.cuda.CUDAGraph()
      # thread_local: other threads (the learner, other hosts) may launch on their streams meanwhile
      with torch.cuda.graph(g, stream=self.stream, capture_error_mode='thread_local'):
        self._g_prev_states, self._g_out = self._device_step(self._g_ids, self._g_env, self.epsilon_counter)
      self._g_actions_pin = torch.zeros([N], dtype=torch.int32).pin_memory()
    self._graph = g

  def _inference_graph(self, env_ids, run_ids, env_outputs, raw_rewards):
    """reference learner.py:711-790 with the device side as one graph replay."""
    pending = None
    with torch.cuda.stream(self.stream):
      if self._graph is None:
        self._build_graph()
      self._begin_batch(env_ids, run_ids, env_outputs, raw_rewards)
      # inputs: host arrays -> pinned staging -> the graph's static device buffers
      srcs = (env_ids.astype(np.int32),) + tuple(np.asarray(x) for x in env_outputs)
      for pin, dst, src in zip(self._g_pin, (self._g_ids,) + tuple(self._g_env), srcs):
        t = torch.from_numpy(np.ascontiguousarray(src))
        if t.numel() >= 65536 and t.is_pinned():
          dst.copy_(t, non_blocking=True)        # pinned observations (the batcher's slabs): DMA straight
        else:
          pin.numpy()[...] = src
          dst.copy_(pin, non_blocking=True)
      self._graph.replay()
      # completed unrolls of training environments, known on the host; positions in the full batch
      tr_pos = np.nonzero(env_ids < self.num_training_envs)[0]
      done_host, pos = self.store.host_advance(env_ids[tr_pos])
      if done_host.size:
        completed_ids, unrolls = self.store.complete(int(done_host.size))
        pending = self._completed_unrolls(completed_ids, unrolls)
        # the state the next unroll starts from = the state this step started from (:825-826)
        pos_dev = torch.as_tensor(tr_pos[pos].astype(np.int64)).to(self.device, non_blocking=True)
        self.first_agent_states.replace(
            completed_ids, utils.pack_sequence_as(self.agent_state_specs,
                                                  [t.index_select(0, pos_dev) for t in self._g_prev_states]),
            check_unique=False)
      self._g_actions_pin.copy_(self._g_out.action, non_blocking=True)
      self.stream.synchronize()
    if pending is not None:
      self.unroll_queue.enqueue_many(pending)                                  # :823-824
    return self._g_actions_pin.numpy().copy()

  def _inference(self, env_ids, run_ids, env_outputs, raw_rewards):
    """reference learner.py:711-790."""
    s = self.settings
    env_ids = np.asarray(env_ids); run_ids = np.asarray(run_ids)
    if self.use_graph and len(env_ids) == self.N:
      return self._inference_graph(env_ids, run_ids, env_outputs, raw_rewards)
    with torch.cuda.stream(self.stream):
      self._begin_batch(env_ids, run_ids, env_outputs, raw_rewards)
      # inference (:760-781): gather previous action / state (one launch), T=1 forward
      n = len(env_ids)
      ids32 = torch.as_tensor(env_ids.astype(np.int32)).to(self.device, non_blocking=True)
      env_dev = utils.EnvOutput(*(torch.as_tensor(np.asarray(x)).to(self.device, non_blocking=True)
                                  for x in env_outputs))
      tables = self._state_tables(self.agent_states)
      prev_actions = torch.empty([n], dtype=torch.int32, device=self.device)
      prev_flat = [torch.empty([n] + list(t.shape[1:]), dtype=t.dtype, device=self.device) for t in tables]
      _lib.rows_multi([(self.actions._state[0], prev_actions, _lib.ROW_GATHER)] +
                      [(t, r, _lib.ROW_GATHER) for t, r in zip(tables, prev_flat)], ids32)
      prev_states = utils.pack_sequence_as(self.agent_state_specs, prev_flat)
      agent_outputs, curr_states = self.agent((prev_actions, env_dev), prev_states)
      agent_outputs = agent_outputs._replace(action=learner.apply_epsilon_greedy(       # :783-787
          agent_outputs.action, ids32, self.num_training_envs, self.num_eval_envs, s.eval_epsilon,
          self.agent._num_actions, generator=self.generator))
      # training environments only go to the unroll store (:792-803)
      tr_pos = np.nonzero(env_ids < self.num_training_envs)[0]
      pending = None
      if tr_pos.size:
        if tr_pos.size == n:
          sel = lambda t: t
          tr_ids = env_ids
        else:
          pos_dev = torch.as_tensor(tr_pos.astype(np.int64)).to(self.device, non_blocking=True)
          sel = lambda t: t.index_select(0, pos_dev)
          tr_ids = env_ids[tr_pos]
        vals = utils.map_structure(sel, (prev_actions, env_dev, agent_outputs))
        completed_ids, unrolls = self.store.append(tr_ids, vals, check_duplicates=False)
        if int(completed_ids.numel()):
          pending = self._completed_unrolls(completed_ids, unrolls)
          self.first_agent_states.replace(completed_ids, self.agent_states.read(completed_ids), check_unique=False)   # :825-826
      # update the current state and action (:829-830): one scatter launch
      curr_flat = [t.contiguous() for t in utils.flatten(curr_states)]
      _lib.rows_multi([(t, r, _lib.ROW_SCATTER) for t, r in zip(tables, curr_flat)] +
                      [(self.actions._state[0], agent_outputs.action.contiguous(), _lib.ROW_SCATTER)], ids32)
      out = agent_outputs.action.cpu()          # D2H + sync of this stream
    if pending is not None:
      self.unroll_queue.enqueue_many(pending)                                  # :823-824
    return out.numpy()


def fill_replay(host, feeder, timeout=None):
  """create_dataset's dequeue (:410-448): moves `get_replay_insertion_batch_size` unrolls from the
  unroll queue into the replay buffer.  Returns False if the queue closed."""
  n = learner.get_replay_insertion_batch_size(feeder.settings)
  try:
    unrolls = host.unroll_queue.dequeue_many(n)
  except utils.QueueClosedError:
    return False
  if torch.cuda.is_available():
    # the unrolls were allocated on the inference stream and are copied into the replay buffer on THIS
    # thread's stream: tell the caching allocator, so that their blocks are not handed back to the
    # inference stream (and overwritten by the next unrolls) while that copy is still queued
    cur = torch.cuda.current_stream()
    for t in utils.flatten(unrolls):
      if isinstance(t, torch.Tensor) and t.is_cuda:
        t.record_stream(cur)
  feeder.insert(learner.Unroll(*unrolls))
  return True


def learner_loop(create_env_fn, create_agent_fn, create_optimizer_fn):
  """reference learner.py:478-900 (one replica)."""
  from seed_rl_b200.agents.vtrace import learner_loop as vloop
  logging.info('Starting learner loop')
  utils.validate_learner_config(FLAGS)
  s = learner.settings_from_flags()
  assert s.n_steps >= 1, '--n_steps < 1 does not make sense.'
  env = create_env_fn(0, FLAGS)
  num_actions = env.action_space.n
  TS = utils.TensorSpec
  env_output_specs = utils.EnvOutput(TS([], 'float32', 'reward'), TS([], 'bool', 'done'),
                                     TS(list(env.observation_space.shape), 'uint8', 'observation'),
                                     TS([], 'bool', 'abandoned'), TS([], 'int32', 'episode_step'))
  agent = create_agent_fn(env_output_specs, num_actions)
  target_agent = create_agent_fn(env_output_specs, num_actions)
  iter_frame_ratio = learner.get_replay_insertion_batch_size(s) * s.unroll_length * FLAGS.num_action_repeats
  final_iteration = int(math.ceil(FLAGS.total_environment_frames / iter_frame_ratio))
  optimizer, learning_rate_fn = create_optimizer_fn(final_iteration)
  step = learner.R2D2LearnerStep(agent, target_agent, optimizer, settings=s)
  os.makedirs(FLAGS.logdir, exist_ok=True)
  ckpt_path = os.path.join(FLAGS.logdir, 'ckpt.pt')
  if os.path.exists(ckpt_path):                                                # :650-654
    logging.info('Restoring checkpoint: %s', ckpt_path)
    d = vloop.restore_checkpoint(ckpt_path, agent, optimizer)
    target_agent.load_state_dict(d['target_agent'])
  summary_writer = utils.SummaryWriter(FLAGS.logdir)
  host = R2D2InferenceHost(agent, FLAGS.num_envs, FLAGS.num_eval_envs, FLAGS.inference_batch_size,
                           env.observation_space.shape, settings=s, num_action_repeats=FLAGS.num_action_repeats,
                           unroll_queue_max_size=FLAGS.unroll_queue_max_size, cuda_graph=FLAGS.inference_cuda_graph)
  replay = utils.PrioritizedReplay(s.replay_buffer_size, host.unroll_specs, s.importance_sampling_exponent)
  feeder = learner.ReplayFeeder(replay, s)
  server = grpc.Server([FLAGS.server_address])
  server.bind(host.inference)
  server.start()
  last_ckpt_time, last_log_time = 0, time.time()
  last_frames = optimizer.iterations * iter_frame_ratio
  max_norm = 0.
  try:
    while optimizer.iterations < final_iteration:
      frames = optimizer.iterations * iter_frame_ratio
      now = time.time()
      if now - last_ckpt_time >= FLAGS.save_checkpoint_secs:                   # :851-853
        vloop.save_checkpoint(ckpt_path, agent, optimizer, extra={'target_agent': target_agent.state_dict()})
        last_ckpt_time = now
      while True:                                                              # :418-436
        if not fill_replay(host, feeder):
          return
        if feeder.ready():
          break
        logging.info('Waiting for the replay buffer to fill up. It currently has %d elements, waiting for at '
                     'least %d elements', replay.num_inserted, s.replay_buffer_min_size)
      _, priorities, indices, norm = step.minimize(feeder.sample())            # :845-846,866
      feeder.update_priorities(indices, priorities)                           # :868
      if now - last_log_time >= 120:                                           # :872-885
        max_norm = max(max_norm, float(norm))
        dt = time.time() - last_log_time
        summary_writer.set_step(frames)
        summary_writer.scalar('num_environment_frames/sec (actors)', (frames - last_frames) / dt)
        summary_writer.scalar('num_environment_frames/sec (learner)', (frames - last_frames) / dt * s.replay_ratio)
        summary_writer.scalar('learning_rate', learning_rate_fn(optimizer.iterations))
        summary_writer.scalar('replay_buffer_num_inserted', replay.num_inserted)
        summary_writer.scalar('unroll_queue_size', host.unroll_queue.size())
        summary_writer.scalar('max_gradient_norm_before_clip', max_norm)
        summary_writer.flush()
        last_log_time, last_frames, max_norm = time.time(), frames, 0.
  finally:
    vloop.save_checkpoint(ckpt_path, agent, optimizer, extra={'target_agent': target_agent.state_dict()})
    server.shutdown()
    host.unroll_queue.close()
    summary_writer.close()
