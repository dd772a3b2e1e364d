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

from seed_rl_b200.agents.r2d2 import learner
from seed_rl_b200.atari import networks
from seed_rl_b200.common import inference_host
from seed_rl_b200.common import utils
from seed_rl_b200.grpc import ops as grpc

FLAGS = flags.FLAGS


class R2D2InferenceHost(inference_host.InferenceHostBase):
  """What the reference builds around `inference` (learner.py:656-793) for one GPU."""

  algorithm = 'R2D2'

  def __init__(self, agent, num_envs, num_eval_envs, inference_batch_size, observation_shape, settings=None,
               num_action_repeats=1, device='cuda', unroll_queue_max_size=100, generator=None, cuda_graph=False,
               epsilon_seed=0):
    """generator: the torch generator epsilon-greedy draws from on the eager path.  cuda_graph: replay
    the device side of every batch of exactly `inference_batch_size` rows as one CUDA graph, with
    epsilon-greedy drawn on the device from Philox keyed by `epsilon_seed` (a different random stream
    than `generator`'s, so the explored actions differ; the distribution is the same).  Other batch
    sizes take the eager path."""
    self.settings = s = settings or learner.default_settings()
    learner.check_bellman_target(s.bellman_target, s.retrace_lambda)
    self.num_envs, self.num_eval_envs = int(num_envs), int(num_eval_envs)
    self.num_training_envs = self.num_envs - self.num_eval_envs                      # :122-123
    if self.num_training_envs <= 0:
      raise ValueError('Total number of environments ({}) should be greater than number of environments '
                       'reserved to eval ({})'.format(num_envs, num_eval_envs))            # :473-476
    self.generator = generator
    TS = utils.TensorSpec
    agent_output_specs = networks.AgentOutput(TS([], 'int32', 'action'), TS([agent._num_actions], 'float32', 'q_values'))
    npix = int(np.prod(observation_shape))
    agent_state_specs = networks.AgentState(
        (TS([networks.LSTM_UNITS], 'float32', 'h'), TS([networks.LSTM_UNITS], 'float32', 'c')),
        TS([npix], 'int32', 'frame_stacking_state') if agent._stack_size > 1 else ())
    # Buffer of incomplete unrolls: training environments only, burn_in overlapping steps (:659-662)
    super(R2D2InferenceHost, self).__init__(
        agent, self.num_envs, inference_batch_size, observation_shape, 'int32', agent_state_specs,
        agent_output_specs, s.unroll_length, num_overlapping_steps=s.burn_in, id_limit=self.num_training_envs,
        num_action_repeats=num_action_repeats, device=device, use_graph=cuda_graph,
        allow_abandoned=s.bootstrap_abandoned,
        info_queue=utils.StructuredFIFOQueue(-1, (TS([], 'int64', 'episode_num_frames'),
                                                  TS([], 'float32', 'episode_returns'),
                                                  TS([], 'float32', 'episode_raw_returns'),
                                                  TS([], 'int32', 'env_ids'))))
    self.unroll_specs = learner.Unroll(agent_state_specs, TS([], 'float32', 'priority'), *self.store.unroll_specs)
    self.unroll_queue = utils.StructuredFIFOQueue(unroll_queue_max_size, self.unroll_specs)   # :686-687
    self.epsilon_seed = int(epsilon_seed)
    # the per-env epsilons (:129-152) of the graph path, built once
    self.envs_epsilon = learner.get_envs_epsilon(torch.arange(self.num_envs, device=self.device),
                                                 self.num_training_envs, self.num_eval_envs,
                                                 s.eval_epsilon).contiguous()

  def _episode_infos(self, done_ids):
    return (super(R2D2InferenceHost, self)._episode_infos(done_ids) +
            (torch.as_tensor(done_ids.astype(np.int32)),))

  def _policy(self, ids32, prev_actions, env_outputs, prev_states, counter):
    """The T=1 forward (:760-781), then epsilon-greedy (:783-787): from `generator` on the eager path,
    from the device counter's Philox stream in the graph."""
    agent_outputs, curr_states = self.agent((prev_actions, env_outputs), prev_states)
    if counter is None:
      return agent_outputs._replace(action=learner.apply_epsilon_greedy(
          agent_outputs.action, ids32, self.num_training_envs, self.num_eval_envs, self.settings.eval_epsilon,
          self.agent._num_actions, generator=self.generator)), curr_states
    learner.device_epsilon_greedy(agent_outputs.action, ids32, self.envs_epsilon, self.agent._num_actions,
                                  self.epsilon_seed, counter)
    return agent_outputs, curr_states

  def _completed_unrolls(self, nc):
    """(:805-824) the completed unrolls with their first agent states and initial priorities from the
    behaviour Q values of the suffix, under the learner's `bellman_target`."""
    s = self.settings
    completed_ids, unrolls = self.store.complete(nc)
    _, unrolled_env, unrolled_agent = unrolls
    first = self.first_agent_states.read(completed_ids)                      # :805
    _, ao_suf = learner.split_structure(tuple(utils.make_time_major(unrolled_agent)), s.burn_in)
    _, env_suf = learner.split_structure(tuple(utils.make_time_major(unrolled_env)), s.burn_in)
    ao = learner.AgentOutput(*ao_suf)
    _, priorities, _ = learner.compute_loss_and_priorities_from_agent_outputs(
        ao, ao, utils.EnvOutput(*env_suf), ao, s.discounting, n_steps=s.n_steps,
        value_function_rescaling_epsilon=s.value_function_rescaling_epsilon, bellman_target=s.bellman_target,
        retrace_lambda=s.retrace_lambda, abandoned=env_suf[3] if s.bootstrap_abandoned else None)
    return completed_ids, learner.Unroll(first, priorities, *unrolls)


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
  assert s.n_steps >= 1, '--n_steps < 1 does not make sense.'       # unused under --bellman_target=retrace
  learner.check_bellman_target(s.bellman_target, s.retrace_lambda)
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
