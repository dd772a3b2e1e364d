"""`learner_loop` -- mirror of reference agents/vtrace/learner.py:170-483: the central
inference closure bound on the RPC server (a6, :349-407), the unroll store / queue plumbing
(a8/a9, :314-336,394-399,418-445) and the training loop (:467-483), for ONE replica
(= one GPU / process; `torchrun` starts one per GPU, each with its own env shard, like the
reference's per-host server/store, :314-416).

Data path per inference batch: actor payloads land in a pinned slab (C++ batcher) ->
one H2D copy per field -> T=1 `seedrl_net_forward` + in-kernel sampling -> scatter into the
HBM-resident UnrollStore -> completed unrolls (already on the GPU) go to the capacity-1
queue -> the learner thread stacks B of them straight into time-major order.
Observations are never copied on the host after the slab (reference: >= 4 host copies).
"""
import collections
import math
import os
import threading
import time

from absl import flags
from absl import logging
import torch

from seed_rl_b200.agents.vtrace import learner as learner_lib
from seed_rl_b200.common import inference_host
from seed_rl_b200.common import utils
from seed_rl_b200.common.parametric_distribution import get_parametric_distribution_for_action_space
from seed_rl_b200.dmlab import networks
from seed_rl_b200.grpc import ops as grpc

FLAGS = flags.FLAGS
Unroll = learner_lib.Unroll


class InferenceHost(inference_host.InferenceHostBase):
  """Everything `create_host` builds in the reference (learner.py:314-413) for one GPU."""

  algorithm = 'VTRACE'

  def __init__(self, agent, num_envs, unroll_length, inference_batch_size, obs_shape,
               num_action_repeats=1, device='cuda', info_queue=None, training_batch_size=None,
               cuda_graph=None, allow_abandoned=False, num_tasks=1):
    """training_batch_size: when given, completed unrolls are gathered straight into the columns
    of preallocated time-major training batches (`self.assembler`, utils.BatchAssembler: zero-copy
    minibatch assembly); otherwise they go through the reference's capacity-1 `unroll_queue` of
    single unrolls and `dequeue_batch` stacks them.  cuda_graph: replay the device side of every
    full batch as one CUDA graph (default: with the assembler); it needs the assembler.
    allow_abandoned: accept abandoned episodes (--bootstrap_abandoned).  num_tasks: the assembler records
    each column's task, env_id % num_tasks (--popart_tasks)."""
    TS = utils.TensorSpec
    agent_output_specs = networks.AgentOutput(
        TS([], 'int64', 'action'), TS([agent._num_actions], 'float32', 'policy_logits'),
        TS([], 'float32', 'baseline'))
    agent_state_specs = (TS([networks.LSTM_UNITS], 'float32', 'h'), TS([networks.LSTM_UNITS], 'float32', 'c'))
    # CUDA-graph replay of the device side of a full inference batch: gather -> T=1 forward ->
    # sample -> write-back -> store append are ~40 small dependent launches whose CPU issue cost,
    # not their GPU time, bounded the step.
    use_graph = bool(training_batch_size) and (cuda_graph is None or bool(cuda_graph))
    # time_major=True: completed unrolls come out as [T+1, n, ...] (no make_time_major pass)
    super(InferenceHost, self).__init__(
        agent, num_envs, inference_batch_size, obs_shape, 'int64', agent_state_specs, agent_output_specs,
        unroll_length, time_major=True, num_action_repeats=num_action_repeats, device=device,
        info_queue=info_queue, use_graph=use_graph, allow_abandoned=allow_abandoned)
    self.unroll_specs = Unroll(agent_state_specs, *self.store.unroll_specs)
    self.unroll_queue = utils.StructuredFIFOQueue(1, self.unroll_specs)      # capacity 1, :336
    self.assembler = None
    if training_batch_size:
      self.assembler = utils.BatchAssembler(self.store._specs, agent_state_specs, unroll_length + 1,
                                            training_batch_size, slots=2, device=device, num_tasks=num_tasks)

  def _policy(self, ids32, prev_actions, env_outputs, prev_states, counter):
    return self.agent(prev_actions, env_outputs, prev_states, is_training=False, rng_counter=counter)

  def _completed_unrolls(self, nc):
    """Into the next columns of the assembler, or (:394-399) one queue item per unroll."""
    if self.assembler is None:
      completed_ids, unrolls = self.store.complete(nc)
      first = self.first_agent_states.read(completed_ids)
      # [T+1, nc, ...] -> [nc, T+1, ...]: the queue splits the batch along dim 0 into single unrolls
      return completed_ids, Unroll(first, *utils.map_structure(lambda t: t.transpose(0, 1), unrolls))

    def on_placed(slot, col0, ids):
      first = self.first_agent_states.read(ids.to(torch.int64))
      for dst, src in zip(self.assembler._states[slot], first):
        dst[col0:col0 + int(ids.numel())].copy_(src)
      self.assembler.place_task_ids(slot, col0, ids)
    completed_ids, _ = self.store.complete_into(nc, self.assembler, on_placed)
    return completed_ids, None


def dequeue_batch(unroll_queue, batch_size):
  """reference learner.py:418-432: B unrolls -> one time-major batch.  Unrolls are already
  [T+1, ...] on the GPU; stacking along dim 1 IS the time-major layout."""
  items = [unroll_queue.dequeue() for _ in range(batch_size)]
  if torch.cuda.is_available():
    # the items were allocated on the inference stream: tell the caching allocator that this
    # stream reads them, so their blocks are not recycled under the (asynchronous) stack below
    cur = torch.cuda.current_stream()
    for it in items:
      for t in utils.flatten(it):
        if isinstance(t, torch.Tensor) and t.is_cuda:
          t.record_stream(cur)
  state = tuple(torch.stack([it.agent_state[k] for it in items]) for k in range(2))
  def stack(field):
    return utils.map_structure(lambda *xs: torch.stack(xs, dim=1),
                               *[getattr(it, field) for it in items])
  return Unroll(state, stack('prev_actions'), stack('env_outputs'), stack('agent_outputs'))


def save_checkpoint(path, agent, optimizer, extra=None):
  """tf.train.CheckpointManager.save analogue (reference learner.py:283-296,470-476): one
  `torch.save` blob {agent: flat fp32 arena + tensor table, optimizer: Adam m / v / iterations}
  written atomically.  NOT interchangeable with the reference's tf.train.Checkpoint files (no
  TensorFlow here); `named_parameters()` gives the Keras-layout tensors by name for conversion."""
  blob = {'agent': agent.state_dict(), 'optimizer': optimizer.state_dict(), 'format': 'seed_rl_b200/1'}
  if extra:
    blob.update(extra)
  torch.save(blob, path + '.tmp')
  os.replace(path + '.tmp', path)


def restore_checkpoint(path, agent, optimizer):
  """ckpt.restore(...).assert_consumed() analogue: raises on a tensor-table mismatch."""
  d = torch.load(path, map_location='cpu', weights_only=False)
  networks.check_popart_state(d['agent'], getattr(agent, 'popart_moments', None) is not None,
                              getattr(agent, 'popart_tasks', 0) or None)
  info = d['agent'].get('param_info')
  if info is not None and [tuple(x) for x in info] != [tuple(x) for x in agent.param_info]:
    raise ValueError('checkpoint %s was written by a different network (tensor table mismatch)' % path)
  agent.load_state_dict(d['agent'])
  optimizer.load_state_dict(d['optimizer'], device=str(agent.device))
  return d


def rank_server_address(address, rank):
  """One server per replica (reference: one per host, learner.py:339-347): replica r binds the
  flag's address with its port (or unix-socket path) offset by r."""
  if rank == 0:
    return address
  if address.startswith('unix:'):
    return '%s.%d' % (address, rank)
  host, _, port = address.rpartition(':')
  return '%s:%d' % (host, int(port) + rank)


def init_replicas():
  """torchrun starts one learner process per GPU (SURVEY 8e); returns (rank, world)."""
  import torch.distributed as td
  world = int(os.environ.get('WORLD_SIZE', '1'))
  rank = int(os.environ.get('RANK', '0'))
  if world > 1 and not td.is_initialized():
    local = int(os.environ.get('LOCAL_RANK', '0'))
    if torch.cuda.is_available():
      torch.cuda.set_device(local)
      td.init_process_group('nccl', device_id=torch.device('cuda', local))
    else:
      td.init_process_group('gloo')
  return rank, world


def assembled_batch(assembler):
  """The zero-copy counterpart of `dequeue_batch`: the next full time-major batch of the
  assembler as an `Unroll` of views (no copy).  Returns (slot, Unroll); call
  assembler.release(slot) after the step that consumes it has been enqueued."""
  slot, state, (prev_actions, env_outputs, agent_outputs) = assembler.get()
  return slot, Unroll(tuple(state), prev_actions, utils.EnvOutput(*env_outputs),
                      networks.AgentOutput(*agent_outputs))


def learner_loop(create_env_fn, create_agent_fn, create_optimizer_fn):
  """reference learner.py:170-483 (one replica per process / GPU)."""
  logging.info('Starting learner loop')
  utils.validate_learner_config(FLAGS)
  rank, world = init_replicas()
  env = create_env_fn(0, FLAGS)
  dist = get_parametric_distribution_for_action_space(env.action_space)
  agent = create_agent_fn(env.action_space, env.observation_space, dist)
  if not hasattr(agent, '_entropy_mul'):
    agent.init_entropy_cost(FLAGS.entropy_cost, FLAGS.entropy_cost_adjustment_speed)
  iter_frame_ratio = FLAGS.batch_size * FLAGS.unroll_length * FLAGS.num_action_repeats
  final_iteration = int(math.ceil(FLAGS.total_environment_frames / iter_frame_ratio))
  optimizer, learning_rate_fn = create_optimizer_fn(final_iteration)
  settings = learner_lib.loss_settings_from_flags()
  # summaries + periodic progress export (learner.py:236-237,280,286,447-465)
  os.makedirs(FLAGS.logdir, exist_ok=True)
  summary_writer = utils.SummaryWriter(FLAGS.logdir) if rank == 0 else None
  logger = utils.ProgressLogger(summary_writer=summary_writer,
                                starting_step=optimizer.iterations * iter_frame_ratio)
  step = learner_lib.LearnerStep(agent, optimizer, dist, settings, logger=logger, grad_reduce=FLAGS.grad_reduce)

  ckpt_path = os.path.join(FLAGS.logdir, 'ckpt.pt')
  init = FLAGS.init_checkpoint or (ckpt_path if os.path.exists(ckpt_path) else None)
  if init:                                                                 # :286-296
    logging.info('Restoring checkpoint: %s', init)
    restore_checkpoint(init, agent, optimizer)
    logger.reset(summary_writer, optimizer.iterations * iter_frame_ratio)

  def save():
    if rank == 0:                      # replicas are bit-identical; one writer, no os.replace race
      save_checkpoint(ckpt_path, agent, optimizer)

  info_specs = (utils.TensorSpec([], 'int64', 'episode_num_frames'),
                utils.TensorSpec([], 'float32', 'episode_returns'),
                utils.TensorSpec([], 'float32', 'episode_raw_returns'))
  info_queue = utils.StructuredFIFOQueue(-1, info_specs)
  assert step.world == world
  per_replica = FLAGS.batch_size // world                                   # :422
  host = InferenceHost(agent, FLAGS.num_envs, FLAGS.unroll_length, FLAGS.inference_batch_size,
                       env.observation_space.shape, FLAGS.num_action_repeats, info_queue=info_queue,
                       training_batch_size=per_replica, allow_abandoned=FLAGS.bootstrap_abandoned,
                       num_tasks=settings.popart_tasks if settings.popart else 1)
  server = grpc.Server([rank_server_address(FLAGS.server_address, rank)])
  server.bind(host.inference)
  server.start()

  def additional_logs():                                                    # :447-463
    if summary_writer:
      summary_writer.scalar('learning_rate', learning_rate_fn(optimizer.iterations))
    n = info_queue.size()
    n -= n % FLAGS.log_episode_frequency
    if n:
      stats = info_queue.dequeue_many(n)
      for key, values in zip(('episode_num_frames', 'episode_return', 'episode_raw_return'), stats):
        for chunk in torch.split(values.float(), FLAGS.log_episode_frequency):
          if summary_writer:
            summary_writer.scalar(key, float(chunk.mean()))
      for fr, ret, raw in zip(*stats):
        logging.info('Return: %f Raw return: %f Frames: %i', float(ret), float(raw), int(fr))

  logger.start(additional_logs)
  last_ckpt_time = 0
  try:
    while optimizer.iterations < final_iteration:                           # :467-476
      now = time.time()
      if now - last_ckpt_time >= FLAGS.save_checkpoint_secs:
        save()
        last_ckpt_time = now
      slot, batch = assembled_batch(host.assembler)
      _, logs = step.minimize(batch, task_ids=host.assembler.task_ids(slot))
      host.assembler.release(slot)
      logger.step_end(logs, None, iter_frame_ratio)                         # :280
  finally:
    logger.shutdown()
    save()
    server.shutdown()
    host.unroll_queue.close()
    host.assembler.close()
    if summary_writer:
      summary_writer.close()
