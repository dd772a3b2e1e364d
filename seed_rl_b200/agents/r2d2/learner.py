"""R2D2 learner -- mirror of the reference's `agents/r2d2/learner.py` (BASELINE cfg 5):

  flags                                            :43-92    (same names and defaults)
  Unroll / SampledUnrolls / EpisodeInfo            :96-112
  get_replay_insertion_batch_size, get_envs_epsilon, apply_epsilon_greedy   :115-177
  compute_loss_and_priorities_from_agent_outputs   :258-330 (+ value rescaling :180-192 and
                                                   n-step Bellman targets :195-255, fused; or,
                                                   opt-in and not in the reference, Retrace(lambda)
                                                   targets with a greedy target policy)
  compute_loss_and_priorities                      :333-386  (burn-in, two unrolls per network)
  minimize (R2D2LearnerStep)                       :581-634  (importance-weighted mean loss,
                                                   global-norm clip :604-609, Keras Adam)
  update_target_agent                              :535-544
  insert / sample / update_priorities of the replay path (create_dataset :389-467, loop :856-885)
                                                   -> ReplayFeeder over common.utils.PrioritizedReplay

Device work per step = 2 burn-in unrolls + 2 suffix unrolls (seedrl_r2d2_net_forward) ->
seedrl_r2d2_loss_fwd_bwd (or seedrl_r2d2_retrace_loss_fwd_bwd) -> seedrl_r2d2_net_backward ->
seedrl_clip_by_global_norm -> seedrl_adam_apply -> priority write-back.  There is no autograd tape.
"""
import collections

from absl import flags
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common import common_flags  # pylint: disable=unused-import
from seed_rl_b200.common import utils

FLAGS = flags.FLAGS
BELLMAN_TARGETS = ('n_step', 'retrace')


def _define(fn, name, default, help_):
  """The V-trace and R2D2 learners are separate binaries in the reference and share flag names
  (batch_size, unroll_length, discounting ...).  When both mirrors are imported into one
  process (the test-suite does) the first definition stands; R2D2 code therefore never reads
  those flags directly but goes through `settings_from_flags` / `default_settings`."""
  common_flags.define_once(fn, name, default, help_)


_define(flags.DEFINE_integer, 'save_checkpoint_secs', 1800, 'Checkpoint save period in seconds.')
_define(flags.DEFINE_integer, 'total_environment_frames', int(1e9), 'Total environment frames to train for.')
_define(flags.DEFINE_integer, 'batch_size', 64, 'Batch size for training.')
_define(flags.DEFINE_float, 'replay_ratio', 1.5, 'Average number of times each observation is replayed and '
        'used for training.')
_define(flags.DEFINE_integer, 'inference_batch_size', -1, 'Batch size for inference, -1 for auto-tune.')
_define(flags.DEFINE_integer, 'unroll_length', 100, 'Unroll length in agent steps.')
_define(flags.DEFINE_integer, 'num_training_tpus', 1, 'Unused: there are no TPUs (kept for flag compatibility).')
_define(flags.DEFINE_integer, 'update_target_every_n_step', 2500,
        'Update the target network at this frequency (expressed in number of training steps)')
_define(flags.DEFINE_integer, 'replay_buffer_size', 100, 'Size of the replay buffer (in number of unrolls stored).')
_define(flags.DEFINE_integer, 'replay_buffer_min_size', 10,
        'Learning only starts when there is at least this number of unrolls in the replay buffer')
_define(flags.DEFINE_float, 'priority_exponent', 0.9, 'Priority exponent used when sampling in the replay buffer.')
_define(flags.DEFINE_integer, 'unroll_queue_max_size', 100, 'Max size of the unroll queue')
_define(flags.DEFINE_integer, 'burn_in', 40, 'Length of the RNN burn-in prefix.')
_define(flags.DEFINE_float, 'importance_sampling_exponent', 0.6,
        'Exponent used when computing the importance sampling correction.')
_define(flags.DEFINE_float, 'clip_norm', 40, 'We clip gradient norm to this value.')
_define(flags.DEFINE_float, 'value_function_rescaling_epsilon', 1e-3, 'Epsilon used for value function rescaling.')
_define(flags.DEFINE_integer, 'n_steps', 5, 'n-step returns: how far ahead we look for computing the Bellman targets.')
_define(flags.DEFINE_float, 'discounting', .997, 'Discounting factor.')
_define(flags.DEFINE_string, 'bellman_target', 'n_step',
        'Bellman targets of the loss: "n_step", the reference\'s n-step double-DQN targets, or "retrace", '
        'Retrace(lambda) targets (Munos et al. 2016) with a target policy greedy in the online network. '
        'Retrace is not in the reference; under it --n_steps is unused.')
_define(flags.DEFINE_float, 'retrace_lambda', 0.95, 'Trace coefficient lambda in [0, 1] of --bellman_target=retrace.')
_define(flags.DEFINE_bool, 'bootstrap_abandoned', False,
        'Accept abandoned episodes (EnvOutput.abandoned: a time limit, not the task, ended them) and '
        'bootstrap from the value of their last observation instead of treating it as terminal '
        '(advantages.py NStep).')
_define(flags.DEFINE_float, 'eval_epsilon', 1e-3, 'Epsilon (as in epsilon-greedy) used for evaluation.')
_define(flags.DEFINE_bool, 'inference_cuda_graph', False,
        'Replay the device side of every full inference batch as one CUDA graph, with epsilon-greedy '
        'drawn on the device from Philox (a different random stream than the torch generator of the '
        'default path, so the explored actions differ).')

AgentOutput = collections.namedtuple('AgentOutput', 'action q_values')

Unroll = collections.namedtuple('Unroll', 'agent_state priority prev_actions env_outputs agent_outputs')
SampledUnrolls = collections.namedtuple('SampledUnrolls', 'unrolls indices importance_weights')
EpisodeInfo = collections.namedtuple('EpisodeInfo', 'num_frames returns raw_returns env_ids')

# flag defaults of the reference (learner.py:47-87)
N_STEPS = 5
VALUE_FUNCTION_RESCALING_EPSILON = 1e-3
RETRACE_LAMBDA = 0.95

R2D2Settings = collections.namedtuple(
    'R2D2Settings',
    'batch_size replay_ratio unroll_length update_target_every_n_step replay_buffer_size '
    'replay_buffer_min_size priority_exponent burn_in importance_sampling_exponent clip_norm '
    'value_function_rescaling_epsilon n_steps discounting eval_epsilon num_training_tpus bellman_target '
    'retrace_lambda bootstrap_abandoned', defaults=(False,))


def default_settings(**kw):
  """The reference's flag defaults (learner.py:47-92), plus the n-step targets of the reference as the
  default `bellman_target`."""
  d = dict(batch_size=64, replay_ratio=1.5, unroll_length=100, update_target_every_n_step=2500,
           replay_buffer_size=100, replay_buffer_min_size=10, priority_exponent=0.9, burn_in=40,
           importance_sampling_exponent=0.6, clip_norm=40., value_function_rescaling_epsilon=1e-3, n_steps=5,
           discounting=.997, eval_epsilon=1e-3, num_training_tpus=1, bellman_target='n_step',
           retrace_lambda=RETRACE_LAMBDA, bootstrap_abandoned=False)
  d.update(kw)
  return R2D2Settings(**d)


def settings_from_flags():
  return R2D2Settings(**{k: getattr(FLAGS, k) for k in R2D2Settings._fields})


def get_replay_insertion_batch_size(settings=None, per_replica=False):
  """reference :115-119."""
  s = settings or settings_from_flags()
  if per_replica:
    return int(s.batch_size / s.replay_ratio / s.num_training_tpus)
  return int(s.batch_size / s.replay_ratio)


def get_envs_epsilon(env_ids, num_training_envs, num_eval_envs, eval_epsilon):
  """reference :129-152: 0.4 ** linspace(1, 8, num_training_envs) for training environments,
  eval_epsilon for eval environments; gathered at env_ids (one-time table + a gather)."""
  dev = env_ids.device if isinstance(env_ids, torch.Tensor) else 'cuda'
  eps = torch.cat([torch.pow(torch.tensor(0.4, dtype=torch.float32),
                             torch.linspace(1., 8., num_training_envs, dtype=torch.float32)),
                   torch.full([num_eval_envs], float(eval_epsilon), dtype=torch.float32)]).to(dev)
  return eps[torch.as_tensor(env_ids).to(dev).long()]


def apply_epsilon_greedy(actions, env_ids, num_training_envs, num_eval_envs, eval_epsilon, num_actions,
                         generator=None):
  """reference :155-177: with probability epsilon(env) the action is replaced by a uniform one."""
  actions = _lib.require_cuda(actions, torch.int32, 'actions')
  B = int(actions.shape[0])
  eps = get_envs_epsilon(env_ids, num_training_envs, num_eval_envs, eval_epsilon).to(actions.device)
  random_actions = torch.randint(0, num_actions, [B], dtype=torch.int32, device=actions.device, generator=generator)
  probs = torch.rand([B], device=actions.device, generator=generator)
  return torch.where(probs < eps, random_actions, actions)


def device_epsilon_greedy(actions, env_ids_i32, envs_epsilon, num_actions, seed, counter):
  """apply_epsilon_greedy in place, capturable in a CUDA graph (seedrl_r2d2_epsilon_greedy):
  actions int32 [B] (greedy on entry), envs_epsilon float32 [num_envs] (the get_envs_epsilon table),
  counter an int64 device scalar: the Philox offset, incremented by the call.  Draws from a
  different random stream than apply_epsilon_greedy, with the same distribution."""
  for t, dt, name in ((actions, torch.int32, 'actions'), (env_ids_i32, torch.int32, 'env_ids'),
                      (envs_epsilon, torch.float32, 'envs_epsilon'), (counter, torch.int64, 'counter')):
    if not (t.is_cuda and t.dtype == dt and t.is_contiguous()):
      raise ValueError('%s must be a contiguous CUDA %s tensor' % (name, dt))
  if env_ids_i32.numel() != actions.numel():
    raise ValueError('env_ids and actions must have the same length')
  _lib.check(_lib.lib().seedrl_r2d2_epsilon_greedy(
      int(actions.numel()), int(num_actions), _lib.ptr(env_ids_i32), _lib.ptr(envs_epsilon),
      int(seed) & 0xFFFFFFFFFFFFFFFF, _lib.ptr(counter), _lib.ptr(actions), _lib.stream_ptr()))


def check_bellman_target(bellman_target, retrace_lambda):
  """Raises ValueError for an unknown target kind or, under 'retrace', a lambda outside [0, 1]."""
  if bellman_target not in BELLMAN_TARGETS:
    raise ValueError('bellman_target must be one of %s, got %r' % (BELLMAN_TARGETS, bellman_target))
  if bellman_target == 'retrace' and not 0. <= float(retrace_lambda) <= 1.:
    raise ValueError('retrace_lambda must be in [0, 1], got %r' % (retrace_lambda,))


def compute_loss_and_priorities_from_agent_outputs(training_agent_output, target_agent_output, env_outputs,
                                                   agent_outputs, gamma, eta=0.9, n_steps=N_STEPS,
                                                   importance_weights=None,
                                                   value_function_rescaling_epsilon=VALUE_FUNCTION_RESCALING_EPSILON,
                                                   bellman_target='n_step', retrace_lambda=RETRACE_LAMBDA,
                                                   abandoned=None):
  """reference :258-330.  Returns (loss [B], priorities [B]); the gradient of
  mean(loss * importance_weights) w.r.t. training_agent_output.q_values (reference :604) is
  returned as the third element (the reference gets it from the tape).

  bellman_target='n_step' is the reference's rule.  'retrace' (not in the reference) replaces the
  n-step targets by Retrace(retrace_lambda) targets whose target policy is greedy in the online
  network, so the trace is retrace_lambda * 1[replayed action == argmax_a Q_online]; n_steps is then
  unused (seedrl_r2d2_retrace_loss_fwd_bwd in include/seedrl_b200.h states the targets).

  abandoned [T,B] (None = none): row i marks the transition into x_i as not real, as
  advantages.py NStep does; targets reaching it bootstrap from x_{i-1} and transition i-1 adds
  nothing to the loss (seedrl_r2d2_loss_fwd_bwd_abandoned)."""
  check_bellman_target(bellman_target, retrace_lambda)
  f32 = torch.float32
  q = _lib.require_cuda(training_agent_output.q_values, f32, 'training q_values')
  qt = _lib.require_cuda(target_agent_output.q_values, f32, 'target q_values')
  act = _lib.require_cuda(agent_outputs.action.to(torch.int64), torch.int64, 'replay actions')
  rew = _lib.require_cuda(env_outputs.reward, f32, 'reward')
  dn = _lib.require_cuda(env_outputs.done, torch.bool, 'done')
  if q.dim() != 3 or tuple(qt.shape) != tuple(q.shape):
    raise ValueError('q_values must be [time, batch, num_actions] for both agents')
  T, B, A = (int(x) for x in q.shape)
  ab = None
  if abandoned is not None:
    ab = _lib.require_cuda(abandoned, torch.bool, 'abandoned')
    if tuple(ab.shape) != (T, B):
      raise ValueError('abandoned has shape %s, expected %s' % (tuple(ab.shape), (T, B)))
  w = None if importance_weights is None else _lib.require_cuda(importance_weights, f32, 'importance_weights')
  L = _lib.lib()
  loss = torch.empty(B, dtype=f32, device=q.device); prio = torch.empty_like(loss)
  dq = torch.empty_like(q)
  if bellman_target == 'retrace':
    scratch = torch.empty(int(L.seedrl_r2d2_retrace_loss_scratch_bytes(T, B)), dtype=torch.uint8, device=q.device)
    tail = (_lib.ptr(w), float(gamma), float(retrace_lambda), float(eta), float(value_function_rescaling_epsilon),
            _lib.ptr(loss), _lib.ptr(prio), _lib.ptr(dq), _lib.ptr(scratch), _lib.stream_ptr())
    if ab is None:
      _lib.check(L.seedrl_r2d2_retrace_loss_fwd_bwd(T, B, A, _lib.ptr(q), _lib.ptr(qt), _lib.ptr(act), _lib.ptr(rew),
                                                    _lib.ptr(dn), *tail))
    else:
      _lib.check(L.seedrl_r2d2_retrace_loss_fwd_bwd_abandoned(T, B, A, _lib.ptr(q), _lib.ptr(qt), _lib.ptr(act),
                                                              _lib.ptr(rew), _lib.ptr(dn), _lib.ptr(ab), *tail))
    return loss, prio, dq
  scratch = torch.empty(int(L.seedrl_r2d2_loss_scratch_bytes(T, B, n_steps)), dtype=torch.uint8, device=q.device)
  tail = (_lib.ptr(w), float(gamma), int(n_steps), float(eta), float(value_function_rescaling_epsilon),
          _lib.ptr(loss), _lib.ptr(prio), _lib.ptr(dq), _lib.ptr(scratch), _lib.stream_ptr())
  if ab is None:
    _lib.check(L.seedrl_r2d2_loss_fwd_bwd(T, B, A, _lib.ptr(q), _lib.ptr(qt), _lib.ptr(act), _lib.ptr(rew),
                                          _lib.ptr(dn), *tail))
  else:
    _lib.check(L.seedrl_r2d2_loss_fwd_bwd_abandoned(T, B, A, _lib.ptr(q), _lib.ptr(qt), _lib.ptr(act), _lib.ptr(rew),
                                                    _lib.ptr(dn), _lib.ptr(ab), *tail))
  return loss, prio, dq


def replay_sample(priorities, num_inserted, num_samples, priority_exp, importance_sampling_exponent,
                  uniforms=None, generator=None):
  """PrioritizedReplay.sample's index / weight part (common/utils.py:327-352) for
  priority_exp != 0.  priorities: float32 [size] on the GPU; returns (indices int64
  [num_samples], weights float32 [num_samples], probabilities [limit])."""
  pr = _lib.require_cuda(priorities, torch.float32, 'priorities')
  limit = min(int(pr.numel()), int(num_inserted))
  if limit <= 0:
    raise ValueError('Cannot sample if replay buffer is empty')
  if uniforms is None:
    uniforms = torch.rand(num_samples, device=pr.device, generator=generator)
  u = _lib.require_cuda(uniforms, torch.float32, 'uniforms')
  idx = torch.empty(num_samples, dtype=torch.int64, device=pr.device)
  wts = torch.empty(num_samples, dtype=torch.float32, device=pr.device)
  probs = torch.empty(limit, dtype=torch.float32, device=pr.device)
  _lib.check(_lib.lib().seedrl_replay_sample(limit, _lib.ptr(pr), float(priority_exp),
                                             float(importance_sampling_exponent), int(num_samples), _lib.ptr(u),
                                             _lib.ptr(idx), _lib.ptr(wts), _lib.ptr(probs), _lib.stream_ptr()))
  return idx, wts, probs


def clip_by_global_norm(flat_grads, clip_norm):
  """tf.clip_by_global_norm over the flat gradient arena, in place.  Returns the global norm."""
  g = _lib.require_cuda(flat_grads, torch.float32, 'gradients')
  L = _lib.lib()
  norm = torch.empty((), dtype=torch.float32, device=g.device)
  scratch = torch.empty(int(L.seedrl_clip_scratch_bytes()), dtype=torch.uint8, device=g.device)
  _lib.check(L.seedrl_clip_by_global_norm(g.numel(), _lib.ptr(g), float(clip_norm), _lib.ptr(norm), _lib.ptr(scratch),
                                          _lib.stream_ptr()))
  return norm


def split_structure(structure, prefix_length):
  """common/utils.py:947-956 (time axis 0): views, no data movement."""
  flat = utils.flatten(structure)
  pre = [None if x is None else x[:prefix_length] for x in flat]
  suf = [None if x is None else x[prefix_length:] for x in flat]
  return utils.pack_sequence_as(structure, pre), utils.pack_sequence_as(structure, suf)


def compute_loss_and_priorities(training_agent, target_agent, agent_state, prev_actions, env_outputs, agent_outputs,
                                gamma, burn_in, importance_weights=None, n_steps=N_STEPS,
                                value_function_rescaling_epsilon=VALUE_FUNCTION_RESCALING_EPSILON,
                                bellman_target='n_step', retrace_lambda=RETRACE_LAMBDA, abandoned=None):
  """reference :333-386.  Time-major inputs with burn_in + unroll_length + 1 rows.  Burn-in
  unrolls update the recurrent state of both networks without gradient (:365-371); the suffix is
  unrolled by the training agent (kept for `backward`) and the target agent.  Returns
  (loss [B], priorities [B], dq [T_suffix, B, A]).  `abandoned` (None = none) has the rows of
  env_outputs; its suffix goes to compute_loss_and_priorities_from_agent_outputs."""
  check_bellman_target(bellman_target, retrace_lambda)     # before any network work
  if burn_in:
    (pa_pre, env_pre), (pa_suf, env_suf) = split_structure((prev_actions, tuple(env_outputs)), burn_in)
    _, ao_suf = split_structure(tuple(agent_outputs), burn_in)
    _, training_state = training_agent((pa_pre, env_pre), agent_state, unroll=True)
    _, target_state = target_agent((pa_pre, env_pre), agent_state, unroll=True)
  else:
    pa_suf, env_suf, ao_suf = prev_actions, tuple(env_outputs), tuple(agent_outputs)
    training_state = target_state = agent_state
  training_out, _ = training_agent((pa_suf, env_suf), training_state, unroll=True, is_training=True)
  target_out, _ = target_agent((pa_suf, env_suf), target_state, unroll=True)
  return compute_loss_and_priorities_from_agent_outputs(
      training_out, target_out, utils.EnvOutput(*env_suf), AgentOutput(*ao_suf), gamma, n_steps=n_steps,
      importance_weights=importance_weights, value_function_rescaling_epsilon=value_function_rescaling_epsilon,
      bellman_target=bellman_target, retrace_lambda=retrace_lambda,
      abandoned=None if abandoned is None else abandoned[burn_in:])


class R2D2LearnerStep(object):
  """`minimize` of reference :581-634 for one replica, plus `update_target_agent` (:535-544)
  on the reference's cadence (:845-846)."""

  def __init__(self, agent, target_agent, optimizer, settings=None, process_group=None):
    self.agent, self.target_agent, self.optimizer = agent, target_agent, optimizer
    self.settings = settings or default_settings()
    check_bellman_target(self.settings.bellman_target, self.settings.retrace_lambda)
    self.pg = process_group
    import torch.distributed as td
    self.world = td.get_world_size(process_group) if (td.is_available() and td.is_initialized()) else 1
    optimizer._create_slots(agent.params)
    self.last_gradient_norm = None

  def update_target_agent(self):
    self.target_agent.assign_from(self.agent)

  def compute_gradients(self, sampled):
    """:596-611.  sampled: SampledUnrolls with time-major unrolls.  Leaves the clipped gradient in
    agent.grads; returns (loss scalar, priorities [B], indices, gradient_norm_before_clip)."""
    u, s = sampled.unrolls, self.settings
    w = _lib.require_cuda(sampled.importance_weights, torch.float32, 'importance_weights')
    loss, priorities, dq = compute_loss_and_priorities(
        self.agent, self.target_agent, u.agent_state, u.prev_actions, u.env_outputs, u.agent_outputs,
        gamma=s.discounting, burn_in=s.burn_in, importance_weights=w, n_steps=s.n_steps,
        value_function_rescaling_epsilon=s.value_function_rescaling_epsilon, bellman_target=s.bellman_target,
        retrace_lambda=s.retrace_lambda, abandoned=u.env_outputs[3] if s.bootstrap_abandoned else None)
    grads = self.agent.backward(dq)
    if s.clip_norm:
      norm = clip_by_global_norm(grads, s.clip_norm)                 # :606-609 (use_norm = the same norm)
    else:
      norm = torch.linalg.vector_norm(grads)
    return (loss * w).mean(), priorities, sampled.indices, norm

  def apply_gradients(self):
    grads = self.agent.grads
    if self.world > 1:
      import torch.distributed as td
      td.all_reduce(grads, op=td.ReduceOp.SUM, group=self.pg)        # replicas SUM (tests/utils_test.py:640-650)
    self.optimizer.apply_gradients(self.agent.params, grads)

  def minimize(self, sampled):
    if self.optimizer.iterations % self.settings.update_target_every_n_step == 0:      # :845-846
      self.update_target_agent()
    loss, priorities, indices, norm = self.compute_gradients(sampled)
    self.apply_gradients()
    self.last_gradient_norm = norm
    return loss, priorities, indices, norm


class ReplayFeeder(object):
  """create_dataset's `dequeue` (:410-461) + the priority write-back of the main loop (:868): insert
  `get_replay_insertion_batch_size` new unrolls, then sample a batch by priority and hand it to
  the learner time-major.  Single-threaded like the reference's (the buffer is not thread-safe)."""

  def __init__(self, replay_buffer, settings=None, generator=None):
    self.replay_buffer = replay_buffer
    self.settings = settings or default_settings()
    self.generator = generator

  def insert(self, unrolls):
    """unrolls: Unroll with env-major tensors [n, T, ...] and priority [n]."""
    return self.replay_buffer.insert(unrolls, unrolls.priority)

  def ready(self):
    return self.replay_buffer.num_inserted >= self.settings.replay_buffer_min_size

  def sample(self, batch_size=None):
    s = self.settings
    indices, weights, unrolls = self.replay_buffer.sample(batch_size or s.batch_size, s.priority_exponent,
                                                          generator=self.generator)
    unrolls = unrolls._replace(prev_actions=utils.make_time_major(unrolls.prev_actions),
                               env_outputs=utils.make_time_major(unrolls.env_outputs),
                               agent_outputs=utils.make_time_major(unrolls.agent_outputs))
    return SampledUnrolls(unrolls, indices, weights)

  def update_priorities(self, indices, priorities):
    self.replay_buffer.update_priorities(indices, priorities)
