"""V-trace learner -- mirror of the reference's `agents/vtrace/learner.py`:

  flags                         learner.py:38-68   (same names and defaults)
  compute_loss                  learner.py:73-159
  Unroll                        learner.py:162-163
  minimize (LearnerStep)        learner.py:255-280
  learner_loop                  learner.py:170-483 (see learner_loop.py for the RPC wiring)

Device work per step = seedrl_net_forward -> seedrl_vtrace_loss_fwd_bwd ->
seedrl_net_backward -> [one NCCL all-reduce(SUM) of the flat gradient arena]
-> seedrl_adam_apply.  There is no autograd tape: the loss kernel emits the analytic
gradient w.r.t. the network outputs and the network backward is an explicit schedule.
"""
import collections
import math

from absl import flags
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common import common_flags  # pylint: disable=unused-import
from seed_rl_b200.common import utils

# Training.
common_flags.define_once(flags.DEFINE_integer, 'save_checkpoint_secs', 1800, 'Checkpoint save period in seconds.')
common_flags.define_once(flags.DEFINE_integer, 'total_environment_frames', int(1e9),
                     'Total environment frames to train for.')
common_flags.define_once(flags.DEFINE_integer, 'batch_size', 32, 'Batch size for training.')
common_flags.define_once(flags.DEFINE_integer, 'inference_batch_size', -1, 'Batch size for inference, -1 for auto-tune.')
common_flags.define_once(flags.DEFINE_integer, 'unroll_length', 100, 'Unroll length in agent steps.')
common_flags.define_once(flags.DEFINE_integer, 'num_training_tpus', 1, 'Unused: there are no TPUs (kept for flag compatibility).')
common_flags.define_once(flags.DEFINE_string, 'init_checkpoint', None,
                    'Path to the checkpoint used to initialize the agent.')
# Loss settings.
common_flags.define_once(flags.DEFINE_float, 'entropy_cost', 0.00025, 'Entropy cost/multiplier.')
common_flags.define_once(flags.DEFINE_float, 'target_entropy', None, 'If not None, the entropy cost is '
                   'automatically adjusted to reach the desired entropy level.')
common_flags.define_once(flags.DEFINE_float, 'entropy_cost_adjustment_speed', 10., 'Controls how fast '
                   'the entropy cost coefficient is adjusted.')
common_flags.define_once(flags.DEFINE_float, 'baseline_cost', .5, 'Baseline cost/multiplier.')
common_flags.define_once(flags.DEFINE_float, 'kl_cost', 0., 'KL(old_policy|new_policy) loss multiplier.')
common_flags.define_once(flags.DEFINE_float, 'discounting', .99, 'Discounting factor.')
common_flags.define_once(flags.DEFINE_float, 'lambda_', 1., 'Lambda.')
common_flags.define_once(flags.DEFINE_float, 'max_abs_reward', 0., 'Maximum absolute reward when calculating loss.'
                   'Use 0. to disable clipping.')
# Logging
common_flags.define_once(flags.DEFINE_integer, 'log_batch_frequency', 100, 'We average that many batches '
                     'before logging batch statistics like entropy.')
common_flags.define_once(flags.DEFINE_integer, 'log_episode_frequency', 1, 'We average that many episodes'
                     ' before logging average episode return and length.')
# flags of this implementation (not in the reference)
common_flags.define_once(flags.DEFINE_enum, 'grad_reduce', 'sum', ['sum', 'mean'],
                  'Cross-replica gradient reduction. The reference SUMs '
                  '(tests/utils_test.py:609-650).')
common_flags.define_once(flags.DEFINE_bool, 'popart', False,
                         'Normalise value targets and advantages with PopArt (popart.py, EMAMeanStd '
                         'statistics, compensation on).')
common_flags.define_once(flags.DEFINE_float, 'popart_beta', 1e-2,
                         'Step size of the PopArt moment EMA (EMAMeanStd beta).')
common_flags.define_once(flags.DEFINE_integer, 'popart_tasks', 1,
                         'With --popart: the number of tasks K (1 to 64), each with its own PopArt statistics and '
                         'compensation.  Environment id i belongs to task i % K, as create_env_fn(i, ...) picks '
                         'levels[i % K].')
common_flags.define_once(flags.DEFINE_bool, 'bootstrap_abandoned', False,
                         'Accept abandoned episodes (EnvOutput.abandoned: a time limit, not the task, ended '
                         'them) and bootstrap from the value of their last observation instead of '
                         'treating it as terminal (advantages.py vtrace / NStep).')

FLAGS = flags.FLAGS

LossSettings = collections.namedtuple(
    'LossSettings',
    'discounting lambda_ baseline_cost entropy_cost kl_cost max_abs_reward '
    'target_entropy entropy_cost_adjustment_speed popart popart_beta bootstrap_abandoned popart_tasks',
    defaults=(False, 1e-2, False, 1))

MAX_POPART_TASKS = 64


def check_loss_settings(settings):
  """Raises ValueError for a PopArt task count outside [1, 64], or above 1 without PopArt."""
  K = settings.popart_tasks
  if not (isinstance(K, int) and 1 <= K <= MAX_POPART_TASKS):
    raise ValueError('popart_tasks must be an integer in [1, %d], got %r' % (MAX_POPART_TASKS, K))
  if K > 1 and not settings.popart:
    raise ValueError('popart_tasks = %d needs popart' % K)


def loss_settings_from_flags():
  return LossSettings(FLAGS.discounting, FLAGS.lambda_, FLAGS.baseline_cost,
                      FLAGS.entropy_cost, FLAGS.kl_cost, FLAGS.max_abs_reward,
                      FLAGS.target_entropy, FLAGS.entropy_cost_adjustment_speed, FLAGS.popart,
                      FLAGS.popart_beta, FLAGS.bootstrap_abandoned, FLAGS.popart_tasks)


def default_loss_settings(**kw):
  d = dict(discounting=.99, lambda_=1., baseline_cost=.5, entropy_cost=0.00025, kl_cost=0.,
           max_abs_reward=0., target_entropy=None, entropy_cost_adjustment_speed=10., popart=False,
           popart_beta=1e-2, bootstrap_abandoned=False, popart_tasks=1)
  d.update(kw)
  return LossSettings(**d)


class _NullLogger(object):
  def log_session(self):
    return []

  def log(self, session, name, value):
    session.append((name, value))


_LOG_NAMES = [  # learner.py:138-157
    ('V/value function', 'v_mean'), ('V/L2 error', 'v_l2_error'),
    ('losses/policy', 'policy'), ('losses/V', 'V'), ('losses/entropy', 'entropy'),
    ('losses/kl', 'kl'), ('losses/total', 'total'),
    ('policy/max_action_abs(before_tanh)', 'max_action_abs'),
    ('policy/entropy', 'mean_entropy'), ('policy/entropy_cost', 'entropy_cost'),
    ('policy/kl(old|new)', 'mean_kl')]
_POPART_LOG_NAMES = [('PopArt/mean', 'popart_mean'), ('PopArt/std', 'popart_std')]   # popart.py:175-176

_scratch_cache = {}


def _loss_scratch(T1, B, A, device, num_tasks=0):
  """num_tasks > 0: the multi-task PopArt scratch."""
  key = (T1, B, A, str(device), num_tasks)
  if key not in _scratch_cache:
    L = _lib.lib()
    n = int(L.seedrl_vtrace_popart_tasks_scratch_bytes(T1, B, A, num_tasks) if num_tasks
            else L.seedrl_vtrace_loss_scratch_bytes(T1, B, A))
    _scratch_cache[key] = torch.zeros(n, dtype=torch.uint8, device=device)   # zeroed ONCE
  return _scratch_cache[key]


def _loss_inputs(learner_logits, learner_baseline, behaviour_logits, actions, rewards, done,
                 entropy_cost_param):
  f32 = torch.float32
  ll = _lib.require_cuda(learner_logits, f32, 'learner_logits')
  lb = _lib.require_cuda(learner_baseline, f32, 'learner_baseline')
  bl = _lib.require_cuda(behaviour_logits, f32, 'behaviour_logits')
  act = _lib.require_cuda(actions, torch.int64, 'actions')
  rew = _lib.require_cuda(rewards, f32, 'rewards')
  dn = _lib.require_cuda(done, torch.bool, 'done')
  ecp = _lib.require_cuda(entropy_cost_param, f32, 'entropy_cost_param')
  if ll.dim() != 3 or lb.dim() != 2:
    raise ValueError('learner outputs must be [T+1,B,A] and [T+1,B]')
  T1, B, A = (int(x) for x in ll.shape)
  for t, shp, nm in ((lb, (T1, B), 'learner_baseline'), (bl, (T1, B, A), 'behaviour_logits'),
                     (act, (T1, B), 'actions'), (rew, (T1, B), 'rewards'), (dn, (T1, B), 'done')):
    if tuple(t.shape) != shp:
      raise ValueError('%s has shape %s, expected %s' % (nm, tuple(t.shape), shp))
  return ll, lb, bl, act, rew, dn, ecp


def _abandoned_input(abandoned, shape):
  """The [T+1,B] abandoned mask as a contiguous CUDA bool tensor, or None."""
  if abandoned is None:
    return None
  ab = _lib.require_cuda(abandoned, torch.bool, 'abandoned')
  if tuple(ab.shape) != tuple(shape):
    raise ValueError('abandoned has shape %s, expected %s' % (tuple(ab.shape), tuple(shape)))
  return ab


def _loss_config(settings):
  return _lib.LossConfig(
      settings.discounting, settings.lambda_, settings.baseline_cost, settings.kl_cost,
      settings.max_abs_reward or 0.0, 1.0, 1.0,     # compute_loss uses vtrace's default clips
      settings.target_entropy or 0.0, 1 if settings.target_entropy else 0,
      settings.entropy_cost_adjustment_speed)


def _loss_outputs(ll, lb, want_vtrace):
  f32 = torch.float32
  T1, B = int(ll.shape[0]), int(ll.shape[1])
  dev = ll.device
  return dict(
      loss_terms=torch.empty(_lib.LOSS_TERMS, dtype=f32, device=dev),
      dlogits=torch.empty_like(ll), dbaseline=torch.empty_like(lb),
      d_entropy_cost_param=torch.empty((), dtype=f32, device=dev),
      vs=torch.empty([T1 - 1, B], dtype=f32, device=dev) if want_vtrace else None,
      pg_advantages=torch.empty([T1 - 1, B], dtype=f32, device=dev) if want_vtrace else None)


def vtrace_loss_fwd_bwd(settings, learner_logits, learner_baseline, behaviour_logits,
                        actions, rewards, done, entropy_cost_param, want_vtrace=False, abandoned=None):
  """The fused kernel of compute_loss (learner.py:82-157) + its gradient.  All inputs
  have T+1 rows.  Returns dict(loss_terms[16], dlogits, dbaseline, d_entropy_cost_param,
  vs, pg_advantages).  `abandoned` [T+1,B] (None = none): transition t with abandoned[t+1]
  bootstraps from V_t instead of being terminal (seedrl_vtrace_loss_fwd_bwd_abandoned)."""
  ll, lb, bl, act, rew, dn, ecp = _loss_inputs(learner_logits, learner_baseline, behaviour_logits, actions,
                                               rewards, done, entropy_cost_param)
  ab = _abandoned_input(abandoned, dn.shape)
  T1, B, A = (int(x) for x in ll.shape)
  cfg = _loss_config(settings)
  out = _loss_outputs(ll, lb, want_vtrace)
  import ctypes
  L = _lib.lib()
  head = (T1, B, A, _lib.ptr(ll), _lib.ptr(lb), _lib.ptr(bl), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(dn))
  tail = (ctypes.byref(cfg), _lib.ptr(ecp), _lib.ptr(out['loss_terms']),
          _lib.ptr(out['dlogits']), _lib.ptr(out['dbaseline']),
          _lib.ptr(out['d_entropy_cost_param']), _lib.ptr(out['vs']),
          _lib.ptr(out['pg_advantages']), _lib.ptr(_loss_scratch(T1, B, A, ll.device)),
          _lib.stream_ptr())
  if ab is None:
    _lib.check(L.seedrl_vtrace_loss_fwd_bwd(*head, *tail))
  else:
    _lib.check(L.seedrl_vtrace_loss_fwd_bwd_abandoned(*head, _lib.ptr(ab), *tail))
  return out


def popart_loss_fwd_bwd(settings, learner_logits, learner_baseline, behaviour_logits, actions, rewards,
                        done, entropy_cost_param, popart_moments, popart_compensation, d_popart_compensation,
                        reduce_moment_sums=None, world=1, want_vtrace=False, abandoned=None, task_ids=None,
                        task_error=None):
  """compute_loss with PopArt (generalized_onpolicy_loss.py:94-133,169-199 around popart.py and
  EMAMeanStd) + its gradient: seedrl_vtrace_popart_loss_fwd, then `reduce_moment_sums` (in-place
  SUM of the two moment sums across the `world` replicas; None for one replica), then
  seedrl_vtrace_popart_update.  Updates popart_moments (mu1, mu2) and popart_compensation
  (sigma, mu) in place and writes d(loss)/d(sigma, mu) to d_popart_compensation.  Returns what
  vtrace_loss_fwd_bwd returns; vs and pg_advantages are in return units.  `abandoned` as in
  vtrace_loss_fwd_bwd.

  With settings.popart_tasks = K > 1: task_ids (int32 CUDA [B], the task of each column) and task_error
  (int32 CUDA [1], set for an id outside [0, K); zero it once and poll it) are required, the three state
  tensors are [K,2], and the call is popart_tasks_loss_fwd_bwd.  With K = 1 they are ignored."""
  if settings.popart_tasks > 1:
    return popart_tasks_loss_fwd_bwd(settings, learner_logits, learner_baseline, behaviour_logits, actions,
                                     rewards, done, entropy_cost_param, popart_moments, popart_compensation,
                                     d_popart_compensation, task_ids, task_error, reduce_moment_sums,
                                     want_vtrace, abandoned)
  ll, lb, bl, act, rew, dn, ecp = _loss_inputs(learner_logits, learner_baseline, behaviour_logits, actions,
                                               rewards, done, entropy_cost_param)
  ab = _abandoned_input(abandoned, dn.shape)
  T1, B, A = (int(x) for x in ll.shape)
  f32 = torch.float32
  for t, nm in ((popart_moments, 'popart_moments'), (popart_compensation, 'popart_compensation'),
                (d_popart_compensation, 'd_popart_compensation')):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == f32 and t.is_contiguous() and t.numel() == 2):
      raise ValueError('%s must be a contiguous float32 CUDA tensor of 2 elements' % nm)
  beta = float(settings.popart_beta)
  if not 0.0 <= beta <= 1.0:
    raise ValueError('popart_beta must be in [0, 1], got %r' % beta)
  cfg = _loss_config(settings)
  out = _loss_outputs(ll, lb, want_vtrace)
  td = torch.empty([T1 - 1, B], dtype=f32, device=ll.device)
  sums = torch.empty(2, dtype=f32, device=ll.device)
  scratch = _loss_scratch(T1, B, A, ll.device)
  import ctypes
  L = _lib.lib()
  head = (T1, B, A, _lib.ptr(ll), _lib.ptr(lb), _lib.ptr(bl), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(dn))
  tail = (ctypes.byref(cfg), _lib.ptr(ecp), _lib.ptr(popart_moments), _lib.ptr(popart_compensation),
          _lib.ptr(out['loss_terms']), _lib.ptr(out['dlogits']), _lib.ptr(out['dbaseline']),
          _lib.ptr(out['d_entropy_cost_param']), _lib.ptr(out['vs']), _lib.ptr(out['pg_advantages']),
          _lib.ptr(td), _lib.ptr(sums), _lib.ptr(scratch), _lib.stream_ptr())
  if ab is None:
    _lib.check(L.seedrl_vtrace_popart_loss_fwd(*head, *tail))
  else:
    _lib.check(L.seedrl_vtrace_popart_loss_fwd_abandoned(*head, _lib.ptr(ab), *tail))
  if reduce_moment_sums is not None:
    reduce_moment_sums(sums)
  _lib.check(L.seedrl_vtrace_popart_update(
      T1, B, int(world), beta, float(settings.baseline_cost), _lib.ptr(lb), _lib.ptr(td), _lib.ptr(sums),
      _lib.ptr(popart_moments), _lib.ptr(popart_compensation), _lib.ptr(out['dbaseline']),
      _lib.ptr(d_popart_compensation), _lib.ptr(out['loss_terms']), _lib.ptr(scratch), _lib.stream_ptr()))
  return out


def popart_tasks_loss_fwd_bwd(settings, learner_logits, learner_baseline, behaviour_logits, actions, rewards,
                              done, entropy_cost_param, popart_moments, popart_compensation, d_popart_compensation,
                              task_ids, task_error, reduce_moment_sums=None, want_vtrace=False, abandoned=None):
  """popart_loss_fwd_bwd with K = settings.popart_tasks tasks: seedrl_vtrace_popart_tasks_loss_fwd, then
  `reduce_moment_sums` (in-place SUM of the float64 [K,3] per-task sums across replicas), then
  seedrl_vtrace_popart_tasks_update.  Column b is normalised with the state of task task_ids[b]."""
  ll, lb, bl, act, rew, dn, ecp = _loss_inputs(learner_logits, learner_baseline, behaviour_logits, actions,
                                               rewards, done, entropy_cost_param)
  ab = _abandoned_input(abandoned, dn.shape)
  T1, B, A = (int(x) for x in ll.shape)
  K = int(settings.popart_tasks)
  f32 = torch.float32
  for t, nm in ((popart_moments, 'popart_moments'), (popart_compensation, 'popart_compensation'),
                (d_popart_compensation, 'd_popart_compensation')):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == f32 and t.is_contiguous() and
            tuple(t.shape) == (K, 2)):
      raise ValueError('%s must be a contiguous float32 CUDA tensor of shape (%d, 2)' % (nm, K))
  if task_ids is None:
    raise ValueError('popart_tasks = %d needs the task_ids of the batch columns' % K)
  tid = _lib.require_cuda(task_ids, torch.int32, 'task_ids')
  if tuple(tid.shape) != (B,):
    raise ValueError('task_ids has shape %s, expected (%d,)' % (tuple(tid.shape), B))
  if not (isinstance(task_error, torch.Tensor) and task_error.is_cuda and task_error.dtype == torch.int32):
    raise ValueError('task_error must be an int32 CUDA tensor')
  beta = float(settings.popart_beta)
  if not 0.0 <= beta <= 1.0:
    raise ValueError('popart_beta must be in [0, 1], got %r' % beta)
  cfg = _loss_config(settings)
  out = _loss_outputs(ll, lb, want_vtrace)
  td = torch.empty([T1 - 1, B], dtype=f32, device=ll.device)
  sums = torch.empty([K, 3], dtype=torch.float64, device=ll.device)
  scratch = _loss_scratch(T1, B, A, ll.device, K)
  import ctypes
  L = _lib.lib()
  _lib.check(L.seedrl_vtrace_popart_tasks_loss_fwd(
      T1, B, A, _lib.ptr(ll), _lib.ptr(lb), _lib.ptr(bl), _lib.ptr(act), _lib.ptr(rew), _lib.ptr(dn),
      _lib.ptr(ab), _lib.ptr(tid), K, ctypes.byref(cfg), _lib.ptr(ecp), _lib.ptr(popart_moments),
      _lib.ptr(popart_compensation), _lib.ptr(out['loss_terms']), _lib.ptr(out['dlogits']),
      _lib.ptr(out['dbaseline']), _lib.ptr(out['d_entropy_cost_param']), _lib.ptr(out['vs']),
      _lib.ptr(out['pg_advantages']), _lib.ptr(td), _lib.ptr(sums), _lib.ptr(task_error), _lib.ptr(scratch),
      _lib.stream_ptr()))
  if reduce_moment_sums is not None:
    reduce_moment_sums(sums)
  _lib.check(L.seedrl_vtrace_popart_tasks_update(
      T1, B, K, beta, float(settings.baseline_cost), _lib.ptr(lb), _lib.ptr(td), _lib.ptr(tid), _lib.ptr(sums),
      _lib.ptr(popart_moments), _lib.ptr(popart_compensation), _lib.ptr(out['dbaseline']),
      _lib.ptr(d_popart_compensation), _lib.ptr(out['loss_terms']), _lib.ptr(scratch), _lib.stream_ptr()))
  out['moment_sums'] = sums
  return out


def popart_task_logs(popart_moments):
  """[(name, device scalar)]: 'PopArt/mean/<k>' and 'PopArt/std/<k>' of every task, from the [K,2] moments
  (the std as the kernels take it: clip(sqrt(mu2 - mu1^2), 1e-6, 1e6), in float64).  No host sync."""
  m = popart_moments.double()
  std = (m[:, 1] - m[:, 0] * m[:, 0]).sqrt().clamp(1e-6, 1e6).float()
  logs = []
  for k in range(int(popart_moments.shape[0])):
    logs += [('PopArt/mean/%d' % k, popart_moments[k, 0]), ('PopArt/std/%d' % k, std[k])]
  return logs


def compute_loss(logger, parametric_action_distribution, agent, agent_state,
                 prev_actions, env_outputs, agent_outputs, settings=None, reduce_moment_sums=None, world=1,
                 task_ids=None):
  """reference learner.py:73-159.  Returns (total_loss, log session).  The gradient of
  total_loss w.r.t. the network outputs is left on the agent for `minimize`.  With
  settings.popart the agent must have enable_popart()'d: its PopArt state is updated here and
  d(loss)/d(sigma, mu) written to its gradient tail; `reduce_moment_sums` and `world` are the
  cross-replica sum of popart_loss_fwd_bwd.  With settings.bootstrap_abandoned the kernels get
  env_outputs.abandoned; without it they get no mask.  With settings.popart_tasks = K > 1, task_ids (int32
  [B]) gives each column's task and is required; with K = 1 it is ignored."""
  settings = settings or loss_settings_from_flags()
  ab = {'abandoned': env_outputs[3]} if settings.bootstrap_abandoned else {}   # EnvOutput.abandoned
  learner_outputs, _ = agent(prev_actions, env_outputs, agent_state,
                             unroll=True, is_training=True)                 # :75-79
  if settings.popart:
    if getattr(agent, 'popart_moments', None) is None:
      raise ValueError('settings.popart needs an agent with enable_popart() called')
    r = popart_loss_fwd_bwd(settings, learner_outputs.policy_logits, learner_outputs.baseline,
                            agent_outputs.policy_logits, agent_outputs.action,
                            env_outputs[0], env_outputs[1], agent.entropy_cost_param,
                            agent.popart_moments, agent.popart_compensation, agent.popart_compensation_grad,
                            reduce_moment_sums, world, task_ids=task_ids,
                            task_error=getattr(agent, 'popart_task_error', None), **ab)
  else:
    r = vtrace_loss_fwd_bwd(settings, learner_outputs.policy_logits, learner_outputs.baseline,
                            agent_outputs.policy_logits, agent_outputs.action,
                            env_outputs[0], env_outputs[1], agent.entropy_cost_param, **ab)
  agent._loss_grads = r
  logger = logger or _NullLogger()
  session = logger.log_session()
  lt = r['loss_terms']
  tasks = settings.popart and settings.popart_tasks > 1
  for name, key in _LOG_NAMES + (_POPART_LOG_NAMES if settings.popart and not tasks else []):
    logger.log(session, name, lt[_lib.LT[key]])
  if tasks:
    for name, value in popart_task_logs(agent.popart_moments):
      logger.log(session, name, value)
  return lt[_lib.LT['total']], session


Unroll = collections.namedtuple(
    'Unroll', 'agent_state prev_actions env_outputs agent_outputs')


def reduce_gradients(flat_grads, world, process_group=None, grad_reduce='sum'):
  """The ONE exchange step of a data-parallel iteration: all-reduce(SUM) of the flat
  gradient arena in place (NCCL over NVLink on GPUs, gloo in the CPU tests).  Returns the
  scale Adam must apply to the reduced gradient: 1 for the reference's semantics --
  every replica's *mean*-loss gradient is SUMMED across replicas
  (reference tests/utils_test.py:609-650: `expected_a = 1 - N*0.2`) -- or 1/world for
  `grad_reduce='mean'`."""
  if grad_reduce not in ('sum', 'mean'):
    raise ValueError('grad_reduce must be "sum" or "mean"')
  if world <= 1:
    return 1.0
  import torch.distributed as td
  td.all_reduce(flat_grads, op=td.ReduceOp.SUM, group=process_group)
  return 1.0 / world if grad_reduce == 'mean' else 1.0


def env_shard(rank, world, num_envs):
  """Environments owned by replica `rank`: {i : i mod world == rank} (SURVEY 8e)."""
  return list(range(rank, num_envs, world))


class LearnerStep(object):
  """`minimize` of reference learner.py:255-280 for one replica (= one GPU/process)."""

  def __init__(self, agent, optimizer, parametric_action_distribution=None, settings=None,
               logger=None, process_group=None, grad_reduce='sum', check_errors_every=64,
               overlap_reduce=True):
    self.agent = agent
    self.overlap_reduce = overlap_reduce
    self._side = self._head_ev = self._head_work = None
    # the kernels' bounded-wait error flag is polled (one 4-byte D2H + stream sync) every
    # `check_errors_every` steps; 0 = never (the caller polls agent.check_errors() itself)
    self.check_errors_every = int(check_errors_every)
    self._steps = 0
    self.optimizer = optimizer
    self.dist = parametric_action_distribution
    self.settings = settings or default_loss_settings()
    check_loss_settings(self.settings)
    self.logger = logger
    self.pg = process_group
    self.grad_reduce = grad_reduce
    import torch.distributed as td
    self.world = td.get_world_size(process_group) if (td.is_available() and td.is_initialized()) else 1
    if not hasattr(agent, '_entropy_mul'):
      agent.init_entropy_cost(self.settings.entropy_cost,
                              self.settings.entropy_cost_adjustment_speed)       # :225-234
    if self.settings.popart and agent.popart_moments is None:
      if optimizer.m is not None:
        raise ValueError('PopArt extends the parameter arena: enable it before the optimizer creates its slots')
      agent.enable_popart(self.settings.popart_tasks)
    elif self.settings.popart and agent.popart_tasks != self.settings.popart_tasks:
      raise ValueError('the agent has %d PopArt tasks; the settings ask for %d'
                       % (agent.popart_tasks, self.settings.popart_tasks))
    optimizer._create_slots(agent.params)                                        # :244-245
    self.last_loss_terms = None

  def _reduce_moment_sums(self, sums):
    import torch.distributed as td
    td.all_reduce(sums, op=td.ReduceOp.SUM, group=self.pg)

  def compute_gradients(self, unroll, task_ids=None):
    """task_ids: int32 [B], the task of each column, required with settings.popart_tasks > 1."""
    loss, logs = compute_loss(self.logger, self.dist, self.agent, unroll.agent_state,
                              unroll.prev_actions, unroll.env_outputs, unroll.agent_outputs,
                              self.settings, self._reduce_moment_sums if self.world > 1 else None,
                              self.world, task_ids=task_ids)
    r = self.agent._loss_grads
    self._head_work = None
    if self.world > 1 and self.overlap_reduce and torch.cuda.is_available():
      # bucket 1 (heads, Dense, LSTM = 94 % of the arena) is all-reduced on a side stream while
      # the convolution torso's backward still runs; bucket 2 follows in apply_gradients
      import torch.distributed as td
      if self._side is None:
        self._side, self._head_ev = torch.cuda.Stream(), torch.cuda.Event()
      grads = self.agent.backward(r['dlogits'], r['dbaseline'], head_ready_event=self._head_ev)
      with torch.cuda.stream(self._side):
        self._side.wait_event(self._head_ev)
        self._head_work = td.all_reduce(grads[:self.agent.grad_split], op=td.ReduceOp.SUM, group=self.pg,
                                        async_op=True)
    else:
      grads = self.agent.backward(r['dlogits'], r['dbaseline'])                   # :264
    grads[self.agent.entropy_cost_param_index] = r['d_entropy_cost_param']
    self.last_loss_terms = r['loss_terms']
    return loss, logs

  def apply_gradients(self):
    grads = self.agent.grads
    if getattr(self, '_head_work', None) is not None:
      import torch.distributed as td
      td.all_reduce(grads[self.agent.grad_split:], op=td.ReduceOp.SUM, group=self.pg)
      self._head_work.wait()              # the compute stream waits for the side-stream bucket
      self._head_work = None
      scale = 1.0 / self.world if self.grad_reduce == 'mean' else 1.0
    else:
      scale = reduce_gradients(grads, self.world, self.pg, self.grad_reduce)
    mul = self.settings.entropy_cost_adjustment_speed
    self.optimizer.apply_gradients(
        self.agent.params, grads, grad_scale=scale,
        clamp_index=self.agent.entropy_cost_param_index,
        clamp_lo=-20.0 / mul, clamp_hi=20.0 / mul)                                # :229-231

  def minimize(self, unroll, task_ids=None):
    loss, logs = self.compute_gradients(unroll, task_ids=task_ids)
    self.apply_gradients()
    self._steps += 1
    if self.check_errors_every and (self._steps == 1 or self._steps % self.check_errors_every == 0):
      self.agent.check_errors()
    return loss, logs


class DeviceFeeder(object):
  """Double-buffered host -> device feed of training batches (the role tf.data prefetching
  onto the accelerator plays for the reference's `minimize(it)`, learner.py:457-466).

  `put(pinned)` enqueues the H2D copies of one batch (a dict of pinned host tensors) on a
  private copy stream into the slot the learner is not using; `get()` returns the dict of
  device tensors of the oldest pending batch and makes the current (compute) stream wait for
  its copies.  While step i trains from one slot, batch i+1 streams into the other, so the
  upload is hidden behind the step instead of serialised in front of it."""

  def __init__(self, example, device='cuda', slots=2):
    self._slots = [{k: torch.empty_like(v, device=device) for k, v in example.items()} for _ in range(slots)]
    self._copied = [torch.cuda.Event() for _ in range(slots)]
    self._consumed = [None] * slots
    self._stream = torch.cuda.Stream(device=device)
    self._put = 0
    self._get = 0

  @property
  def slots(self):
    return self._slots

  def put(self, pinned):
    if self._put - self._get >= len(self._slots):
      raise RuntimeError('DeviceFeeder: every slot holds an unconsumed batch')
    s = self._put % len(self._slots)
    with torch.cuda.stream(self._stream):
      if self._consumed[s] is not None:
        self._stream.wait_event(self._consumed[s])     # the step that read this slot has finished
      for k, v in pinned.items():
        self._slots[s][k].copy_(v, non_blocking=True)
      self._copied[s].record(self._stream)
    self._put += 1

  def get(self):
    if self._get >= self._put:
      raise RuntimeError('DeviceFeeder: no batch pending')
    s = self._get % len(self._slots)
    torch.cuda.current_stream().wait_event(self._copied[s])
    self._get += 1
    return s, self._slots[s]

  def done_with(self, slot):
    """Call after the step that consumed `slot` has been enqueued on the compute stream."""
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream())
    self._consumed[slot] = ev
