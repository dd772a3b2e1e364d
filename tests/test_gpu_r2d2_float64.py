"""The R2D2 learner step at the `bench.py --agent r2d2` shape (B = 64, burn-in 40 + unroll 100 + 1 = 141 rows of
84x84x1 frames stacked 4, A = 18, learner.default_settings()) against a float64 reference that makes the GPU's
discrete decisions (tests/r2d2_float64_reference.py), in gemm_mode 'simt', 'tc3', and 'tc3' with lstm_mode 'tc3'.

Why conditioned.  The step is piecewise smooth: every ReLU switches its derivative at zero and the double-DQN target
takes an argmax.  A random-init net at this shape has units within fp32 / bf16x3 rounding of their kink, so an
unconditioned reference jumps by more than the kernels' arithmetic error: perturbing every parameter by 2^-16 moves
the float64 gradients by up to 1.5e-2 (value/hidden/kernel) and 8.7e-3 (advantage/hidden/kernel), 2^-20 by 4.4e-3 on
body/dense/kernel.  Those jumps are ReLU masks flipping, not greedy actions (none flips).  After
R2D2LearnerStep.compute_gradients the online agent's (101, 64) workspace still holds the suffix forward;
seedrl_debug_r2d2_net_views locates its post-ReLU buffers, the masks are those > 0, and the greedy action is the
first maximum of the GPU's online q (dueling_fwd_kernel's rule).  The float64 reference evaluates each ReLU of its
suffix unroll as z * mask and takes that greedy action; it is then smooth, and its response to a relative
perturbation delta of the parameters (both networks), h0 and c0 is linear in delta:
test_conditioned_reference_is_linear_in_the_perturbation shows it from 2^-24 to 2^-16.

Bars, per stage (q, target q, dq, loss, priorities, norm before the clip, each of the 18 gradient tensors after the
clip, the Adam update of each tensor): error = max|gpu - ref| / max|ref| (relative difference for scalars),
bar = max(FLOOR, C x m), one C and one FLOOR for every stage and mode, where m is measured:
  * 'simt': the distance to float64 of the float32 reference under the same decisions -- the fp32 rounding of an
    independent implementation of the same step;
  * bf16x3 ('tc3', and the 'tc3' recurrence): the larger of that and the float64 reference's response to a 2^-16
    relative perturbation (N(0, 1) multipliers) of the parameters, h0 and c0, the size of a bf16x3 operand's
    rounding.  Both terms are needed: the contractions round their operands to bf16x3, everything else (the
    accumulators, the LSTM cell, the loss kernel's TD errors, dq) rounds to fp32 as in 'simt'.
C = 8 as in test_gpu_lstm_recurrence.py: the kernels round at every layer and time step while each measure perturbs
once.  Measured on an H100 the worst stage sits at 5.1x its measure ('simt' body/conv0/kernel, whose weight
gradient sums 2.6 M positions in a different order than the CPU) and every other below 3x.
The Adam update compared is the GPU's parameters after apply_gradients minus before, with the half ulp that storing
the fp32 parameter rounds allowed element-wise (the reference's update is taken before that rounding).
"""
import ctypes

import numpy as np
import pytest
import torch

import r2d2_float64_reference as RF

pytestmark = pytest.mark.gpu

C = 8
FLOOR = 1e-6
A, OBS, S, B = 18, (84, 84, 1), 4, 64
LR, ADAM_EPS = 0.00048, 1e-3            # bench.py: Adam(0.00048, epsilon=1e-3)
DELTA = 2.0 ** -16
MODES = {'simt': ('simt', 'tiled'), 'tc3': ('tc3', 'tiled'), 'tc3-lstm-tc3': ('tc3', 'tc3')}
_cache = {}


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _problem():
  """The case of test_gpu_fullsize_r2d2.py: params seed 5, target seed 6, batch seed 21."""
  if 'problem' not in _cache:
    from oracle import r2d2_learner_oracle as RL, r2d2_net_oracle as NO
    from seed_rl_b200.agents.r2d2 import learner
    ls = learner.default_settings()
    T = ls.burn_in + ls.unroll_length + 1
    _cache['problem'] = (NO.init_params(A, OBS, S, seed=5), NO.init_params(A, OBS, S, seed=6),
                         RL.synthetic_replay_batch(T, B, A, OBS, seed=21, done_p=0.01), ls,
                         RF.settings(A, S, ls, LR, ADAM_EPS))
  return _cache['problem']


def _gpu_step(gemm_mode, lstm_mode):
  """One R2D2LearnerStep.compute_gradients + apply_gradients; -> numpy results and the GPU's decisions."""
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils

  class Recorded(networks.DuelingLSTMDQNNet):
    """Keeps the q of its last call and the dq of its last backward."""

    def __call__(self, *args, **kw):
      out = super().__call__(*args, **kw)
      self.last_q = out[0].q_values
      return out

    def backward(self, dq):
      self.last_dq = dq.clone()
      return super().backward(dq)

  params, tparams, b, ls, _ = _problem()
  T, Bb = b['reward'].shape
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  agent = Recorded(A, OBS, S, gemm_mode=gemm_mode, lstm_mode=lstm_mode); agent.load_named_parameters(params)
  target = Recorded(A, OBS, S, gemm_mode=gemm_mode, lstm_mode=lstm_mode); target.load_named_parameters(tparams)
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(LR, epsilon=ADAM_EPS), settings=ls)
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']), torch.zeros(T, Bb, dtype=torch.bool).cuda(),
                        torch.zeros(T, Bb, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
  unrolls = learner.Unroll(state, None, c(b['prev_actions']), env, learner.AgentOutput(c(b['action']), None))
  sampled = learner.SampledUnrolls(unrolls, c(b['indices']), c(b['importance_weights']))
  loss, priorities, _, gnorm = step.compute_gradients(sampled)
  agent.check_errors(); target.check_errors()
  Ts = T - ls.burn_in
  N = Ts * Bb
  ws = agent.workspace(Ts, Bb)

  def view(index, shape):
    off, nb = ctypes.c_size_t(), ctypes.c_size_t()
    _lib.check(_lib.lib().seedrl_debug_r2d2_net_views(agent._h, Ts, Bb, index, ctypes.byref(off), ctypes.byref(nb)))
    assert nb.value == 4 * int(np.prod(shape))
    return ws[off.value:off.value + nb.value].view(torch.float32).reshape(shape)
  masks = dict(conv0=view(0, (N, 20, 20, 32)), conv1=view(1, (N, 9, 9, 64)), conv2=view(2, (N, 7, 7, 64)),
               dense=view(3, (N, 512 + 1 + A))[:, :512], value=view(4, (N, 512)), advantage=view(5, (N, 512)))
  masks = {k: (v > 0).cpu().numpy() for k, v in masks.items()}
  q = agent.last_q.cpu().numpy()
  out = dict(q=q, target_q=target.last_q.cpu().numpy(), dq=agent.last_dq.cpu().numpy(), total=float(loss),
             priorities=priorities.cpu().numpy(), norm=float(gnorm),
             grads={k: v.cpu().numpy().copy() for k, v in agent.named_gradients().items()},
             masks=masks, greedy=q.argmax(-1))
  before = {k: v.cpu().numpy().copy() for k, v in agent.named_parameters().items()}
  step.apply_gradients()
  after = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  out['update'] = {k: before[k].astype(np.float64) - after[k] for k in before}
  out['after'] = after
  del agent, target, step, sampled, unrolls, env, state, ws
  torch.cuda.empty_cache()
  return out


def _run(mode):
  """The GPU step of `mode`, the float64 reference under its decisions and the measured m (cached)."""
  if mode in _cache:
    return _cache[mode]
  params, tparams, b, _, st = _problem()
  gpu = _gpu_step(*MODES[mode])
  cond = dict(masks=gpu['masks'], greedy=gpu['greedy'])
  ref = RF.step(params, tparams, b, st, torch.float64, **cond)
  m = _stages(RF.step(params, tparams, b, st, torch.float32, **cond), ref)
  probes = {}
  if mode != 'simt':
    deltas = (2.0 ** -24, 2.0 ** -20, DELTA) if mode == 'tc3' else (DELTA,)
    for d in deltas:
      probes[d] = RF.step(*RF.perturbed(params, tparams, b, d), st, torch.float64, **cond)
    m16 = _stages(probes[DELTA], ref)
    m = {k: max(m[k], m16[k]) for k in m}
  _cache[mode] = (gpu, ref, m, probes)
  return _cache[mode]


def _stages(x, ref):
  """{stage: error of x against ref}; x is a reference result or the GPU's."""
  e = dict(q=_relmax(x['q'], ref['q']), target_q=_relmax(x['target_q'], ref['target_q']),
           dq=_relmax(x['dq'], ref['dq']), loss=abs(x['total'] - ref['total']) / abs(ref['total']),
           priorities=_relmax(x['priorities'], ref['priorities']), norm=abs(x['norm'] - ref['norm']) / ref['norm'])
  for k in ref['grads']:
    e['grad ' + k] = _relmax(x['grads'][k] * x.get('scale', 1.0), ref['grads'][k] * ref['scale'])
  for k in ref['update']:
    d = np.abs(x['update'][k] - ref['update'][k])
    if 'after' in x:     # the GPU's parameters are stored in fp32: half an ulp of each is rounding, not error
      d = np.maximum(d - 0.5 * np.spacing(np.abs(x['after'][k])), 0.0)
    e['adam ' + k] = float(d.max() / (np.abs(ref['update'][k]).max() + 1e-30))
  return e


@pytest.mark.parametrize('mode', list(MODES))
def test_r2d2_step_matches_float64_under_its_own_decisions(mode):
  gpu, ref, ms, _ = _run(mode)
  errs = _stages(gpu, ref)
  T, Bb = ref['q'].shape[:2]
  print('R2D2 FLOAT64 %s (suffix %dx%d, C = %g, floor %.0e, m = %s): error / bar' %
        (mode, T, Bb, C, FLOOR, 'float32 reference' if mode == 'simt' else 'max(float32 reference, 2^-16 response)'))
  bad = []
  for k in errs:
    bar = max(FLOOR, C * ms[k])
    print('  %-34s %.2e / %.2e' % (k, errs[k], bar))
    if not errs[k] <= bar:
      bad.append((k, errs[k], bar))
  assert not bad, bad


def test_conditioned_reference_is_linear_in_the_perturbation():
  """Under the 'tc3' step's decisions the float64 reference's response grows 16x per 16x of perturbation, in every
  stage: no decision is left unshared, so the bf16x3 bars measure arithmetic.  The Adam updates are fp32
  (optim_oracle.keras_adam_step), below the resolution of a 2^-24 response, and are checked from 2^-20."""
  _, ref, _, probes = _run('tc3')
  resp = {d: _stages(p, ref) for d, p in probes.items()}
  d24, d20, d16 = sorted(resp)
  print('R2D2 FLOAT64 conditioned response at 2^-24 / 2^-20 / 2^-16')
  bad = []
  for k in resp[d16]:
    r = (resp[d24][k], resp[d20][k], resp[d16][k])
    print('  %-34s %.2e %.2e %.2e' % ((k,) + r))
    first = 1 if k.startswith('adam ') else 0
    if not all(8 <= r[i + 1] / max(r[i], 1e-300) <= 32 for i in range(first, 2)):
      bad.append((k, r))
  assert not bad, bad
