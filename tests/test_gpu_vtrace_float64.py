"""The V-trace learner step at the test_gpu_fullsize.py shape (T = 20, B = 64, 84x84x4 frames, A = 18, params seed 1,
synthetic_batch seed 1234, h0 / c0 ~ N(0, 1)) against a float64 reference that makes the GPU's ReLU and max-pool
decisions (tests/vtrace_float64_reference.py): ImpalaDeep in conv_mode 'simt', 'tc3', 'tc3p' and 'tc3p' with the
'tc3' recurrence, ImpalaShallow in 'simt' and 'tc3'.

Why conditioned.  The step is piecewise smooth: a random-init net at this shape has ReLU units and max-pool windows
within fp32 / bf16x3 rounding of their kink, and a reference that makes its own decisions jumps there by more than
the kernels' arithmetic (the fp32 oracle's gradients move by up to 5.1e-3 under a 1e-6 parameter perturbation,
which is why test_gpu_fullsize.py's gradient bars are 4-8x that).  After LearnerStep.compute_gradients the agent's
(21, 64) workspace still holds the forward; seedrl_debug_net_views locates the buffers that carry each decision: the 14 ReLU masks and
3 pool-tap tensors of ImpalaDeep, the 3 masks of ImpalaShallow.  A second forward on the same workspace must leave
them bit-identical (the backward overwrites none of them, and the step is deterministic).  The float64 reference
evaluates each ReLU as z * mask and each pool as a gather at the GPU's tap; it is then smooth in the parameters,
and test_conditioned_reference_is_linear_in_the_perturbation shows it for 'tc3p'.

The decisions are checked before they are shared: wherever the GPU's mask or tap differs from the one the float64
reference would make, the unit must be a near-tie, |z_64| (ReLU) or max - x_64[gpu tap] (pool) within that layer's
activation bar times the layer's max-abs.  A mask read from the wrong plane, or a tap from the wrong window, fails.

Bars, per stage (logits, baseline, loss and the continuous logged terms, dlogits, dbaseline, every viewed activation,
the 39 gradients, the Adam update of the 39 tensors and entropy_cost_param): error = max|gpu - ref| / max|ref|
(relative difference for scalars), bar = max(FLOOR, C x m), the rule and constants of test_gpu_r2d2_float64.py:
  * 'simt': m = the distance to float64 of the float32 reference under the same decisions;
  * bf16x3 modes: m = the larger of that and the float64 reference's response to a 2^-16 relative perturbation
    (N(0, 1) multipliers) of the parameters, h0 and c0.
A post-ReLU view (tc3p's c0 / o0 / c1, the shallow convs, Dense) is compared with z x mask.  The Adam update is the
GPU's parameters after apply_gradients minus before, with the half ulp of the stored fp32 parameter allowed.
"""
import ctypes

import numpy as np
import pytest
import torch

import vtrace_float64_reference as RF

pytestmark = pytest.mark.gpu

C = 8
FLOOR = 1e-6
A, OBS, T, B = 18, (84, 84, 4), 20, 64
DELTA = 2.0 ** -16
MODES = {'deep-simt': ('deep', 'simt', 'tiled'), 'deep-tc3': ('deep', 'tc3', 'tiled'),
         'deep-tc3p': ('deep', 'tc3p', 'tiled'), 'deep-tc3p-lstm-tc3': ('deep', 'tc3p', 'tc3'),
         'shallow-simt': ('shallow', 'simt', 'tiled'), 'shallow-tc3': ('shallow', 'tc3', 'tiled')}
_cache = {}


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _problem(net):
  if net not in _cache:
    from oracle import learner_oracle, loss_oracle, net_oracle
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    b = learner_oracle.synthetic_batch(T, B, A, OBS, seed=1234)
    rng = np.random.default_rng(5)
    b['h0'] = rng.normal(size=b['h0'].shape).astype(np.float32)
    b['c0'] = rng.normal(size=b['c0'].shape).astype(np.float32)
    _cache[net] = (net_oracle.init_params(net, A, OBS, seed=1), b, loss_oracle.default_config())
  return _cache[net]


def _view_names(net, conv_mode):
  """[(view index, reference name, post-ReLU?)]; pools carry the name of their taps."""
  if net == 'shallow':
    return [(0, 'conv0', True), (1, 'conv1', True), (2, 'dense', True)]
  out = []
  for s in range(3):
    for j, k in enumerate(('p', 'c0', 'o0', 'c1')):
      out.append((5 * s + j, 'stack%d/%s' % (s, k), conv_mode == 'tc3p' and k != 'p'))
    out.append((5 * s + 4, 'stack%d/pool' % s, False))
  return out + [(15, 'o1', False), (16, 'dense', True)]


def _shape(net, name, N):
  if name == 'dense':
    return (N, 256)
  if net == 'shallow':
    return (N, 20, 20, 16) if name == 'conv0' else (N, 9, 9, 32)
  hw, c = (11, 32) if name == 'o1' else ((42, 16), (21, 32), (11, 32))[int(name[5])]
  return (N, hw, hw, c)


def _read_views(agent, net, T1, Bn, ws=None):
  """{reference name: the GPU buffer as a CPU array} (fp32 NHWC / decoded planes / uint8 taps) of the (T1, Bn)
  workspace `ws` (default: the agent's own)."""
  from seed_rl_b200 import _lib
  L = _lib.lib()
  ws = agent.workspace(T1, Bn) if ws is None else ws
  N = T1 * Bn
  out = {}
  for i, name, _ in _view_names(net, agent.conv_mode):
    off, nb, fmt = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int()
    _lib.check(L.seedrl_debug_net_views(agent._h, T1, Bn, i, ctypes.byref(off), ctypes.byref(nb), ctypes.byref(fmt)))
    raw = ws[off.value:off.value + nb.value]
    shape = _shape(net, name, N)
    if name == 'dense':
      y = raw.view(torch.float32).reshape(N, -1)[:, :256]
    elif fmt.value == 1:
      y = torch.empty(shape, dtype=torch.float32, device=ws.device)
      _lib.check(L.seedrl_debug_from_planes(N, shape[1], shape[2], shape[3], _lib.ptr(raw), _lib.ptr(y),
                                            _lib.stream_ptr()))
    else:
      y = raw.view(torch.float32 if fmt.value == 0 else torch.uint8).reshape(shape)
    out[name] = y.cpu().numpy()
  return out


def _gpu_step(net, conv_mode, lstm_mode):
  """One LearnerStep.compute_gradients + apply_gradients; -> numpy results and the GPU's decisions."""
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda

  base = networks.ImpalaDeep if net == 'deep' else networks.ImpalaShallow

  class Recorded(base):
    """Keeps the outputs of its last call."""

    def __call__(self, *args, **kw):
      out = super().__call__(*args, **kw)
      self.last = out[0]
      return out

  params, b, cfg = _problem(net)
  agent = Recorded(A, OBS, conv_mode=conv_mode, lstm_mode=lstm_mode)
  agent.load_named_parameters(params)
  step = learner.LearnerStep(agent, optimizers.Adam(RF.LR, beta_1=RF.BETA1, epsilon=RF.ADAM_EPS),
                             settings=learner.default_loss_settings())
  u = _batch_to_cuda(b)
  loss, _ = step.compute_gradients(u)
  agent.check_errors()
  T1, Bn = b['reward'].shape
  r = agent._loss_grads
  lt = r['loss_terms'].cpu().numpy()
  names = dict(learner._LOG_NAMES)
  views = _read_views(agent, net, T1, Bn)
  out = dict(logits=agent.last.policy_logits.cpu().numpy(), baseline=agent.last.baseline.cpu().numpy(),
             total=float(loss), logs={k: float(lt[_lib.LT[names[k]]]) for k in names
                                      if k != 'policy/max_action_abs(before_tanh)'},
             dlogits=r['dlogits'].cpu().numpy(), dbaseline=r['dbaseline'].cpu().numpy(),
             grads={k: v.cpu().numpy().copy() for k, v in agent.named_gradients().items()})
  # the decisions of a second forward on the same workspace are the step's: the backward wrote none of them
  agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True, is_training=True)
  again = _read_views(agent, net, T1, Bn)
  for k in views:
    np.testing.assert_array_equal(again[k], views[k], err_msg='view %s changed' % k)
  del again
  out['post'] = {name: p for _, name, p in _view_names(net, conv_mode)}
  out['views'] = {k: v for k, v in views.items() if not k.endswith('/pool')}
  out['masks'] = {k: v > 0 for k, v in out['views'].items()}
  out['taps'] = {k: v for k, v in views.items() if k.endswith('/pool')}
  before = {k: v.cpu().numpy().copy() for k, v in agent.named_parameters().items()}
  before['entropy_cost_param'] = agent.entropy_cost_param.cpu().numpy().copy()
  step.apply_gradients()
  after = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  after['entropy_cost_param'] = agent.entropy_cost_param.cpu().numpy()
  out['update'] = {k: before[k].astype(np.float64) - after[k] for k in before}
  out['after'] = after
  del agent, step, u
  torch.cuda.empty_cache()
  return out


def _shape_views(x, gpu):
  """The reference's activations in the form of the GPU's views: z, or z x (GPU mask) for a post-ReLU view."""
  return {k: x['acts'][k] * gpu['masks'][k] if gpu['post'][k] else x['acts'][k] for k in gpu['views']}


def _stages(x, ref, gpu):
  """{stage: error of x against ref}; x is a reference result or the GPU's."""
  e = dict(logits=_relmax(x['logits'], ref['logits']), baseline=_relmax(x['baseline'], ref['baseline']),
           loss=abs(x['total'] - ref['total']) / abs(ref['total']))
  for k in ref['logs']:
    e['log ' + k] = abs(x['logs'][k] - ref['logs'][k]) / max(abs(ref['logs'][k]), 1e-30)
  e['dlogits'] = _relmax(x['dlogits'], ref['dlogits'])
  e['dbaseline'] = _relmax(x['dbaseline'], ref['dbaseline'])
  xv = x['views'] if 'views' in x else _shape_views(x, gpu)
  rv = _shape_views(ref, gpu)
  for k in rv:
    e['act ' + k] = _relmax(xv[k], rv[k])
  for k in ref['grads']:
    if k != 'entropy_cost_param':
      e['grad ' + k] = _relmax(x['grads'][k], ref['grads'][k])
  for k in ref['update']:
    d = np.abs(x['update'][k] - ref['update'][k])
    if 'after' in x:     # the GPU's parameters are stored in fp32: half an ulp of each is rounding, not error
      d = np.maximum(d - 0.5 * np.spacing(np.abs(x['after'][k])), 0.0)
    e['adam ' + k] = float(d.max() / (np.abs(ref['update'][k]).max() + 1e-30))
  return e


def _run(mode):
  """The GPU step of `mode` against the float64 reference under its decisions: stage errors, measures and the
  near-tie report (cached per module; the large arrays are dropped)."""
  if mode in _cache:
    return _cache[mode]
  net, conv_mode, lstm_mode = MODES[mode]
  params, b, cfg = _problem(net)
  gpu = _gpu_step(net, conv_mode, lstm_mode)
  cond = dict(masks=gpu['masks'], taps=gpu['taps'])
  ref = RF.step(net, params, b, cfg, torch.float64, **cond)
  errs = _stages(gpu, ref, gpu)
  m = _stages(RF.step(net, params, b, cfg, torch.float32, **cond), ref, gpu)
  resp = {}
  if conv_mode != 'simt':
    deltas = (2.0 ** -24, 2.0 ** -20, DELTA) if mode == 'deep-tc3p' else (DELTA,)
    for d in deltas:
      resp[d] = _stages(RF.step(net, *RF.perturbed(params, b, d), cfg, torch.float64, **cond), ref, gpu)
    m = {k: max(m[k], resp[DELTA][k]) for k in m}
  bars = {k: max(FLOOR, C * m[k]) for k in m}
  # near-ties: where the GPU decided otherwise than the float64 reference would, in units of the layer's bar
  ties = {}
  rv = _shape_views(ref, gpu)
  for k, v in ref['ties'].items():
    stage = 'act ' + (k.replace('pool', 'p'))
    scale = np.abs(rv[stage[4:]]).max()
    ties[k] = (v.size, float(v.max() / scale) if v.size else 0.0, bars[stage])
  _cache[mode] = (errs, m, bars, ties, resp)
  return _cache[mode]


@pytest.mark.parametrize('mode', list(MODES))
def test_vtrace_step_matches_float64_under_its_own_decisions(mode):
  errs, _, bars, ties, _ = _run(mode)
  print('VTRACE FLOAT64 %s (T=%d B=%d, C = %g, floor %.0e, m = %s): error / bar' %
        (mode, T, B, C, FLOOR, 'float32 reference' if mode.endswith('simt') else
         'max(float32 reference, 2^-16 response)'))
  bad = []
  for k in errs:
    print('  %-48s %.2e / %.2e' % (k, errs[k], bars[k]))
    if not errs[k] <= bars[k]:
      bad.append((k, errs[k], bars[k]))
  print('  decisions the GPU made otherwise than float64: count, worst distance to the tie / the layer bar')
  for k, (n, worst, bar) in ties.items():
    print('  %-48s %6d  %.2e / %.2e' % (k, n, worst, bar))
    if not worst <= bar:
      bad.append(('decision ' + k, n, worst, bar))
  assert not bad, bad


def test_conditioned_reference_is_linear_in_the_perturbation():
  """Under the 'tc3p' step's decisions the float64 reference's response grows 16x per 16x of perturbation, in every
  stage: no decision is left unshared, so the bf16x3 bars measure arithmetic.  The Adam updates are fp32
  (optim_oracle.keras_adam_step), below the resolution of a 2^-24 response, and are checked from 2^-20; an update
  whose 2^-16 response stays within 8 fp32 ulps is saturated (lr_t sign(g) with beta_1 = 0) and is skipped.  Stages
  the perturbation does not reach (the kl terms with kl_cost = 0, the entropy cost and its update) respond with 0."""
  _, _, _, _, resp = _run('deep-tc3p')
  d24, d20, d16 = sorted(resp)
  print('VTRACE FLOAT64 conditioned response at 2^-24 / 2^-20 / 2^-16')
  bad = []
  for k in resp[d16]:
    r = (resp[d24][k], resp[d20][k], resp[d16][k])
    print('  %-48s %.2e %.2e %.2e' % ((k,) + r))
    if r == (0.0, 0.0, 0.0) and ('kl' in k or 'entropy_cost' in k):
      continue
    if k.startswith('adam ') and r[2] < 8 * 2.0 ** -23:
      continue        # every element's |g| >> eps / sqrt(1 - beta_2): the update is lr_t sign(g) to fp32 rounding
    first = 1 if k.startswith('adam ') else 0
    if not all(8 <= r[i + 1] / max(r[i], 1e-300) <= 32 for i in range(first, 2)):
      bad.append((k, r))
  assert not bad, bad
