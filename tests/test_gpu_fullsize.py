"""Network parity at the BASELINE sizes (VERDICT r1 "what's weak" #2): the CUDA learner step
against the CPU oracle (`oracle/learner_oracle.CpuLearner`, the restatement of reference
agents/vtrace/learner.py:73-159,255-280 + dmlab/networks.py:26-171) at

  * T=20, B=64  (BASELINE cfg 4's per-GPU slice / cfg 2 shape): loss, learner logits and
    baseline, and ALL 39 gradient tensors (+ entropy_cost_param);
  * T=20, B=256 (cfg 3): forward outputs and final LSTM state.

At these sizes the 512-position conv tiles wrap many frames, split-K runs all its splits, the
deferred weight-gradient partial buffer is full and the persistent LSTM runs all 21 grid
barriers -- the toy-size tests in test_gpu_parity.py exercise none of that.

Tolerances (stated, per mode):
  forward outputs   2e-4 of the tensor's max-abs (+2e-5 abs)
  loss              2e-4 relative
  gradients         per tensor max|a-w| / max|w| <= GRAD_TOL[mode], or 4x the oracle's own
                    sensitivity to a 1e-6 relative parameter perturbation where the step is
                    ill-conditioned (same rule as test_gpu_parity.py:476-496).

The oracle's OWN gradients (a CPU computation) move by up to 5.1e-3 (max-rel) under a 1e-6
relative parameter perturbation at this size -- the step is piecewise smooth (ReLU masks, max-pool
argmax, rho clipping) and a random-init net sits on many of the kinks.  bf16x3 ('tc3'/'tc3p') carries
~2^-16 relative rounding per product, so those modes are asserted at 5e-3 (or 4x sensitivity), not at
the fp32 path's 2e-3: that is what the arithmetic can meet, and it is stated rather than hidden.
'tc3p' additionally STORES every 16/32-channel activation and gradient as a bf16 hi+lo pair
(2^-17 = 7.6e-6 relative, i.e. 7.6x the 1e-6 probe perturbation the sensitivity is measured with),
so its bound is 8x the oracle's sensitivity (the oracle itself moves 2.1e-3 / 5.1e-3 under the probe
on the two most sensitive tensors).
"""
import numpy as np
import pytest
import torch

from oracle import learner_oracle, loss_oracle, net_oracle

pytestmark = pytest.mark.gpu

A = 18
OBS = (84, 84, 4)
# fp32 SIMT: summation order only.  tc3 / tc3p: bf16x3 split operands (~2^-16 per product).
GRAD_TOL = {'simt': 2e-3, 'tc3': 5e-3, 'tc3p': 5e-3}
SENS_MULT = {'simt': 4, 'tc3': 4, 'tc3p': 8}
MODES = ['simt', 'tc3', 'tc3p']

_cache = {}


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _oracle_step(T, B):
  """CPU oracle once per (T, B): loss, outputs, gradients and their sensitivity."""
  key = ('step', T, B)
  if key in _cache:
    return _cache[key]
  torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
  params = net_oracle.init_params('deep', A, OBS, seed=1)
  cfg = loss_oracle.default_config()
  cpu = learner_oracle.CpuLearner('deep', A, OBS, cfg, params=params)
  b = learner_oracle.synthetic_batch(T, B, A, OBS, seed=1234)
  total, _, g, aux = cpu.grads(b)
  logits = aux['logits'].detach().numpy().copy()
  baseline = aux['baseline'].detach().numpy().copy()
  # the oracle's own sensitivity to a 1e-6 relative parameter perturbation
  prng = np.random.default_rng(0)
  with torch.no_grad():
    for k, v in cpu.params.items():
      v.mul_(torch.as_tensor(1 + 1e-6 * prng.normal(size=tuple(v.shape)).astype(np.float32)))
  _, _, g_pert, _ = cpu.grads(b)
  sens = {k: _relmax(g_pert[k], g[k]) for k in g}
  _cache[key] = (params, b, float(total), logits, baseline, g, sens)
  return _cache[key]


def _agent(mode, params):
  from seed_rl_b200.dmlab import networks
  try:
    agent = networks.ImpalaDeep(A, OBS, conv_mode=mode)
  except ValueError:
    pytest.skip('conv_mode %s not built' % mode)
  agent.load_named_parameters(params)
  return agent


@pytest.mark.parametrize('mode', MODES)
def test_learner_step_T20_B64_matches_oracle(mode):
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from test_gpu_parity import _batch_to_cuda
  T, B = 20, 64
  params, b, total, logits, baseline, g, sens = _oracle_step(T, B)
  agent = _agent(mode, params)
  step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                             settings=learner.default_loss_settings())
  u = _batch_to_cuda(b)
  loss, _ = step.compute_gradients(u)
  agent.check_errors()
  out = agent._loss_grads
  assert abs(float(loss) - total) < 2e-4 * max(1.0, abs(total)), (float(loss), total)
  # learner outputs of the training forward
  lo, _ = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
  e_log = _relmax(lo.policy_logits.cpu().numpy(), logits)
  e_base = _relmax(lo.baseline.cpu().numpy(), baseline)
  mine = agent.named_gradients()
  errs, bad = {}, []
  for k in g:
    if k == 'entropy_cost_param':
      continue
    errs[k] = _relmax(mine[k].cpu().numpy(), g[k])
    tol = max(GRAD_TOL[mode], SENS_MULT[mode] * sens[k])
    if not errs[k] <= tol:
      bad.append((k, errs[k], tol))
  worst = max(errs, key=errs.get)
  print('FULLSIZE %s T=20 B=64: loss %.6f vs %.6f; logits %.2e baseline %.2e; worst grad %s %.2e '
        '(oracle 1e-6-perturbation sensitivity there %.2e; max sensitivity %.2e)' %
        (mode, float(loss), total, e_log, e_base, worst, errs[worst], sens[worst], max(sens.values())))
  assert e_log < 2e-4 and e_base < 2e-4, (e_log, e_base)
  assert len(errs) == 39
  assert not bad, bad
  np.testing.assert_allclose(float(mine['entropy_cost_param']), float(g['entropy_cost_param']),
                             rtol=1e-3, atol=1e-9)
  del out


def _oracle_forward(T, B):
  key = ('fwd', T, B)
  if key in _cache:
    return _cache[key]
  params = net_oracle.init_params('deep', A, OBS, seed=1)
  b = learner_oracle.synthetic_batch(T, B, A, OBS, seed=4321)
  rng = np.random.default_rng(5)
  b['h0'] = rng.normal(size=b['h0'].shape).astype(np.float32)
  b['c0'] = rng.normal(size=b['c0'].shape).astype(np.float32)
  pt = net_oracle.to_torch(params)
  with torch.no_grad():
    logits, baseline, (h, c) = net_oracle.unroll(
        'deep', pt, torch.as_tensor(b['prev_actions']), torch.as_tensor(b['reward']),
        torch.as_tensor(b['done']), torch.as_tensor(b['observation']),
        (torch.as_tensor(b['h0']), torch.as_tensor(b['c0'])), A)
  _cache[key] = (params, b, logits.numpy(), baseline.numpy(), h.numpy(), c.numpy())
  return _cache[key]


@pytest.mark.parametrize('mode', MODES)
def test_forward_T20_B256_matches_oracle(mode):
  """BASELINE cfg 3 shape: 5 376 frames per unroll batch (M = 5 376 rows through the GEMMs,
  ~10^8 tall-image positions through the first stack's convs)."""
  from test_gpu_parity import _batch_to_cuda
  T, B = 20, 256
  params, b, logits, baseline, h, c = _oracle_forward(T, B)
  agent = _agent(mode, params)
  u = _batch_to_cuda(b)
  out, (h2, c2) = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True, is_training=True)
  agent.check_errors()
  errs = dict(logits=_relmax(out.policy_logits.cpu().numpy(), logits),
              baseline=_relmax(out.baseline.cpu().numpy(), baseline),
              h=_relmax(h2.cpu().numpy(), h), c=_relmax(c2.cpu().numpy(), c))
  print('FULLSIZE %s T=20 B=256 forward: %s' % (mode, {k: '%.2e' % v for k, v in errs.items()}))
  assert max(errs.values()) < 2e-4, errs
  del agent
  torch.cuda.empty_cache()
