"""GPU: the tensor-core LSTM recurrence, lstm_mode 'tc3' (csrc/lstm_tc.cu).  It computes the recurrent
products h[t-1] U and dZ[t+1] U^T on wgmma in bf16x3 (hi*hi + lo*hi + hi*lo, fp32 accumulation) and is
otherwise the tiled recurrence (lstm_mode 'tiled'): same cell, done-resets and workspace.

  * parity with 'tiled' on the same parameters and inputs, random (h0, c0) and resets inside the unroll:
    ImpalaShallow (LSTM(256)) and DuelingLSTMDQNNet (LSTM(512)), forward and backward.  Bars: outputs and
    final (h, c) within 2e-4 of their max-abs (bf16x3 is ~2^-16 relative per product), the whole gradient
    arena within 1e-3 relative L2;
  * full-size learner steps with the 'tc3' recurrence against the CPU oracle, under the rules of
    test_gpu_fullsize.py / test_gpu_fullsize_r2d2.py for the step's conv / GEMM mode;
  * bit-identical repeats; the InferenceHost CUDA-graph path; switching modes on a live agent.
"""
import threading
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

A, OBS = 18, (84, 84, 4)
R_A, R_OBS, R_S = 6, (36, 36, 1), 4


def _relmax(x, y):
  x = x.double(); y = y.double()
  return float((x - y).abs().max() / (y.abs().max() + 1e-30))


def _rel_l2(x, y):
  x = x.double(); y = y.double()
  return float((x - y).norm() / (y.norm() + 1e-30))


def _impala_batch(T, B):
  from oracle import learner_oracle
  from test_gpu_parity import _batch_to_cuda
  b = learner_oracle.synthetic_batch(T, B, A, seed=5)
  b['done'][min(1, T), 0] = True
  if T >= 3:
    b['done'][T - 1, B // 2] = True
  rng = np.random.default_rng(1)
  b['h0'] = rng.normal(size=b['h0'].shape).astype(np.float32)
  b['c0'] = rng.normal(size=b['c0'].shape).astype(np.float32)
  return _batch_to_cuda(b)


def _impala_run(agent, u):
  """forward (learner outputs, final state) + the V-trace step's backward: (logits, h, c, loss, grads)"""
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  step = learner.LearnerStep(agent, optimizers.Adam(1e-3))
  out, (h, c) = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
  loss, _ = step.compute_gradients(u)
  agent.check_errors()
  return out.policy_logits.clone(), h.clone(), c.clone(), float(loss), agent.grads.clone()


def _r2d2_inputs(T, B):
  from oracle import r2d2_learner_oracle as RL
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import utils
  b = RL.synthetic_replay_batch(T, B, R_A, R_OBS, seed=B, done_p=0.2)
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']),
                        torch.zeros(T, B, dtype=torch.bool).cuda(), torch.zeros(T, B, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
  dq = torch.randn(T, B, R_A, device='cuda', generator=torch.Generator(device='cuda').manual_seed(2))
  return (c(b['prev_actions']), env), state, dq


def _r2d2_run(agent, inputs):
  x, state, dq = inputs
  out, st = agent(x, state, unroll=True, is_training=True)
  agent.backward(dq)
  agent.check_errors()
  return out.q_values.clone(), st.core_state[0].clone(), st.core_state[1].clone(), agent.grads.clone()


# ---- 1. parity with the tiled recurrence -----------------------------------------------------------------
@pytest.mark.parametrize('T,B', [(6, 5), (3, 70), (1, 3), (20, 64), (5, 256), (4, 300)])
def test_impala_tc3_recurrence_matches_tiled(T, B):
  from seed_rl_b200.dmlab import networks
  u = _impala_batch(T, B)
  res = {m: _impala_run(networks.ImpalaShallow(A, OBS, seed=2, lstm_mode=m), u) for m in ('tiled', 'tc3')}
  a, p = res['tiled'], res['tc3']
  for i, name in enumerate(('logits', 'h', 'c')):
    assert _relmax(p[i], a[i]) <= 2e-4, (name, _relmax(p[i], a[i]))
  assert abs(p[3] - a[3]) <= 2e-4 * max(1.0, abs(a[3])), (p[3], a[3])
  assert _rel_l2(p[4], a[4]) <= 1e-3, _rel_l2(p[4], a[4])


@pytest.mark.parametrize('T,B', [(5, 40), (3, 64), (4, 9), (2, 100)])
def test_r2d2_tc3_recurrence_matches_tiled(T, B):
  from seed_rl_b200.atari import networks
  inputs = _r2d2_inputs(T, B)
  res = {m: _r2d2_run(networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, seed=11, lstm_mode=m), inputs)
         for m in ('tiled', 'tc3')}
  a, p = res['tiled'], res['tc3']
  for i, name in enumerate(('q_values', 'h', 'c')):
    assert _relmax(p[i], a[i]) <= 2e-4, (name, _relmax(p[i], a[i]))
  assert _rel_l2(p[3], a[3]) <= 1e-3, _rel_l2(p[3], a[3])


# ---- 2. full size against the CPU oracle -----------------------------------------------------------------
def test_impala_tc3p_step_T20_B64_with_tc3_recurrence_matches_oracle():
  """test_gpu_fullsize.py's learner step in conv mode 'tc3p' with the recurrence on the tensor cores:
  loss, learner outputs and all 39 gradient tensors under that file's rule for 'tc3p'."""
  import test_gpu_fullsize as F
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda
  params, b, total, logits, baseline, g, sens = F._oracle_step(20, 64)
  agent = networks.ImpalaDeep(A, OBS, conv_mode='tc3p', lstm_mode='tc3')
  agent.load_named_parameters(params)
  step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                             settings=learner.default_loss_settings())
  u = _batch_to_cuda(b)
  loss, _ = step.compute_gradients(u)
  agent.check_errors()
  assert abs(float(loss) - total) < 2e-4 * max(1.0, abs(total)), (float(loss), total)
  lo, _ = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
  e_log = F._relmax(lo.policy_logits.cpu().numpy(), logits)
  e_base = F._relmax(lo.baseline.cpu().numpy(), baseline)
  mine = agent.named_gradients()
  errs, bad = {}, []
  for k in g:
    if k == 'entropy_cost_param':
      continue
    errs[k] = F._relmax(mine[k].cpu().numpy(), g[k])
    tol = max(F.GRAD_TOL['tc3p'], F.SENS_MULT['tc3p'] * sens[k])
    if not errs[k] <= tol:
      bad.append((k, errs[k], tol))
  worst = max(errs, key=errs.get)
  print('FULLSIZE tc3p + lstm tc3 T=20 B=64: loss %.6f vs %.6f; logits %.2e baseline %.2e; worst grad %s %.2e'
        % (float(loss), total, e_log, e_base, worst, errs[worst]))
  assert e_log < 2e-4 and e_base < 2e-4, (e_log, e_base)
  assert len(errs) == 39
  assert not bad, bad


def test_r2d2_step_B64_with_tc3_recurrence_matches_oracle():
  """test_gpu_fullsize_r2d2.py's learner step (B = 64, 141 rows) with the recurrence on the tensor cores:
  loss, priorities, gradients under that file's 'tc3' rule, parameters after one Adam step.

  Two tensors do not meet that rule and are held to 1e-2 instead: the advantage stream's hidden layer
  (kernel 6.4e-3, bias 6.7e-3 measured on an H100; 1.3e-3 with the fp32 recurrence, oracle 1e-6 response
  1.6e-4).  The cause is the step's kinks, not arithmetic: the fp32 oracle makes its own ReLU decisions, and
  units that sit within rounding of zero take the other side in the oracle than on the GPU.  Perturbing every
  parameter by 2^-16 moves the float64 gradient of this tensor by 8.7e-3 with the decisions free, and by 5.2e-5
  with them held.  test_gpu_r2d2_float64.py runs this same step against a float64 reference that shares the
  GPU's ReLU masks and greedy actions: there advantage/hidden/kernel is 3.9e-5 and the bias 2.0e-5 off, against
  bars of 4.1e-4 and 2.8e-4.  This test keeps pinning the wiring to the oracle; that one pins the precision.
  Every other tensor meets max(6e-3, 4x the oracle's response)."""
  import test_gpu_fullsize_r2d2 as F
  from oracle import optim_oracle
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils
  st, params, tparams, b, total, prio, g, norm, sens = F._r2d2_oracle()
  T, B = b['reward'].shape
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  agent = networks.DuelingLSTMDQNNet(F.R_A, F.R_OBS, F.R_S, lstm_mode='tc3'); agent.load_named_parameters(params)
  target = networks.DuelingLSTMDQNNet(F.R_A, F.R_OBS, F.R_S, lstm_mode='tc3'); target.load_named_parameters(tparams)
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(F.R_LR, epsilon=F.R_EPS), settings=st)
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']), torch.zeros(T, B, dtype=torch.bool).cuda(),
                        torch.zeros(T, B, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
  unrolls = learner.Unroll(state, None, c(b['prev_actions']), env, learner.AgentOutput(c(b['action']), None))
  sampled = learner.SampledUnrolls(unrolls, c(b['indices']), c(b['importance_weights']))
  loss, priorities, _, gnorm = step.compute_gradients(sampled)
  agent.check_errors(); target.check_errors()
  e_loss = abs(float(loss) - total) / max(1.0, abs(total))
  e_prio = F._relmax(priorities.cpu().numpy(), prio)
  e_norm = abs(float(gnorm) - norm) / norm
  scale = np.float32(st.clip_norm / max(norm, st.clip_norm))
  mine = agent.named_gradients()
  bad = []
  print('FULLSIZE R2D2 lstm tc3 T=%d B=%d: loss %.1e priorities %.1e norm %.1e' % (T, B, e_loss, e_prio, e_norm))
  for k in g:
    err = F._relmax(mine[k].cpu().numpy(), g[k] * scale)
    tol = max(F.R_TOL['tc3'], F.SENS_MULT * sens[k], 1e-2 if k.startswith('advantage/hidden/') else 0.0)
    print('  %-28s %.2e  (bar %.1e, oracle 1e-6 response %.1e)' % (k, err, tol, sens[k]))
    if not err <= tol:
      bad.append((k, err, tol))
  assert e_loss < 1e-3 and e_prio < 2e-3 and e_norm < 5e-3, (e_loss, e_prio, e_norm)
  assert not bad, bad
  # one Adam step moves each parameter at most lr_t / eps per unit of gradient error away from the oracle's
  before = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  step.apply_gradients()
  after = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  lr_t = F.R_LR * np.sqrt(1 - 0.999) / (1 - 0.9)
  for k in g:
    z = np.zeros_like(before[k])
    ref = optim_oracle.keras_adam_step(before[k], g[k] * scale, z, z, 0, F.R_LR, eps=F.R_EPS)[0]
    gerr = float(np.abs(mine[k].cpu().numpy() - g[k] * scale).max())
    d = float(np.abs(after[k] - ref).max())
    assert d <= 1.01 * 0.1 * lr_t / F.R_EPS * gerr + 1e-7 * np.abs(before[k]).max() + 1e-9, (k, d, gerr)
  del agent, target, step, sampled, unrolls, env, state, mine
  torch.cuda.empty_cache()


# ---- 3. determinism --------------------------------------------------------------------------------------
@pytest.mark.parametrize('net,T,B', [('impala', 5, 64), ('impala', 5, 70), ('r2d2', 4, 64), ('r2d2', 4, 9)])
def test_tc3_recurrence_is_bit_reproducible(net, T, B):
  if net == 'impala':
    from seed_rl_b200.dmlab import networks
    agent, inputs, run = networks.ImpalaShallow(A, OBS, seed=2, lstm_mode='tc3'), _impala_batch(T, B), _impala_run
  else:
    from seed_rl_b200.atari import networks
    agent, inputs, run = (networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, seed=11, lstm_mode='tc3'), _r2d2_inputs(T, B),
                          _r2d2_run)
  r0, r1 = run(agent, inputs), run(agent, inputs)
  for x, y in zip(r0, r1):
    if isinstance(x, float):
      assert x == y
    else:
      assert torch.equal(x, y)


# ---- 4. the InferenceHost CUDA-graph path ----------------------------------------------------------------
def test_tc3_graph_inference_is_consistent_with_training_unroll():
  """Full inference batches on the host's CUDA-graph path (T1 = 1) with an assembler, ImpalaDeep in mode
  'tc3': every assembled batch replayed through the training unroll (mode 'tc3') from its stored first
  state reproduces the logits and baselines stored at inference time."""
  from seed_rl_b200.agents.vtrace import learner_loop
  from seed_rl_b200.common import utils
  from seed_rl_b200.dmlab import networks
  from test_gpu_inference import _env_batch
  num_envs, T, N, B = 6, 3, 3, 4
  agent = networks.ImpalaDeep(A, OBS, seed=3, lstm_mode='tc3')
  host = learner_loop.InferenceHost(agent, num_envs, T, N, OBS, training_batch_size=B)
  assert host.use_graph
  batches = []

  def learner_thread():
    try:
      while True:
        slot, u = learner_loop.assembled_batch(host.assembler)
        batches.append(utils.map_structure(lambda t: t.clone(), tuple(u)))
        host.assembler.release(slot)
    except utils.QueueClosedError:
      return
  th = threading.Thread(target=learner_thread); th.start()
  rng = np.random.default_rng(0)
  run_ids = rng.integers(1, 2**40, num_envs)
  for step in range(9):
    for ids in (np.array([0, 1, 2], np.int32), np.array([5, 3, 4], np.int32)):
      host.inference(ids, run_ids[ids], _env_batch(rng, ids, step), np.zeros(len(ids), np.float32))
  torch.cuda.synchronize()
  assert host._graph is not None
  for _ in range(100):
    if len(batches) == 3:
      break
    time.sleep(0.05)
  host.assembler.close(); th.join(10)
  assert len(batches) == 3                     # 12 completed unrolls of 4 + 1 rows
  for bt in batches:
    u = learner_loop.Unroll(*bt)
    out, _ = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
    np.testing.assert_allclose(out.policy_logits.cpu().numpy(), u.agent_outputs.policy_logits.cpu().numpy(),
                               rtol=2e-4, atol=2e-5)
    np.testing.assert_allclose(out.baseline.cpu().numpy(), u.agent_outputs.baseline.cpu().numpy(),
                               rtol=2e-4, atol=2e-5)
  agent.check_errors()


# ---- 5. switching modes, errors --------------------------------------------------------------------------
def test_impala_switch_tiled_tc3_tiled_on_live_agent():
  from seed_rl_b200 import _lib
  from seed_rl_b200.dmlab import networks
  u = _impala_batch(4, 70)
  agent = networks.ImpalaShallow(A, OBS, seed=2)
  res = []
  for mode in (2, 3, 2):
    _lib.check(_lib.lib().seedrl_net_set_lstm_mode(agent._h, mode))
    res.append(_impala_run(agent, u))
  for x, y in zip(res[0], res[2]):
    assert x == y if isinstance(x, float) else torch.equal(x, y)
  assert not torch.equal(res[0][0], res[1][0])         # mode 3 did run its own arithmetic
  assert _relmax(res[1][0], res[0][0]) <= 2e-4


def test_r2d2_switch_tiled_tc3_tiled_on_live_agent():
  from seed_rl_b200 import _lib
  from seed_rl_b200.atari import networks
  inputs = _r2d2_inputs(3, 40)
  agent = networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, seed=11)
  res = []
  for mode in (2, 3, 2):
    _lib.check(_lib.lib().seedrl_r2d2_net_set_lstm_mode(agent._h, mode))
    res.append(_r2d2_run(agent, inputs))
  for x, y in zip(res[0], res[2]):
    assert torch.equal(x, y)
  assert _relmax(res[1][0], res[0][0]) <= 2e-4


def test_unknown_lstm_modes_are_rejected():
  from seed_rl_b200 import _lib
  from seed_rl_b200.atari import networks as atari_networks
  from seed_rl_b200.dmlab import networks
  with pytest.raises(ValueError, match='tc3'):
    networks.ImpalaShallow(A, OBS, lstm_mode='tc')
  with pytest.raises(ValueError, match='tc3'):
    atari_networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, lstm_mode='stepwise')
  with pytest.raises(ValueError, match='tc3'):
    networks.ImpalaShallow(A, OBS, lstm_mode='stepwise')
  with pytest.raises(ValueError, match='tc3'):
    networks.ImpalaShallow(A, OBS, lstm_mode='persistent')
  with pytest.raises(ValueError, match='tc3'):
    atari_networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, lstm_mode='persistent')
  agent = networks.ImpalaShallow(A, OBS, lstm_mode='tc3')
  assert _lib.lib().seedrl_net_set_lstm_mode(agent._h, 4) != 0
  r2d2 = atari_networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, lstm_mode='tc3')
  assert _lib.lib().seedrl_r2d2_net_set_lstm_mode(r2d2._h, 0) != 0
  for mode in (0, 1):                  # only 2 (tiled) and 3 (tc3) exist
    assert _lib.lib().seedrl_net_set_lstm_mode(agent._h, mode) == 3        # SEEDRL_ERR_INVALID_ARGUMENT
    assert _lib.lib().seedrl_r2d2_net_set_lstm_mode(r2d2._h, mode) == 3
  assert r2d2.lstm_mode == 'tc3' and agent.lstm_mode == 'tc3'
