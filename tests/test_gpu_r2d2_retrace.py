"""GPU: the opt-in Retrace(lambda) loss of the R2D2 learner (seedrl_r2d2_retrace_loss_fwd_bwd) against the
float64 oracle of tests/retrace_oracle.py, which tests/test_r2d2_retrace.py pins to the reference's own
n-step targets in their two reductions.

  * the kernel at (T, B, A) = (16, 6, 18), (101, 64, 18), (4, 2, 3) for lambda in {0, 0.95, 1} and Q values of
    scale 1 and 1e-3, to rtol 2e-5 (loss, priorities) and 2e-4 (dq) and within the per-sequence float64 bars of
    test_gpu_r2d2_loss_float64.py; lambda = 0 bit-equal to the n-step kernel at n_steps = 1; repeat launches bit-identical; bad arguments
    refused with nothing launched;
  * one learner step with bellman_target='retrace' at the `bench.py --agent r2d2` shape against
    CpuR2D2Learner, with the tolerance rule of test_gpu_fullsize_r2d2.py;
  * R2D2InferenceHost under 'retrace' hands the replay the initial priorities the oracle computes, within the
    float64 bar of test_gpu_r2d2_loss_float64.py.
"""
import math

import numpy as np
import pytest
import torch

import retrace_oracle as RO
import test_gpu_r2d2_loss_float64 as LF
from oracle import optim_oracle

pytestmark = pytest.mark.gpu

c = lambda a: torch.as_tensor(np.asarray(a)).cuda()


def _inputs(T, B, A, seed, p_greedy=0.7, q=1.0):
  """q: the scale of the Q values."""
  rng = np.random.default_rng(seed)
  tq = (rng.normal(size=(T, B, A)) * q).astype(np.float32)
  gq = (rng.normal(size=(T, B, A)) * 3 * q).astype(np.float32)
  ra = np.where(rng.random((T, B)) < p_greedy, tq.argmax(-1), rng.integers(0, A, (T, B))).astype(np.int64)
  r = rng.normal(size=(T, B)).astype(np.float32)
  d = rng.random((T, B)) < 0.1
  w = (rng.random(B) + 0.1).astype(np.float32)
  return tq, gq, ra, r, d, w


def _loss(tq, gq, ra, r, d, w, **kw):
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  env = utils.EnvOutput(c(r), c(d), None, None, None)
  out = learner.compute_loss_and_priorities_from_agent_outputs(
      learner.AgentOutput(None, c(tq)), learner.AgentOutput(None, c(gq)), env, learner.AgentOutput(c(ra), None),
      0.997, importance_weights=c(w), **kw)
  return [x.cpu().numpy() for x in out]


@pytest.mark.parametrize('q', [1.0, 1e-3])
@pytest.mark.parametrize('lam', [0.0, 0.95, 1.0])
@pytest.mark.parametrize('T,B,A', [(16, 6, 18), (101, 64, 18), (4, 2, 3)])
def test_retrace_loss_vs_float64(T, B, A, lam, q):
  tq, gq, ra, r, d, w = _inputs(T, B, A, seed=T + A, q=q)
  loss, prio, dq = _loss(tq, gq, ra, r, d, w, bellman_target='retrace', retrace_lambda=lam)
  want_loss, want_prio, _, want_dq = RO.loss_and_priorities(tq, gq, ra, r, d, 0.997, lam, importance_weights=w)
  np.testing.assert_allclose(loss, want_loss, rtol=2e-5, atol=1e-6 * q)
  np.testing.assert_allclose(prio, want_prio, rtol=2e-5, atol=1e-6 * q)
  np.testing.assert_allclose(dq, want_dq, rtol=2e-4, atol=1e-6 * q)
  LF.check_outputs(dict(loss=loss, priorities=prio, dq=dq), (tq, gq, ra, r, d, w), 'retrace', lam, 0.997, 0.9, 1e-3)
  if lam == 0.0:
    for got, want in zip((loss, prio, dq), _loss(tq, gq, ra, r, d, w, n_steps=1)):
      np.testing.assert_array_equal(got, want)
  # repeat launches are bit-identical
  for got, again in zip((loss, prio, dq), _loss(tq, gq, ra, r, d, w, bellman_target='retrace', retrace_lambda=lam)):
    np.testing.assert_array_equal(got, again)


def test_retrace_loss_refuses_bad_arguments_without_launch():
  from seed_rl_b200 import _lib
  L = _lib.lib()
  T, B, A = 8, 4, 5
  tq, gq, ra, r, d, w = (c(x) for x in _inputs(T, B, A, seed=1))
  d8 = d.to(torch.uint8)
  loss, prio, dq = torch.zeros(B).cuda(), torch.zeros(B).cuda(), torch.full((T, B, A), 7.).cuda()
  scratch = torch.zeros(int(L.seedrl_r2d2_retrace_loss_scratch_bytes(T, B)), dtype=torch.uint8).cuda()
  ins = [tq, gq, ra, r, d8, w]
  outs = [loss, prio, dq, scratch]

  def call(T=T, lam=0.5, null=None):
    p = [None if i == null else _lib.ptr(x) for i, x in enumerate(ins + outs)]
    return L.seedrl_r2d2_retrace_loss_fwd_bwd(T, B, A, *p[:6], 0.997, lam, 0.9, 1e-3, *p[6:], _lib.stream_ptr())
  torch.cuda.synchronize()
  n0 = _lib.launch_count()
  for kw in (dict(T=1), dict(lam=-1e-3), dict(lam=1.5), dict(lam=math.nan), dict(null=0), dict(null=1),
             dict(null=2), dict(null=3), dict(null=4), dict(null=6), dict(null=7), dict(null=8), dict(null=9)):
    assert call(**kw) == 3, kw
  torch.cuda.synchronize()
  assert _lib.launch_count() == n0
  assert float(dq.min()) == 7. and float(loss.abs().max()) == 0.
  assert call() == 0 and _lib.launch_count() == n0 + 1
  torch.cuda.synchronize()


# ---- one learner step at the bench.py --agent r2d2 shape ----------------------------------------------------
R_A, R_OBS, R_S, R_B = 18, (84, 84, 1), 4, 64
R_LR, R_EPS = 0.00048, 1e-3
R_TOL = {'simt': 2e-3, 'tc3': 6e-3}
SENS_MULT = 4
_cache = {}


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _oracle_step(st):
  if 'r2d2' in _cache:
    return _cache['r2d2']
  from oracle import r2d2_learner_oracle as RL, r2d2_net_oracle as NO
  T = st.burn_in + st.unroll_length + 1
  params = NO.init_params(R_A, R_OBS, R_S, seed=5)
  tparams = NO.init_params(R_A, R_OBS, R_S, seed=6)
  b = RL.synthetic_replay_batch(T, R_B, R_A, R_OBS, seed=21, done_p=0.01)
  kw = dict(gamma=st.discounting, burn_in=st.burn_in, n_steps=st.n_steps, clip_norm=st.clip_norm, lr=R_LR, eps=R_EPS,
            target_params=tparams, bellman_target='retrace', retrace_lambda=st.retrace_lambda)
  # the replayed actions: greedy in the online network on most rows, so that traces run over several rows
  cpu = RO.CpuR2D2Learner(R_A, R_OBS, R_S, params=params, **kw)
  with torch.no_grad():        # the online Q values do not depend on the replayed actions
    greedy = RO.compute_loss_and_priorities(cpu.params, cpu.target, b, R_A, R_S, st.discounting, st.burn_in,
                                            bellman_target='retrace')[2]['q'].numpy().argmax(-1)
  rng = np.random.default_rng(3)
  suf = b['action'][st.burn_in:]
  b['action'][st.burn_in:] = np.where(rng.random(suf.shape) < 0.8, greedy, suf).astype(np.int32)
  total, _, prio, g, norm, _ = cpu.grads(b)
  prng = np.random.default_rng(0)
  pert = RO.CpuR2D2Learner(R_A, R_OBS, R_S, params={k: (v * (1 + 1e-6 * prng.normal(size=v.shape))).astype(np.float32)
                                                    for k, v in params.items()}, **kw)
  g2 = pert.grads(b)[3]
  sens = {k: _relmax(g2[k], g[k]) for k in g}
  _cache['r2d2'] = (params, tparams, b, total, prio, g, norm, sens, float((b['action'][st.burn_in:] == greedy).mean()))
  return _cache['r2d2']


@pytest.mark.parametrize('mode', ['simt', 'tc3'])
def test_retrace_learner_step_B64_matches_oracle(mode):
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils
  st = learner.default_settings(bellman_target='retrace')
  params, tparams, b, total, prio, g, norm, sens, frac_greedy = _oracle_step(st)
  T, B = b['reward'].shape
  agent = networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, gemm_mode=mode); agent.load_named_parameters(params)
  target = networks.DuelingLSTMDQNNet(R_A, R_OBS, R_S, gemm_mode=mode); target.load_named_parameters(tparams)
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(R_LR, epsilon=R_EPS), settings=st)
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']), torch.zeros(T, B, dtype=torch.bool).cuda(),
                        torch.zeros(T, B, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']))
  unrolls = learner.Unroll(state, None, c(b['prev_actions']), env, learner.AgentOutput(c(b['action']), None))
  sampled = learner.SampledUnrolls(unrolls, c(b['indices']), c(b['importance_weights']))
  loss, priorities, _, gnorm = step.compute_gradients(sampled)
  agent.check_errors(); target.check_errors()
  e_loss = abs(float(loss) - total) / max(1.0, abs(total))
  e_prio = _relmax(priorities.cpu().numpy(), prio)
  e_norm = abs(float(gnorm) - norm) / norm
  scale = np.float32(st.clip_norm / max(norm, st.clip_norm))
  mine = agent.named_gradients()
  assert len(mine) == 18 and set(mine) == set(g)
  errs = {k: _relmax(mine[k].cpu().numpy(), g[k] * scale) for k in g}
  bars = {k: max(R_TOL[mode], SENS_MULT * sens[k]) for k in g}
  print('RETRACE R2D2 %s T=%d B=%d lambda=%.2f (%.0f%% greedy rows): loss %.6f vs %.6f (%.1e); priorities %.1e; '
        'norm %.4f vs %.4f (%.1e)' % (mode, T, B, st.retrace_lambda, 100 * frac_greedy, float(loss), total, e_loss,
                                      e_prio, float(gnorm), norm, e_norm))
  for k in g:
    print('  %-28s %.2e  (bar %.1e)' % (k, errs[k], bars[k]))
  assert e_loss < 1e-3 and e_prio < 2e-3 and e_norm < 5e-3, (e_loss, e_prio, e_norm)
  assert not [k for k in g if not errs[k] <= bars[k]], errs
  before = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  step.apply_gradients()
  after = {k: v.cpu().numpy() for k, v in agent.named_parameters().items()}
  lr_t = R_LR * np.sqrt(1 - 0.999) / (1 - 0.9)
  for k in g:
    z = np.zeros_like(before[k])
    own = optim_oracle.keras_adam_step(before[k], mine[k].cpu().numpy(), z, z, 0, R_LR, eps=R_EPS)[0]
    np.testing.assert_allclose(after[k], own, rtol=0, atol=1e-3 * lr_t * 3.2 + 1e-7 * np.abs(before[k]).max(),
                               err_msg=k)
    ref = optim_oracle.keras_adam_step(before[k], g[k] * scale, z, z, 0, R_LR, eps=R_EPS)[0]
    gerr = float(np.abs(mine[k].cpu().numpy() - g[k] * scale).max())
    d = float(np.abs(after[k] - ref).max())
    assert d <= 1.01 * 0.1 * lr_t / R_EPS * gerr + 1e-7 * np.abs(before[k]).max() + 1e-9, (k, d, gerr)
  del agent, target, step, sampled, unrolls, env, state, mine
  torch.cuda.empty_cache()


def test_retrace_inference_host_initial_priorities():
  """R2D2InferenceHost with bellman_target='retrace': the initial priority of every completed unroll is the
  oracle's, from the behaviour Q values of its suffix (the same values as online and target)."""
  from seed_rl_b200.agents.r2d2 import learner, learner_loop
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import utils
  A, obs, S = 6, (36, 36, 1), 4
  st = learner.default_settings(batch_size=6, unroll_length=6, burn_in=2, bellman_target='retrace',
                                retrace_lambda=0.9)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=1, gemm_mode='simt')
  host = learner_loop.R2D2InferenceHost(agent, num_envs=6, num_eval_envs=1, inference_batch_size=3,
                                        observation_shape=obs, settings=st,
                                        generator=torch.Generator(device='cuda').manual_seed(0))
  rng = np.random.default_rng(0)
  run_ids = rng.integers(1, 2**40, 6)
  for step_i in range(19):
    for ids in (np.array([0, 1, 2], np.int32), np.array([5, 3, 4], np.int32)):
      n = len(ids)
      env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), rng.random(n) < 0.15,
                            rng.integers(0, 256, (n,) + obs, dtype=np.uint8), np.zeros(n, bool),
                            np.full(n, step_i, np.int32))
      host.inference(ids, run_ids[ids], env, np.zeros(n, np.float32))
  torch.cuda.synchronize()
  n = host.unroll_queue.size()
  assert n >= 10
  greedy_rows = 0
  for _ in range(n):
    u = host.unroll_queue.dequeue()
    q = u.agent_outputs.q_values[st.burn_in:].cpu().numpy()[:, None]
    a = u.agent_outputs.action[st.burn_in:].cpu().numpy()[:, None].astype(np.int64)
    greedy_rows += int((a == q.argmax(-1)).sum())
    r, d = (x[st.burn_in:].cpu().numpy()[:, None] for x in (u.env_outputs.reward, u.env_outputs.done))
    _, prio, _, _ = RO.loss_and_priorities(q, q, a, r, d, st.discounting, st.retrace_lambda)
    np.testing.assert_allclose(float(u.priority), float(prio[0]), rtol=1e-4, atol=1e-6)
    # and within the float64 bar of test_gpu_r2d2_loss_float64.py
    LF.check_outputs(dict(priorities=np.array([float(u.priority)])), (q, q, a, r, d, None), 'retrace',
                     st.retrace_lambda, st.discounting, 0.9, st.value_function_rescaling_epsilon)
  assert greedy_rows > 0
