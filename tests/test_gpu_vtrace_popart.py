"""The V-trace learner's PopArt (--popart) on the GPU: seedrl_vtrace_popart_loss_fwd (both kernel forms) and
seedrl_vtrace_popart_update against the float64 composition of tests/popart_reference.py, the identity at
beta = 0, exact invariance under power-of-two reward scaling, the preserved predictions, and the learner step
(with Adam on the compensation, determinism and a checkpoint round trip).

Bars: error = max|gpu - ref64| / max|ref64| (relative difference for scalars); bar = max(1e-5, 8 m), m = the same
error of the float32 composition, so that a stage whose float32 arithmetic is itself ill-conditioned (the
mean of e V, a difference of return-sized numbers) is held to what float32 can do."""
import os

import numpy as np
import pytest
import torch

import popart_reference as PR
from seed_rl_b200 import _lib
from seed_rl_b200.agents.vtrace import learner

pytestmark = pytest.mark.gpu

T = 20


def _batch(B, A, seed, reward_scale=300.0, reward_offset=500.0):
  g = np.random.default_rng(seed)
  T1 = T + 1
  return dict(
      ll=(g.standard_normal((T1, B, A)) * 2).astype(np.float32),
      lb=(g.standard_normal((T1, B)) * 3).astype(np.float32),
      bl=(g.standard_normal((T1, B, A)) * 2).astype(np.float32),
      act=g.integers(0, A, (T1, B)).astype(np.int64),
      rew=(g.standard_normal((T1, B)) * reward_scale + reward_offset).astype(np.float32),
      done=g.random((T1, B)) < 0.05)


def _settings(beta=1e-2, **kw):
  return learner.default_loss_settings(popart=True, popart_beta=beta, **kw)


def _run(settings, b, state, stream=1, ecp=-0.8):
  """One phase 1 + phase 2 on the GPU -> (outputs dict of numpy, new state [4])."""
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  try:
    d = {k: torch.as_tensor(v).cuda() for k, v in b.items()}
    mom = torch.tensor(state[:2], dtype=torch.float32).cuda()
    comp = torch.tensor(state[2:], dtype=torch.float32).cuda()
    dcomp = torch.zeros(2, dtype=torch.float32).cuda()
    out = learner.popart_loss_fwd_bwd(settings, d['ll'], d['lb'], d['bl'], d['act'], d['rew'], d['done'],
                                      torch.tensor(ecp, dtype=torch.float32).cuda(), mom, comp, dcomp,
                                      want_vtrace=True)
    torch.cuda.synchronize()
  finally:
    _lib.lib().seedrl_debug_set_loss_stream(1)
  res = {k: v.cpu().numpy() for k, v in out.items() if v is not None}
  res['dcomp'] = dcomp.cpu().numpy()
  return res, np.concatenate([mom.cpu().numpy(), comp.cpu().numpy()])


def _err(x, ref):
  x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
  if ref.ndim == 0:
    return abs(float(x) - float(ref)) / max(abs(float(ref)), 1e-30)
  return float(np.abs(x - ref).max() / max(np.abs(ref).max(), 1e-30))


def _check(name, gpu, r64, r32):
  e, m = _err(gpu, r64), _err(r32, r64)
  bar = max(1e-5, 8 * m)
  assert e <= bar, '%s: error %.3g > bar %.3g (float32 reference %.3g)' % (name, e, bar, m)


@pytest.mark.parametrize('stream', [0, 1])
@pytest.mark.parametrize('A', [9, 18])
@pytest.mark.parametrize('B', [64, 256, 4096, 65536])
def test_phases_against_float64(B, A, stream):
  settings = _settings(beta=0.05)
  cfg = settings
  state = np.array([0.0, 1.0, 1.0, 0.0], np.float32)
  for step in range(3):
    b = _batch(B, A, seed=1000 * step + B + A)
    gpu, new_state = _run(settings, b, state, stream)
    args = (cfg, b['ll'], b['lb'], b['bl'], b['act'], b['rew'], b['done'], np.float32(-0.8), state, 0.05)
    r64 = PR.loss_and_grads(*args, FT=np.float64)
    r32 = PR.loss_and_grads(*args, FT=np.float32)
    tag = 'B=%d A=%d stream=%d step %d ' % (B, A, stream, step)
    for k in ('policy', 'V', 'entropy', 'kl', 'total', 'v_mean', 'v_l2_error', 'mean_entropy', 'popart_mean',
              'popart_std'):
      _check(tag + k, gpu['loss_terms'][_lib.LT[k]], r64['terms'][k], r32['terms'][k])
    _check(tag + 'vs', gpu['vs'], r64['vs'], r32['vs'])
    _check(tag + 'pg_advantages', gpu['pg_advantages'], r64['pg_adv'], r32['pg_adv'])
    _check(tag + 'dlogits', gpu['dlogits'], r64['dlogits'], r32['dlogits'])
    _check(tag + 'dbaseline', gpu['dbaseline'], r64['dbaseline'], r32['dbaseline'])
    for i, k in enumerate(('d sigma', 'd mu')):
      _check(tag + k, gpu['dcomp'][i], r64['dcomp'][i], r32['dcomp'][i])
    for i, k in enumerate(('mu1', 'mu2', 'sigma', 'mu')):
      _check(tag + k, new_state[i], r64['state'][i], r32['state'][i])
    assert not gpu['dlogits'][-1].any() and not gpu['dbaseline'][-1].any()
    state = new_state
  assert state[1] > 1e4        # the moments followed returns of order 1e3


@pytest.mark.parametrize('case', ['b1e-2', 'b3e-4', 'b1'])
def test_phases_against_reference_golden(case):
  """Each step of tests/golden/popart_golden.npz (the unmodified reference PopArt and EMAMeanStd around the
  reference V-trace, over numpy float32), from the state the reference held before it."""
  d = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'popart_golden.npz'))
  discounting, lambda_, baseline_cost = (float(x) for x in d['cfg'])
  settings = _settings(beta=float(d['%s_beta' % case]), discounting=discounting, lambda_=lambda_,
                       baseline_cost=baseline_cost)
  k = 0
  while '%s_%d_ll' % (case, k) in d:
    p = '%s_%d_' % (case, k)
    b = dict(ll=d[p + 'll'], lb=d[p + 'lb'], bl=d[p + 'bl'], act=d[p + 'act'], rew=d[p + 'rew'], done=d[p + 'done'])
    gpu, new_state = _run(settings, b, d[p + 'state_before'])
    lt = gpu['loss_terms']
    for name, x, ref in (('vs', gpu['vs'], d[p + 'vs']), ('pg_adv', gpu['pg_advantages'], d[p + 'pg_adv']),
                         ('state', new_state, d[p + 'state_after']),
                         ('policy', lt[_lib.LT['policy']], d[p + 'policy_loss']),
                         ('V', lt[_lib.LT['V']], d[p + 'v_loss']),
                         ('PopArt/mean', lt[_lib.LT['popart_mean']], d[p + 'PopArt__mean']),
                         ('PopArt/std', lt[_lib.LT['popart_std']], d[p + 'PopArt__std'])):
      x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
      if name == 'state':
        err = float((np.abs(x - ref) / np.abs(ref)).max())
      else:
        err = float(np.abs(x - ref).max() / np.abs(ref).max())
      assert err <= 1e-4, '%s%s: %.3g' % (p, name, err)    # the float64 composition's own distance bar
    k += 1
  assert k >= 3


def test_moments_of_all_replicas():
  """world = 2: the moment sums of a second replica's batch, added in by `reduce_moment_sums`, give the state
  of one process on both batches side by side; this replica's gradients are those of its own batch with the
  statistics of both."""
  B, A = 256, 18
  b1, b2 = _batch(B, A, seed=31), _batch(B, A, seed=32)
  state = np.array([150.0, 4.0e4, 0.9, 0.1], np.float32)
  settings = _settings(beta=0.1)
  other = {}

  def run(b, reduce_moment_sums, world):
    d = {k: torch.as_tensor(v).cuda() for k, v in b.items()}
    mom = torch.tensor(state[:2]).cuda()
    comp = torch.tensor(state[2:]).cuda()
    dcomp = torch.zeros(2).cuda()
    out = learner.popart_loss_fwd_bwd(settings, d['ll'], d['lb'], d['bl'], d['act'], d['rew'], d['done'],
                                      torch.tensor(-0.8).cuda(), mom, comp, dcomp, reduce_moment_sums, world)
    torch.cuda.synchronize()
    return out, np.concatenate([mom.cpu().numpy(), comp.cpu().numpy()]), dcomp.cpu().numpy()
  run(b2, lambda sums: other.setdefault('sums', sums.clone()), 1)
  out, new_state, dcomp = run(b1, lambda sums: sums.add_(other['sums']), 2)
  both = {k: np.concatenate([b1[k], b2[k]], axis=1) for k in b1}
  args = (settings, both['ll'], both['lb'], both['bl'], both['act'], both['rew'], both['done'], np.float32(-0.8),
          state, 0.1)
  r64, r32 = PR.loss_and_grads(*args, FT=np.float64), PR.loss_and_grads(*args, FT=np.float32)
  for i in range(4):
    _check('state %d' % i, new_state[i], r64['state'][i], r32['state'][i])
  N = 2 * B * T
  s1, s2 = (float(x) for x in PR.moment_sums(settings, *(both[k] for k in ('ll', 'lb', 'bl', 'act', 'rew', 'done')),
                                                state)[:2])
  args1 = (settings, b1['ll'], b1['lb'], b1['bl'], b1['act'], b1['rew'], b1['done'], np.float32(-0.8), state, 0.1)
  m64 = PR.loss_and_grads(*args1, FT=np.float64, global_means=(s1 / N, s2 / N))
  m32 = PR.loss_and_grads(*args1, FT=np.float32, global_means=(s1 / N, s2 / N))
  _check('dbaseline', out['dbaseline'].cpu().numpy(), m64['dbaseline'], m32['dbaseline'])
  for i in range(2):
    _check('dcomp %d' % i, dcomp[i], m64['dcomp'][i], m32['dcomp'][i])


@pytest.mark.parametrize('stream', [0, 1])
@pytest.mark.parametrize('B', [64, 4096])
def test_beta0_initial_state_matches_plain_kernel(B, stream):
  A = 18
  b = _batch(B, A, seed=7)
  gpu, new_state = _run(_settings(beta=0.0), b, np.array([0, 1, 1, 0], np.float32), stream)
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  try:
    d = {k: torch.as_tensor(v).cuda() for k, v in b.items()}
    plain = learner.vtrace_loss_fwd_bwd(learner.default_loss_settings(), d['ll'], d['lb'], d['bl'], d['act'],
                                        d['rew'], d['done'], torch.tensor(-0.8).cuda(), want_vtrace=True)
    torch.cuda.synchronize()
  finally:
    _lib.lib().seedrl_debug_set_loss_stream(1)
  np.testing.assert_array_equal(gpu['dlogits'], plain['dlogits'].cpu().numpy())
  np.testing.assert_array_equal(gpu['dbaseline'], plain['dbaseline'].cpu().numpy())
  np.testing.assert_array_equal(gpu['vs'], plain['vs'].cpu().numpy())
  np.testing.assert_array_equal(gpu['pg_advantages'], plain['pg_advantages'].cpu().numpy())
  np.testing.assert_array_equal(new_state, np.array([0, 1, 1, 0], np.float32))
  lt = plain['loss_terms'].cpu().numpy()
  np.testing.assert_allclose(gpu['loss_terms'][:12], lt[:12], rtol=2e-6, atol=0)
  assert gpu['loss_terms'][_lib.LT['popart_mean']] == 0.0 and gpu['loss_terms'][_lib.LT['popart_std']] == 1.0


@pytest.mark.parametrize('stream', [0, 1])
def test_power_of_two_scale_invariance(stream):
  B, A, c = 4096, 18, np.float32(2.0 ** 10)
  b = _batch(B, A, seed=11)
  state = np.array([350.0, 2.0e5, 0.8, 0.3], np.float32)
  settings = _settings(beta=0.05)
  g1, s1 = _run(settings, b, state, stream)
  b2 = dict(b, rew=b['rew'] * c)
  g2, s2 = _run(settings, b2, np.array([state[0] * c, state[1] * c * c, state[2], state[3]], np.float32), stream)
  for k in ('dlogits', 'dbaseline', 'dcomp'):
    np.testing.assert_array_equal(g1[k], g2[k], err_msg=k)
  np.testing.assert_array_equal(s1[2:], s2[2:])
  np.testing.assert_array_equal(g1['vs'] * c, g2['vs'])
  assert s1[0] * c == s2[0] and s1[1] * c * c == s2[1]


def test_update_preserves_predictions():
  B, A = 4096, 9
  b = _batch(B, A, seed=5)
  state = np.array([120.0, 3.0e4, 1.3, -0.2], np.float32)
  _, new = _run(_settings(beta=0.3), b, state)

  def u(st):
    st = st.astype(np.float64)
    s = np.sqrt(st[1] - st[0] ** 2)
    return s * (st[2] * b['lb'].astype(np.float64) + st[3]) + st[0]
  before, after = u(state), u(new)
  assert abs(new[0] - state[0]) > 1.0          # the statistics moved
  assert np.abs(after - before).max() <= 1e-5 * np.abs(before).max()


def _agent_and_step(conv_mode, seed=0):
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  agent = networks.ImpalaDeep(18, seed=seed, conv_mode=conv_mode, lstm_mode='tc3' if conv_mode == 'tc3p' else 'tiled')
  opt = optimizers.Adam(1e-3)
  step = learner.LearnerStep(agent, opt, settings=_settings(beta=0.05), check_errors_every=0)
  return agent, opt, step


def _unroll(B, seed):
  g = np.random.default_rng(seed)
  T1 = T + 1
  frames = torch.as_tensor(g.integers(0, 256, (T1, B, 84, 84, 4), dtype=np.uint8)).cuda()
  from seed_rl_b200.common import utils
  from seed_rl_b200.dmlab import networks
  env = utils.EnvOutput(torch.as_tensor((g.standard_normal((T1, B)) * 300 + 500).astype(np.float32)).cuda(),
                        torch.as_tensor(g.random((T1, B)) < 0.05).cuda(), frames,
                        torch.zeros(T1, B, dtype=torch.bool).cuda(), torch.zeros(T1, B, dtype=torch.int32).cuda())
  ao = networks.AgentOutput(torch.as_tensor(g.integers(0, 18, (T1, B))).cuda(),
                            torch.as_tensor(g.standard_normal((T1, B, 18)).astype(np.float32)).cuda(),
                            torch.zeros((T1, B)).cuda())
  state = (torch.zeros(B, 256).cuda(), torch.zeros(B, 256).cuda())
  return learner.Unroll(state, torch.as_tensor(g.integers(0, 18, (T1, B))).cuda(), env, ao)


def test_only_the_compensation_is_in_the_trained_arena():
  """popart_test.py test_variables on the learner: of the four PopArt variables, sigma and mu are the two
  entries appended to the parameter table, inside the arena Adam and the gradient all-reduce cover; mu1 and mu2
  are a buffer of their own.  The network's table, offsets and grad_split are those of an agent without PopArt."""
  from seed_rl_b200.dmlab import networks
  plain = networks.ImpalaDeep(18, seed=0)
  agent, opt, step = _agent_and_step('simt')
  plain.init_entropy_cost(step.settings.entropy_cost, step.settings.entropy_cost_adjustment_speed)
  n = len(plain.param_info)
  assert agent.param_info[:n] == plain.param_info and agent.grad_split == plain.grad_split
  extra = agent.param_info[n:]
  assert [x[0] for x in extra] == ['popart/compensation_std', 'popart/compensation_mean']
  assert [x[2] for x in extra] == [plain.arena_floats, plain.arena_floats + 1]
  assert agent.params.numel() == opt.m.numel() == agent.grads.numel() > plain.arena_floats + 1
  np.testing.assert_array_equal(agent.popart_compensation.cpu().numpy(), [1, 0])
  lo, hi = agent.params.data_ptr(), agent.params.data_ptr() + 4 * agent.params.numel()
  assert not lo <= agent.popart_moments.data_ptr() < hi
  np.testing.assert_array_equal(agent.popart_moments.cpu().numpy(), [0, 1])
  assert torch.equal(agent.params[:plain.arena_floats], plain.params)


@pytest.mark.parametrize('conv_mode', ['simt', 'tc3p'])
def test_learner_step_against_float64_composition(conv_mode):
  """One ImpalaDeep learner step at T = 20, B = 64: the loss gradients the step hands to the network backward,
  the compensation gradients in the gradient tail and the stored state, against the float64 composition on the
  network outputs of that step; then Adam moves the compensation from (sigma+, mu+)."""
  agent, opt, step = _agent_and_step(conv_mode)
  for it in range(3):
    un = _unroll(64, seed=it)
    state = np.concatenate([agent.popart_moments.cpu().numpy(), agent.popart_compensation.cpu().numpy()])
    ecp = float(agent.entropy_cost_param)
    step.compute_gradients(un)
    out, _ = agent(un.prev_actions, un.env_outputs, un.agent_state, unroll=True)
    r = agent._loss_grads
    lt = r['loss_terms'].cpu().numpy()
    args = (step.settings, out.policy_logits.cpu().numpy(), out.baseline.cpu().numpy(),
            un.agent_outputs.policy_logits.cpu().numpy(), un.agent_outputs.action.cpu().numpy(),
            un.env_outputs[0].cpu().numpy(), un.env_outputs[1].cpu().numpy(), ecp, state, 0.05)
    r64, r32 = PR.loss_and_grads(*args, FT=np.float64), PR.loss_and_grads(*args, FT=np.float32)
    tag = '%s step %d ' % (conv_mode, it)
    _check(tag + 'dlogits', r['dlogits'].cpu().numpy(), r64['dlogits'], r32['dlogits'])
    _check(tag + 'dbaseline', r['dbaseline'].cpu().numpy(), r64['dbaseline'], r32['dbaseline'])
    _check(tag + 'total', lt[0], r64['terms']['total'], r32['terms']['total'])
    tail = agent.popart_compensation_grad.cpu().numpy()
    for i in range(2):
      _check(tag + 'dcomp %d' % i, tail[i], r64['dcomp'][i], r32['dcomp'][i])
    new_state = np.concatenate([agent.popart_moments.cpu().numpy(), agent.popart_compensation.cpu().numpy()])
    for i in range(4):
      _check(tag + 'state %d' % i, new_state[i], r64['state'][i], r32['state'][i])
    step.apply_gradients()
    after = agent.popart_compensation.cpu().numpy()
    assert np.all(np.abs(after - new_state[2:]) <= 3e-3) and np.any(after != new_state[2:])


def test_learner_runs_are_deterministic_and_resume_from_checkpoint(tmp_path):
  from seed_rl_b200.agents.vtrace import learner_loop
  unrolls = [_unroll(16, seed=100 + i) for i in range(4)]

  def run(n, agent_opt_step=None):
    agent, opt, step = agent_opt_step or _agent_and_step('tc3p')
    for un in unrolls[:n]:
      step.minimize(un)
    torch.cuda.synchronize()
    return agent, opt, step
  a1, o1, _ = run(4)
  a2, o2, _ = run(4)
  assert torch.equal(a1.params, a2.params) and torch.equal(a1.popart_moments, a2.popart_moments)
  a3, o3, _ = run(2)
  path = os.path.join(str(tmp_path), 'ckpt.pt')
  learner_loop.save_checkpoint(path, a3, o3)
  a4, o4, s4 = _agent_and_step('tc3p', seed=1)
  learner_loop.restore_checkpoint(path, a4, o4)
  for un in unrolls[2:]:
    s4.minimize(un)
  torch.cuda.synchronize()
  assert torch.equal(a1.params, a4.params) and torch.equal(a1.popart_moments, a4.popart_moments)
  assert torch.equal(o1.m, o4.m) and torch.equal(o1.v, o4.v)
