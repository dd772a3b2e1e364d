"""Multi-task PopArt (--popart_tasks) on the GPU: seedrl_vtrace_popart_tasks_loss_fwd (both kernel forms, chosen
with seedrl_debug_set_loss_stream) and seedrl_vtrace_popart_tasks_update against the float64 per-task
composition of tests/popart_tasks_reference.py; bit-identity with the single-task entry points at one task;
absent tasks; per-task scale invariance; preserved predictions; two replicas with different task mixes; the
ImpalaDeep learner step; and the error flag for a task id outside [0, K).

Bars as in tests/test_gpu_vtrace_popart.py: error = max|gpu - ref64| / max|ref64|, bar = max(1e-5, 8 m), m the
same error of the float32 composition.  Per-task quantities are checked task by task, each on its own scale."""
import os

import numpy as np
import pytest
import torch

import popart_tasks_reference as PT
from seed_rl_b200 import _lib
from seed_rl_b200.agents.vtrace import learner

pytestmark = pytest.mark.gpu

T = 20


def _batch(B, A, seed, ids, scales):
  g = np.random.default_rng(seed)
  T1 = T + 1
  scale = np.asarray(scales, np.float32)[ids]
  return dict(
      ll=(g.standard_normal((T1, B, A)) * 2).astype(np.float32),
      lb=(g.standard_normal((T1, B)) * 3).astype(np.float32),
      bl=(g.standard_normal((T1, B, A)) * 2).astype(np.float32),
      act=g.integers(0, A, (T1, B)).astype(np.int64),
      rew=((g.standard_normal((T1, B)) * 0.6 + 1.0) * scale).astype(np.float32),
      done=g.random((T1, B)) < 0.05)


def _uneven_ids(B, K, seed):
  """Task k draws a share proportional to 1 / (k + 1)."""
  p = 1.0 / np.arange(1, K + 1)
  return np.random.default_rng(seed).choice(K, size=B, p=p / p.sum()).astype(np.int32)


def _settings(K, beta=0.05, **kw):
  return learner.default_loss_settings(popart=True, popart_beta=beta, popart_tasks=K, **kw)


def _run(settings, b, states, ids, stream=1, ecp=-0.8, abandoned=None, reduce_moment_sums=None):
  """Both phases through the multi-task entry points -> (outputs of numpy, new states [K,4], task_error)."""
  K = settings.popart_tasks
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  try:
    d = {k: torch.as_tensor(v).cuda() for k, v in b.items()}
    st = torch.as_tensor(np.asarray(states, np.float32)).cuda()
    mom, comp = st[:, :2].contiguous(), st[:, 2:].contiguous()
    dcomp = torch.zeros(K, 2, dtype=torch.float32).cuda()
    err = torch.zeros(1, dtype=torch.int32).cuda()
    ab = None if abandoned is None else torch.as_tensor(abandoned).cuda()
    out = learner.popart_tasks_loss_fwd_bwd(
        settings, d['ll'], d['lb'], d['bl'], d['act'], d['rew'], d['done'], torch.tensor(ecp).cuda(), mom, comp,
        dcomp, torch.as_tensor(ids).cuda(), err, reduce_moment_sums, want_vtrace=True, abandoned=ab)
    torch.cuda.synchronize()
  finally:
    _lib.lib().seedrl_debug_set_loss_stream(1)
  res = {k: v.cpu().numpy() for k, v in out.items() if v is not None}
  res['dcomp'] = dcomp.cpu().numpy()
  return res, np.concatenate([mom.cpu().numpy(), comp.cpu().numpy()], 1), int(err.item())


def _err(x, ref):
  x, ref = np.asarray(x, np.float64), np.asarray(ref, np.float64)
  if ref.ndim == 0:
    return abs(float(x) - float(ref)) / max(abs(float(ref)), 1e-30)
  return float(np.abs(x - ref).max() / max(np.abs(ref).max(), 1e-30))


def _check(name, gpu, r64, r32):
  e, m = _err(gpu, r64), _err(r32, r64)
  bar = max(1e-5, 8 * m)
  assert e <= bar, '%s: error %.3g > bar %.3g (float32 reference %.3g)' % (name, e, bar, m)


def _check_against(tag, gpu, state, r64, r32, ids, K):
  for k in ('policy', 'V', 'entropy', 'kl', 'total', 'v_mean', 'v_l2_error', 'mean_entropy'):
    _check(tag + k, gpu['loss_terms'][_lib.LT[k]], r64['terms'][k], r32['terms'][k])
  assert gpu['loss_terms'][_lib.LT['popart_mean']] == 0 and gpu['loss_terms'][_lib.LT['popart_std']] == 0
  for k in range(K):
    cols = ids == k
    t = tag + 'task %d ' % k
    for j, nm in enumerate(('mu1', 'mu2', 'sigma', 'mu')):
      _check(t + nm, state[k, j], r64['state'][k, j], r32['state'][k, j])
    for j, nm in enumerate(('d sigma', 'd mu')):
      if cols.any():
        _check(t + nm, gpu['dcomp'][k, j], r64['dcomp'][k, j], r32['dcomp'][k, j])
      else:
        assert gpu['dcomp'][k, j] == 0 and not np.signbit(gpu['dcomp'][k, j])
    if cols.any():
      for key, rk in (('vs', 'vs'), ('pg_advantages', 'pg_adv'), ('dbaseline', 'dbaseline'), ('dlogits', 'dlogits')):
        _check(t + key, gpu[key][:, cols], r64[rk][:, cols], r32[rk][:, cols])
      for j, nm in enumerate(('sum vs', 'sum vs^2', 'rows')):
        _check(t + nm, gpu['moment_sums'][k, j], r64['sums'][k, j], r32['sums'][k, j])
  assert not gpu['dlogits'][-1].any() and not gpu['dbaseline'][-1].any()


@pytest.mark.parametrize('stream', [0, 1])
@pytest.mark.parametrize('K', [3, 30])
@pytest.mark.parametrize('B', [64, 4096, 65536])
def test_phases_against_float64(B, K, stream):
  settings = _settings(K)
  ids = _uneven_ids(B, K, seed=B + K)
  scales = 10.0 ** np.linspace(0, 3, K)          # returns from ~1 to ~1e3 across the tasks
  states = np.tile(np.array([0.0, 1.0, 1.0, 0.0], np.float32), (K, 1))
  ab = None
  for step in range(3):
    b = _batch(B, 9, seed=1000 * step + B + K, ids=ids, scales=scales)
    if B == 4096 and step == 2:                    # the abandoned mask composes with the tasks
      ab = np.random.default_rng(3).random((T + 1, B)) < 0.02
      b['done'] = b['done'] | ab
    gpu, new, err = _run(settings, b, states, ids, stream, abandoned=ab)
    assert err == 0
    if ab is not None:
      # masked transitions take vs_t = u_t with their column's task state and pg_adv_t = 0; every row still
      # counts in its task's moments
      mask = ab[1:]
      st = states[ids].astype(np.float64)
      s = np.sqrt(st[:, 1] - st[:, 0] ** 2)
      u = s * (st[:, 2] * b['lb'][:-1].astype(np.float64) + st[:, 3]) + st[:, 0]
      assert mask.any() and np.all(gpu['pg_advantages'][mask] == 0)
      np.testing.assert_allclose(gpu['vs'][mask], u[mask], rtol=1e-6, atol=1e-6 * np.abs(u).max())
      np.testing.assert_array_equal(gpu['moment_sums'][:, 2], T * np.bincount(ids, minlength=K))
      assert np.isfinite(new).all()
      continue
    args = (settings, b['ll'], b['lb'], b['bl'], b['act'], b['rew'], b['done'], np.float32(-0.8), states, ids, 0.05)
    r64, r32 = PT.loss_and_grads(*args, FT=np.float64), PT.loss_and_grads(*args, FT=np.float32)
    _check_against('B=%d K=%d stream=%d step %d ' % (B, K, stream, step), gpu, new, r64, r32, ids, K)
    states = new


@pytest.mark.parametrize('stream', [0, 1])
@pytest.mark.parametrize('abandoned', [False, True])
@pytest.mark.parametrize('B', [64, 65536])
def test_one_task_equals_single_task_entry_points(B, abandoned, stream):
  """K = 1, every id 0: the multi-task entry points give the single-task ones' outputs bit for bit."""
  b = _batch(B, 9, seed=7, ids=np.zeros(B, np.int32), scales=[300.0])
  ab = (np.random.default_rng(8).random((T + 1, B)) < 0.02) if abandoned else None
  if ab is not None:
    b['done'] = b['done'] | ab
  state = np.array([40.0, 2500.0, 1.1, -0.05], np.float32)
  new_out, new_state, err = _run(_settings(1), b, state[None], np.zeros(B, np.int32), stream, abandoned=ab)
  assert err == 0
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  try:
    d = {k: torch.as_tensor(v).cuda() for k, v in b.items()}
    mom, comp = torch.tensor(state[:2]).cuda(), torch.tensor(state[2:]).cuda()
    dcomp = torch.zeros(2).cuda()
    old = learner.popart_loss_fwd_bwd(_settings(1), d['ll'], d['lb'], d['bl'], d['act'], d['rew'], d['done'],
                                      torch.tensor(-0.8).cuda(), mom, comp, dcomp, want_vtrace=True,
                                      abandoned=None if ab is None else torch.as_tensor(ab).cuda())
    torch.cuda.synchronize()
  finally:
    _lib.lib().seedrl_debug_set_loss_stream(1)
  for k in ('loss_terms', 'dlogits', 'dbaseline', 'd_entropy_cost_param', 'vs', 'pg_advantages'):
    np.testing.assert_array_equal(new_out[k], old[k].cpu().numpy(), err_msg=k)
  np.testing.assert_array_equal(new_out['dcomp'][0], dcomp.cpu().numpy())
  np.testing.assert_array_equal(new_state[0], np.concatenate([mom.cpu().numpy(), comp.cpu().numpy()]))


@pytest.mark.parametrize('stream', [0, 1])
def test_absent_task_keeps_its_state_and_gets_zero_gradient(stream):
  K, B = 5, 4096
  ids = _uneven_ids(B, K, seed=1)
  ids[ids == 3] = 0
  states = np.array([[3.0, 20.0, 1.2, 0.1], [30.0, 1500.0, 0.9, -0.2], [0.5, 2.0, 1.0, 0.0],
                     [7.0, 60.0, 1.3, 0.4], [300.0, 1.5e5, 1.1, 0.05]], np.float32)
  b = _batch(B, 9, seed=2, ids=ids, scales=[3.0, 30.0, 1.0, 10.0, 300.0])
  gpu, new, err = _run(_settings(K), b, states, ids, stream)
  assert err == 0
  np.testing.assert_array_equal(new[3], states[3])
  assert np.all(gpu['dcomp'][3] == 0) and not np.signbit(gpu['dcomp'][3]).any()
  np.testing.assert_array_equal(gpu['moment_sums'][3], [0, 0, 0])
  assert np.all(new[[0, 1, 2, 4], 0] != states[[0, 1, 2, 4], 0])


@pytest.mark.parametrize('stream', [0, 1])
def test_per_task_scale_invariance(stream):
  """Task 1's rewards x 2^10, its mu1 x 2^10 and mu2 x 2^20: every gradient is bit-identical, every other task's
  state is bit-identical, and task 1's moments scale exactly."""
  K, B, c = 4, 65536, np.float32(2.0 ** 10)
  ids = _uneven_ids(B, K, seed=4)
  states = np.array([[5.0, 40.0, 1.1, 0.1], [50.0, 3000.0, 0.8, -0.3], [1.0, 3.0, 1.0, 0.0],
                     [200.0, 5e4, 1.2, 0.2]], np.float32)
  b = _batch(B, 9, seed=9, ids=ids, scales=[5.0, 50.0, 1.0, 200.0])
  g1, s1, _ = _run(_settings(K), b, states, ids, stream)
  b2 = dict(b, rew=np.where(ids[None, :] == 1, b['rew'] * c, b['rew']).astype(np.float32))
  st2 = states.copy()
  st2[1, 0] *= c
  st2[1, 1] *= c * c
  g2, s2, _ = _run(_settings(K), b2, st2, ids, stream)
  for k in ('dlogits', 'dbaseline', 'dcomp'):
    np.testing.assert_array_equal(g1[k], g2[k], err_msg=k)
  np.testing.assert_array_equal(s1[[0, 2, 3]], s2[[0, 2, 3]])
  np.testing.assert_array_equal(s1[1, 2:], s2[1, 2:])
  assert s1[1, 0] * c == s2[1, 0] and s1[1, 1] * c * c == s2[1, 1]


def test_update_preserves_each_tasks_predictions():
  K, B = 3, 4096
  ids = _uneven_ids(B, K, seed=6)
  states = np.array([[120.0, 3.0e4, 1.3, -0.2], [2.0, 9.0, 0.7, 0.3], [-40.0, 5000.0, 1.0, 0.0]], np.float32)
  b = _batch(B, 9, seed=5, ids=ids, scales=[500.0, 3.0, 60.0])
  _, new, _ = _run(_settings(K, beta=0.3), b, states, ids)

  def u(st, cols):
    st = st.astype(np.float64)
    s = np.sqrt(st[1] - st[0] ** 2)
    return s * (st[2] * b['lb'][:, cols].astype(np.float64) + st[3]) + st[0]
  for k in range(K):
    cols = ids == k
    before, after = u(states[k], cols), u(new[k], cols)
    assert new[k, 0] != states[k, 0]
    assert np.abs(after - before).max() <= 1e-5 * np.abs(before).max(), k


@pytest.mark.parametrize('stream', [0, 1])
def test_two_replicas_with_different_task_mixes(stream):
  """Replica A has tasks 0 and 1, replica B tasks 0 and 2: the per-task sums, SUM-joined between the phases,
  give both replicas the state one process reaches on both batches side by side."""
  K, B = 3, 4096
  ids_a = np.where(np.arange(B) % 3 == 0, 1, 0).astype(np.int32)
  ids_b = np.where(np.arange(B) % 5 == 0, 2, 0).astype(np.int32)
  states = np.array([[10.0, 200.0, 1.0, 0.0], [1.0, 5.0, 1.1, 0.1], [100.0, 2e4, 0.9, -0.1]], np.float32)
  ba = _batch(B, 9, seed=11, ids=ids_a, scales=[10.0, 1.0, 100.0])
  bb = _batch(B, 9, seed=12, ids=ids_b, scales=[10.0, 1.0, 100.0])
  seen = {}

  def capture(name):
    def f(s):
      seen[name] = s.clone()
    return f
  _run(_settings(K), ba, states, ids_a, stream, reduce_moment_sums=capture('a'))
  _run(_settings(K), bb, states, ids_b, stream, reduce_moment_sums=capture('b'))
  _, sa, _ = _run(_settings(K), ba, states, ids_a, stream, reduce_moment_sums=lambda s: s.add_(seen['b']))
  _, sb, _ = _run(_settings(K), bb, states, ids_b, stream, reduce_moment_sums=lambda s: s.add_(seen['a']))
  np.testing.assert_array_equal(sa, sb)
  both = {k: np.concatenate([ba[k], bb[k]], 1) for k in ba}
  _, s1, _ = _run(_settings(K), both, states, np.concatenate([ids_a, ids_b]), stream)
  np.testing.assert_allclose(sa, s1, rtol=1e-6)
  assert (seen['a'][2] == 0).all() and (seen['b'][1] == 0).all()
  assert sa[1, 0] != states[1, 0] and sa[2, 0] != states[2, 0]


@pytest.mark.parametrize('stream', [0, 1])
def test_out_of_range_task_id_sets_the_error_flag(stream):
  K, B = 3, 4096
  ids = _uneven_ids(B, K, seed=13)
  b = _batch(B, 9, seed=14, ids=ids, scales=[1.0, 1.0, 1.0])
  states = np.tile(np.array([0.0, 1.0, 1.0, 0.0], np.float32), (K, 1))
  _, _, err = _run(_settings(K), b, states, ids, stream)
  assert err == 0
  bad = ids.copy()
  bad[17], bad[4000] = K, -1
  _, new, err = _run(_settings(K), b, states, bad, stream)
  assert err == 1 and np.isfinite(new).all()


# ---- the ImpalaDeep learner step -------------------------------------------------------------------------------
K_STEP = 4


def _agent_and_step(conv_mode, seed=0):
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  agent = networks.ImpalaDeep(18, seed=seed, conv_mode=conv_mode, lstm_mode='tc3' if conv_mode == 'tc3p' else 'tiled')
  opt = optimizers.Adam(1e-3)
  step = learner.LearnerStep(agent, opt, settings=_settings(K_STEP), check_errors_every=1)
  return agent, opt, step


def _unroll(B, seed):
  g = np.random.default_rng(seed)
  T1 = T + 1
  from seed_rl_b200.common import utils
  from seed_rl_b200.dmlab import networks
  ids = _uneven_ids(B, K_STEP, seed)
  scale = np.asarray([3.0, 30.0, 300.0, 1000.0], np.float32)[ids]
  frames = torch.as_tensor(g.integers(0, 256, (T1, B, 84, 84, 4), dtype=np.uint8)).cuda()
  env = utils.EnvOutput(torch.as_tensor((g.standard_normal((T1, B)) * 0.5 + 1.0).astype(np.float32) * scale).cuda(),
                        torch.as_tensor(g.random((T1, B)) < 0.05).cuda(), frames,
                        torch.zeros(T1, B, dtype=torch.bool).cuda(), torch.zeros(T1, B, dtype=torch.int32).cuda())
  ao = networks.AgentOutput(torch.as_tensor(g.integers(0, 18, (T1, B))).cuda(),
                            torch.as_tensor(g.standard_normal((T1, B, 18)).astype(np.float32)).cuda(),
                            torch.zeros((T1, B)).cuda())
  state = (torch.zeros(B, 256).cuda(), torch.zeros(B, 256).cuda())
  return learner.Unroll(state, torch.as_tensor(g.integers(0, 18, (T1, B))).cuda(), env, ao), torch.as_tensor(ids).cuda()


def _agent_state(agent):
  return np.concatenate([agent.popart_moments.cpu().numpy(), agent.popart_compensation.cpu().numpy()], 1)


@pytest.mark.parametrize('conv_mode', ['simt', 'tc3p'])
def test_learner_step_against_float64_composition(conv_mode):
  agent, opt, step = _agent_and_step(conv_mode)
  n = agent.param_info.index(('popart/compensation_std/0', (), agent.arena_floats))
  assert [x[0] for x in agent.param_info[n:n + 4]] == ['popart/compensation_std/0', 'popart/compensation_mean/0',
                                                       'popart/compensation_std/1', 'popart/compensation_mean/1']
  assert tuple(agent.popart_moments.shape) == (K_STEP, 2)
  for it in range(3):
    un, ids = _unroll(64, seed=it)
    states = _agent_state(agent)
    ecp = float(agent.entropy_cost_param)
    _, logs = step.compute_gradients(un, task_ids=ids)
    names = [x[0] for x in logs]
    assert 'PopArt/mean/3' in names and 'PopArt/std/0' in names and 'PopArt/mean' not in names
    out, _ = agent(un.prev_actions, un.env_outputs, un.agent_state, unroll=True)
    r = agent._loss_grads
    args = (step.settings, out.policy_logits.cpu().numpy(), out.baseline.cpu().numpy(),
            un.agent_outputs.policy_logits.cpu().numpy(), un.agent_outputs.action.cpu().numpy(),
            un.env_outputs[0].cpu().numpy(), un.env_outputs[1].cpu().numpy(), ecp, states, ids.cpu().numpy(), 0.05)
    r64, r32 = PT.loss_and_grads(*args, FT=np.float64), PT.loss_and_grads(*args, FT=np.float32)
    gpu = {k: v.cpu().numpy() for k, v in r.items() if v is not None}
    gpu['dcomp'] = agent.popart_compensation_grad.cpu().numpy()
    gpu['vs'], gpu['pg_advantages'] = r64['vs'], r64['pg_adv']   # the learner step does not request them
    _check_against('%s step %d ' % (conv_mode, it), gpu, _agent_state(agent), r64, r32, ids.cpu().numpy(), K_STEP)
    step.apply_gradients()
    agent.check_errors()


def test_learner_runs_are_deterministic_and_resume_from_checkpoint(tmp_path):
  from seed_rl_b200.agents.vtrace import learner_loop
  unrolls = [_unroll(16, seed=100 + i) for i in range(4)]

  def run(n, agent_opt_step=None):
    agent, opt, step = agent_opt_step or _agent_and_step('tc3p')
    for un, ids in unrolls[:n]:
      step.minimize(un, task_ids=ids)
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
  for un, ids in unrolls[2:]:
    s4.minimize(un, task_ids=ids)
  torch.cuda.synchronize()
  assert torch.equal(a1.params, a4.params) and torch.equal(a1.popart_moments, a4.popart_moments)
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  other = networks.ImpalaDeep(18, seed=0, conv_mode='tc3p', lstm_mode='tc3')
  learner.LearnerStep(other, optimizers.Adam(1e-3), settings=_settings(3), check_errors_every=0)
  with pytest.raises(ValueError, match='4 PopArt tasks'):
    learner_loop.restore_checkpoint(path, other, optimizers.Adam(1e-3))


def test_learner_step_reports_an_out_of_range_task_id():
  agent, opt, step = _agent_and_step('simt')
  un, ids = _unroll(16, seed=3)
  step.minimize(un, task_ids=ids)
  bad = ids.clone()
  bad[5] = K_STEP
  with pytest.raises(RuntimeError, match='task id outside'):
    step.minimize(un, task_ids=bad)
  with pytest.raises(ValueError, match='task_ids'):
    step.minimize(un)
