"""GPU: abandoned episodes in the V-trace and R2D2 loss kernels and the inference host.

1. Bit-identity: the _abandoned entry points with a NULL and an all-zero mask equal the existing ones exactly
   (V-trace small and TMA-streamed kernels, with and without PopArt; R2D2 n-step n = 1..5 and Retrace).
2. Float64 (tests/abandoned_float64_reference.py) with random masks at the first, interior and last
   transitions next to terminated rows: loss terms, dlogits, dbaseline, vs and pg advantages (through
   tests/vtrace_float64_reference.py with its V-trace replaced by the masked one), PopArt vs / moments, R2D2
   loss, priorities and dq.  Masked rows: dq, dbaseline and pg advantages exactly 0.
3. Truncation: rows before an abandonment at transition k equal the unroll cut to rows 0..k.
4. Learner steps with bootstrap_abandoned: the V-trace LearnerStep's output gradients against the float64 loss
   on the agent's own outputs (PopArt on: bit-equal to the masked PopArt loss on them, and unlike the unmasked
   one); R2D2's compute_gradients passes the replayed abandoned column (its priorities equal the masked loss's,
   differ from the unmasked loss's, and masked dq rows are 0).
5. The inference host (V-trace eager, R2D2 eager and CUDA-graph; the two paths share _begin_batch): the
   reference actor's abandonment sequence is accepted with allow_abandoned (and R2D2's completed unrolls hold
   the abandoned column as sent), rejected without it, and abandoned without done raises."""
import ctypes

import numpy as np
import pytest
import torch

import abandoned_float64_reference as R
import vtrace_float64_reference as VR
from seed_rl_b200 import _lib
from seed_rl_b200.agents.r2d2 import learner as r2d2_learner
from seed_rl_b200.agents.vtrace import learner

pytestmark = pytest.mark.gpu

A = 18
STREAM_TS = (1, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 256)   # every lanes-per-column width of the scan


@pytest.fixture(autouse=True)
def _stream_default():
  yield
  _lib.lib().seedrl_debug_set_loss_stream(1)


def _vtrace_batch(T1, B, seed, ab_p=0.05):
  rng = np.random.default_rng(seed)
  done, ab = R.masks(T1, B, seed + 1, p_abandoned=ab_p)
  return dict(ll=rng.normal(size=(T1, B, A)).astype(np.float32), lb=rng.normal(size=(T1, B)).astype(np.float32),
              bl=rng.normal(size=(T1, B, A)).astype(np.float32), act=rng.integers(0, A, (T1, B)),
              rew=rng.normal(size=(T1, B)).astype(np.float32), done=done, ab=ab)


def _cuda(b):
  return {k: torch.as_tensor(v).cuda() for k, v in b.items()}


ECP = -0.8


def _settings(**kw):
  return learner.default_loss_settings(discounting=0.97, lambda_=0.95, kl_cost=0.01, **kw)


def _plain(b, ab, null_entry=False):
  """vtrace_loss_fwd_bwd; null_entry: the _abandoned entry point with a NULL mask."""
  ecp = torch.tensor(ECP, device='cuda')
  if not null_entry:
    return learner.vtrace_loss_fwd_bwd(_settings(), b['ll'], b['lb'], b['bl'], b['act'], b['rew'], b['done'], ecp,
                                       want_vtrace=True, abandoned=ab)
  T1, B, _ = b['ll'].shape
  cfg = learner._loss_config(_settings())
  out = learner._loss_outputs(b['ll'], b['lb'], True)
  P = _lib.ptr
  _lib.check(_lib.lib().seedrl_vtrace_loss_fwd_bwd_abandoned(
      T1, B, A, P(b['ll']), P(b['lb']), P(b['bl']), P(b['act']), P(b['rew']), P(b['done']), None,
      ctypes.byref(cfg), P(ecp), P(out['loss_terms']), P(out['dlogits']), P(out['dbaseline']),
      P(out['d_entropy_cost_param']), P(out['vs']), P(out['pg_advantages']),
      P(learner._loss_scratch(T1, B, A, b['ll'].device)), _lib.stream_ptr()))
  return out


def _popart(b, ab, null_entry=False):
  mom = torch.tensor([0.3, 2.0], device='cuda'); comp = torch.tensor([1.2, -0.1], device='cuda')
  dcomp = torch.zeros(2, device='cuda')
  ecp = torch.tensor(ECP, device='cuda')
  if null_entry:
    # the popart entry point with a NULL mask: through the ctypes symbol, swapped in for the old one
    L = _lib.lib()
    orig = L.seedrl_vtrace_popart_loss_fwd

    def fwd(*a):
      return L.seedrl_vtrace_popart_loss_fwd_abandoned(*a[:9], None, *a[9:])
    L.seedrl_vtrace_popart_loss_fwd = fwd
    try:
      out = learner.popart_loss_fwd_bwd(_settings(popart=True), b['ll'], b['lb'], b['bl'], b['act'], b['rew'],
                                        b['done'], ecp, mom, comp, dcomp, want_vtrace=True)
    finally:
      L.seedrl_vtrace_popart_loss_fwd = orig
  else:
    out = learner.popart_loss_fwd_bwd(_settings(popart=True), b['ll'], b['lb'], b['bl'], b['act'], b['rew'],
                                      b['done'], ecp, mom, comp, dcomp, want_vtrace=True, abandoned=ab)
  out.update(mom=mom, comp=comp, dcomp=dcomp)
  return out


def _bits(x):
  return x.detach().cpu().contiguous().view(torch.int32).numpy()


# ---- 1. bit-identity ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('popart', [False, True])
@pytest.mark.parametrize('stream', [0, 1])
@pytest.mark.parametrize('B', [64, 256, 65536])
def test_vtrace_null_and_zero_mask_bit_identical(B, stream, popart):
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  b = _cuda(_vtrace_batch(21, B, seed=B + stream))
  b['done'] = b['done'] & ~b['ab']
  run = _popart if popart else _plain
  base = run(b, None)
  for got in (run(b, None, null_entry=True), run(b, torch.zeros_like(b['ab']))):
    for k, v in base.items():
      if v is not None:
        np.testing.assert_array_equal(_bits(got[k]), _bits(v), err_msg=k)


R2D2_RUNS = [('n_step', n) for n in (1, 2, 3, 4, 5)] + [('retrace', 0.95)]


def _r2d2(inp, rule, param, ab, null_entry=False):
  q, qt, act, rew, done, _, w = (torch.as_tensor(x).cuda() for x in inp)
  kw = dict(bellman_target=rule, importance_weights=w)
  if rule == 'n_step':
    kw['n_steps'] = param
  else:
    kw['retrace_lambda'] = param
  ao = r2d2_learner.AgentOutput(act, q)
  env = type('E', (), {'reward': rew, 'done': done})
  if not null_entry:
    return r2d2_learner.compute_loss_and_priorities_from_agent_outputs(
        ao, r2d2_learner.AgentOutput(act, qt), env, ao, 0.997, abandoned=ab, **kw)
  L = _lib.lib()
  names = ('seedrl_r2d2_loss_fwd_bwd', 'seedrl_r2d2_retrace_loss_fwd_bwd')
  orig = [getattr(L, n) for n in names]
  for n in names:
    fa = getattr(L, n + '_abandoned')
    setattr(L, n, lambda *a, fa=fa: fa(*a[:8], None, *a[8:]))
  try:
    return r2d2_learner.compute_loss_and_priorities_from_agent_outputs(
        ao, r2d2_learner.AgentOutput(act, qt), env, ao, 0.997, **kw)
  finally:
    for n, f in zip(names, orig):
      setattr(L, n, f)


@pytest.mark.parametrize('rule,param', R2D2_RUNS)
def test_r2d2_null_and_zero_mask_bit_identical(rule, param):
  inp = R.r2d2_inputs(101, 64, A, seed=3)
  base = _r2d2(inp, rule, param, None)
  for got in (_r2d2(inp, rule, param, None, null_entry=True),
              _r2d2(inp, rule, param, torch.zeros(101, 64, dtype=torch.bool, device='cuda'))):
    for x, y in zip(got, base):
      np.testing.assert_array_equal(_bits(x), _bits(y))


# ---- 2. float64 with random masks --------------------------------------------------------------------------------
def _relmax(a, w):
  a, w = np.asarray(a, np.float64), np.asarray(w, np.float64)
  return np.abs(a - w).max() / max(np.abs(w).max(), 1e-30)


def _vtrace_float64(bn, monkeypatch, ecp=ECP):
  monkeypatch.setattr(VR, 'vtrace_from_importance_weights', R.masked_vtrace(bn['ab'][1:]))
  return VR.loss_and_grads(_settings(), bn['ll'], bn['lb'], bn['bl'], bn['act'], bn['rew'], bn['done'], ecp,
                           torch.float64)


def _check_vtrace(got, ref, ab):
  total, logs, dl, db, _, vs, pg = ref
  assert _relmax(got['vs'].cpu(), vs) < 1e-5
  assert _relmax(got['pg_advantages'].cpu(), pg) < 1e-5
  assert _relmax(got['dbaseline'].cpu(), db) < 1e-5
  assert _relmax(got['dlogits'].cpu(), dl) < 2e-4
  lt = got['loss_terms'].cpu().numpy()
  for name, key in learner._LOG_NAMES:
    w = float(logs[name])
    assert abs(lt[_lib.LT[key]] - w) <= 1e-4 * max(abs(w), 1e-2), (name, lt[_lib.LT[key]], w)
  m = ab[1:]
  assert m.any()
  assert np.all(got['dbaseline'].cpu().numpy()[:-1][m] == 0)
  assert np.all(got['pg_advantages'].cpu().numpy()[m] == 0)


def _float64_cases():
  cases = [(21, 64, 0), (21, 256, 0), (21, 65536, 1), (21, 256, 1)]
  return cases + [(T + 1, 512, 1) for T in STREAM_TS]


@pytest.mark.parametrize('T1,B,stream', _float64_cases())
def test_vtrace_against_float64(T1, B, stream, monkeypatch):
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  bn = _vtrace_batch(T1, B, seed=T1 * 7 + B)
  got = _plain(_cuda(bn), torch.as_tensor(bn['ab']).cuda())
  _check_vtrace(got, _vtrace_float64(bn, monkeypatch), bn['ab'])


@pytest.mark.parametrize('B,stream', [(64, 0), (65536, 1)])
def test_vtrace_popart_against_float64(B, stream):
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  T1 = 21
  bn = _vtrace_batch(T1, B, seed=B + 11)
  got = _popart(_cuda(bn), torch.as_tensor(bn['ab']).cuda())
  mu1, mu2, sigma, mu = 0.3, 2.0, 1.2, -0.1
  s = min(max(np.sqrt(np.float64(np.float32(mu2)) - np.float64(np.float32(mu1)) ** 2), 1e-6), 1e6)
  u = s * (np.float64(np.float32(sigma)) * bn['lb'] + np.float64(np.float32(mu))) + np.float64(np.float32(mu1))
  lsm = lambda x: x - np.log(np.exp(x - x.max(-1, keepdims=True)).sum(-1, keepdims=True)) - x.max(-1, keepdims=True)
  a = bn['act'][:-1, :, None]
  lr = (np.take_along_axis(lsm(bn['ll'][:-1].astype(np.float64)), a, -1) -
        np.take_along_axis(lsm(bn['bl'][:-1].astype(np.float64)), a, -1))[..., 0]
  vs, pg = R.vtrace(lr, 0.97 * (1.0 - bn['done'][1:]), bn['rew'][1:], u[:-1], u[-1], bn['ab'][1:], lambda_=0.95)
  assert _relmax(got['vs'].cpu(), vs) < 1e-5
  assert _relmax(got['pg_advantages'].cpu(), pg) < 1e-5
  m = bn['ab'][1:]
  assert np.all(got['pg_advantages'].cpu().numpy()[m] == 0)
  np.testing.assert_allclose(got['vs'].cpu().numpy()[m], u[:-1][m], rtol=1e-6, atol=1e-6 * np.abs(u).max())
  beta = 1e-2
  mu1n = mu1 + beta * (vs.mean() - mu1)
  mu2n = mu2 + beta * ((vs * vs).mean() - mu2)
  np.testing.assert_allclose(got['mom'].cpu().numpy(), [mu1n, mu2n], rtol=1e-5)


@pytest.mark.parametrize('rule,param', R2D2_RUNS + [('retrace', 1.0)])
def test_r2d2_against_float64(rule, param):
  T, B = 101, 64
  inp = R.r2d2_inputs(T, B, A, seed=17)
  q, qt, act, rew, done, ab, w = inp
  loss, prio, dq = _r2d2(inp, rule, param, torch.as_tensor(ab).cuda())
  ref = R.r2d2_loss(q, qt, act, rew, done, ab, 0.997, rule, param, weights=w)
  assert _relmax(loss.cpu(), ref['loss']) < 1e-4
  assert _relmax(prio.cpu(), ref['priorities']) < 1e-4
  assert _relmax(dq.cpu(), ref['dq']) < 1e-4
  masked = np.zeros((T, B), bool)
  masked[:-1] = ab[1:]
  assert masked.any() and np.all(dq.cpu().numpy()[masked] == 0)


# ---- 3. truncation equivalence -----------------------------------------------------------------------------------
@pytest.mark.parametrize('B,stream,k', [(64, 0, 9), (512, 1, 12), (64, 0, 1)])
def test_vtrace_truncation_equivalence(B, stream, k):
  _lib.lib().seedrl_debug_set_loss_stream(stream)
  T1 = 21
  bn = _vtrace_batch(T1, B, seed=5, ab_p=0.0)
  bn['ab'][:] = False
  bn['ab'][k + 1] = True
  bn['done'][k + 1] = True
  full = _plain(_cuda(bn), torch.as_tensor(bn['ab']).cuda())
  cut = {key: (v[:k + 1] if key != 'ab' else None) for key, v in bn.items()}
  short = _plain(_cuda({key: v for key, v in cut.items() if v is not None}), None)
  for key in ('vs', 'pg_advantages'):
    np.testing.assert_allclose(full[key].cpu().numpy()[:k], short[key].cpu().numpy()[:k], rtol=1e-5,
                               atol=1e-5 * float(short[key].abs().max()))


@pytest.mark.parametrize('rule,param', [('n_step', 1), ('n_step', 3), ('n_step', 5), ('retrace', 0.95)])
def test_r2d2_truncation_equivalence(rule, param):
  T, B, k = 101, 64, 60
  q, qt, act, rew, done, ab, w = R.r2d2_inputs(T, B, A, seed=23)
  ab[:] = False
  ab[k + 1] = True
  done[k + 1] = True
  _, _, dq_full = _r2d2((q, qt, act, rew, done, ab, w), rule, param, torch.as_tensor(ab).cuda())
  cut = tuple(x[:k + 1] for x in (q, qt, act, rew, done, ab)) + (w,)
  _, _, dq_cut = _r2d2(cut, rule, param, None)
  # dq rows < k are -w td / B of the targets of rows <= k
  np.testing.assert_allclose(dq_full.cpu().numpy()[:k], dq_cut.cpu().numpy()[:k], rtol=1e-5,
                             atol=1e-5 * float(dq_cut.abs().max()))


# ---- 4. learner steps --------------------------------------------------------------------------------------------
@pytest.mark.parametrize('popart', [False, True])
def test_vtrace_learner_step_passes_the_mask(popart, monkeypatch):
  from seed_rl_b200.common import optimizers, utils
  from seed_rl_b200.dmlab import networks
  T1, B, obs = 6, 4, (84, 84, 4)
  rng = np.random.default_rng(2)
  done, ab = R.masks(T1, B, 3)
  c = lambda x: torch.as_tensor(x).cuda()
  env = utils.EnvOutput(c(rng.normal(size=(T1, B)).astype(np.float32)), c(done),
                        c(rng.integers(0, 256, (T1, B) + obs, dtype=np.uint8)), c(ab),
                        torch.zeros(T1, B, dtype=torch.int32, device='cuda'))
  ao = networks.AgentOutput(c(rng.integers(0, A, (T1, B))), c(rng.normal(size=(T1, B, A)).astype(np.float32)),
                            torch.zeros(T1, B, device='cuda'))
  state = (torch.zeros(B, 256, device='cuda'), torch.zeros(B, 256, device='cuda'))
  un = learner.Unroll(state, c(rng.integers(0, A, (T1, B))), env, ao)
  agent = networks.ImpalaDeep(A, obs, seed=0, conv_mode='simt')
  step = learner.LearnerStep(agent, optimizers.Adam(1e-4), settings=_settings(popart=popart, bootstrap_abandoned=True),
                             check_errors_every=0)
  with torch.no_grad():
    outs, _ = agent(un.prev_actions, env, state, unroll=True, is_training=True)
    ll, lb = outs.policy_logits.clone(), outs.baseline.clone()
  ecp = agent.entropy_cost_param.clone()
  if popart:
    mom, comp = agent.popart_moments.clone(), agent.popart_compensation.clone()
  step.compute_gradients(un)
  r = agent._loss_grads
  if popart:
    # the step's output gradients are those of the PopArt loss on its own outputs, with the mask
    args = (step.settings, ll, lb, ao.policy_logits, ao.action, env.reward, env.done, ecp)
    want = learner.popart_loss_fwd_bwd(*args, mom.clone(), comp.clone(), torch.zeros(2, device='cuda'),
                                       abandoned=env.abandoned)
    plain = learner.popart_loss_fwd_bwd(*args, mom.clone(), comp.clone(), torch.zeros(2, device='cuda'))
    for k in ('dlogits', 'dbaseline'):
      np.testing.assert_array_equal(_bits(r[k]), _bits(want[k]), err_msg=k)
    assert not torch.equal(r['dbaseline'], plain['dbaseline'])
    return
  bn = dict(ll=ll.cpu().numpy(), lb=lb.cpu().numpy(), bl=ao.policy_logits.cpu().numpy(), act=ao.action.cpu().numpy(),
            rew=env.reward.cpu().numpy(), done=done, ab=ab)
  ref = _vtrace_float64(bn, monkeypatch, float(ecp))
  assert _relmax(r['dbaseline'].cpu(), ref[3]) < 1e-5
  assert _relmax(r['dlogits'].cpu(), ref[2]) < 2e-4
  assert np.all(r['dbaseline'].cpu().numpy()[:-1][ab[1:]] == 0)


@pytest.mark.parametrize('rule', ['n_step', 'retrace'])
def test_r2d2_learner_step_passes_the_mask(rule):
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils
  Ar, obs, S, T, B, burn = 6, (36, 36, 1), 4, 12, 3, 4
  st = r2d2_learner.default_settings(burn_in=burn, unroll_length=T - burn - 1, bellman_target=rule,
                                     bootstrap_abandoned=True)
  rng = np.random.default_rng(4)
  done, ab = R.masks(T, B, 5)
  ab[burn + 2] = True
  done |= ab
  c = lambda x: torch.as_tensor(x).cuda()
  env = utils.EnvOutput(c(rng.normal(size=(T, B)).astype(np.float32)), c(done),
                        c(rng.integers(0, 256, (T, B) + obs, dtype=np.uint8)), c(ab),
                        torch.zeros(T, B, dtype=torch.int32, device='cuda'))
  agent = networks.DuelingLSTMDQNNet(Ar, obs, S, seed=1, gemm_mode='simt')
  target = networks.DuelingLSTMDQNNet(Ar, obs, S, seed=2, gemm_mode='simt')
  state = agent.initial_state(B)
  act = c(rng.integers(0, Ar, (T, B)).astype(np.int32))
  un = r2d2_learner.Unroll(state, torch.zeros(B, device='cuda'), c(rng.integers(0, Ar, (T, B)).astype(np.int32)), env,
                           r2d2_learner.AgentOutput(act, torch.zeros(T, B, Ar, device='cuda')))
  w = torch.ones(B, device='cuda')
  step = r2d2_learner.R2D2LearnerStep(agent, target, optimizers.Adam(1e-4), settings=st)
  loss, prio, _, _ = step.compute_gradients(r2d2_learner.SampledUnrolls(un, torch.arange(B), w))
  _, want_prio, dq = r2d2_learner.compute_loss_and_priorities(
      agent, target, state, un.prev_actions, env, un.agent_outputs, gamma=st.discounting, burn_in=burn,
      importance_weights=w, n_steps=st.n_steps, bellman_target=rule, retrace_lambda=st.retrace_lambda,
      abandoned=env.abandoned)
  np.testing.assert_array_equal(_bits(prio), _bits(want_prio))
  masked = np.zeros((T - burn, B), bool)
  masked[:-1] = ab[burn + 1:]
  assert masked.any() and np.all(dq.cpu().numpy()[masked] == 0)
  _, plain_prio, _ = r2d2_learner.compute_loss_and_priorities(
      agent, target, state, un.prev_actions, env, un.agent_outputs, gamma=st.discounting, burn_in=burn,
      importance_weights=w, n_steps=st.n_steps, bellman_target=rule, retrace_lambda=st.retrace_lambda)
  assert not torch.equal(plain_prio, want_prio)


# ---- 5. inference host -------------------------------------------------------------------------------------------
def _actor_sequence(obs, n_envs, steps, abandon_at, seed):
  """Per step, one EnvOutput for envs 0..n_envs-1: env 0 hits a time limit at step `abandon_at` (the reference
  actor's sequence: the final observation with done=False and its reward, then the reset observation with
  done=True, abandoned=True and reward 0)."""
  from seed_rl_b200.common import utils
  rng = np.random.default_rng(seed)
  seq = []
  for s in range(steps):
    rew = rng.normal(size=n_envs).astype(np.float32)
    done = np.zeros(n_envs, bool); ab = np.zeros(n_envs, bool)
    if s == abandon_at + 1:
      done[0] = ab[0] = True
      rew[0] = 0.
    seq.append(utils.EnvOutput(rew, done, rng.integers(0, 256, (n_envs,) + obs, dtype=np.uint8), ab,
                               np.full(n_envs, s, np.int32)))
  return seq


def _vtrace_host(allow, graph):   # eager only
  from seed_rl_b200.agents.vtrace import learner_loop
  from seed_rl_b200.dmlab import networks
  obs = (84, 84, 4)
  agent = networks.ImpalaDeep(A, obs, seed=3)
  return learner_loop.InferenceHost(agent, 2, 3, 2, obs, allow_abandoned=allow), obs


def _r2d2_host(allow, graph):
  from seed_rl_b200.agents.r2d2 import learner_loop
  from seed_rl_b200.atari import networks
  obs = (36, 36, 1)
  st = r2d2_learner.default_settings(burn_in=1, unroll_length=3, bootstrap_abandoned=allow)
  agent = networks.DuelingLSTMDQNNet(6, obs, 4, seed=1, gemm_mode='simt')
  return learner_loop.R2D2InferenceHost(agent, num_envs=3, num_eval_envs=1, inference_batch_size=2,
                                        observation_shape=obs, settings=st, unroll_queue_max_size=-1,
                                        cuda_graph=graph), obs


@pytest.mark.parametrize('agent,graph', [('vtrace', False), ('r2d2', False), ('r2d2', True)])
def test_inference_host_abandonment(agent, graph):
  make = _vtrace_host if agent == 'vtrace' else _r2d2_host
  ids, run_ids = np.array([0, 1], np.int32), np.array([7, 8], np.int64)
  raw = np.zeros(2, np.float32)
  # accepted, and the completed unroll's abandoned column is the one sent
  host, obs = make(True, graph)
  # the V-trace host's unroll is 3 + 1 rows: 3 steps complete none (its capacity-1 queue has no consumer here)
  n_steps = 3 if agent == 'vtrace' else 7
  seq = _actor_sequence(obs, 2, n_steps, abandon_at=1, seed=0)
  for env in seq:
    host.inference(ids, run_ids, env, raw)
  torch.cuda.synchronize()
  if agent == 'r2d2':
    got = host.unroll_queue.dequeue_many(host.unroll_queue.size())
    col = got.env_outputs.abandoned.cpu().numpy()
    steps = got.env_outputs.episode_step.cpu().numpy()
    assert col.shape == steps.shape and col.sum() >= 1
    assert np.all(steps[col] == 2)                       # only env 0's reset row was sent abandoned
  # abandoned without done raises, before any table is touched
  bad = seq[2]._replace(done=np.zeros(2, bool), abandoned=np.array([True, False]))
  before = host.env_run_ids.copy()
  with pytest.raises(ValueError):
    host.inference(ids, run_ids + 1, bad, raw)
  np.testing.assert_array_equal(host.env_run_ids, before)
  # without the flag it raises as before
  host, obs = make(False, graph)
  host.inference(ids, run_ids, seq[0], raw)
  host.inference(ids, run_ids, seq[1], raw)
  with pytest.raises(ValueError, match='Abandoned done states are not supported'):
    host.inference(ids, run_ids, seq[2], raw)
