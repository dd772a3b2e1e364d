"""GPU parity tests proper: every CUDA entry point, through the C-ABI, against the CPU
oracle on the same seeded inputs, against the committed golden fixtures, and -- at the
BASELINE sizes -- through size-independent properties.  Run with `-m gpu` on an H100.

Stated tolerances (fp32):
  V-trace / losses          rtol=atol=1e-5   (expf ulp differences x 20-step accumulation)
  action indices            bit-exact (injected Gumbel noise)
  network activations       rtol 2e-4, atol 2e-5 vs torch-CPU fp32 (different summation order,
                            x*(1/255) vs x/255)
  network gradients         rtol 2e-3 of the tensor's max-abs (long reductions)
  Adam                      rtol=1e-6 atol=1e-7 per step
"""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import learner_oracle, loss_oracle, net_oracle, optim_oracle, store_oracle, vtrace_oracle
from test_oracle_golden import (FULL_EXPECT, FULL_ROWS, OVERLAP_EXPECT, OVERLAP_ROWS)

pytestmark = pytest.mark.gpu

G = np.load(os.path.join(os.path.dirname(__file__), 'golden', 'vtrace_golden.npz'))


def _cuda(x):
  return torch.as_tensor(np.asarray(x)).cuda()


def _inputs(prefix):
  names = ['target_action_log_probs', 'behaviour_action_log_probs', 'discounts', 'rewards',
           'values', 'bootstrap_value']
  return {n: G['%s_%s' % (prefix, n)].astype(np.float32) for n in names}


def _relerr(a, b):
  a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
  return float(np.abs(a - b).max() / (np.abs(b).max() + 1e-30))


# ---------------------------------------------------------------- (a1) V-trace
def test_vtrace_golden_known_answer():
  from seed_rl_b200.common import vtrace
  i = {k: _cuda(v) for k, v in _inputs('A').items()}
  r = vtrace.from_importance_weights(**i, clip_rho_threshold=3.7, clip_pg_rho_threshold=2.2)
  np.testing.assert_allclose(r.vs.cpu().numpy(), G['A_gt_vs'], rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r.pg_advantages.cpu().numpy(), G['A_gt_pg'], rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r.vs.cpu().numpy(), G['A_ref_vs'], rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('case,kw', [
    ('B1', {}),
    ('B2', dict(clip_rho_threshold=None, clip_pg_rho_threshold=None)),
    ('B3', dict(clip_rho_threshold=3.7, clip_pg_rho_threshold=2.2, lambda_=0.9))])
def test_vtrace_cfg1_T20_B64(case, kw):
  from seed_rl_b200.common import vtrace
  i = {k: _cuda(v) for k, v in _inputs('B').items()}
  r = vtrace.from_importance_weights(**i, **kw)
  np.testing.assert_allclose(r.vs.cpu().numpy(), G[case + '_ref_vs'], rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r.pg_advantages.cpu().numpy(), G[case + '_ref_pg'], rtol=1e-5, atol=1e-5)


def test_vtrace_lambda_done_and_trailing_dims_and_ragged():
  from seed_rl_b200.common import vtrace
  v = G['C_values']
  disc = (0.99 * (~G['C_done'])).astype(np.float32)
  r = vtrace.from_importance_weights(_cuda(G['C_tlp']), _cuda(G['C_blp']), _cuda(disc),
                                     _cuda(G['C_rewards']), _cuda(v[:-1]), _cuda(v[-1]), lambda_=0.95)
  np.testing.assert_allclose(r.vs.cpu().numpy(), G['C_adv_targets'], rtol=1e-5, atol=1e-5)
  i = {k: _cuda(G['D_' + k]) for k in ['target_action_log_probs', 'behaviour_action_log_probs',
                                        'discounts', 'rewards', 'values', 'bootstrap_value']}
  r = vtrace.from_importance_weights(**i)
  assert tuple(r.vs.shape) == (7, 3, 2)
  np.testing.assert_allclose(r.vs.cpu().numpy(), G['D_ref_vs'], rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r.pg_advantages.cpu().numpy(), G['D_ref_pg'], rtol=1e-5, atol=1e-5)
  # ragged sizes incl. T not a multiple of the prefetch chunk, B not a multiple of the block
  rng = np.random.default_rng(5)
  for T, B in [(1, 1), (3, 7), (20, 129), (33, 1000), (100, 5)]:
    a = dict(target_action_log_probs=rng.uniform(-2, 2, (T, B)), behaviour_action_log_probs=rng.uniform(-2, 2, (T, B)),
             discounts=0.99 * (rng.random((T, B)) < 0.9), rewards=rng.normal(size=(T, B)),
             values=rng.normal(size=(T, B)), bootstrap_value=rng.normal(size=(B,)))
    a = {k: x.astype(np.float32) for k, x in a.items()}
    want = vtrace_oracle.from_importance_weights(**a, lambda_=0.97)
    got = vtrace.from_importance_weights(**{k: _cuda(x) for k, x in a.items()}, lambda_=0.97)
    np.testing.assert_allclose(got.vs.cpu().numpy(), want.vs, rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(got.pg_advantages.cpu().numpy(), want.pg_advantages, rtol=1e-5, atol=1e-5)
  # empty
  e = torch.zeros([0, 4]).cuda()
  r = vtrace.from_importance_weights(e, e, e, e, e, torch.zeros([4]).cuda())
  assert tuple(r.vs.shape) == (0, 4)
  with pytest.raises(ValueError):
    vtrace.from_importance_weights(e, e, e, e, e, torch.zeros([1, 4]).cuda())


def test_vtrace_full_size_properties():
  """Size-independent properties at a streaming size (B = 2^18 columns)."""
  from seed_rl_b200.common import vtrace
  g = torch.Generator(device='cuda').manual_seed(0)
  T, B = 20, 1 << 18
  tlp = torch.rand(T, B, device='cuda', generator=g) * 4 - 2
  rew = torch.randn(T, B, device='cuda', generator=g)
  val = torch.randn(T, B, device='cuda', generator=g)
  boot = torch.randn(B, device='cuda', generator=g)
  disc = torch.full((T, B), 0.99, device='cuda')
  # on-policy (rho=1), lambda=1, no clipping: vs_t == n-step discounted return + bootstrap
  r = vtrace.from_importance_weights(tlp, tlp, disc, rew, val, boot)
  ret = boot.clone()
  rets = []
  for t in range(T - 1, -1, -1):
    ret = rew[t] + 0.99 * ret
    rets.append(ret)
  want = torch.stack(rets[::-1])
  assert float((r.vs - want).abs().max()) < 2e-4
  # discount 0 everywhere: vs = V + rho_clipped*(r - V), pg = rho_clipped*(r - V)
  blp = torch.rand(T, B, device='cuda', generator=g) * 4 - 2
  r = vtrace.from_importance_weights(tlp, blp, torch.zeros_like(disc), rew, val, boot)
  rho = torch.exp(tlp - blp).clamp(max=1.0)
  assert float((r.pg_advantages - rho * (rew - val)).abs().max()) < 1e-5
  assert float((r.vs - (val + rho * (rew - val))).abs().max()) < 1e-5
  # column independence: permuting columns permutes outputs
  perm = torch.randperm(B, device='cuda')
  r1 = vtrace.from_importance_weights(tlp, blp, disc, rew, val, boot)
  r2 = vtrace.from_importance_weights(tlp[:, perm], blp[:, perm], disc[:, perm], rew[:, perm],
                                      val[:, perm], boot[perm])
  assert torch.equal(r1.vs[:, perm], r2.vs)


# ---------------------------------------------------------------- (a3) categorical
def test_categorical_log_prob_entropy_sample():
  from seed_rl_b200.common import parametric_distribution as pd
  T, B, A = 7, 2, 3            # reference tests/vtrace_test.py:88-115
  logits = np.arange(T * B * A, dtype=np.float32).reshape(T, B, A) + 10
  actions = np.random.default_rng(0).integers(0, A - 1, size=(T, B)).astype(np.int32)
  d = pd.categorical_distribution(A, 'int32')
  got = d.log_prob(_cuda(logits), _cuda(actions)).cpu().numpy()
  np.testing.assert_allclose(got, vtrace_oracle.categorical_log_prob(logits, actions), rtol=1e-5, atol=1e-5)
  rng = np.random.default_rng(1)
  for N, A in [(1, 1), (64, 18), (1000, 9), (5, 40)]:
    lg = (rng.normal(size=(N, A)) * 3).astype(np.float32)
    act = rng.integers(0, A, N)
    d = pd.categorical_distribution(A, 'int64')
    np.testing.assert_allclose(d.log_prob(_cuda(lg), _cuda(act)).cpu().numpy(),
                               vtrace_oracle.categorical_log_prob(lg, act), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(d.entropy(_cuda(lg)).cpu().numpy(),
                               vtrace_oracle.categorical_entropy(lg), rtol=1e-5, atol=1e-5)
    noise = rng.gumbel(size=(N, A)).astype(np.float32)
    got = d.sample(_cuda(lg), gumbel_noise=_cuda(noise)).cpu().numpy()
    assert got.dtype == np.int64
    np.testing.assert_array_equal(got, vtrace_oracle.categorical_sample_from_noise(lg, noise))  # bit-exact
  # Philox path: frequencies follow softmax (statistical, like reference utils_test.py:353-365)
  lg = np.log(np.array([[0.1, 0.2, 0.3, 0.4]], np.float32)).repeat(200000, 0)
  s = pd.categorical_distribution(4, 'int64').sample(_cuda(lg), seed=7, offset=3).cpu().numpy()
  freq = np.bincount(s, minlength=4) / len(s)
  np.testing.assert_allclose(freq, [0.1, 0.2, 0.3, 0.4], atol=0.01)


# ---------------------------------------------------------------- (a2) fused loss
def _loss_case(T1, B, A, seed, **cfgkw):
  rng = np.random.default_rng(seed)
  return dict(
      ll=rng.normal(size=(T1, B, A)).astype(np.float32), lb=rng.normal(size=(T1, B)).astype(np.float32),
      bl=rng.normal(size=(T1, B, A)).astype(np.float32), act=rng.integers(0, A, (T1, B)),
      rew=(rng.normal(size=(T1, B)) * 2).astype(np.float32), done=rng.random((T1, B)) < 0.1), cfgkw


@pytest.mark.parametrize('T1,B,A,kw', [
    (21, 64, 18, {}),
    (21, 64, 18, dict(kl_cost=0.3, entropy_cost=0.01, max_abs_reward=1.0, target_entropy=1.5, lambda_=0.9)),
    (2, 1, 1, {}), (6, 3, 5, dict(kl_cost=0.1)), (21, 70, 18, {}), (101, 33, 9, {}), (4, 257, 2, {})])
def test_vtrace_loss_fwd_bwd_vs_oracle(T1, B, A, kw):
  from seed_rl_b200.agents.vtrace import learner
  c, _ = _loss_case(T1, B, A, 11)
  cfg = loss_oracle.default_config(**kw)
  total, logs, dl, db, dep, aux = loss_oracle.loss_and_grads(cfg, c['ll'], c['lb'], c['bl'], c['act'], c['rew'], c['done'])
  st = learner.default_loss_settings(**kw)
  ecp = torch.tensor(np.log(cfg.entropy_cost) / cfg.entropy_cost_adjustment_speed, dtype=torch.float32).cuda()
  for _ in range(2):   # second launch exercises the self-resetting scratch
    r = learner.vtrace_loss_fwd_bwd(st, _cuda(c['ll']), _cuda(c['lb']), _cuda(c['bl']), _cuda(c['act']),
                                    _cuda(c['rew']), _cuda(c['done']), ecp, want_vtrace=True)
  lt = r['loss_terms'].cpu().numpy()
  from seed_rl_b200 import _lib
  names = {'losses/total': 'total', 'losses/policy': 'policy', 'losses/V': 'V', 'losses/entropy': 'entropy',
           'losses/kl': 'kl', 'V/value function': 'v_mean', 'V/L2 error': 'v_l2_error',
           'policy/entropy': 'mean_entropy', 'policy/entropy_cost': 'entropy_cost',
           'policy/kl(old|new)': 'mean_kl', 'policy/max_action_abs(before_tanh)': 'max_action_abs'}
  for k, key in names.items():
    np.testing.assert_allclose(lt[_lib.LT[key]], logs[k], rtol=2e-5, atol=2e-6, err_msg=k)
  np.testing.assert_allclose(r['vs'].cpu().numpy(), aux['vs'].numpy(), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r['pg_advantages'].cpu().numpy(), aux['pg_advantages'].numpy(), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r['dlogits'].cpu().numpy(), dl, rtol=1e-4, atol=1e-7)
  np.testing.assert_allclose(r['dbaseline'].cpu().numpy(), db, rtol=1e-4, atol=1e-7)
  np.testing.assert_allclose(float(r['d_entropy_cost_param']), dep, rtol=1e-4, atol=1e-8)
  assert float(r['dlogits'][-1].abs().max()) == 0.0 and float(r['dbaseline'][-1].abs().max()) == 0.0


@pytest.mark.parametrize('T1,B,A,kw', [
    (6, 2368, 18, {}),                      # BB=8 (TMA box <= 256 floats), 296 tiles
    (21, 2368, 9, {}), (5, 1184, 19, dict(kl_cost=0.2)),   # DMLab / football action counts
    (21, 3552, 18, dict(kl_cost=0.3, entropy_cost=0.01, max_abs_reward=1.0, target_entropy=1.5, lambda_=0.9)),
    (101, 4736, 18, {}),                    # BB=8, 592 tiles: four per CTA, ring wraps
    (11, 1184, 6, dict(kl_cost=0.1)),       # BB=8
    (9, 2960, 15, {}),                      # BB=16, 185 tiles, run-time A
    (3, 592, 2, {})])                       # BB=4, T=2
def test_vtrace_loss_streaming_kernel_vs_oracle(T1, B, A, kw):
  """Large aligned batches take vtrace_loss_stream_kernel (TMA bulk-copy ring, persistent
  CTAs): same parity bar against the oracle as vtrace_loss_kernel, the two kernels agree
  with each other to fp32 summation-order noise, and the result is deterministic."""
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.vtrace import learner
  c, _ = _loss_case(T1, B, A, 13)
  cfg = loss_oracle.default_config(**kw)
  total, logs, dl, db, dep, aux = loss_oracle.loss_and_grads(cfg, c['ll'], c['lb'], c['bl'], c['act'], c['rew'], c['done'])
  st = learner.default_loss_settings(**kw)
  ecp = torch.tensor(np.log(cfg.entropy_cost) / cfg.entropy_cost_adjustment_speed, dtype=torch.float32).cuda()
  args = [_cuda(c[k]) for k in ('ll', 'lb', 'bl', 'act', 'rew', 'done')]
  res = {}
  try:
    for stream in (0, 1, 1):
      _lib.check(_lib.lib().seedrl_debug_set_loss_stream(stream))
      r = learner.vtrace_loss_fwd_bwd(st, *args, ecp, want_vtrace=True)
      torch.cuda.synchronize()
      res.setdefault(stream, []).append({k: v.clone() for k, v in r.items() if torch.is_tensor(v)})
  finally:
    _lib.check(_lib.lib().seedrl_debug_set_loss_stream(1))
  r, r_again, old = res[1][0], res[1][1], res[0][0]
  lt = r['loss_terms'].cpu().numpy()
  for k, key in {'losses/total': 'total', 'losses/policy': 'policy', 'losses/V': 'V', 'losses/entropy': 'entropy',
                 'losses/kl': 'kl', 'V/value function': 'v_mean', 'V/L2 error': 'v_l2_error',
                 'policy/entropy': 'mean_entropy', 'policy/kl(old|new)': 'mean_kl',
                 'policy/max_action_abs(before_tanh)': 'max_action_abs'}.items():
    np.testing.assert_allclose(lt[_lib.LT[key]], logs[k], rtol=3e-5, atol=3e-6, err_msg=k)
  np.testing.assert_allclose(r['vs'].cpu().numpy(), aux['vs'].numpy(), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r['pg_advantages'].cpu().numpy(), aux['pg_advantages'].numpy(), rtol=1e-5, atol=1e-5)
  np.testing.assert_allclose(r['dlogits'].cpu().numpy(), dl, rtol=1e-4, atol=1e-9)
  np.testing.assert_allclose(r['dbaseline'].cpu().numpy(), db, rtol=1e-4, atol=1e-9)
  np.testing.assert_allclose(float(r['d_entropy_cost_param']), dep, rtol=1e-4, atol=1e-8)
  assert float(r['dlogits'][-1].abs().max()) == 0.0 and float(r['dbaseline'][-1].abs().max()) == 0.0
  for k in ('dlogits', 'dbaseline', 'vs', 'pg_advantages'):
    np.testing.assert_allclose(r[k].cpu().numpy(), old[k].cpu().numpy(), rtol=1e-4,
                               atol=1e-5 if k in ('vs', 'pg_advantages') else 1e-9, err_msg=k)
    assert torch.equal(r[k], r_again[k]), k
  assert torch.equal(r['loss_terms'], r_again['loss_terms'])


def test_vtrace_loss_large_batch_properties():
  """B = 16384 (4096 CTAs): gradient rows sum to zero over actions (softmax Jacobian),
  loss is invariant to a per-row logit shift, partial reduction is deterministic."""
  from seed_rl_b200.agents.vtrace import learner
  g = torch.Generator(device='cuda').manual_seed(1)
  T1, B, A = 21, 16384, 18
  ll = torch.randn(T1, B, A, device='cuda', generator=g); lb = torch.randn(T1, B, device='cuda', generator=g)
  bl = torch.randn(T1, B, A, device='cuda', generator=g)
  act = torch.randint(0, A, (T1, B), device='cuda', generator=g)
  rew = torch.randn(T1, B, device='cuda', generator=g); done = torch.rand(T1, B, device='cuda', generator=g) < 0.02
  st = learner.default_loss_settings()
  ecp = torch.tensor(np.log(st.entropy_cost) / 10.0, dtype=torch.float32).cuda()
  r1 = learner.vtrace_loss_fwd_bwd(st, ll, lb, bl, act, rew, done, ecp)
  l1 = r1['loss_terms'].clone(); d1 = r1['dlogits'].clone()
  assert float(d1.sum(-1).abs().max()) < 1e-9
  r2 = learner.vtrace_loss_fwd_bwd(st, ll + torch.randn(T1, B, 1, device='cuda', generator=g), lb, bl, act, rew, done, ecp)
  assert abs(float(r2['loss_terms'][0] - l1[0])) < 1e-4 * max(1.0, abs(float(l1[0])))
  r3 = learner.vtrace_loss_fwd_bwd(st, ll, lb, bl, act, rew, done, ecp)
  assert torch.equal(r3['loss_terms'], l1) and torch.equal(r3['dlogits'], d1)


# ---------------------------------------------------------------- (a4) Adam
def test_adam_keras_semantics():
  from seed_rl_b200.common import optimizers
  rng = np.random.default_rng(2)
  n = 100003
  p = rng.normal(size=n).astype(np.float32); m = np.zeros(n, np.float32); v = np.zeros(n, np.float32)
  opt = optimizers.Adam(optimizers.PolynomialDecay(4.8e-4, 1000, 0.0), beta_1=0.0, epsilon=3.125e-7)
  pc = _cuda(p)
  for it in range(5):
    g = rng.normal(size=n).astype(np.float32) * 0.1
    lr = optim_oracle.polynomial_decay(4.8e-4, it, 1000)
    p, m, v = optim_oracle.keras_adam_step(p, g, m, v, it, lr, 0.0, 0.999, 3.125e-7)
    opt.apply_gradients(pc, _cuda(g))
    np.testing.assert_allclose(pc.cpu().numpy(), p, rtol=1e-6, atol=1e-7)
  np.testing.assert_allclose(opt.m.cpu().numpy(), m, rtol=1e-6, atol=1e-9)
  np.testing.assert_allclose(opt.v.cpu().numpy(), v, rtol=1e-6, atol=1e-12)
  # beta1 != 0, grad_scale, clamp
  opt = optimizers.Adam(1e-2)
  pc = torch.ones(8).cuda(); g = torch.full((8,), 4.0).cuda()
  opt.apply_gradients(pc, g, grad_scale=0.25, clamp_index=3, clamp_lo=0.995, clamp_hi=2.0)
  p2, _, _ = optim_oracle.keras_adam_step(np.ones(8), np.ones(8), np.zeros(8), np.zeros(8), 0, 1e-2)
  want = p2.copy(); want[3] = 0.995
  np.testing.assert_allclose(pc.cpu().numpy(), want, rtol=1e-6)


# ---------------------------------------------------------------- single kernels
def _conv_ref(x, w, b, mode):
  xt = torch.as_tensor(x)
  if mode == 2:
    xt = xt.float() / 255.0
  elif mode == 1:
    xt = torch.relu(xt)
  return net_oracle._conv_nhwc(xt, torch.as_tensor(w), None if b is None else torch.as_tensor(b), 1, True)


@pytest.mark.parametrize('cin,cout,mode,N,H,W', [
    (4, 16, 2, 3, 84, 84), (16, 16, 1, 5, 42, 42), (16, 32, 0, 2, 42, 42), (32, 32, 1, 7, 21, 21),
    (32, 32, 0, 9, 11, 11), (32, 16, 0, 2, 42, 42), (16, 16, 0, 1, 5, 3), (32, 32, 1, 40, 11, 11),
    (4, 16, 0, 2, 9, 84)])
def test_conv3x3_kernel(cin, cout, mode, N, H, W):
  from seed_rl_b200 import _lib
  rng = np.random.default_rng(cin * 100 + cout + H)
  x = rng.integers(0, 256, (N, H, W, cin), dtype=np.uint8) if mode == 2 else rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  b = rng.normal(size=(cout,)).astype(np.float32)
  mask = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  res = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  want = _conv_ref(x, w, b, mode).numpy()
  out = torch.full((N, H, W, cout), float('nan')).cuda()
  xc, wc, bc = _cuda(x), _cuda(w), _cuda(b)
  _lib.check(_lib.lib().seedrl_debug_conv3x3(cin, cout, mode, N, H, W, _lib.ptr(xc), _lib.ptr(wc), _lib.ptr(bc),
                                             None, None, _lib.ptr(out), _lib.stream_ptr()))
  np.testing.assert_allclose(out.cpu().numpy(), want, rtol=2e-4, atol=2e-5)
  mc, rc = _cuda(mask), _cuda(res)
  _lib.check(_lib.lib().seedrl_debug_conv3x3(cin, cout, mode, N, H, W, _lib.ptr(xc), _lib.ptr(wc), _lib.ptr(bc),
                                             _lib.ptr(mc), _lib.ptr(rc), _lib.ptr(out), _lib.stream_ptr()))
  np.testing.assert_allclose(out.cpu().numpy(), np.where(mask > 0, want, 0) + res, rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize('cin,cout,mode,N,H,W', [
    (4, 16, 2, 3, 84, 84), (16, 16, 1, 5, 42, 42), (16, 32, 0, 2, 42, 42), (32, 32, 1, 7, 21, 21),
    (32, 32, 0, 400, 11, 11), (4, 16, 0, 2, 7, 5)])
def test_conv3x3_wgrad_and_dgrad_kernels(cin, cout, mode, N, H, W):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  rng = np.random.default_rng(cin + cout + N)
  x = rng.integers(0, 256, (N, H, W, cin), dtype=np.uint8) if mode == 2 else rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xt = torch.as_tensor(x)
  xin = (xt.float() / 255.0) if mode == 2 else (torch.relu(xt) if mode == 1 else xt)
  xin = xin.clone().requires_grad_(True)
  wt_ = torch.tensor(w, requires_grad=True); bt = torch.zeros(cout, requires_grad=True)
  y = net_oracle._conv_nhwc(xin, wt_, bt, 1, True)
  (y * torch.as_tensor(dy)).sum().backward()
  pb = int(L.seedrl_debug_wgrad_partial_bytes())
  partial = torch.empty(pb // 4, device='cuda')
  dw = torch.full((3, 3, cin, cout), float('nan')).cuda(); db = torch.full((cout,), float('nan')).cuda()
  xc, dyc = _cuda(x), _cuda(dy)
  _lib.check(L.seedrl_debug_conv3x3_wgrad(cin, cout, mode, N, H, W, _lib.ptr(xc), _lib.ptr(dyc), _lib.ptr(dw),
                                          _lib.ptr(db), _lib.ptr(partial), pb, _lib.stream_ptr()))
  assert _relerr(dw.cpu().numpy(), wt_.grad.numpy()) < 2e-4
  assert _relerr(db.cpu().numpy(), bt.grad.numpy()) < 2e-4
  if mode != 2 and (cout, cin) in [(16, 16), (32, 16), (32, 32)]:
    wc = _cuda(w); wtc = torch.empty(9 * cin * cout).cuda()
    dx = torch.full((N, H, W, cin), float('nan')).cuda()
    _lib.check(L.seedrl_debug_conv3x3_flip(cin, cout, _lib.ptr(wc), _lib.ptr(wtc), _lib.stream_ptr()))
    _lib.check(L.seedrl_debug_conv3x3(cout, cin, 0, N, H, W, _lib.ptr(dyc), _lib.ptr(wtc), None, None, None,
                                      _lib.ptr(dx), _lib.stream_ptr()))
    assert _relerr(dx.cpu().numpy(), xin.grad.numpy()) < 2e-4


@pytest.mark.parametrize('N,H,W,C', [(3, 84, 84, 16), (2, 42, 42, 32), (5, 21, 21, 32), (2, 7, 5, 16)])
def test_maxpool_tf_same(N, H, W, C):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  rng = np.random.default_rng(H)
  x = rng.normal(size=(N, H, W, C)).astype(np.float32)
  xt = torch.tensor(x, requires_grad=True)
  y = net_oracle._maxpool_same_nhwc(xt)
  Ho, Wo = y.shape[1], y.shape[2]
  assert (Ho, Wo) == (-(-H // 2), -(-W // 2))
  dy = rng.normal(size=tuple(y.shape)).astype(np.float32)
  (y * torch.as_tensor(dy)).sum().backward()
  xc = _cuda(x); yc = torch.empty(N, Ho, Wo, C).cuda(); idx = torch.empty(N, Ho, Wo, C, dtype=torch.uint8).cuda()
  _lib.check(L.seedrl_debug_maxpool(0, N, H, W, C, _lib.ptr(xc), _lib.ptr(yc), _lib.ptr(idx), _lib.stream_ptr()))
  np.testing.assert_array_equal(yc.cpu().numpy(), y.detach().numpy())
  dx = torch.empty(N, H, W, C).cuda(); dyc = _cuda(dy)
  _lib.check(L.seedrl_debug_maxpool(1, N, H, W, C, _lib.ptr(dyc), _lib.ptr(dx), _lib.ptr(idx), _lib.stream_ptr()))
  np.testing.assert_allclose(dx.cpu().numpy(), xt.grad.numpy(), rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize('ta,tb,M,N,K', [(0, 0, 130, 70, 50), (1, 0, 256, 18, 1344), (0, 1, 64, 256, 1024),
                                         (1, 1, 33, 65, 17), (0, 0, 1, 1, 1), (0, 0, 1344, 256, 3872)])
def test_sgemm_kernel(ta, tb, M, N, K):
  from seed_rl_b200 import _lib
  rng = np.random.default_rng(M + N + K)
  A = rng.normal(size=(K, M) if ta else (M, K)).astype(np.float32)
  B = rng.normal(size=(N, K) if tb else (K, N)).astype(np.float32)
  bias = rng.normal(size=(N,)).astype(np.float32); mask = rng.normal(size=(M, N)).astype(np.float32)
  C0 = rng.normal(size=(M, N)).astype(np.float32)
  Am = np.maximum(A, 0); opA = Am.T if ta else Am; opB = B.T if tb else B
  want = np.where(mask > 0, np.maximum(opA.astype(np.float64) @ opB + bias, 0), 0) + C0
  Cc = _cuda(C0)
  ac, bc, biasc, maskc = _cuda(A), _cuda(B), _cuda(bias), _cuda(mask)
  _lib.check(_lib.lib().seedrl_debug_sgemm(ta, tb, M, N, K, _lib.ptr(ac), A.shape[1], _lib.ptr(bc), B.shape[1],
                                           _lib.ptr(Cc), N, _lib.ptr(biasc), _lib.ptr(maskc), N, 1, 1, 1,
                                           _lib.stream_ptr()))
  assert _relerr(Cc.cpu().numpy(), want) < 1e-5


# rows x width of the value head at the R2D2 suffix (101 x 64) and full (141 x 64) unroll, a row count that is odd
# and not a multiple of 128 or 8, a width that is not a multiple of 32, tiny shapes
@pytest.mark.parametrize('path,rows,width', [('rowdot', 6464, 512), ('rowdot', 9024, 512), ('rowdot', 6463, 500),
                                             ('rowdot', 37, 31), ('colsum', 6464, 512), ('colsum', 9024, 512),
                                             ('colsum', 6463, 512), ('colsum', 6465, 500), ('colsum', 33, 31)])
def test_sgemm_n1_paths(path, rows, width):
  """The two N = 1 paths of sgemm, which an epilogue flag turns off (test_sgemm_kernel sets them all):
  rowdot_kernel, C[rows] = X w + bias (the value head), and the weighted colsum_kernel, C[width] = X^T d (its weight
  gradient).  Each element within 1e-5 of the sum of the absolute products it adds, against float64: a dropped row
  or column term is ~1/rows (1/width) of that."""
  from seed_rl_b200 import _lib
  rng = np.random.default_rng(rows * 7 + width)
  X = rng.normal(size=(rows, width)).astype(np.float32)
  v = rng.normal(size=width if path == 'rowdot' else rows).astype(np.float32)
  bias = rng.normal(size=1).astype(np.float32)
  X64, v64 = X.astype(np.float64), v.astype(np.float64)
  out = _cuda(np.full(rows if path == 'rowdot' else width + 1, np.nan, np.float32))
  Xc, vc, biasc = _cuda(X), _cuda(v), _cuda(bias)
  if path == 'rowdot':
    want, scale = X64 @ v64 + bias[0], np.abs(X64) @ np.abs(v64) + abs(float(bias[0]))
    args = (0, 0, rows, 1, width, _lib.ptr(Xc), width, _lib.ptr(vc), 1, _lib.ptr(out), 1, _lib.ptr(biasc))
  else:
    want, scale = X64.T @ v64, np.abs(X64).T @ np.abs(v64)
    args = (1, 0, width, 1, rows, _lib.ptr(Xc), width, _lib.ptr(vc), 1, _lib.ptr(out), 1, None)
  _lib.check(_lib.lib().seedrl_debug_sgemm(*args, None, 0, 0, 0, 0, _lib.stream_ptr()))
  got = out.cpu().numpy()
  if path == 'colsum':
    assert np.isnan(got[width])                         # nothing written past the output
    got = got[:width]
  err = np.abs(got.astype(np.float64) - want) / scale
  assert err.max() < 1e-5, (float(err.max()), int(err.argmax()))


# ---------------------------------------------------------------- (a5) network
def _make_agent(net, A, seed=0):
  from seed_rl_b200.dmlab import networks
  cls = networks.ImpalaDeep if net == 'deep' else networks.ImpalaShallow
  agent = cls(A, (84, 84, 4), seed=seed)
  params = net_oracle.init_params(net, A, (84, 84, 4), seed=seed + 1)
  agent.load_named_parameters(params)
  return agent, params


def _batch_to_cuda(b):
  from seed_rl_b200.common import utils
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.dmlab import networks
  T1, B = b['reward'].shape
  env = utils.EnvOutput(_cuda(b['reward']), _cuda(b['done']), _cuda(b['observation']),
                        torch.zeros(T1, B, dtype=torch.bool).cuda(), torch.zeros(T1, B, dtype=torch.int32).cuda())
  ao = networks.AgentOutput(_cuda(b['action']), _cuda(b['behaviour_logits']), _cuda(b['behaviour_baseline']))
  return learner.Unroll((_cuda(b['h0']), _cuda(b['c0'])), _cuda(b['prev_actions']), env, ao)


# The shallow net's (T, B) cover the recurrence's batch-tile classes; at B = 300 the tiled LSTM kernel takes its
# non-cooperative launch (10 forward / 13 BPTT batch tiles x 16 unit groups > 132 SMs).
@pytest.mark.parametrize('net,T,B', [('deep', 3, 2), ('shallow', 3, 2), ('deep', 1, 5), ('shallow', 6, 5),
                                     ('shallow', 3, 70), ('shallow', 1, 3), ('shallow', 20, 64),
                                     ('shallow', 5, 256), ('shallow', 4, 300)])
def test_network_forward_matches_oracle(net, T, B):
  A = 18
  agent, params = _make_agent(net, A)
  assert len(agent.trainable_variables) == (39 if net == 'deep' else 13)
  b = learner_oracle.synthetic_batch(T, B, A, seed=3)
  b['done'][1, 0] = True
  rng = np.random.default_rng(9)
  b['h0'] = rng.normal(size=b['h0'].shape).astype(np.float32)
  b['c0'] = rng.normal(size=b['c0'].shape).astype(np.float32)
  u = _batch_to_cuda(b)
  pt = net_oracle.to_torch(params)
  logits, baseline, (h, c) = net_oracle.unroll(
      net, pt, torch.as_tensor(b['prev_actions']), torch.as_tensor(b['reward']), torch.as_tensor(b['done']),
      torch.as_tensor(b['observation']), (torch.as_tensor(b['h0']), torch.as_tensor(b['c0'])), A)
  noise = rng.gumbel(size=(T + 1, B, A)).astype(np.float32)
  out, (h2, c2) = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True, gumbel_noise=_cuda(noise))
  np.testing.assert_allclose(out.policy_logits.cpu().numpy(), logits.numpy(), rtol=2e-4, atol=2e-5)
  np.testing.assert_allclose(out.baseline.cpu().numpy(), baseline.numpy(), rtol=2e-4, atol=2e-5)
  np.testing.assert_allclose(h2.cpu().numpy(), h.numpy(), rtol=2e-4, atol=2e-5)
  np.testing.assert_allclose(c2.cpu().numpy(), c.numpy(), rtol=2e-4, atol=2e-5)
  # action indices: bit-exact given the kernel's own logits + injected noise
  want = vtrace_oracle.categorical_sample_from_noise(out.policy_logits.cpu().numpy(), noise)
  np.testing.assert_array_equal(out.action.cpu().numpy(), want)
  # T=1 path (inference): unroll=False on the first row reproduces row 0
  env0 = type(u.env_outputs)(*(t[0] for t in u.env_outputs))
  o1, _ = agent(u.prev_actions[0], env0, u.agent_state)
  np.testing.assert_allclose(o1.policy_logits.cpu().numpy(), logits[0].numpy(), rtol=2e-4, atol=2e-5)


@pytest.mark.parametrize('net,T,B', [('deep', 4, 3), ('shallow', 4, 3), ('shallow', 4, 300)])
def test_learner_step_gradients_and_update_match_oracle(net, T, B):
  """compute_loss -> backward -> Adam against the CPU learner (oracle) for 3 steps."""
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  A = 18
  agent, params = _make_agent(net, A)
  kw = dict(kl_cost=0.05, entropy_cost=0.01, target_entropy=2.0)
  cfg = loss_oracle.default_config(**kw)
  cpu = learner_oracle.CpuLearner(net, A, (84, 84, 4), cfg, lr=4.8e-4, beta1=0.0, eps=3.125e-7,
                                  decay_steps=100, params=params)
  opt = optimizers.Adam(optimizers.PolynomialDecay(4.8e-4, 100, 0.0), beta_1=0.0, epsilon=3.125e-7)
  step = learner.LearnerStep(agent, opt, settings=learner.default_loss_settings(**kw))
  for it in range(3):
    b = learner_oracle.synthetic_batch(T, B, A, seed=100 + it)
    b['done'][2, 1] = True
    # like with like: both sides start every iteration from the CPU learner's parameters
    # (Adam normalises gradients, so fp32 noise on near-zero gradients would otherwise
    # make the two trajectories drift by O(lr) per step).
    agent.load_named_parameters({k: v.detach().numpy() for k, v in cpu.params.items()})
    agent.entropy_cost_param.copy_(cpu.entropy_cost_param.detach())
    total, logs, g, _ = cpu.grads(b)
    u = _batch_to_cuda(b)
    loss, _ = step.compute_gradients(u)
    assert abs(float(loss) - float(total)) < 2e-4 * max(1.0, abs(float(total)))
    mine = agent.named_gradients()
    # The loss is only piecewise smooth (rho clipping, ReLU, max-pool argmax), so some
    # states are ill-conditioned: measure the ORACLE's own sensitivity to a 1e-6 relative
    # parameter perturbation and accept the larger of 2e-3 and 4x that per tensor.
    saved = {k: v.detach().clone() for k, v in cpu.params.items()}
    prng = np.random.default_rng(it)
    with torch.no_grad():
      for k, v in cpu.params.items():
        v.mul_(torch.as_tensor(1 + 1e-6 * prng.normal(size=tuple(v.shape)).astype(np.float32)))
    _, _, g_pert, _ = cpu.grads(b)
    with torch.no_grad():
      for k, v in cpu.params.items():
        v.copy_(saved[k])
    bad = []
    for k in g:
      if k == 'entropy_cost_param':
        continue
      err = _relerr(mine[k].cpu().numpy(), g[k])
      tol = max(2e-3, 4 * _relerr(g_pert[k], g[k]))
      if err > tol:
        bad.append((k, err, tol))
    assert not bad, (it, bad)
    np.testing.assert_allclose(float(mine['entropy_cost_param']), float(g['entropy_cost_param']), rtol=1e-3, atol=1e-9)
    # optimizer parity on IDENTICAL inputs: the GPU's own arena, gradient and slots through
    # the Keras-Adam oracle must reproduce the fused kernel's update.
    p0 = agent.params.cpu().numpy(); g0 = agent.grads.cpu().numpy()
    m0 = opt.m.cpu().numpy(); v0 = opt.v.cpu().numpy()
    lr = optim_oracle.polynomial_decay(4.8e-4, opt.iterations, 100)
    wp, wm, wv = optim_oracle.keras_adam_step(p0, g0, m0, v0, opt.iterations, lr, 0.0, 0.999, 3.125e-7)
    idx = agent.entropy_cost_param_index
    wp[idx] = np.clip(wp[idx], -2.0, 2.0)
    step.apply_gradients()
    np.testing.assert_allclose(agent.params.cpu().numpy(), wp, rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(opt.v.cpu().numpy(), wv, rtol=1e-6, atol=1e-30)
    cpu.step(b)
  assert opt.iterations == 3


def test_full_size_step_runs_and_is_deterministic():
  """BASELINE cfg 4 shape (ImpalaDeep, T=20, B=64): finite, reproducible, loss drops on a
  repeated batch."""
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  A = 18
  b = learner_oracle.synthetic_batch(20, 64, A, seed=1234)
  u = _batch_to_cuda(b)
  outs = []
  for rep in range(2):
    agent, _ = _make_agent('deep', A)
    step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7))
    losses = [float(step.minimize(u)[0]) for _ in range(3)]
    assert all(np.isfinite(losses))
    outs.append((losses, agent.params.clone()))
  assert outs[0][0] == outs[1][0] and torch.equal(outs[0][1], outs[1][1])   # deterministic kernels
  assert torch.isfinite(outs[0][1]).all()


# ---------------------------------------------------------------- (a7/a8) store
def _drive_gpu(store, rows, batch):
  out = []
  for i in range(0, len(rows) - len(rows) % batch, batch):
    chunk = rows[i:i + batch]
    rs = np.array([c[0] for c in chunk]); ids = np.array([c[1] for c in chunk], np.int32)
    vals = np.array([c[2] for c in chunk], np.int32)
    store.reset(ids[rs])
    cid, un = store.append(ids, torch.as_tensor(vals))
    out.append((cid.cpu().tolist(), un.cpu().tolist()))
  return out


def test_unroll_store_reference_sequences():
  """reference tests/utils_test.py:70-271 replayed on the GPU store."""
  from seed_rl_b200.common import utils
  s = utils.UnrollStore(4, 3, utils.TensorSpec([], 'int32', 'x'))
  assert _drive_gpu(s, FULL_ROWS, 3) == FULL_EXPECT
  s = utils.UnrollStore(2, 2, utils.TensorSpec([], 'int32', 'x'), num_overlapping_steps=2)
  assert _drive_gpu(s, OVERLAP_ROWS, 2) == OVERLAP_EXPECT
  s = utils.UnrollStore(2, 3, utils.TensorSpec([], 'int32', 'x'))
  with pytest.raises(ValueError):
    s.append(np.array([1, 1], np.int32), torch.tensor([42, 43], dtype=torch.int32))


def test_unroll_store_observation_rows_vs_oracle_and_time_major():
  from seed_rl_b200.common import utils
  rng = np.random.default_rng(0)
  num_envs, T = 12, 4
  specs = (utils.TensorSpec([], 'int64', 'a'), utils.TensorSpec([84, 84, 4], 'uint8', 'obs'),
           utils.TensorSpec([3], 'float32', 'f'), utils.TensorSpec([], 'bool', 'd'))
  gpu = utils.UnrollStore(num_envs, T, specs)
  gtm = utils.UnrollStore(num_envs, T, specs, time_major=True)
  cpu = store_oracle.UnrollStore(num_envs, T, [((), np.int64), ((84, 84, 4), np.uint8), ((3,), np.float32), ((), np.bool_)])
  for step in range(13):
    ids = rng.permutation(num_envs)[:rng.integers(1, num_envs + 1)].astype(np.int32)
    vals = [rng.integers(0, 100, len(ids)), rng.integers(0, 256, (len(ids), 84, 84, 4), dtype=np.uint8),
            rng.normal(size=(len(ids), 3)).astype(np.float32), rng.random(len(ids)) < 0.5]
    cid, un = gpu.append(ids, tuple(torch.as_tensor(v) for v in vals))
    cid2, un2 = gtm.append(ids, tuple(torch.as_tensor(v) for v in vals))
    wid, wun = cpu.append(ids, vals)
    assert cid.cpu().tolist() == wid.tolist()
    for a, t, w in zip(un, un2, wun):
      np.testing.assert_array_equal(a.cpu().numpy(), w)
      np.testing.assert_array_equal(t.cpu().numpy(), np.swapaxes(w, 0, 1))   # == make_time_major


def test_aggregator_reference_sequence():
  """reference tests/utils_test.py:276-286."""
  from seed_rl_b200.common import utils
  agg = utils.Aggregator(4, utils.TensorSpec([], 'int32', 'x'))
  assert agg.read([0, 1, 2, 3]).cpu().tolist() == [0, 0, 0, 0]
  agg.add([0, 1], torch.tensor([42, 43], dtype=torch.int32))
  assert agg.read([0, 1, 2, 3]).cpu().tolist() == [42, 43, 0, 0]
  agg.reset([0])
  assert agg.read([0, 1, 2, 3]).cpu().tolist() == [0, 43, 0, 0]
  agg.replace([0, 2], torch.tensor([1, 2], dtype=torch.int32))
  assert agg.read([0, 1, 2, 3]).cpu().tolist() == [1, 43, 2, 0]
  with pytest.raises(ValueError):
    agg.replace([1, 1], torch.tensor([1, 2], dtype=torch.int32))


def test_native_library_is_what_ran():
  from seed_rl_b200 import _lib
  assert _lib.launch_count() > 0
  maps = open('/proc/self/maps').read()
  assert 'libseedrl_b200.so' in maps
