"""GPU: ImpalaDeep on frames of 1 to 16 channels (grayscale, stacked RGB, GFootball-sized stacks,
odd channel counts and row pitches that are not a multiple of 16 bytes), in 'simt' and 'tc3p':
a learner step against the CPU oracle (structure and tolerances of test_gpu_dmlab_shape.py), bit-
identical repeats, the fused first-layer kernels on their own against float64, and a T=1 inference
batch whose sampled actions follow the oracle's logits exactly."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import learner_oracle, loss_oracle, net_oracle

pytestmark = pytest.mark.gpu

# (H, W, C): 84x84 grayscale (row pitch 84 B), the 72x96x16 GFootball stack, four stacked RGB frames,
# RGBD-sized 6 channels, and an odd everything (pitch 35*7 = 245 B)
SHAPES = [(84, 84, 1), (72, 96, 16), (84, 84, 12), (60, 80, 6), (21, 35, 7)]
TOLS = {'simt': (2e-5, 2e-3), 'tc3p': (2e-4, 1e-2)}
# On the grayscale batch the oracle's own gradients move by up to 1e-3 (L2-relative) when its conv
# kernels get random 1e-6 relative noise (max-pool near-ties at this tiny T*B), so fp32 rounding
# differences alone reach a few 1e-3 there; the other shapes stay below 4e-4 in 'simt'.
GTOL_ILL_CONDITIONED = {(84, 84, 1): 5e-3}


def _step(obs, mode, params, b):
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda
  agent = networks.ImpalaDeep(params['policy_logits/bias'].shape[0], obs, conv_mode=mode)
  agent.load_named_parameters(params)
  step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7))
  u = _batch_to_cuda(b)
  loss, _ = step.compute_gradients(u)
  agent.check_errors()
  grads = {k: v.cpu().numpy().copy() for k, v in agent.named_gradients().items()}
  out, _ = agent(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
  return float(loss), out.policy_logits.cpu().numpy(), grads


@pytest.mark.parametrize('mode', ['simt', 'tc3p'])
@pytest.mark.parametrize('obs', SHAPES)
def test_learner_step_matches_oracle_and_repeats_bitwise(obs, mode):
  A, T, B = 7, 4, 3
  ftol, gtol = TOLS[mode]
  gtol = max(gtol, GTOL_ILL_CONDITIONED.get(obs, 0.0))
  params = net_oracle.init_params('deep', A, obs, seed=1)
  assert params['stack0/conv/kernel'].shape == (3, 3, obs[2], 16) and len(params) == 39
  cpu = learner_oracle.CpuLearner('deep', A, obs, loss_oracle.default_config(), params=params)
  b = learner_oracle.synthetic_batch(T, B, A, obs, seed=100 + obs[2])
  total, _, g, aux = cpu.grads(b)
  loss, logits, mine = _step(obs, mode, params, b)
  assert abs(loss - float(total)) < 2e-4 * max(1.0, abs(float(total)))
  lg = aux['logits'].detach().numpy()
  assert np.abs(logits - lg).max() < ftol * max(1.0, np.abs(lg).max())
  errs = {}
  for k in g:
    if k != 'entropy_cost_param':
      a, w = mine[k].astype(np.float64), g[k].astype(np.float64)
      assert a.shape == w.shape, k
      errs[k] = float(np.linalg.norm(a - w) / (np.linalg.norm(w) + 1e-30))
  assert len(errs) == 39
  bad = {k: v for k, v in errs.items() if not v < gtol}
  print('OBS_CHANNELS %s %s: max L2-rel grad err %.3g' % (obs, mode, max(errs.values())))
  assert not bad, bad
  loss2, logits2, mine2 = _step(obs, mode, params, b)
  assert loss2 == loss
  np.testing.assert_array_equal(logits2, logits)
  for k in mine:
    np.testing.assert_array_equal(mine2[k], mine[k], err_msg=k)


def _planes(x):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  N, H, W, C = x.shape
  out = torch.zeros(int(L.seedrl_debug_planes_bytes(N, H, W, C)), dtype=torch.uint8, device='cuda')
  xc = torch.as_tensor(np.ascontiguousarray(x, np.float32)).cuda()
  _lib.check(L.seedrl_debug_to_planes(N, H, W, C, 0, _lib.ptr(xc), _lib.ptr(out), _lib.stream_ptr()))
  return out


def _from_planes(p, N, H, W, C):
  from seed_rl_b200 import _lib
  y = torch.full((N, H, W, C), float('nan'), device='cuda')
  _lib.check(_lib.lib().seedrl_debug_from_planes(N, H, W, C, _lib.ptr(p), _lib.ptr(y), _lib.stream_ptr()))
  torch.cuda.synchronize()
  return y.cpu().numpy()


@pytest.mark.parametrize('N,H,W,C', [(3, 84, 84, 1), (2, 72, 96, 16), (2, 84, 84, 12), (3, 60, 80, 6),
                                     (4, 21, 35, 7), (2, 9, 107, 2), (2, 17, 30, 9)])
def test_fused_first_layer_kernels_match_float64(N, H, W, C):
  """seedrl_debug_conv0pool_c: pooled raw / ReLU planes to 2e-4 of max-abs (bf16x3 weights, exact
  frames), arg-max taps exact wherever the window's top two are apart; then
  seedrl_debug_first_wgrad_pooled_c on those taps: dW [3,3,C,16] and db against float64 (pooled
  gradient exactly representable in bf16, so only fp32 summation order differs)."""
  from seed_rl_b200 import _lib
  L = _lib.lib()
  rng = np.random.default_rng(N * 100 + C)
  fr = rng.integers(0, 256, (N, H, W, C), dtype=np.uint8)
  w = (rng.normal(size=(3, 3, C, 16)) * 0.3).astype(np.float32)
  bias = rng.normal(size=16).astype(np.float32)
  Ho, Wo = (H + 1) // 2, (W + 1) // 2
  nb = int(L.seedrl_debug_planes_bytes(N, Ho, Wo, 16))
  raw = torch.full((nb,), 0xFF, dtype=torch.uint8, device='cuda'); relu = raw.clone()
  idx = torch.full((N, Ho, Wo, 16), 255, dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  c = lambda a: torch.as_tensor(a).cuda()
  frd, wd, bd = c(fr), c(w), c(bias)
  _lib.check(L.seedrl_debug_conv0pool_c(N, H, W, C, _lib.ptr(frd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(raw),
                                        _lib.ptr(relu), _lib.ptr(idx), _lib.ptr(err), _lib.stream_ptr()))
  torch.cuda.synchronize()
  assert int(err.item()) == 0
  x = torch.as_tensor(fr.astype(np.float64) / 255.0).permute(0, 3, 1, 2)
  y = F.conv2d(x, torch.as_tensor(w.astype(np.float64)).permute(3, 2, 0, 1), torch.as_tensor(bias.astype(np.float64)),
               padding=1)
  pt = max((Ho - 1) * 2 + 3 - H, 0) // 2; pl = max((Wo - 1) * 2 + 3 - W, 0) // 2
  pb = max((Ho - 1) * 2 + 3 - H - pt, 0); pr = max((Wo - 1) * 2 + 3 - W - pl, 0)
  win = F.pad(y, (pl, pr, pt, pb), value=float('-inf')).unfold(2, 3, 2).unfold(3, 3, 2).reshape(N, 16, Ho, Wo, 9)
  want, arg = win.max(dim=-1)
  want = want.permute(0, 2, 3, 1).numpy(); arg = arg.permute(0, 2, 3, 1).numpy()
  srt = np.sort(win.numpy(), axis=-1)
  clear = np.transpose(srt[..., -1] - srt[..., -2], (0, 2, 3, 1)) > 1e-3 * np.abs(want).max()
  got = _from_planes(raw, N, Ho, Wo, 16)
  assert np.abs(got - want).max() <= 2e-4 * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()
  assert np.abs(_from_planes(relu, N, Ho, Wo, 16) - np.maximum(want, 0)).max() <= 2e-4 * np.abs(want).max()
  taps = idx.cpu().numpy()
  np.testing.assert_array_equal(taps[clear], arg[clear].astype(np.uint8))
  assert clear.mean() > 0.9
  # ---- weight gradient from the pooled gradient and the kernel's own taps ----
  gq = rng.normal(size=(N, Ho, Wo, 16)).astype(np.float32)
  gq = (gq.view(np.uint32) & 0xFFFF0000).view(np.float32)          # exact in bf16: hi + lo == g
  gp = _planes(gq)
  dw = torch.full((3, 3, C, 16), float('nan'), device='cuda'); db = torch.full((16,), float('nan'), device='cuda')
  part = torch.empty(3 * 132 * (9 * C * 16 + 16), dtype=torch.float32, device='cuda')
  _lib.check(L.seedrl_debug_first_wgrad_pooled_c(N, H, W, C, _lib.ptr(frd), _lib.ptr(gp), _lib.ptr(idx), _lib.ptr(dw),
                                                 _lib.ptr(db), _lib.ptr(part), part.numel() * 4, _lib.stream_ptr()))
  torch.cuda.synchronize()
  xp = np.pad(fr.astype(np.float64) / 255.0, ((0, 0), (1, 1), (1, 1), (0, 0)))
  nn_, qh, qw, co = np.meshgrid(np.arange(N), np.arange(Ho), np.arange(Wo), np.arange(16), indexing='ij')
  ph = 2 * qh - pt + taps.astype(np.int64) // 3; pw = 2 * qw - pl + taps.astype(np.int64) % 3
  ref = np.zeros((3, 3, C, 16))
  g64 = gq.astype(np.float64)
  for kh in range(3):
    for kw in range(3):
      X = xp[nn_, ph + kh, pw + kw]                                # [N,Ho,Wo,16(co),C]
      ref[kh, kw] = np.einsum('nhwo,nhwoc->co', g64, X)
  got_dw = dw.cpu().numpy()
  assert np.abs(got_dw - ref).max() <= 1e-5 * np.abs(ref).max(), np.abs(got_dw - ref).max() / np.abs(ref).max()
  np.testing.assert_allclose(db.cpu().numpy(), g64.sum(axis=(0, 1, 2)), rtol=1e-5, atol=1e-5 * np.abs(g64).sum() / 16)


@pytest.mark.parametrize('mode', ['simt', 'tc3p'])
@pytest.mark.parametrize('obs', [(84, 84, 1), (72, 96, 16), (84, 84, 12), (21, 35, 7)])
def test_inference_batch_with_gumbel_noise_follows_oracle(obs, mode):
  """One T=1 inference batch through InferenceHost (the observation shape travels through its specs
  and store untouched), then the same batch through the agent with injected Gumbel noise: every
  sampled action equals argmax(oracle logits + noise)."""
  from seed_rl_b200.agents.vtrace import learner_loop
  from seed_rl_b200.dmlab import networks
  A, n = 9, 6
  params = net_oracle.init_params('deep', A, obs, seed=5)
  agent = networks.ImpalaDeep(A, obs, conv_mode=mode)
  agent.load_named_parameters(params)
  host = learner_loop.InferenceHost(agent, n, 3, n, obs)
  rng = np.random.default_rng(obs[2])
  from seed_rl_b200.common import utils
  env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), np.zeros(n, bool),
                        rng.integers(0, 256, (n,) + obs, dtype=np.uint8), np.zeros(n, bool), np.zeros(n, np.int32))
  ids = np.arange(n, dtype=np.int32)
  act = host.inference(ids, np.arange(1, n + 1, dtype=np.int64), env, np.zeros(n, np.float32))
  torch.cuda.synchronize()
  assert act.shape == (n,) and (0 <= act).all() and (act < A).all()
  h0 = np.zeros((n, 256), np.float32)
  prev = np.zeros((1, n), np.int64)
  with torch.no_grad():
    want, _, _ = net_oracle.unroll('deep', net_oracle.to_torch(params), torch.as_tensor(prev),
                                   torch.as_tensor(env.reward[None]), torch.as_tensor(env.done[None]),
                                   torch.as_tensor(env.observation[None]), (torch.as_tensor(h0), torch.as_tensor(h0)), A)
  want = want[0].numpy()
  noise = -np.log(-np.log(rng.uniform(1e-6, 1.0, (n, A)))).astype(np.float32)
  c = lambda a: torch.as_tensor(a).cuda()
  out, _ = agent(c(prev[0]), (c(env.reward), c(env.done), c(env.observation)), (c(h0), c(h0)),
                 gumbel_noise=c(noise))
  # the host sampled from the same logits (no noise injected there): its logits are the agent's
  np.testing.assert_allclose(out.policy_logits.cpu().numpy(), want, rtol=0, atol=TOLS[mode][0] * max(1.0, np.abs(want).max()))
  z = want + noise
  srt = np.sort(z, axis=-1)
  assert (srt[:, -1] - srt[:, -2] > 1e-3).all()                  # no near-tie decides an action
  np.testing.assert_array_equal(out.action.cpu().numpy(), z.argmax(-1))
