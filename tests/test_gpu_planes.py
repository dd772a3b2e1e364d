"""GPU: the plane-tensor convolution path (csrc/conv_planes.cu, conv_mode 'tc3p') kernel by kernel
against float64 references: the HBM operand format itself, the TMA-fed wgmma forward /
data-gradient conv with every epilogue option (bias, ReLU mask, residual, raw / ReLU'd / fp32
outputs), the weight + bias gradient, and max-pool forward / backward -- then one toy-size
learner step against the CPU oracle (the BASELINE-size step is in test_gpu_fullsize.py).

Tolerance: bf16x3 split operands => 2e-4 of the output's max-abs per kernel (same bar as the 'tc3'
kernels, test_gpu_zz_tc.py)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 2e-4


def _L():
  from seed_rl_b200 import _lib
  return _lib, _lib.lib()


def _planes_buf(N, H, W, C, fill=None):
  _lib, L = _L()
  nb = int(L.seedrl_debug_planes_bytes(N, H, W, C))
  assert nb > 0
  t = torch.empty(nb, dtype=torch.uint8, device='cuda')
  if fill is not None:
    t.fill_(fill)
  return t


def _to_planes(x, relu=0):
  """x: numpy fp32 [N,H,W,C] -> plane tensor (device bytes)."""
  _lib, L = _L()
  N, H, W, C = x.shape
  out = _planes_buf(N, H, W, C, fill=0xFF)      # poison: every byte must be written
  xc = torch.as_tensor(np.ascontiguousarray(x, np.float32)).cuda()
  _lib.check(L.seedrl_debug_to_planes(N, H, W, C, relu, _lib.ptr(xc), _lib.ptr(out), _lib.stream_ptr()))
  return out


def _from_planes(p, N, H, W, C):
  _lib, L = _L()
  y = torch.full((N, H, W, C), float('nan'), device='cuda')
  _lib.check(L.seedrl_debug_from_planes(N, H, W, C, _lib.ptr(p), _lib.ptr(y), _lib.stream_ptr()))
  torch.cuda.synchronize()
  return y.cpu().numpy()


def _bf16_bits(a):
  """round-to-nearest-even bf16 bit patterns of fp32 array a (numpy restatement)."""
  u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
  r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
  return r


def test_plane_format_is_pinned_bytewise():
  """The HBM format (DESIGN 3): position s = (n*(H+1) + h + 1)*(W+2) + w + 1, planes [C/8][Lp][8]
  bf16, hi planes then lo planes (lo = bf16(v - hi)), zeros at every padding position."""
  rng = np.random.default_rng(0)
  N, H, W, C = 3, 5, 4, 16
  x = rng.normal(size=(N, H, W, C)).astype(np.float32)
  p = _to_planes(x)
  torch.cuda.synchronize()
  raw = p.cpu().numpy().view(np.uint16)
  G = C // 8
  Lp = raw.size // (2 * G * 8)
  assert Lp % 64 == 0 and Lp >= N * (H + 1) * (W + 2) + 2 * (W + 2) + 2
  planes = raw.reshape(2 * G, Lp, 8)
  want = np.zeros((2 * G, Lp, 8), np.uint16)
  hi = _bf16_bits(x)
  hif = (hi.astype(np.uint32) << 16).view(np.float32)
  lo = _bf16_bits(x - hif)
  for n in range(N):
    for h in range(H):
      for w in range(W):
        s = (n * (H + 1) + h + 1) * (W + 2) + w + 1
        for g in range(G):
          want[g, s] = hi[n, h, w, g * 8:(g + 1) * 8]
          want[G + g, s] = lo[n, h, w, g * 8:(g + 1) * 8]
  np.testing.assert_array_equal(planes, want)
  back = _from_planes(p, N, H, W, C)
  assert np.abs(back - x).max() <= 2.0 ** -16 * np.abs(x).max()


def _ref_conv(x, w, bias):
  """float64 'same' 3x3 conv, NHWC x, HWIO w."""
  xt = torch.as_tensor(x, dtype=torch.float64).permute(0, 3, 1, 2)
  wt = torch.as_tensor(w, dtype=torch.float64).permute(3, 2, 0, 1)
  y = F.conv2d(xt, wt, None if bias is None else torch.as_tensor(bias, dtype=torch.float64), padding=1)
  return y.permute(0, 2, 3, 1).numpy()


CONV_CASES = [
    # cin, cout, N, H, W
    (16, 16, 3, 11, 13), (16, 32, 2, 42, 42), (32, 16, 2, 21, 21), (32, 32, 5, 11, 11),
    (32, 32, 1, 1, 1), (16, 16, 2, 3, 130),
    (16, 16, 84, 42, 42),       # > 2*148 tiles of 512: the NSUB = 4 path
    (32, 32, 330, 21, 21)]


@pytest.mark.parametrize('cin,cout,N,H,W', CONV_CASES)
def test_convp_forward_all_epilogues(cin, cout, N, H, W):
  _lib, L = _L()
  rng = np.random.default_rng(cin + cout + N + H)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  bias = rng.normal(size=cout).astype(np.float32)
  res = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  msk = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xin = _to_planes(x)
  resp = _to_planes(res)
  mskp = _to_planes(msk, relu=1)                      # the ReLU'd forward activation is the mask
  wq = torch.empty(2 * 9 * cin * cout * 2, dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  wc, bc = torch.as_tensor(w).cuda(), torch.as_tensor(bias).cuda()

  def run(bias_t, mask_t, res_t, want_raw, want_relu, want_nhwc, flip=0, wsrc=None, ci=cin, co=cout):
    out_raw = _planes_buf(N, H, W, co, fill=0xFF) if want_raw else None
    out_relu = _planes_buf(N, H, W, co, fill=0xFF) if want_relu else None
    out_nhwc = torch.full((N, H, W, co), float('nan'), device='cuda') if want_nhwc else None
    _lib.check(L.seedrl_debug_convp(ci, co, N, H, W, _lib.ptr(xin if wsrc is None else wsrc[1]),
                                    _lib.ptr(wc if wsrc is None else wsrc[0]), _lib.ptr(bias_t), _lib.ptr(mask_t),
                                    _lib.ptr(res_t), flip, _lib.ptr(out_raw), _lib.ptr(out_relu), _lib.ptr(out_nhwc),
                                    _lib.ptr(wq), _lib.ptr(err), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    return out_raw, out_relu, out_nhwc

  base = _ref_conv(x, w, bias)
  scale = np.abs(base).max()
  # (1) bias only, fp32 NHWC output (the max-pool / Dense consumer)
  _, _, y = run(bc, None, None, False, False, True)
  assert np.abs(y.cpu().numpy() - base).max() < TOL * scale
  # (2) bias + residual -> raw planes + ReLU'd planes (o0 = conv01(relu(c0)) + p)
  raw, relu, _ = run(bc, None, resp, True, True, False)
  want = base + res
  got = _from_planes(raw, N, H, W, cout)
  assert np.abs(got - want).max() < TOL * max(scale, np.abs(want).max())
  gotr = _from_planes(relu, N, H, W, cout)
  assert np.abs(gotr - np.maximum(want, 0)).max() < TOL * max(scale, np.abs(want).max())
  # padding positions of a produced plane tensor are zeros (the next conv's halo), byte for byte:
  # re-encoding the decoded tensor must reproduce the produced bytes up to the hi/lo re-split
  ref_bytes = _to_planes(got)
  torch.cuda.synchronize()
  a16 = raw.cpu().numpy().view(np.uint16); b16 = ref_bytes.cpu().numpy().view(np.uint16)
  zero_mask = (b16.reshape(-1, 8) == 0).all(axis=1)
  assert (a16.reshape(-1, 8)[zero_mask] == 0).all()
  # (3) ReLU'd output only (c0 = relu(conv00(relu(p))))
  _, relu, _ = run(bc, None, None, False, True, False)
  gotr = _from_planes(relu, N, H, W, cout)
  assert np.abs(gotr - np.maximum(base, 0)).max() < TOL * scale
  # (4) data gradient: flipped weights, ReLU mask, residual.  dy has `cout` channels, dx `cin`.
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  dyp = _to_planes(dy)
  mk_in = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  rs_in = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  mk_p, rs_p = _to_planes(mk_in, relu=1), _to_planes(rs_in)
  raw, _, _ = run(None, mk_p, rs_p, True, False, False, flip=1, wsrc=(wc, dyp), ci=cout, co=cin)
  wflip = np.ascontiguousarray(w[::-1, ::-1].transpose(0, 1, 3, 2))       # [kh,kw,co,ci] flipped
  dx = _ref_conv(dy, wflip, None)
  want = np.where(mk_in > 0, dx, 0) + rs_in
  got = _from_planes(raw, N, H, W, cin)
  assert np.abs(got - want).max() < TOL * max(np.abs(dx).max(), np.abs(want).max())


WGRAD_CASES = [(16, 16, 3, 11, 13), (16, 32, 2, 42, 42), (32, 32, 4, 21, 21), (32, 32, 2, 1, 1),
               (16, 16, 300, 42, 42), (32, 32, 700, 11, 11)]


@pytest.mark.parametrize('cin,cout,N,H,W', WGRAD_CASES)
def test_wgradp_matches_float64(cin, cout, N, H, W):
  _lib, L = _L()
  rng = np.random.default_rng(cin * 3 + cout + N)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xp, dyp = _to_planes(x), _to_planes(dy)
  dw = torch.full((3, 3, cin, cout), float('nan'), device='cuda')
  db = torch.full((cout,), float('nan'), device='cuda')
  partial = torch.empty(148 * (9 * cin * cout + cout), device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  outs = []
  for _ in range(2):
    _lib.check(L.seedrl_debug_wgradp(cin, cout, N, H, W, _lib.ptr(xp), _lib.ptr(dyp), _lib.ptr(dw), _lib.ptr(db),
                                     _lib.ptr(partial), partial.numel() * 4, _lib.ptr(err), _lib.stream_ptr()))
    torch.cuda.synchronize()
    outs.append((dw.cpu().numpy().copy(), db.cpu().numpy().copy()))
  assert int(err.item()) == 0
  xt = torch.as_tensor(x, dtype=torch.float64).permute(0, 3, 1, 2)
  wt = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, requires_grad=True)
  bt = torch.zeros(cout, dtype=torch.float64, requires_grad=True)
  y = F.conv2d(xt, wt, bt, padding=1)
  y.backward(torch.as_tensor(dy, dtype=torch.float64).permute(0, 3, 1, 2))
  want_w = wt.grad.permute(2, 3, 1, 0).numpy()
  want_b = bt.grad.numpy()
  got_w, got_b = outs[0]
  assert np.abs(got_w - want_w).max() < TOL * np.abs(want_w).max()
  assert np.abs(got_b - want_b).max() < TOL * max(np.abs(want_b).max(), np.sqrt(N * H * W))
  assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])    # deterministic


@pytest.mark.parametrize('N,H,W,C', [(3, 84, 84, 16), (2, 42, 42, 32), (5, 21, 21, 32), (2, 7, 10, 16), (1, 1, 1, 16)])
def test_poolp_forward_backward(N, H, W, C):
  """TF 'SAME' 3x3/2 max-pool: raw + ReLU'd plane outputs and argmax taps equal the fp32 kernel's
  (itself pinned against the oracle in test_gpu_parity.py); backward gathers through the taps."""
  _lib, L = _L()
  rng = np.random.default_rng(N + H + C)
  x = rng.normal(size=(N, H, W, C)).astype(np.float32)
  Ho, Wo = (H + 1) // 2, (W + 1) // 2
  xc = torch.as_tensor(x).cuda()
  y_ref = torch.empty(N, Ho, Wo, C, device='cuda'); idx_ref = torch.empty(N, Ho, Wo, C, dtype=torch.uint8, device='cuda')
  _lib.check(L.seedrl_debug_maxpool(0, N, H, W, C, _lib.ptr(xc), _lib.ptr(y_ref), _lib.ptr(idx_ref), _lib.stream_ptr()))
  raw, relu = _planes_buf(N, Ho, Wo, C, fill=0xFF), _planes_buf(N, Ho, Wo, C, fill=0xFF)
  idx = torch.full((N, Ho, Wo, C), 255, dtype=torch.uint8, device='cuda')
  _lib.check(L.seedrl_debug_poolp(0, N, H, W, C, _lib.ptr(xc), _lib.ptr(raw), _lib.ptr(relu), None, _lib.ptr(idx),
                                  _lib.stream_ptr()))
  torch.cuda.synchronize()
  assert torch.equal(idx, idx_ref)
  yr = y_ref.cpu().numpy()
  assert np.abs(_from_planes(raw, N, Ho, Wo, C) - yr).max() <= 2.0 ** -16 * np.abs(yr).max()
  assert np.abs(_from_planes(relu, N, Ho, Wo, C) - np.maximum(yr, 0)).max() <= 2.0 ** -16 * np.abs(yr).max()
  # backward
  dy = rng.normal(size=(N, Ho, Wo, C)).astype(np.float32)
  dyp = _to_planes(dy)
  dyq = torch.as_tensor(_from_planes(dyp, N, Ho, Wo, C)).cuda()      # the hi+lo value the kernel sees
  dx_ref = torch.empty(N, H, W, C, device='cuda')
  _lib.check(L.seedrl_debug_maxpool(1, N, H, W, C, _lib.ptr(dyq), _lib.ptr(dx_ref), _lib.ptr(idx_ref), _lib.stream_ptr()))
  dx_nhwc = torch.full((N, H, W, C), float('nan'), device='cuda')
  _lib.check(L.seedrl_debug_poolp(1, N, H, W, C, _lib.ptr(dyp), None, None, _lib.ptr(dx_nhwc), _lib.ptr(idx),
                                  _lib.stream_ptr()))
  dx_pl = _planes_buf(N, H, W, C, fill=0xFF)
  _lib.check(L.seedrl_debug_poolp(1, N, H, W, C, _lib.ptr(dyp), _lib.ptr(dx_pl), None, None, _lib.ptr(idx),
                                  _lib.stream_ptr()))
  torch.cuda.synchronize()
  ref = dx_ref.cpu().numpy()
  assert np.abs(dx_nhwc.cpu().numpy() - ref).max() <= 1e-6 * max(1.0, np.abs(ref).max())
  assert np.abs(_from_planes(dx_pl, N, H, W, C) - ref).max() <= 2.0 ** -15 * max(1.0, np.abs(ref).max())


def test_network_step_planes_matches_fp32_oracle():
  """ImpalaDeep learner step in conv_mode 'tc3p' on the toy batch of test_gpu_zz_tc.py: same bar
  as 'tc3' (loss 2e-4, every gradient tensor 1e-2 L2-relative; the oracle itself moves 4.6e-3
  when its conv operands are rounded to hi+lo bf16)."""
  from test_gpu_zz_tc import _step_errors
  loss, total, errs = _step_errors('tc3p')
  print('TC3P_NET max L2-rel vs fp32 oracle: %.3g' % max(errs.values()))
  assert abs(loss - total) < 2e-4 * max(1.0, abs(total))
  bad = {k: v for k, v in errs.items() if not v < 1e-2}
  assert not bad, bad


def test_inference_step_planes_matches_tc3():
  """T=1 forward (central inference shape, B=64): 'tc3p' logits agree with the fp32 SIMT path."""
  from oracle import learner_oracle, net_oracle
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda
  A = 18
  params = net_oracle.init_params('deep', A, (84, 84, 4), seed=1)
  b = learner_oracle.synthetic_batch(0, 64, A, seed=3)
  u = _batch_to_cuda(b)
  outs = {}
  for mode in ('simt', 'tc3p'):
    ag = networks.ImpalaDeep(A, (84, 84, 4), conv_mode=mode)
    ag.load_named_parameters(params)
    o, _ = ag(u.prev_actions, u.env_outputs, u.agent_state, unroll=True, is_training=True)
    ag.check_errors()
    outs[mode] = o.policy_logits.cpu().numpy()
  assert np.abs(outs['tc3p'] - outs['simt']).max() < 2e-4 * np.abs(outs['simt']).max()


@pytest.mark.parametrize('T,B', [(3, 2), (20, 8)])
def test_first_layer_fused_kernels_match_dense_path(T, B):
  """csrc/conv_first.cu -- forward: first conv + bias + max-pool in one wgmma kernel (im2col in
  shared memory, pooled planes + arg-max taps out); backward: weight gradient of the first conv
  gathered from the POOLED gradient and the taps -- against the path they replace (staged wgmma
  conv -> fp32 NHWC -> pool kernel; pool backward -> full-resolution gradient -> dense weight-gradient
  conv).  Same arithmetic (bf16x3 products, fp32 accumulation), different summation order: loss,
  learner outputs agree to 1e-5 and every gradient tensor to 2e-3 of its max-abs (3e-2 in the conv
  stacks, whose gradients are sums over 10^5..10^6 cancelling terms even on these tiny batches; a wrong tap or channel would be an O(1) error; a pooling near-tie may also route one
  gradient element to the neighbouring tap).  The oracle comparison at full size is test_gpu_fullsize.py."""
  from oracle import learner_oracle, loss_oracle, net_oracle
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda
  A = 18
  params = net_oracle.init_params('deep', A, (84, 84, 4), seed=2)
  u = _batch_to_cuda(learner_oracle.synthetic_batch(T, B, A, seed=11))
  grads, outs, losses = {}, {}, {}
  try:
    for dense in (1, 0):
      _lib.check(_lib.lib().seedrl_debug_set_first_layer_dense(dense))
      ag = networks.ImpalaDeep(A, (84, 84, 4), conv_mode='tc3p')
      ag.load_named_parameters(params)
      st = learner.LearnerStep(ag, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7),
                               settings=learner.default_loss_settings())
      loss, _ = st.compute_gradients(u)
      ag.check_errors()
      losses[dense] = float(loss)
      grads[dense] = {k: v.cpu().numpy().copy() for k, v in ag.named_gradients().items()}
      o, _ = ag(u.prev_actions, u.env_outputs, u.agent_state, unroll=True)
      outs[dense] = o.policy_logits.cpu().numpy()
  finally:
    _lib.check(_lib.lib().seedrl_debug_set_first_layer_dense(0))
  assert abs(losses[0] - losses[1]) < 1e-5 * max(1.0, abs(losses[1]))
  assert np.abs(outs[0] - outs[1]).max() < 1e-5 * np.abs(outs[1]).max()
  for k in grads[0]:
    a, w = grads[0][k], grads[1][k]
    # the first conv's own kernel / bias gradient: exact fp32 products and a different summation
    # tree in the gather vs bf16x3 split of a 75 %-zero full-resolution gradient in the dense path
    # (both are sums of ~10^6 cancelling terms)
    tol = 3e-2 if k.startswith('stack') else 2e-3     # conv stacks: sums over 10^5..10^6 cancelling terms
    assert np.abs(a - w).max() <= tol * np.abs(w).max() + 1e-12, (k, np.abs(a - w).max() / np.abs(w).max())


@pytest.mark.parametrize('N,H,W', [(3, 84, 84), (2, 72, 96), (5, 21, 24), (1, 7, 8), (149, 84, 84)])
def test_conv0pool_fused_first_layer(N, H, W):
  """conv0pool_kernel (first conv on uint8 frames + bias + TF-SAME 3x3/2 max-pool, one kernel)
  against float64 conv + pool: pooled values to 2e-4 of max-abs (bf16x3 weights, exact frames),
  ReLU'd copy, arg-max taps (wherever the runner-up is not within rounding), and every padding
  byte of both plane tensors written as zero (buffers are poisoned first)."""
  _lib, L = _L()
  rng = np.random.default_rng(N + H)
  fr = rng.integers(0, 256, (N, H, W, 4), dtype=np.uint8)
  w = (rng.normal(size=(3, 3, 4, 16)) * 0.3).astype(np.float32)
  b = rng.normal(size=16).astype(np.float32)
  Ho, Wo = (H + 1) // 2, (W + 1) // 2
  raw, relu = _planes_buf(N, Ho, Wo, 16, fill=0xFF), _planes_buf(N, Ho, Wo, 16, fill=0xFF)
  idx = torch.full((N, Ho, Wo, 16), 255, dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  c = lambda a: torch.as_tensor(a).cuda()
  frd, wd, bd = c(fr), c(w), c(b)
  _lib.check(L.seedrl_debug_conv0pool(N, H, W, _lib.ptr(frd), _lib.ptr(wd), _lib.ptr(bd), _lib.ptr(raw), _lib.ptr(relu),
                                      _lib.ptr(idx), _lib.ptr(err), _lib.stream_ptr()))
  torch.cuda.synchronize()
  assert int(err.item()) == 0
  x = torch.as_tensor(fr.astype(np.float64) / 255.0).permute(0, 3, 1, 2)
  y = F.conv2d(x, torch.as_tensor(w.astype(np.float64)).permute(3, 2, 0, 1), torch.as_tensor(b.astype(np.float64)), padding=1)
  pt = max((Ho - 1) * 2 + 3 - H, 0) // 2; pl = max((Wo - 1) * 2 + 3 - W, 0) // 2
  pb = max((Ho - 1) * 2 + 3 - H - pt, 0); pr = max((Wo - 1) * 2 + 3 - W - pl, 0)
  yp = F.pad(y, (pl, pr, pt, pb), value=float('-inf'))
  win = yp.unfold(2, 3, 2).unfold(3, 3, 2).reshape(N, 16, Ho, Wo, 9)           # taps kh*3+kw
  want, arg = win.max(dim=-1)
  want = want.permute(0, 2, 3, 1).numpy(); arg = arg.permute(0, 2, 3, 1).numpy()
  srt = np.sort(win.numpy(), axis=-1)
  clear = np.transpose(srt[..., -1] - srt[..., -2], (0, 2, 3, 1)) > 1e-3 * np.abs(want).max()
  got = _from_planes(raw, N, Ho, Wo, 16)
  assert np.abs(got - want).max() <= TOL * np.abs(want).max(), np.abs(got - want).max() / np.abs(want).max()
  gr = _from_planes(relu, N, Ho, Wo, 16)
  assert np.abs(gr - np.maximum(want, 0)).max() <= TOL * np.abs(want).max()
  np.testing.assert_array_equal(idx.cpu().numpy()[clear], arg[clear].astype(np.uint8))
  # padding positions: the plane tensors must equal what to_planes writes (zeros outside pixels)
  for buf, ref in ((raw, got), (relu, gr)):
    again = _to_planes(ref.astype(np.float32))
    d = (buf.view(torch.int16).float() - again.view(torch.int16).float()).abs()
    # identical wherever padding; pixels may differ in the lo plane's last bits only
    a16 = buf.view(torch.uint16).cpu().numpy(); b16 = again.view(torch.uint16).cpu().numpy()
    assert not (a16 == 0xFFFF).all() and (a16[b16 == 0] == 0).mean() > 0.999
