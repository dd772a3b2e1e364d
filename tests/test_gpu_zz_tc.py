"""GPU: the wgmma (tensor-core) 3x3 convolution kernels against the CPU oracle.

Two operand modes:
  split=0  bf16 operands, fp32 accumulation: 1.5e-2 of the output's max-abs per kernel
           (each product carries ~2^-8 relative rounding; K <= 288 terms)
  split=1  bf16x3 (v = hi + lo; hi*hi + lo*hi + hi*lo): fp32-faithful, 2e-4 per kernel
Runs last (file name) because a broken tensor-core kernel can poison the CUDA context for
later tests.  (tools/tc_probe.py runs each case in its own process.)  The kernels' shared-memory
descriptors are fixed to the documented layout; the entry point's `variant` argument must be 0, and
test_abi.py checks that any other value is refused.
"""
import numpy as np
import pytest
import torch

from oracle import net_oracle

pytestmark = pytest.mark.gpu

TOL = {0: 1.5e-2, 1: 2e-4}
CASES = [(16, 16, 1, 5, 42, 42), (16, 32, 0, 2, 42, 42), (32, 32, 1, 7, 21, 21),
         (32, 32, 0, 9, 11, 11), (32, 16, 0, 2, 42, 42), (16, 16, 0, 1, 5, 3),
         (32, 32, 1, 300, 11, 11), (4, 16, 2, 3, 84, 84), (4, 16, 2, 11, 9, 7), (16, 16, 1, 64, 42, 42)]


def _ref(x, w, b, mode):
  xt = torch.as_tensor(x)
  if mode == 1:
    xt = torch.relu(xt)
  if mode == 2:
    xt = xt.float() / 255.0
  return net_oracle._conv_nhwc(xt, torch.as_tensor(w), None if b is None else torch.as_tensor(b), 1, True)


def _run(cin, cout, mode, N, H, W, x, w, b, mask, res, flip, split=0):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  c = lambda a: None if a is None else torch.as_tensor(np.asarray(a)).cuda()
  xc, wc, bc, mc, rc = c(x), c(w), c(b), c(mask), c(res)
  out = torch.full((N, H, W, cout), float('nan')).cuda()
  wq = torch.empty(2 * 9 * max(cin, 16) * cout * 2, dtype=torch.uint8).cuda()
  err = torch.zeros(1, dtype=torch.int32).cuda()
  _lib.check(L.seedrl_debug_conv3x3_tc(cin, cout, mode, split, N, H, W, _lib.ptr(xc), _lib.ptr(wc),
                                       _lib.ptr(bc), _lib.ptr(mc), _lib.ptr(rc), _lib.ptr(out), flip,
                                       0, _lib.ptr(wq), _lib.ptr(err), _lib.stream_ptr()))
  torch.cuda.synchronize()
  return out.cpu().numpy(), int(err.item())


def _run_wgrad(cin, cout, mode, N, H, W, x, dy, split=0):
  from seed_rl_b200 import _lib
  L = _lib.lib()
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  xc, dyc = c(x), c(dy)
  pb = int(L.seedrl_debug_wgrad_partial_bytes())
  partial = torch.empty(pb // 4, device='cuda')
  dw = torch.full((3, 3, cin, cout), float('nan')).cuda(); db = torch.full((cout,), float('nan')).cuda()
  err = torch.zeros(1, dtype=torch.int32).cuda()
  _lib.check(L.seedrl_debug_conv3x3_wgrad_tc(cin, cout, mode, split, N, H, W, _lib.ptr(xc), _lib.ptr(dyc),
                                             _lib.ptr(dw), _lib.ptr(db), _lib.ptr(partial), pb,
                                             _lib.ptr(err), _lib.stream_ptr()))
  torch.cuda.synchronize()
  return dw.cpu().numpy(), db.cpu().numpy(), int(err.item())


def _relerr(a, b):
  return float(np.nanmax(np.abs(np.nan_to_num(a, nan=1e30) - b)) / (np.abs(b).max() + 1e-30))


@pytest.fixture(params=[512, 256, 128])
def conv_tile(request):
  from seed_rl_b200 import _lib
  _lib.check(_lib.lib().seedrl_debug_set_conv_tile(request.param))
  yield request.param
  _lib.check(_lib.lib().seedrl_debug_set_conv_tile(512))


@pytest.mark.parametrize('split', [0, 1])
@pytest.mark.parametrize('cin,cout,mode,N,H,W', CASES)
def test_conv3x3_tc_forward(cin, cout, mode, N, H, W, split, conv_tile):
  rng = np.random.default_rng(cin * 100 + cout + H)
  if mode == 2:
    x = rng.integers(0, 256, (N, H, W, cin), dtype=np.uint8)
  else:
    x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  b = rng.normal(size=(cout,)).astype(np.float32)
  mask = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  res = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  want = _ref(x, w, b, mode).numpy()
  got, err = _run(cin, cout, mode, N, H, W, x, w, b, None, None, 0, split)
  assert err == 0 and _relerr(got, want) < TOL[split]
  got, err = _run(cin, cout, mode, N, H, W, x, w, b, mask, res, 0, split)
  assert err == 0 and _relerr(got, np.where(mask > 0, want, 0) + res) < TOL[split]


@pytest.mark.parametrize('split', [0, 1])
@pytest.mark.parametrize('cin,cout,N,H,W', [(16, 16, 5, 42, 42), (16, 32, 2, 42, 42), (32, 32, 7, 21, 21)])
def test_conv3x3_tc_data_gradient(cin, cout, N, H, W, split, conv_tile):
  """dX = tc_conv(dY, flipped/transposed weights) == autograd of the forward conv."""
  rng = np.random.default_rng(cin + cout)
  x = torch.tensor(rng.normal(size=(N, H, W, cin)).astype(np.float32), requires_grad=True)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  y = net_oracle._conv_nhwc(x, torch.as_tensor(w), None, 1, True)
  (y * torch.as_tensor(dy)).sum().backward()
  got, err = _run(cout, cin, 0, N, H, W, dy, w, None, None, None, 1, split)
  assert err == 0 and _relerr(got, x.grad.numpy()) < TOL[split]


@pytest.fixture(params=[512, 256, 128])
def wgrad_chunk(request):
  from seed_rl_b200 import _lib
  _lib.check(_lib.lib().seedrl_debug_set_wgrad_chunk(request.param))
  yield request.param
  _lib.check(_lib.lib().seedrl_debug_set_wgrad_chunk(256))


@pytest.mark.parametrize('split', [0, 1])
@pytest.mark.parametrize('cin,cout,mode,N,H,W', [(32, 32, 1, 3, 21, 21), (32, 32, 0, 40, 11, 11), (16, 16, 1, 5, 42, 42),
                                                 (16, 32, 0, 2, 42, 42), (32, 32, 1, 700, 21, 21), (32, 32, 0, 1, 4, 4),
                                                 (4, 16, 2, 3, 84, 84), (4, 16, 2, 40, 9, 7), (16, 16, 1, 300, 42, 42)])
def test_conv3x3_tc_weight_gradient(cin, cout, mode, N, H, W, split, wgrad_chunk):
  """dW, db on the tensor cores (MN-major operands, one register accumulator per kernel row with
  the three taps of the row stacked along N) == autograd.  mode 2 = uint8 frames / 255."""
  rng = np.random.default_rng(cin + cout + N)
  if mode == 2:
    x = rng.integers(0, 256, (N, H, W, cin), dtype=np.uint8)
  else:
    x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xin = torch.relu(torch.as_tensor(x)) if mode == 1 else torch.as_tensor(x)
  if mode == 2:
    xin = xin.float() / 255.0
  wt = torch.zeros(3, 3, cin, cout, requires_grad=True); bt = torch.zeros(cout, requires_grad=True)
  (net_oracle._conv_nhwc(xin, wt, bt, 1, True) * torch.as_tensor(dy)).sum().backward()
  dw, db, err = _run_wgrad(cin, cout, mode, N, H, W, x, dy, split)
  assert err == 0
  assert _relerr(dw, wt.grad.numpy()) < TOL[split]
  assert _relerr(db, bt.grad.numpy()) < 1e-4      # bias gradient is summed in fp32
  dw2, db2, _ = _run_wgrad(cin, cout, mode, N, H, W, x, dy, split)
  assert np.array_equal(dw, dw2) and np.array_equal(db, db2)   # deterministic


def _step_errors(conv_mode):
  from oracle import learner_oracle, loss_oracle
  from seed_rl_b200.agents.vtrace import learner
  from seed_rl_b200.common import optimizers
  from seed_rl_b200.dmlab import networks
  from test_gpu_parity import _batch_to_cuda
  A, T, B = 18, 4, 3
  params = net_oracle.init_params('deep', A, (84, 84, 4), seed=1)
  agent = networks.ImpalaDeep(A, (84, 84, 4), conv_mode=conv_mode)
  agent.load_named_parameters(params)
  cfg = loss_oracle.default_config()
  cpu = learner_oracle.CpuLearner('deep', A, (84, 84, 4), cfg, params=params)
  b = learner_oracle.synthetic_batch(T, B, A, seed=100)
  total, _, g, _ = cpu.grads(b)
  step = learner.LearnerStep(agent, optimizers.Adam(4.8e-4, beta_1=0.0, epsilon=3.125e-7))
  loss, _ = step.compute_gradients(_batch_to_cuda(b))
  mine = agent.named_gradients()
  errs = {}
  for k in g:
    if k != 'entropy_cost_param':
      a, w = mine[k].cpu().numpy().astype(np.float64), g[k].astype(np.float64)
      errs[k] = float(np.linalg.norm(a - w) / (np.linalg.norm(w) + 1e-30))
  return float(loss), float(total), errs


def test_network_step_bf16x3_matches_fp32_oracle():
  """ImpalaDeep learner step with every 16/32-channel conv (fwd, dgrad, wgrad) on wgmma in
  bf16x3 mode: the loss matches the fp32 CPU oracle to 2e-4 and all 39 gradient tensors to
  1e-2 L2-relative.  (Each bf16x3 kernel is within 2e-4 -- tests above.  This tiny
  3-unroll random batch amplifies operand rounding by ~2-3 orders of magnitude: the CPU
  oracle itself moves by 4.6e-3 when its conv operands are rounded to hi+lo bf16, which is
  exactly what the GPU shows: 5.1e-3.  The fp32 SIMT path stays the 2e-3 max-rel parity
  path in test_gpu_parity.)"""
  loss, total, errs = _step_errors('tc3')
  assert abs(loss - total) < 2e-4 * max(1.0, abs(total))
  bad = {k: v for k, v in errs.items() if not v < 1e-2}
  print('TC3_NET max L2-rel vs fp32 oracle: %.3g' % max(errs.values()))
  assert not bad, bad


def test_network_step_plain_bf16_is_reported_not_parity():
  """Plain bf16 operands ('tc'): per-kernel error is 2e-3 (tests above), but through 15
  conv layers forward and backward on a 3-unroll random batch the gradient of the first
  stack deviates ~10-15% (L2) from fp32 -- the CPU oracle with the same operand rounding
  (net_oracle.CONV_OPERAND_DTYPE=bfloat16) shows the same level, so this is what bf16
  operands cost, not a kernel defect.  That is why bf16x3 is the parity mode; this test only
  bounds the deviation and prints it."""
  loss, total, errs = _step_errors('tc')
  print('TC_NET (plain bf16) max L2-rel vs fp32 oracle: %.3g' % max(errs.values()))
  assert abs(loss - total) < 2e-2 * max(1.0, abs(total))
  assert max(errs.values()) < 0.5
  heads = [v for k, v in errs.items() if k.split('/')[0] in ('policy_logits', 'baseline', 'core')]
  assert max(heads) < 3e-2


# ---------------------------------------------------------------- dense GEMMs on wgmma
GEMM_CASES = [
    # ta, tb, M, N, K, epilogue
    (0, 0, 1344, 256, 3872, dict(bias=True, relu=True, a_relu=True)),     # Dense(256) forward (split-K)
    (0, 0, 300, 1024, 275, dict(bias=True)),                               # LSTM input projection, lda = 275
    (1, 0, 275, 1024, 333, {}),                                            # xc^T dz (TA, unaligned ld)
    (1, 0, 3872, 256, 1344, dict(a_relu=True)),                            # Dense weight gradient
    (0, 1, 1344, 3872, 256, dict(mask=True)),                              # Dense data gradient (TB)
    (0, 1, 200, 256, 1024, dict(mask=True, accumulate=True)),
    (1, 1, 129, 40, 100, dict(bias=True)),
    (0, 0, 64, 16, 32, {}), (0, 0, 130, 19, 70, dict(relu=True)), (0, 1, 65, 300, 33, {}),
    (1, 0, 256, 16, 60000, {}),                                            # im2col weight gradient: 128 K-slices (wide reduce)
    (0, 0, 128, 32, 40000, dict(bias=True, relu=True, accumulate=True))]


@pytest.mark.parametrize('split', [0, 1])
@pytest.mark.parametrize('ta,tb,M,N,K,epi', GEMM_CASES)
def test_gemm_tc_matches_numpy(ta, tb, M, N, K, epi, split):
  """C = op(A) op(B) with fp32 storage on the tensor cores (K-major / MN-major operand
  layouts chosen by the storage order, split-K, fused epilogue) against float64 numpy."""
  from seed_rl_b200 import _lib
  L = _lib.lib()
  rng = np.random.default_rng(M + 3 * N + 7 * K + ta + 2 * tb)
  A = rng.normal(size=(K, M) if ta else (M, K)).astype(np.float32)
  B = rng.normal(size=(N, K) if tb else (K, N)).astype(np.float32)
  bias = rng.normal(size=N).astype(np.float32) if epi.get('bias') else None
  mask = rng.normal(size=(M, N + 3)).astype(np.float32) if epi.get('mask') else None
  C0 = rng.normal(size=(M, N + 5)).astype(np.float32)          # ldc > N: the padding must survive
  a64 = A.astype(np.float64).T if ta else A.astype(np.float64)
  if epi.get('a_relu'):
    a64 = np.maximum(a64, 0)
  b64 = B.astype(np.float64).T if tb else B.astype(np.float64)
  want = a64 @ b64
  scale = np.abs(want).max()
  if bias is not None:
    want = want + bias
  if epi.get('relu'):
    want = np.maximum(want, 0)
  if mask is not None:
    want = np.where(mask[:, :N] > 0, want, 0)
  if epi.get('accumulate'):
    want = want + C0[:, :N]
  c = lambda a: None if a is None else torch.as_tensor(a).cuda()
  Ac, Bc, bc, mc, Cc = c(A), c(B), c(bias), c(mask), c(C0)
  ws = torch.empty(48 << 18, device='cuda')                     # 48 MB of fp32
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  outs = []
  for _ in range(2):
    Cc.copy_(torch.as_tensor(C0))
    _lib.check(L.seedrl_debug_gemm_tc(ta, tb, split, M, N, K, _lib.ptr(Ac), A.shape[1], _lib.ptr(Bc), B.shape[1],
                                      _lib.ptr(Cc), N + 5, _lib.ptr(bc), _lib.ptr(mc), N + 3,
                                      int(bool(epi.get('relu'))), int(bool(epi.get('accumulate'))),
                                      int(bool(epi.get('a_relu'))), _lib.ptr(ws), ws.numel() * 4, _lib.ptr(err),
                                      _lib.stream_ptr()))
    torch.cuda.synchronize()
    outs.append(Cc.cpu().numpy().copy())
  assert int(err.item()) == 0
  got = outs[0]
  assert np.array_equal(got[:, N:], C0[:, N:])                  # nothing written past column N
  assert np.array_equal(outs[0], outs[1])                       # deterministic (split-K in slice order)
  assert np.abs(got[:, :N] - want).max() < TOL[split] * scale


# ---------------------------------------------------------------- bias gradients (column sums)
@pytest.mark.parametrize('M,N,ld,use_ws', [
    (537600, 16, 16, True),      # shallow net conv 8x8/4 bias gradient at T=20, B=64 (row-slab path)
    (108864, 32, 32, True), (6464, 2048, 2048, True), (1344, 1024, 1024, True), (100003, 64, 64, True),
    (9024 * 49, 64, 64, True), (70001, 4, 4, True),
    (537600, 16, 16, False),     # same matrix without scratch: one CTA per 32 columns
    (1344, 18, 18, True), (1000, 32, 40, True), (21, 1, 1, True)])
def test_colsum_matches_float64(M, N, ld, use_ws):
  """out[n] = sum_m X[m, n] against a float64 sum; the slab path is deterministic and never writes
  outside its partials."""
  from seed_rl_b200 import _lib
  L = _lib.lib()
  g = torch.Generator(device='cuda').manual_seed(M + N)
  X = torch.randn(M, ld, device='cuda', generator=g) + 0.25
  ws = torch.full((1 << 20,), float('nan'), device='cuda') if use_ws else None
  outs = []
  for _ in range(2):
    out = torch.full((N + 3,), 7.0, device='cuda')
    _lib.check(L.seedrl_debug_colsum(M, N, _lib.ptr(X), ld, _lib.ptr(out), _lib.ptr(ws),
                                     ws.numel() * 4 if use_ws else 0, _lib.stream_ptr()))
    torch.cuda.synchronize()
    outs.append(out.cpu().numpy().copy())
  want = X[:, :N].double().sum(0).cpu().numpy()
  scale = float(X[:, :N].double().abs().sum(0).max())
  assert np.array_equal(outs[0], outs[1])
  assert np.all(outs[0][N:] == 7.0)
  assert np.abs(outs[0][:N] - want).max() < 2e-6 * scale
