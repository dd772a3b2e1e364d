"""The 'valid' strided convolutions of the R2D2 body (atari/networks.py:228-238: 8x8/4 -> 32, 4x4/2 -> 64,
3x3/1 -> 64) and of the IMPALA shallow net (8x8/4 -> 16, 4x4/2 -> 32), one layer at a time through
seedrl_debug_strided_conv (the calls csrc/r2d2_net.cu and csrc/net.cu make for a layer), against float64
torch: conv2d + bias + ReLU, its weight / bias gradient and its input gradient masked by the ReLU'd input.

Sizes: the benchmarked unrolls (R2D2 burn-in 40 x 64 = 2 560 and suffix 101 x 64 = 6 464 frames; shallow net
T+1 = 21 x 64 = 1 344 and 21 x 256 = 5 376 frames), one and three frames, geometries the gathered operand
cannot take (the materialised path must run, and is asserted to), frames whose last rows / columns no window
covers, and one forward just under the R2D2 net's 8 000 000-row cap.

Every output is poisoned with NaN first (every element must be written; the columns of a padded leading
dimension past C_out must stay untouched), every run is repeated (bit-identical), and the gathered operand
must give the materialised one's result bit for bit.

Bars (DESIGN.md section 2): wgmma bf16x3 max|a-w| <= 2e-4 max|w|, bf16 1.5e-2 max|w|; fp32 SIMT rtol 2e-4,
atol 2e-5 element-wise (as test_gpu_parity.py::test_conv3x3_kernel) for the forward and the data gradient.
The SIMT weight and bias gradients reduce over all M = N Ho Wo positions (2.6 M at the R2D2 suffix) with one
fp32 accumulator per output: a float32 running sum of 2.6 M products of u8/255 frames and a zero-mean
gradient lands 1e-2 .. 5e-2 away from the float64 sum (2.4e-4 relative on an entry of magnitude 26, measured
with numpy's sequential float32 cumsum), so an element-wise 2e-4 bar measures the fp32 summation order, not
the kernel.  Those two tensors are held to 2e-4 of their max-abs instead, the bar of the bf16x3 path.
"""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from seed_rl_b200 import _lib

WS_BYTES = 48 << 20          # gemm_tc_workspace_bytes()
MODES = (0, 1, 2)            # SIMT sgemm, bf16 gemm_tc, bf16x3 gemm_tc
NAME = {0: 'simt', 1: 'bf16', 2: 'bf16x3'}
REL_BAR = {1: 1.5e-2, 2: 2e-4}
CHUNK = 256                  # frames per float64 reference chunk (bounds host memory)


def _geom(H, W, K, S):
  return (H - K) // S + 1, (W - K) // S + 1


def _x_float(x):
  return torch.as_tensor(x).double() / 255.0 if x.dtype == np.uint8 else torch.as_tensor(x).double()


def _reference(x, w, b, dy, mask, S, ops):
  """float64 torch over frame chunks: y = relu(conv(x) + b) [M, cout], dW (HWIO), db, dx [N,H,W,C]."""
  N, H, W, C = x.shape
  K, cout = w.shape[0], w.shape[3]
  Ho, Wo = _geom(H, W, K, S)
  wt = torch.as_tensor(w).double().permute(3, 2, 0, 1).contiguous()         # OIHW
  bt = torch.as_tensor(b).double()
  y, dx = [], []
  dw = torch.zeros_like(wt)
  db = torch.zeros(cout, dtype=torch.float64)
  for n0 in range(0, N, CHUNK):
    xs = _x_float(x[n0:n0 + CHUNK]).permute(0, 3, 1, 2)                      # NCHW
    if 0 in ops:
      y.append(torch.relu(F.conv2d(xs, wt, bt, stride=S)).permute(0, 2, 3, 1).reshape(-1, cout))
    if 1 in ops or 2 in ops:
      g = torch.as_tensor(dy[n0 * Ho * Wo:(n0 + CHUNK) * Ho * Wo]).double().reshape(-1, Ho, Wo, cout)
      g = g.permute(0, 3, 1, 2)
      if 1 in ops:
        dw += torch.nn.grad.conv2d_weight(xs, wt.shape, g, stride=S)
        db += g.sum((0, 2, 3))
      if 2 in ops:
        d = torch.nn.grad.conv2d_input(xs.shape, wt, g, stride=S).permute(0, 2, 3, 1)
        dx.append(torch.where(torch.as_tensor(mask[n0:n0 + CHUNK]) > 0, d, torch.zeros((), dtype=d.dtype)))
  ref = {}
  if 0 in ops:
    ref[0] = torch.cat(y).numpy()
  if 1 in ops:
    ref[1] = (dw.permute(2, 3, 1, 0).reshape(K * K * C, cout).numpy(), db.numpy())
  if 2 in ops:
    ref[2] = torch.cat(dx).numpy()
  return ref


def _call(op, mode, gather, x, N, H, W, C, K, S, cout, w, b, dy, mask, out, ldo, dbias, col):
  L = _lib.lib()
  flag, gathered = torch.zeros(1, dtype=torch.int32, device='cuda'), ctypes.c_int(-1)
  ws = _call.ws
  xp = None if x is None else ctypes.c_void_p(x.data_ptr())
  _lib.check(L.seedrl_debug_strided_conv(op, mode, gather, int(x is not None and x.dtype == torch.uint8), N, H, W, C,
                                         K, S, cout, xp, _lib.ptr(w), _lib.ptr(b), _lib.ptr(dy), _lib.ptr(mask),
                                         _lib.ptr(out), ldo, _lib.ptr(dbias), _lib.ptr(col),
                                         0 if col is None else col.numel() * 4, _lib.ptr(ws), WS_BYTES,
                                         _lib.ptr(flag), ctypes.byref(gathered), _lib.stream_ptr()))
  torch.cuda.synchronize()
  assert int(flag.item()) == 0
  return gathered.value


def _err(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _check(name, mode, got, want, reduction):
  """The bar of `mode` for one tensor; prints the worst relative error."""
  assert np.isfinite(got).all(), name
  err = _err(got, want)
  if mode == 0 and not reduction:
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-5, err_msg=name)
    bar = 2e-4
  else:
    bar = 2e-4 if mode == 0 else REL_BAR[mode]
    assert err <= bar, (name, err, bar)
  return '%s %.1e/%.2g' % (name, err, bar)


def _run_case(N, H, W, C, K, S, cout, u8, ops, x_offset=0, expect_gather=None, uncovered=False, seed=0):
  """All modes, gathered and materialised, every op in `ops`, against one float64 reference."""
  rng = np.random.default_rng(seed + N + H + C + cout)
  Ho, Wo = _geom(H, W, K, S)
  M, KC = N * Ho * Wo, K * K * C
  if u8:
    x = rng.integers(0, 256, (N, H, W, C), dtype=np.uint8)
  else:
    x = np.maximum(rng.normal(size=(N, H, W, C)), 0).astype(np.float32)   # a ReLU'd activation: ~half exact zeros
  w = (rng.normal(size=(K, K, C, cout)) / np.sqrt(KC)).astype(np.float32)
  b = (0.1 * rng.normal(size=cout)).astype(np.float32)
  # the gradient that reaches a ReLU'd layer output is zero wherever that output is
  dy = (rng.normal(size=(M, cout)) * (rng.random((M, cout)) < 0.6)).astype(np.float32) if ops != (0,) else None
  mask = x if 2 in ops else None
  ref = _reference(x, w, b, dy, mask, S, ops)
  if uncovered:
    # pixels below the last window row / right of the last window column get no gradient at all
    assert (Ho - 1) * S + K < H or (Wo - 1) * S + K < W
    assert not ref[2][:, (Ho - 1) * S + K:].any() and not ref[2][:, :, (Wo - 1) * S + K:].any()

  xc = torch.as_tensor(x).cuda()
  if x_offset:
    # the same tensor starting 4 bytes past a 16-byte boundary
    buf = torch.empty(x.size + 4, dtype=xc.dtype, device='cuda')
    xc = buf[1:1 + x.size].view(x.shape).copy_(xc)
  wc, bc = torch.as_tensor(w).cuda(), torch.as_tensor(b).cuda()
  dyc = None if dy is None else torch.as_tensor(dy).cuda()
  mc = None if mask is None else torch.as_tensor(mask).cuda()
  col = torch.empty(M * KC, device='cuda')
  _call.ws = torch.empty(WS_BYTES // 4, device='cuda')
  nan = float('nan')
  report = []
  for op in ops:
    for mode in MODES:
      res = {}
      for gather in ((1, 0) if mode else (0,)):
        runs = []
        for _ in range(2):
          if op == 2:
            out = torch.full((N, H, W, C), nan, device='cuda')
            g = _call(2, mode, gather, None, N, H, W, C, K, S, cout, wc, None, dyc, mc, out, 0, None, col)
            runs.append((out,))
          else:
            rows, ldo = (M, cout + 4) if op == 0 else (KC, cout + 4)
            out = torch.full((rows, ldo), nan, device='cuda')
            dbias = torch.full((cout,), nan, device='cuda') if op == 1 else None
            g = _call(op, mode, gather, xc, N, H, W, C, K, S, cout, wc, bc, dyc, None, out, ldo, dbias, col)
            assert bool(torch.isnan(out[:, cout:]).all()), 'padding columns written'
            runs.append((out[:, :cout].contiguous(),) + ((dbias,) if op == 1 else ()))
          if op != 2 and gather and expect_gather is not None:
            assert g == expect_gather, (op, mode, g)
          if op == 2 or not gather or mode == 0:
            assert g == 0
        for t0, t1 in zip(*runs):
          assert torch.equal(t0, t1), 'two runs differ (op %d mode %d gather %d)' % (op, mode, gather)
        res[(gather, g)] = runs[0]
      if len(res) == 2 and (1, 1) in res:       # gathered and materialised both ran
        for t0, t1 in zip(res[(1, 1)], res[(0, 0)]):
          assert torch.equal(t0, t1), 'gathered != materialised (op %d mode %d)' % (op, mode)
      got = [t.cpu().numpy() for t in next(iter(res.values()))]
      if op == 0:
        report.append(_check('fwd/' + NAME[mode], mode, got[0], ref[0], False))
      elif op == 1:
        report.append(_check('dW/' + NAME[mode], mode, got[0], ref[1][0], True))
        report.append(_check('db/' + NAME[mode], mode, got[1], ref[1][1], True))
      else:
        report.append(_check('dx/' + NAME[mode], mode, got[0], ref[2], False))
        if uncovered:
          d = got[0]
          assert not d[:, (Ho - 1) * S + K:].any() and not d[:, :, (Wo - 1) * S + K:].any()
  print('STRIDED N=%d %dx%dx%d %s -> %dx%dx%d (K%d/S%d): %s' % (N, H, W, C, 'u8' if u8 else 'f32', Ho, Wo, cout,
                                                                 K, S, '; '.join(report)))
  del col, xc, dyc, mc
  _call.ws = None
  torch.cuda.empty_cache()


# (H, W, C, K, S, cout, u8, ops) of the R2D2 body on 84x84 frames stacked 4
R2D2 = {'conv1': (84, 84, 4, 8, 4, 32, True, (0, 1)),
        'conv2': (20, 20, 32, 4, 2, 64, False, (0, 1, 2)),
        'conv3': (9, 9, 64, 3, 1, 64, False, (0, 1, 2))}


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1, 3, 2560, 6464])
@pytest.mark.parametrize('layer', sorted(R2D2))
def test_r2d2_body_layer_vs_float64(layer, N):
  H, W, C, K, S, cout, u8, ops = R2D2[layer]
  _run_case(N, H, W, C, K, S, cout, u8, ops)


@pytest.mark.gpu
@pytest.mark.parametrize('N', [1344, 5376])
@pytest.mark.parametrize('layer', ['conv0', 'conv1'])
def test_shallow_net_layer_vs_float64(layer, N):
  if layer == 'conv0':
    _run_case(N, 84, 84, 4, 8, 4, 16, True, (0, 1), expect_gather=1)
  else:
    _run_case(N, 20, 20, 16, 4, 2, 32, False, (0, 1, 2), expect_gather=1)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['u8_c1', 'u8_72x96x3', 'f32_offset4'])
def test_fallback_geometries_materialise(case):
  """Geometries conv_gather_setup refuses: the materialised im2col (4-channel vectors or scalar) runs."""
  if case == 'u8_c1':                # W*C = 84: 8-byte groups straddle rows
    _run_case(37, 84, 84, 1, 8, 4, 32, True, (0, 1), expect_gather=0)
  elif case == 'u8_72x96x3':         # S*C = 12: im2col_kernel<true, 1>
    _run_case(29, 72, 96, 3, 8, 4, 32, True, (0, 1), expect_gather=0)
  else:                              # 16-byte loads impossible: x 4 bytes past alignment
    _run_case(50, 20, 20, 32, 4, 2, 64, False, (0, 1), x_offset=1, expect_gather=0)


@pytest.mark.gpu
@pytest.mark.parametrize('case', ['u8_85x83', 'f32_85x83', 'f32_10x9'])
def test_uncovered_remainders(case):
  """(H-K) or (W-K) not a multiple of S: the last rows / columns are in no window; their data gradient is 0."""
  if case == 'u8_85x83':             # conv1 on 85x83 frames: 20x19 outputs, row 84 / columns 80-82 unread
    _run_case(41, 85, 83, 4, 8, 4, 32, True, (0, 1), expect_gather=0)
  elif case == 'f32_85x83':          # 4x4/2 on 85x83x16: row 84 and column 82 uncovered; gathered
    _run_case(23, 85, 83, 16, 4, 2, 32, False, (0, 1, 2), expect_gather=1, uncovered=True)
  else:                              # conv2 of the 44x40 R2D2 net: 10x9x32 -> 4x3x64, column 8 uncovered
    _run_case(333, 10, 9, 32, 4, 2, 64, False, (0, 1, 2), expect_gather=1, uncovered=True)


@pytest.mark.gpu
def test_conv1_forward_near_r2d2_row_cap():
  """seedrl_r2d2_net_forward takes up to 8 000 000 conv1 rows: 19 999 frames give 7 999 600 (62 497 tiles of
  128 rows along grid.y for gemm_tc, 124 994 tiles of 64 rows for the SIMT sgemm, past grid.y's 65 535).
  float64 reference on 20 000 random rows, every row of the last frame and of the 128-row tiles holding the
  last frame's first row and the last row."""
  N, H, W, C, K, S, cout = 19999, 84, 84, 4, 8, 4, 32
  Ho, Wo = _geom(H, W, K, S)
  M, KC = N * Ho * Wo, K * K * C
  assert M < 8000000 <= M + Ho * Wo
  rng = np.random.default_rng(8)
  x = rng.integers(0, 256, (N, H, W, C), dtype=np.uint8)
  w = (rng.normal(size=(K, K, C, cout)) / np.sqrt(KC)).astype(np.float32)
  b = (0.1 * rng.normal(size=cout)).astype(np.float32)
  first_last = (N - 1) * Ho * Wo
  rows = np.unique(np.concatenate([
      rng.choice(M, 20000, replace=False), np.arange(first_last, M),
      np.arange(first_last // 128 * 128, first_last // 128 * 128 + 128), np.arange((M - 1) // 128 * 128, M)]))
  n, r = rows // (Ho * Wo), rows % (Ho * Wo)
  ho, wo = r // Wo, r % Wo
  hh = ho[:, None] * S + np.arange(K)[None]                          # [R, K]
  ww = wo[:, None] * S + np.arange(K)[None]
  patches = x[n[:, None, None], hh[:, :, None], ww[:, None, :]].astype(np.float64) / 255.0   # [R, K, K, C]
  want = np.maximum(patches.reshape(len(rows), KC) @ w.reshape(KC, cout).astype(np.float64) + b, 0)
  xc, wc, bc = torch.as_tensor(x).cuda(), torch.as_tensor(w).cuda(), torch.as_tensor(b).cuda()
  rows_c = torch.as_tensor(rows).cuda()
  col = torch.empty(M * KC, device='cuda')
  _call.ws = torch.empty(WS_BYTES // 4, device='cuda')
  report, kept = [], {}
  for mode, gather in ((0, 0), (2, 1), (2, 0), (1, 1)):
    outs = []
    for _ in range(2):
      out = torch.full((M, cout), float('nan'), device='cuda')
      g = _call(0, mode, gather, xc, N, H, W, C, K, S, cout, wc, bc, None, None, out, cout, None, col)
      assert g == gather
      assert not bool(torch.isnan(out).any()), 'rows left unwritten'
      outs.append(out)
    assert torch.equal(outs[0], outs[1])
    got = outs[0][rows_c].cpu().numpy()
    del outs[1]
    if mode == 2:
      if gather:
        kept[2] = outs[0]
      else:
        assert torch.equal(kept.pop(2), outs[0]), 'gathered != materialised'
    if mode == 0:
      np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-5)
      report.append('simt %.1e' % _err(got, want))
    else:
      err = _err(got, want)
      assert err <= REL_BAR[mode], (mode, err)
      report.append('%s%s %.1e/%.2g' % (NAME[mode], '/gather' if gather else '', err, REL_BAR[mode]))
    del outs
  print('STRIDED cap N=%d M=%d rows checked %d: %s' % (N, M, len(rows), '; '.join(report)))
  del col, xc, kept
  _call.ws = None
  torch.cuda.empty_cache()


def test_strided_conv_refuses_bad_arguments():
  """CPU: refusals are argument errors (code 3), raised before anything is launched."""
  L = _lib.lib()
  p = ctypes.c_void_p(16)
  args = lambda op, mode, N, col_bytes, ldo: (op, mode, 1, 1, N, 84, 84, 4, 8, 4, 32, p, p, p, p, p, p, ldo, p, p,
                                              col_bytes, None, 0, None, None, None)
  assert L.seedrl_debug_strided_conv(*args(3, 2, 1, 1 << 30, 32)) == 3        # op
  assert L.seedrl_debug_strided_conv(*args(0, 3, 1, 1 << 30, 32)) == 3        # mode
  assert L.seedrl_debug_strided_conv(*args(0, 2, 0, 1 << 30, 32)) == 3        # N
  assert L.seedrl_debug_strided_conv(*args(0, 2, 1, 1 << 30, 31)) == 3        # ldo < cout
  assert L.seedrl_debug_strided_conv(*args(0, 0, 1, 100, 32)) == 3            # SIMT: column scratch too small
  assert L.seedrl_debug_strided_conv(*args(2, 2, 1, 100, 0)) == 3             # data gradient: column scratch
