"""GPU: wgradp_kernel's pipeline.  Each K chunk copies x and dy once, plus a halo, into 2..6 smem
stages; A is built in registers with its kw shift, B's kh shift is a descriptor offset, and for
16-channel inputs three warpgroups per M-tile each take one kh of every chunk.  These shapes reach
the schedules the learner's own shapes do not:

  * CTAs that walk more chunks than there are stages, at every (cin, cout)
  * chunk counts that are not a multiple of the grid, and fewer chunks than SMs
  * 200-pixel rows, where the dy halo (2 * PW positions) is longer than the chunk itself
  * odd PW (row pitch W + 2), so the kh and kw shifts are not multiples of 8 positions
  * dy with a nonzero mean, so the bias gradient (the constant-fragment row) is large

Each case is checked against float64, checked to be bit-identical across two runs, and checked to
leave the error flag at 0.  The learner's own shapes are checked against float64 at the benchmark's
batch too."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_planes import TOL, _L, _to_planes

pytestmark = pytest.mark.gpu

CASES = [
    # cin, cout, N, H, W, dy mean      K chunks / CTAs (132 SMs), chunk KC, stages
    (16, 16, 200, 42, 42, 0.0),      # 1479 / 132 (11 or 12 per CTA), 256, 5
    (16, 32, 100, 42, 42, 0.0),      # 1479 / 132, 128, 6
    (32, 32, 500, 21, 21, 0.0),      # 1977 / 132, 128, 5
    (32, 32, 300, 11, 11, 0.5),      # 366 / 132, 128, 6
    (16, 16, 2, 21, 21, 0.5),        # 5 / 5, PW = 23
    (16, 32, 5, 11, 13, 0.0),        # 8 / 8, PW = 15
    (32, 32, 3, 11, 11, 0.0),        # 4 / 4, PW = 13
    (16, 16, 3, 5, 200, 0.0),        # 15 / 15, 2 * PW = 404 > KC = 256, 3
    (16, 32, 4, 4, 200, 0.5),        # 34 / 34, 2 * PW > KC = 128, 3
    (32, 32, 6, 5, 200, 0.0),        # 59 / 59, 2 * PW > KC = 128, 2
    (32, 32, 40, 6, 200, 0.0),       # 444 / 132, 128, 2
    (16, 16, 30, 17, 35, 0.0),       # 79 / 79, PW = 37
]


def _wgradp(cin, cout, N, H, W, xp, dyp, runs=2):
  _lib, L = _L()
  dw = torch.full((3, 3, cin, cout), float('nan'), device='cuda')
  db = torch.full((cout,), float('nan'), device='cuda')
  partial = torch.empty(148 * (9 * cin * cout + cout), device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  outs = []
  for _ in range(runs):
    _lib.check(L.seedrl_debug_wgradp(cin, cout, N, H, W, _lib.ptr(xp), _lib.ptr(dyp), _lib.ptr(dw), _lib.ptr(db),
                                     _lib.ptr(partial), partial.numel() * 4, _lib.ptr(err), _lib.stream_ptr()))
    torch.cuda.synchronize()
    outs.append((dw.cpu().numpy().copy(), db.cpu().numpy().copy()))
  assert int(err.item()) == 0
  return outs


def _want(x, dy, device):
  xt = torch.as_tensor(x, dtype=torch.float64, device=device).permute(0, 3, 1, 2)
  cin, cout = x.shape[3], dy.shape[3]
  wt = torch.zeros(cout, cin, 3, 3, dtype=torch.float64, device=device, requires_grad=True)
  bt = torch.zeros(cout, dtype=torch.float64, device=device, requires_grad=True)
  y = F.conv2d(xt, wt, bt, padding=1)
  y.backward(torch.as_tensor(dy, dtype=torch.float64, device=device).permute(0, 3, 1, 2))
  return wt.grad.permute(2, 3, 1, 0).cpu().numpy(), bt.grad.cpu().numpy()


@pytest.mark.parametrize('cin,cout,N,H,W,mean', CASES)
def test_wgradp_pipeline(cin, cout, N, H, W, mean):
  rng = np.random.default_rng(cin * 7 + cout + N + W)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  dy = (rng.normal(size=(N, H, W, cout)) + mean).astype(np.float32)
  outs = _wgradp(cin, cout, N, H, W, _to_planes(x), _to_planes(dy))
  assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
  want_w, want_b = _want(x, dy, 'cpu')
  got_w, got_b = outs[0]
  assert np.abs(got_w - want_w).max() < TOL * np.abs(want_w).max()
  assert np.abs(got_b - want_b).max() < TOL * max(np.abs(want_b).max(), np.sqrt(N * H * W))


# the learner step's wgradp launches at the benchmark batch (T + 1 = 21 frames x 64 unrolls), with
# post-ReLU activations as x
@pytest.mark.parametrize('cin,cout,H', [(16, 16, 42), (16, 32, 42), (32, 32, 21), (32, 32, 11)])
def test_wgradp_learner_shapes(cin, cout, H):
  N = 21 * 64
  g = torch.Generator(device='cuda').manual_seed(cin + cout + H)
  x = torch.relu(torch.randn(N, H, H, cin, device='cuda', generator=g)).cpu().numpy()
  dy = (torch.randn(N, H, H, cout, device='cuda', generator=g) * 1e-3).cpu().numpy()
  outs = _wgradp(cin, cout, N, H, H, _to_planes(x), _to_planes(dy))
  assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
  want_w, want_b = _want(x, dy, 'cuda')
  got_w, got_b = outs[0]
  assert np.abs(got_w - want_w).max() < TOL * np.abs(want_w).max()
  assert np.abs(got_b - want_b).max() < TOL * np.abs(want_b).max()
