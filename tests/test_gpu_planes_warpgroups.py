"""GPU: convp_kernel's block scheduling.  Four MMA + epilogue warpgroups take a CTA's 64-position
blocks round-robin over its tiles, through 2..4 smem stages, and each warpgroup releases a stage
exactly once per tile.  These shapes reach the schedules the learner's own shapes do not:

  * NSUB = 2 (small batches): fewer tiles than SMs, and a tile count that is not a multiple of
    the grid, so CTAs own different numbers of tiles
  * CTAs that walk more tiles than there are stages (NSUB = 4 with 4 stages, NSUB = 2 with 3, NSUB = 1
    with 2)
  * NSUB = 1 (images too wide for 256-position tiles): 2 blocks per tile, so half the warpgroups have
    no block in a tile
  * the fp32 NHWC output at 11x11

Every case runs the bias + ReLU-mask + residual epilogue with all three outputs (raw planes, ReLU'd
planes, fp32 NHWC) against float64, checks that every padding position of the plane outputs is
written as zero, and runs twice: both runs must be bit-identical."""
import numpy as np
import pytest
import torch

from test_gpu_planes import TOL, _L, _from_planes, _planes_buf, _ref_conv, _to_planes

pytestmark = pytest.mark.gpu

CASES = [
    # cin, cout, N, H, W               tiles / CTAs (132 SMs), tile size, stages
    (16, 16, 2, 21, 21),           # 6 / 6, NSUB = 2, 4 stages
    (32, 32, 250, 11, 11),         # 154 / 132, NSUB = 2, 3 stages
    (32, 32, 252, 21, 21),         # 500 / 132 (up to 4 tiles per CTA), NSUB = 2, 3 stages
    (16, 16, 200, 42, 42),         # 740 / 132 (up to 6 tiles per CTA), NSUB = 4, 4 stages
    (16, 32, 3, 4, 200),           # 14 / 14, NSUB = 2, 4 stages
    (32, 16, 40, 6, 200),          # 224 / 132, NSUB = 2, 2 stages
    (32, 32, 2, 5, 200),           # 24 / 24, NSUB = 1, 2 stages
    (32, 32, 60, 5, 200),          # 573 / 132 (up to 5 tiles per CTA), NSUB = 1, 2 stages
]


def _pixel_positions(N, H, W):
  n, h, w = np.meshgrid(np.arange(N), np.arange(H), np.arange(W), indexing='ij')
  return ((n * (H + 1) + h + 1) * (W + 2) + w + 1).ravel()


@pytest.mark.parametrize('cin,cout,N,H,W', CASES)
def test_convp_warpgroup_schedule(cin, cout, N, H, W):
  _lib, L = _L()
  rng = np.random.default_rng(3 * cin + cout + N + W)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  bias = rng.normal(size=cout).astype(np.float32)
  res = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  msk = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xin, resp, mskp = _to_planes(x), _to_planes(res), _to_planes(msk, relu=1)
  wq = torch.empty(2 * 9 * cin * cout * 2, dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  wc, bc = torch.as_tensor(w).cuda(), torch.as_tensor(bias).cuda()

  runs = []
  for _ in range(2):
    raw = _planes_buf(N, H, W, cout, fill=0xFF)
    relu = _planes_buf(N, H, W, cout, fill=0xFF)
    nhwc = torch.full((N, H, W, cout), float('nan'), device='cuda')
    _lib.check(L.seedrl_debug_convp(cin, cout, N, H, W, _lib.ptr(xin), _lib.ptr(wc), _lib.ptr(bc), _lib.ptr(mskp),
                                    _lib.ptr(resp), 0, _lib.ptr(raw), _lib.ptr(relu), _lib.ptr(nhwc), _lib.ptr(wq),
                                    _lib.ptr(err), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert int(err.item()) == 0
    runs.append((raw, relu, nhwc))
  for a, b in zip(*runs):
    assert torch.equal(a, b)                                # bit-identical, padding bytes included

  raw, relu, nhwc = runs[0]
  base = _ref_conv(x, w, bias)
  want = np.where(msk > 0, base, 0) + res
  scale = max(np.abs(base).max(), np.abs(want).max())
  assert np.abs(_from_planes(raw, N, H, W, cout) - want).max() < TOL * scale
  assert np.abs(_from_planes(relu, N, H, W, cout) - np.maximum(want, 0)).max() < TOL * scale
  assert np.abs(nhwc.cpu().numpy() - want).max() < TOL * scale
  # every storage position that is not a pixel is zero in every plane (the next conv's halo)
  pad = np.ones(int(L.seedrl_debug_planes_bytes(N, H, W, cout)) // (4 * cout), bool)
  pad[_pixel_positions(N, H, W)] = False
  for buf in (raw, relu):
    planes = buf.cpu().numpy().view(np.uint16).reshape(2 * (cout // 8), -1, 8)
    assert (planes[:, pad] == 0).all()
