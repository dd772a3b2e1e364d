"""GPU: convp_kernel epilogue combinations the ImpalaDeep step launches most, which
test_gpu_planes.py::test_convp_forward_all_epilogues does not cover on their own:

  * ReLU mask without residual            (data gradients of conv11 and conv01)
  * residual with raw planes only         (conv11 of every stack but the last)
  * residual with fp32 NHWC only          (conv11 of the last stack)

each against a float64 reference, and each run twice: the two outputs must be bit-identical.
Shapes reach the NSUB = 4 and 2 variants, CTAs owning several tiles (odd and even counts) and a
single-tile launch.  Same tolerance as test_gpu_planes.py (bf16x3 split operands)."""
import numpy as np
import pytest
import torch

from test_gpu_planes import TOL, _L, _from_planes, _planes_buf, _ref_conv, _to_planes

pytestmark = pytest.mark.gpu

CASES = [
    # cin, cout, N, H, W
    (16, 16, 84, 42, 42),      # NSUB = 4, several tiles per CTA
    (32, 32, 330, 21, 21),     # NSUB = 4, 32 channels
    (16, 32, 2, 42, 42),
    (32, 16, 9, 21, 21),       # small batch: NSUB = 2
    (32, 32, 5, 11, 11),
    (16, 16, 1, 1, 1),         # one tile
]


@pytest.mark.parametrize('cin,cout,N,H,W', CASES)
def test_convp_epilogue_combinations(cin, cout, N, H, W):
  _lib, L = _L()
  rng = np.random.default_rng(7 * cin + cout + N + H)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
  bias = rng.normal(size=cout).astype(np.float32)
  res = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  xin, resp = _to_planes(x), _to_planes(res)
  wq = torch.empty(2 * 9 * cin * cout * 2, dtype=torch.uint8, device='cuda')
  err = torch.zeros(1, dtype=torch.int32, device='cuda')
  wc, bc = torch.as_tensor(w).cuda(), torch.as_tensor(bias).cuda()

  def run(src, ci, co, bias_t, mask_t, res_t, raw, nhwc, flip):
    outs = []
    for _ in range(2):
      out_raw = _planes_buf(N, H, W, co, fill=0xFF) if raw else None
      out_nhwc = torch.full((N, H, W, co), float('nan'), device='cuda') if nhwc else None
      _lib.check(L.seedrl_debug_convp(ci, co, N, H, W, _lib.ptr(src), _lib.ptr(wc), _lib.ptr(bias_t),
                                      _lib.ptr(mask_t), _lib.ptr(res_t), flip, _lib.ptr(out_raw), None,
                                      _lib.ptr(out_nhwc), _lib.ptr(wq), _lib.ptr(err), _lib.stream_ptr()))
      torch.cuda.synchronize()
      assert int(err.item()) == 0
      outs.append((out_raw if raw else out_nhwc).cpu().numpy())
    assert np.array_equal(outs[0], outs[1])                 # deterministic, padding bytes included
    return outs[0]

  base = _ref_conv(x, w, bias)
  want = base + res
  scale = max(np.abs(base).max(), np.abs(want).max())
  # residual, raw planes only
  raw = run(xin, cin, cout, bc, None, resp, True, False, 0)
  got = _from_planes(torch.as_tensor(raw).cuda(), N, H, W, cout)
  assert np.abs(got - want).max() < TOL * scale
  # residual, fp32 NHWC only
  y = run(xin, cin, cout, bc, None, resp, False, True, 0)
  assert np.abs(y - want).max() < TOL * scale
  # data gradient: ReLU mask without residual
  dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
  mk_in = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  dyp, mk_p = _to_planes(dy), _to_planes(mk_in, relu=1)
  raw = run(dyp, cout, cin, None, mk_p, None, True, False, 1)
  wflip = np.ascontiguousarray(w[::-1, ::-1].transpose(0, 1, 3, 2))
  dx = _ref_conv(dy, wflip, None)
  want = np.where(mk_in > 0, dx, 0)
  got = _from_planes(torch.as_tensor(raw).cuda(), N, H, W, cin)
  assert np.abs(got - want).max() < TOL * np.abs(dx).max()
