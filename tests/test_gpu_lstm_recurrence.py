"""The LSTM recurrence on its own (seedrl_debug_lstm_forward / _backward: the calls the networks make, csrc/lstm.cu)
in every lstm_mode against a float64 Keras LSTMCell with done-resets, forward and BPTT.

Modes: 2 tiled, 3 tiled on wgmma bf16x3 ('tc3'), at H = 256 (IMPALA) and H = 512 (R2D2).

Reference: `ref_forward` / `ref_backward` below, the schedule of tests/test_backward_formulas.py in float64 on the
same fp32 inputs the GPU gets; `test_reference_matches_torch_float64_autograd` checks it against torch autograd
through oracle/net_oracle.lstm_cell.

Bars (DESIGN.md's sensitivity rule).  For each output (gates, hs, cs, hp, final (h, c), dz, and dU = hp^T dz taken
in float64 from the GPU's hp and dz) the error is max|gpu - ref| / max|ref|.  The response is the same measure
between the reference and the reference run on U, x W + b, h0 and c0 each multiplied by (1 +- 2^-24) (mode 2,
fp32 rounding) or (1 +- 2^-16) (mode 3), random signs.  The bar is
max(FLOOR, K x response) with K = SENS_MULT and FLOOR below, one pair for every case.  The kernels round at every
step while the probe perturbs the inputs once, so K leaves room for accumulation over 141 steps.

The bf16x3 bars are loose.  The 2^-16 probe is coarser than the arithmetic (a hi + lo pair keeps an operand to
about 2^-17 and the products accumulate in fp32): measured on an H100, 'tc3' sits about 100x under its bars
(hs 2.2e-6 against 2.3e-4 at H = 512, T1 = 141, B = 64).  Dropping one of the three bf16x3 products still fails
them (the forward lo(h) hi(U) product by 6x on gates at 1 x 64; the BPTT hi(dZ) lo(U) partner by 1.0x to 5.4x on
dz / dU, only where T1 > 1), but a defect worth a fraction of one lo product would pass.

Also checked: nothing is written outside the outputs (every output has a NaN-filled extra time step and extra rows
that must stay NaN, and every element inside must be written); two calls are bit-identical, also when a call in
another mode used the workspace in between; the error flag stays 0; H = 128 and one row past each mode's batch
limit are refused with nothing launched, and so is every mode but 2 and 3.
"""
import zlib

import numpy as np
import pytest
import torch

SENS_MULT = 8
FLOOR = 2e-6


def _eps(mode):
  """Relative input perturbation of the response: fp32 rounding, or the bf16x3 model."""
  return 2.0 ** -16 if mode == 3 else 2.0 ** -24

OUTPUTS = ('gates', 'hs', 'cs', 'hp', 'h_T', 'c_T', 'dz', 'dU')
INVALID_ARGUMENT = 3


# ---- float64 reference -----------------------------------------------------------------------------------
def _sig(x):
  return 0.5 * (1.0 + np.tanh(0.5 * x))        # 1 / (1 + e^-x), without overflow warnings at |x| ~ 100


def ref_forward(U, done, xwb, h0, c0):
  """Keras LSTMCell(H) over T1 steps with done-resets; returns (gates, cs, hs, hp) [T1, B, 4H / H]."""
  T1, B, H4 = xwb.shape
  H = H4 // 4
  gates = np.empty((T1, B, H4)); cs = np.empty((T1, B, H)); hs = np.empty((T1, B, H)); hp = np.empty((T1, B, H))
  hp[0] = np.where(done[0][:, None], 0.0, h0)
  for t in range(T1):
    zt = xwb[t] + hp[t] @ U
    gi, gf, gg, go = _sig(zt[:, :H]), _sig(zt[:, H:2 * H]), np.tanh(zt[:, 2 * H:3 * H]), _sig(zt[:, 3 * H:])
    cprev = np.where(done[t][:, None], 0.0, c0 if t == 0 else cs[t - 1])
    cs[t] = gf * cprev + gi * gg
    hs[t] = go * np.tanh(cs[t])
    gates[t] = np.concatenate([gi, gf, gg, go], 1)
    if t + 1 < T1:
      hp[t + 1] = np.where(done[t + 1][:, None], 0.0, hs[t])
  return gates, cs, hs, hp


def ref_backward(U, done, gates, cs, c0, dhs):
  """BPTT of ref_forward for d loss / d hs = dhs: d loss / d (x W + b) [T1, B, 4H]."""
  T1, B, H = cs.shape
  dz = np.empty((T1, B, 4 * H))
  dhrec = dcn = None
  for t in range(T1 - 1, -1, -1):
    gi, gf, gg, go = np.split(gates[t], 4, 1)
    cut = done[t + 1][:, None] if t + 1 < T1 else None
    dh = dhs[t].copy()
    if dhrec is not None:
      dh += np.where(cut, 0.0, dhrec)
    tc = np.tanh(cs[t])
    dc = dh * go * (1 - tc * tc)
    if dcn is not None:
      dc += np.where(cut, 0.0, dcn)
    cprev = np.where(done[t][:, None], 0.0, c0 if t == 0 else cs[t - 1])
    dz[t] = np.concatenate([dc * gg * gi * (1 - gi), dc * cprev * gf * (1 - gf), dc * gi * (1 - gg * gg),
                            dh * tc * go * (1 - go)], 1)
    dcn = dc * gf
    dhrec = dz[t] @ U.T
  return dz


def _dU(hp, dz):
  return hp.reshape(-1, hp.shape[-1]).T @ dz.reshape(-1, dz.shape[-1])


def ref_all(U, done, xwb, h0, c0, dhs):
  gates, cs, hs, hp = ref_forward(U, done, xwb, h0, c0)
  dz = ref_backward(U, done, gates, cs, c0, dhs)
  return dict(gates=gates, hs=hs, cs=cs, hp=hp, h_T=hs[-1], c_T=cs[-1], dz=dz, dU=_dU(hp, dz))


def _relmax(a, ref):
  return float(np.abs(np.asarray(a, np.float64) - ref).max() / max(np.abs(ref).max(), 1e-300))


# ---- inputs ----------------------------------------------------------------------------------------------
def _orthogonal(rng, H):
  """Keras Orthogonal() for a [H, 4H] kernel: orthonormal rows."""
  q, r = np.linalg.qr(rng.normal(size=(4 * H, H)))
  return (q * np.sign(np.diag(r))).T


def _resets(rng, T1, B, pattern):
  done = np.zeros((T1, B), bool)
  if pattern == 'tail':
    # only the rows of the last partial tile (of 8 rows: also inside the last tile of 16, 32 and 64 rows)
    lo = B - (B % 8 or 8)
    done[:, lo:] = rng.random((T1, B - lo)) < 0.5
    return done
  done[:] = rng.random((T1, B)) < (0.2 if pattern == 'mixed' else 0.01)
  done[0, ::3] = True                                 # resets at t = 0 replace h0 and c0
  done[-1, 1::4] = True                               # a reset at the last step
  if B > 2:
    done[:, 2] = True                                 # a row that resets on every step
  for r in range(5, B - 8, 16):                       # rows r and r + 8 of one 16-row group: different resets
    done[:, r] = np.arange(T1) % 2 == 0
    done[:, r + 8] = False
  return done


def make_inputs(H, T1, B, pattern, regime, seed):
  """fp32 inputs (numpy) of one case."""
  rng = np.random.default_rng(seed)
  U = _orthogonal(rng, H)
  if regime == 'saturated':                           # |x W + b| up to 100: expf(-z) overflows in the sigmoid
    xwb = rng.uniform(-100.0, 100.0, size=(T1, B, 4 * H))
  else:
    xwb = rng.normal(size=(T1, B, 4 * H))
    xwb[..., H:2 * H] += 3.0 if regime == 'long' else 1.0   # forget bias: Keras unit_forget_bias, or +3
  h0 = rng.uniform(-1.0, 1.0, size=(B, H))
  c0 = rng.normal(size=(B, H)) * (5.0 if regime == 'long' else 1.0)
  dhs = rng.normal(size=(T1, B, H))
  f = lambda a: np.ascontiguousarray(a, np.float32)
  return dict(U=f(U), done=_resets(rng, T1, B, pattern), xwb=f(xwb), h0=f(h0), c0=f(c0), dhs=f(dhs))


def reference_and_responses(inp, epss):
  """(reference outputs, {eps: {output: response}}) of one case, float64."""
  d = {k: (v.astype(np.float64) if v.dtype == np.float32 else v) for k, v in inp.items()}
  ref = ref_all(d['U'], d['done'], d['xwb'], d['h0'], d['c0'], d['dhs'])
  resp = {}
  for eps in sorted(set(epss)):
    rng = np.random.default_rng(12345)
    p = {k: d[k] * (1.0 + eps * rng.choice([-1.0, 1.0], size=d[k].shape)) for k in ('U', 'xwb', 'h0', 'c0')}
    out = ref_all(p['U'], d['done'], p['xwb'], p['h0'], p['c0'], d['dhs'])
    resp[eps] = {k: _relmax(out[k], ref[k]) for k in OUTPUTS}
  return ref, resp


# ---- CPU: the reference against torch float64 autograd ------------------------------------------------------
def test_reference_matches_torch_float64_autograd():
  from oracle import net_oracle
  H, T1, B = 256, 6, 5
  inp = make_inputs(H, T1, B, 'mixed', 'keras', seed=3)
  inp['done'][2, 1] = True
  d = {k: (v.astype(np.float64) if v.dtype == np.float32 else v) for k, v in inp.items()}
  assert d['done'].any() and not d['done'].all()
  ref = ref_all(d['U'], d['done'], d['xwb'], d['h0'], d['c0'], d['dhs'])
  # x = x W + b with W = I, b = 0: the gradient with respect to x is dz
  p = {'core/kernel': torch.eye(4 * H, dtype=torch.float64),
       'core/recurrent_kernel': torch.tensor(d['U'], requires_grad=True),
       'core/bias': torch.zeros(4 * H, dtype=torch.float64)}
  x = torch.tensor(d['xwb'], requires_grad=True)
  h, c = torch.tensor(d['h0']), torch.tensor(d['c0'])
  hs, cs = [], []
  for t in range(T1):
    m = torch.tensor(d['done'][t])[:, None]
    h = torch.where(m, torch.zeros_like(h), h); c = torch.where(m, torch.zeros_like(c), c)
    h, c = net_oracle.lstm_cell(p, x[t], h, c)
    hs.append(h); cs.append(c)
  hs, cs = torch.stack(hs), torch.stack(cs)
  (hs * torch.tensor(d['dhs'])).sum().backward()
  np.testing.assert_allclose(ref['hs'], hs.detach().numpy(), rtol=1e-12, atol=1e-13)
  np.testing.assert_allclose(ref['cs'], cs.detach().numpy(), rtol=1e-12, atol=1e-13)
  np.testing.assert_allclose(ref['dz'], x.grad.numpy(), rtol=1e-10, atol=1e-12)
  np.testing.assert_allclose(ref['dU'], p['core/recurrent_kernel'].grad.numpy(), rtol=1e-10, atol=1e-12)


# ---- batch limits of the launchers --------------------------------------------------------------------------
def batch_limit(mode, H, bwd):
  """The largest batch each launcher takes (lstm_tiled.cu, lstm_tc.cu)."""
  def fits(B):
    if mode == 2:          # at most 64 tiles of at most 32 rows, fewer rows where shared memory runs out
      KC = min(4 * H, 1024)
      smem = lambda r: 4 * ((4 * H * 16 + KC * r + 16 * r * 16 + r * 16) if bwd else (H * 64 + H * r + 8 * r * 64 + r * 16))
      tiles = max(1, min(8, 132 // (H // 16)))
      rb = min(32, max(8, -(-(-(-B // tiles)) // 8) * 8))
      while rb > 8 and smem(rb) > 220 * 1024:
        rb -= 8
      return smem(rb) <= 220 * 1024 and -(-B // rb) <= 64
    return -(-B // 64) <= 64   # mode 3: at most 64 tiles of 64 rows
  lo, hi = 1, 1 << 16
  assert fits(lo) and not fits(hi)
  while hi - lo > 1:
    mid = (lo + hi) // 2
    lo, hi = (mid, hi) if fits(mid) else (lo, mid)
  return lo


def test_batch_limits():
  """The limits the launchers are pinned to (CPU restatement; the GPU tests below run at and one past them)."""
  assert [batch_limit(2, H, b) for H in (256, 512) for b in (False, True)] == [2048, 1536, 1024, 1024]
  assert [batch_limit(3, H, b) for H in (256, 512) for b in (False, True)] == [4096] * 4


# ---- GPU ---------------------------------------------------------------------------------------------------
def _lib():
  from seed_rl_b200 import _lib as L
  return L


class Runner:
  """Device buffers of one case, with a NaN guard (one extra time step of B + 8 rows) after every output."""

  def __init__(self, inp, ws_bytes):
    self.T1, self.B, self.H = inp['xwb'].shape[0], inp['xwb'].shape[1], inp['U'].shape[0]
    dev = lambda a: torch.as_tensor(a).cuda()
    self.U, self.h0, self.c0, self.dhs = dev(inp['U']), dev(inp['h0']), dev(inp['c0']), dev(inp['dhs'])
    self.done = dev(inp['done'].astype(np.uint8))
    self.xwb = dev(inp['xwb'])
    self.ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    self.flag = torch.zeros(1, dtype=torch.int32, device='cuda')

  def guarded(self, width):
    n = self.T1 * self.B * width
    buf = torch.full((n + (self.B + 8) * width,), float('nan'), device='cuda')
    return buf, buf[:n].view(self.T1, self.B, width)

  def forward(self, mode):
    L = _lib()
    H = self.H
    bufs = {k: self.guarded(w) for k, w in (('z', 4 * H), ('hs', H), ('cs', H), ('hp', H))}
    bufs['z'][1].copy_(self.xwb)
    rc = L.lib().seedrl_debug_lstm_forward(
        mode, H, self.T1, self.B, L.ptr(self.U), L.ptr(self.done), L.ptr(bufs['z'][1]),
        L.ptr(self.h0), L.ptr(self.c0), L.ptr(bufs['hs'][1]), L.ptr(bufs['cs'][1]), L.ptr(bufs['hp'][1]),
        L.ptr(self.ws), self.ws.numel(), L.ptr(self.flag), L.stream_ptr())
    return rc, bufs

  def backward(self, mode, gates, cs):
    L = _lib()
    buf = self.guarded(4 * self.H)
    rc = L.lib().seedrl_debug_lstm_backward(
        mode, self.H, self.T1, self.B, L.ptr(self.U), L.ptr(self.done), L.ptr(gates),
        L.ptr(cs), L.ptr(self.c0), L.ptr(self.dhs), L.ptr(buf[1]), L.ptr(self.ws), self.ws.numel(),
        L.ptr(self.flag), L.stream_ptr())
    return rc, buf

  def step(self, mode, bptt=True):
    """forward, then BPTT from its gates and cs: {name: (guarded buffer, view)}."""
    rc, bufs = self.forward(mode)
    _lib().check(rc)
    if bptt:
      rc, bufs['dz'] = self.backward(mode, bufs['z'][1], bufs['cs'][1])
      _lib().check(rc)
    torch.cuda.synchronize()
    assert int(self.flag.item()) == 0, 'a barrier wait expired'
    for k, (buf, view) in bufs.items():
      n = view.numel()
      assert torch.isnan(buf[n:]).all(), '%s: written past its end (time step T1 / rows past B)' % k
      assert torch.isfinite(view).all(), '%s: an element is not written or not finite' % k
    return bufs


def _ws_bytes(H, T1, B):
  return max(_lib().lib().seedrl_debug_lstm_workspace_bytes(m, H, T1, B) for m in (2, 3))


def _gpu_outputs(bufs):
  f = lambda k: bufs[k][1].double().cpu().numpy()
  out = dict(gates=f('z'), hs=f('hs'), cs=f('cs'), hp=f('hp'))
  out.update(h_T=out['hs'][-1], c_T=out['cs'][-1])
  if 'dz' in bufs:
    out.update(dz=f('dz'), dU=_dU(out['hp'], f('dz')))
  return out


def _check(tag, eps, got, ref, resp, outputs=OUTPUTS):
  bad, line = [], []
  for k in outputs:
    err = _relmax(got[k], ref[k])
    bar = max(FLOOR, SENS_MULT * resp[eps][k])
    line.append('%s %.2e/%.2e' % (k, err, bar))
    if not err <= bar:
      bad.append((k, err, bar))
  print('LSTMREC %s: %s' % (tag, '  '.join(line)))
  assert not bad, bad


# (name, T1, B, pattern, regime, hidden sizes)
CASES = [
    ('infer_1x1', 1, 1, 'mixed', 'keras', (256, 512)),
    ('infer_1x64', 1, 64, 'mixed', 'keras', (256, 512)),
    ('infer_1x256', 1, 256, 'mixed', 'keras', (256, 512)),
    ('infer_2x256', 2, 256, 'mixed', 'keras', (256, 512)),
    ('learn_21x64', 21, 64, 'mixed', 'keras', (256, 512)),
    ('learn_21x256', 21, 256, 'mixed', 'keras', (256, 512)),
    ('learn_141x64', 141, 64, 'mixed', 'keras', (256, 512)),
    ('long_141x64', 141, 64, 'sparse', 'long', (256, 512)),
    ('saturated_5x100', 5, 100, 'mixed', 'saturated', (256, 512)),
    ('ragged_3x65', 3, 65, 'tail', 'keras', (256, 512)),
    ('ragged_3x100', 3, 100, 'tail', 'keras', (256, 512)),
    ('ragged_4x129', 4, 129, 'tail', 'keras', (256, 512)),
    ('ragged_3x300', 3, 300, 'mixed', 'keras', (256, 512)),
    ('noncoop_3x320', 3, 320, 'mixed', 'keras', (512,)),      # tc3: 5 tiles x 32 unit groups > 132 SMs
    ('noncoop_3x1024', 3, 1024, 'mixed', 'keras', (512,)),
    ('noncoop_3x640', 3, 640, 'tail', 'keras', (256,)),       # tc3: 10 tiles x 16 unit groups
]
ARMS = {256: (2, 3), 512: (2, 3)}    # lstm modes
GRID = [(name, H, mode) for name, _, _, _, _, Hs in CASES for H in Hs for mode in ARMS[H]]
_CACHE = {}


def _case(name, H):
  """fp32 inputs, reference and responses of one case (the last one is kept: the grid runs case by case)."""
  key = (name, H)
  if key not in _CACHE:
    _CACHE.clear()
    _, T1, B, pattern, regime, _ = next(c for c in CASES if c[0] == name)
    inp = make_inputs(H, T1, B, pattern, regime, seed=zlib.crc32(('%s/%d' % key).encode()))
    _CACHE[key] = (inp,) + reference_and_responses(inp, [_eps(mode) for mode in ARMS[H]])
  return _CACHE[key]


@pytest.mark.gpu
@pytest.mark.parametrize('name,H,mode', GRID, ids=['%s-H%d-mode%d' % arm for arm in GRID])
def test_recurrence_matches_float64(name, H, mode):
  inp, ref, resp = _case(name, H)
  T1, B = inp['xwb'].shape[:2]
  r = Runner(inp, _ws_bytes(H, T1, B))
  first = r.step(mode)
  _check('mode %d H %d %dx%d %s' % (mode, H, T1, B, name), _eps(mode), _gpu_outputs(first), ref, resp)
  # bit-identical on a repeat after a call in another mode on the same workspace and error flag
  r.step(3 if mode != 3 else 2)
  again = r.step(mode)
  for k in first:
    assert torch.equal(first[k][0].nan_to_num(7.0), again[k][0].nan_to_num(7.0)), k


@pytest.mark.gpu
@pytest.mark.parametrize('H,mode', [(256, 2), (256, 3), (512, 2), (512, 3)])
def test_largest_batch(H, mode):
  """The forward at its mode's largest batch, the BPTT at its own (from the reference's forward, rounded to fp32,
  where that batch is past the forward's limit)."""
  T1 = 2
  bf, bb = batch_limit(mode, H, False), batch_limit(mode, H, True)
  for B, part in ((bf, 'forward'), (bb, 'bptt')):
    inp = make_inputs(H, T1, B, 'mixed', 'keras', seed=B)
    ref, resp = reference_and_responses(inp, [_eps(mode)])
    r = Runner(inp, _ws_bytes(H, T1, B))
    if part == 'forward':
      got = _gpu_outputs(r.step(mode, bptt=False))
      _check('largest batch mode %d H %d %dx%d forward' % (mode, H, T1, B), _eps(mode), got, ref, resp,
             ('gates', 'hs', 'cs', 'hp', 'h_T', 'c_T'))
    else:
      f32 = lambda a: torch.as_tensor(a.astype(np.float32)).cuda()
      gates, cs = f32(ref['gates']), f32(ref['cs'])
      rc, dz = r.backward(mode, gates, cs)
      _lib().check(rc)
      torch.cuda.synchronize()
      assert int(r.flag.item()) == 0
      n = dz[1].numel()
      assert torch.isnan(dz[0][n:]).all() and torch.isfinite(dz[1]).all()
      got = dz[1].double().cpu().numpy()
      _check('largest batch mode %d H %d %dx%d bptt' % (mode, H, T1, B), _eps(mode), dict(dz=got, dU=_dU(ref['hp'], got)),
             ref, resp, ('dz', 'dU'))


@pytest.mark.gpu
@pytest.mark.parametrize('H,mode', [(256, 2), (256, 3), (512, 2), (512, 3)])
def test_one_row_past_the_limit_is_refused(H, mode):
  L = _lib()
  for bwd in (False, True):
    B = batch_limit(mode, H, bwd) + 1
    inp = make_inputs(H, 1, B, 'mixed', 'keras', seed=1)
    r = Runner(inp, _ws_bytes(H, 1, B))
    gates = torch.rand(1, B, 4 * H, device='cuda')
    torch.cuda.synchronize()
    n0 = L.launch_count()
    rc, bufs = r.backward(mode, gates, gates[..., :H].contiguous()) if bwd else r.forward(mode)
    torch.cuda.synchronize()
    assert rc == INVALID_ARGUMENT, (bwd, B, rc)
    assert L.launch_count() == n0
    assert int(r.flag.item()) == 0
    if bwd:
      assert torch.isnan(bufs[0]).all()
    else:
      assert torch.equal(bufs['z'][1], r.xwb)
      assert all(torch.isnan(bufs[k][0]).all() for k in ('hs', 'cs', 'hp'))


@pytest.mark.gpu
@pytest.mark.parametrize('mode', [2, 3])
def test_bad_hidden_size_and_arguments_are_refused(mode):
  L = _lib()
  T1, B = 2, 8
  r = Runner(make_inputs(256, T1, B, 'mixed', 'keras', seed=2), _ws_bytes(256, T1, B))
  z, o = r.xwb.clone(), torch.full((T1, B, 256), float('nan'), device='cuda')
  need = L.lib().seedrl_debug_lstm_workspace_bytes(mode, 256, T1, B)
  assert need > 0

  def fwd(H, ws_bytes=r.ws.numel(), m=mode):
    return L.lib().seedrl_debug_lstm_forward(m, H, T1, B, L.ptr(r.U), L.ptr(r.done), L.ptr(z),
                                             L.ptr(r.h0), L.ptr(r.c0), L.ptr(o), L.ptr(o), L.ptr(o), L.ptr(r.ws),
                                             ws_bytes, L.ptr(r.flag), L.stream_ptr())

  def bwd(H, ws_bytes=r.ws.numel(), m=mode):
    return L.lib().seedrl_debug_lstm_backward(m, H, T1, B, L.ptr(r.U), L.ptr(r.done), L.ptr(z), L.ptr(o),
                                              L.ptr(r.c0), L.ptr(r.dhs), L.ptr(z), L.ptr(r.ws), ws_bytes,
                                              L.ptr(r.flag), L.stream_ptr())
  torch.cuda.synchronize()
  n0 = L.launch_count()
  assert fwd(128) == INVALID_ARGUMENT and bwd(128) == INVALID_ARGUMENT          # H = 128 (buffers hold H = 256)
  assert fwd(256, ws_bytes=need - 1) == INVALID_ARGUMENT and bwd(256, ws_bytes=need - 1) == INVALID_ARGUMENT
  for m in (0, 1, 4, -1):                                                       # only the tiled and tc3 recurrences
    assert L.lib().seedrl_debug_lstm_workspace_bytes(m, 256, T1, B) == 0
    assert fwd(256, m=m) == INVALID_ARGUMENT and bwd(256, m=m) == INVALID_ARGUMENT
  torch.cuda.synchronize()
  assert L.launch_count() == n0
  assert torch.equal(z, r.xwb) and torch.isnan(o).all() and int(r.flag.item()) == 0
