"""seedrl_adam_apply (csrc/optim_kernels.cu) on its own against the Keras dense Adam update evaluated in float64:

    m' = m + (s g - m)(1 - b1);   v' = v + ((s g)^2 - v)(1 - b2);   p' = p - (m' lr_t) / (sqrt(v') + eps)

(oracle/optim_oracle.py's form), where s is grad_scale, and lr_t, eps, s and the fp32 subtractions 1 - b1, 1 - b2 are
the fp32 constants the kernel receives.  The reference takes the fp32 p, g, m, v the kernel read.  Over a run of
steps each step's reference starts from the GPU's own state after the previous step, so errors do not compound.

Bars, per element, forward-error bounds with u = 2^-24 and TINY = 2^-149 (the fp32 subnormal step: the kernel is
built without flush-to-zero, and s g squared underflows for |s g| below about 1e-23):
  * m', v': |gpu - ref| <= K u (sum of the magnitudes of the terms the formula adds) + K TINY, the terms being
    m, (s g)(1 - b1), m (1 - b1) for m' and v, (s g)^2 (1 - b2), v (1 - b2) for v';
  * p': compared with p - D, D recomputed in float64 from the GPU's own m' and v'.  The bar is
    half an ulp of the stored p' (the final subtraction) + K u |D| + K TINY (the four roundings of D).
K = 4, the count of roundings in each formula.  Calibrated with the fp32 numpy form of the same update (one rounding
per operation, no fused multiply-add), which test_bars_hold_for_the_fp32_numpy_form checks on the CPU: over the
vtrace and r2d2 hyperparameters, 20 steps of 200 011 elements and gradients from 1e-30 to 1e15, its worst element
comes to 2.6 u (m'), 3.6 u (v': (s g)^2 is itself rounded) and 3.5 u (D) of those sums of magnitudes.

1 - b2 in fp32 is exact (Sterbenz: b2 is within a factor of 2 of 1), 1 - fp32(0.999) = 0.000999987125; rounding
the decimal 1 - 0.999 = 0.001 instead moves v' by 1.3e-5 relative, far over the bar.

Sizes: the live parameter arenas (ImpalaDeep with and without its PopArt tail, ImpalaShallow, the R2D2 net, read from
seedrl_*_arena_floats), 4 (1056 x 256 + 1) + {0, 1, 2, 3} -- at 1056 blocks (8 per SM) of 256 threads, one float4
more than the grid covers in one pass, so thread 0 takes a second float4, with every tail length -- and n = 1 to 7.
"""
import ctypes

import numpy as np
import pytest

U = 2.0 ** -24
TINY = 2.0 ** -149
K = 4.0
STEPS = 20
SCALES = (1.0, 0.5, 0.25, 0.125)
ERR_INVALID_ARGUMENT = 3
ONE_PASS = 1056 * 256                      # float4s the capped grid covers in one pass
# name -> (beta_1, beta_2, epsilon, learning rate at `iterations`): bench.py's two optimizers
HPARAMS = {'vtrace': (0.0, 0.999, 3.125e-7, lambda it: 4.8e-4 * (1.0 - min(it, 10 ** 6) / 10 ** 6)),
           'r2d2': (0.9, 0.999, 1e-3, lambda it: 4.8e-4)}
SIZES = (['deep', 'deep-popart', 'shallow', 'r2d2'] + ['pass2+%d' % r for r in range(4)] +
         ['n%d' % n for n in range(1, 8)])
f32, f64 = np.float32, np.float64


def _lr_t(hp, it):
  from oracle import optim_oracle
  b1, b2, _, lr = HPARAMS[hp]
  return float(optim_oracle.keras_adam_lr_t(it, lr(it), b1, b2))


def _size(name):
  """-> (n, the indices of the arena no tensor covers: padding that gets a zero gradient forever)."""
  if name.startswith('pass2+'):
    return 4 * (ONE_PASS + 1) + int(name[6:]), np.zeros(0, np.int64)
  if name.startswith('n'):
    return int(name[1:]), np.zeros(0, np.int64)
  if name == 'r2d2':
    from seed_rl_b200.atari import networks
    net = networks.DuelingLSTMDQNNet(18, (84, 84, 1), 4)
  else:
    from seed_rl_b200.dmlab import networks
    net = (networks.ImpalaShallow if name == 'shallow' else networks.ImpalaDeep)(18, (84, 84, 4))
    if name == 'deep-popart':
      net.enable_popart()
  n = int(net.params.numel())
  assert n == net.arena_floats + (64 if name == 'deep-popart' else 0)
  used = np.zeros(n, bool)
  for _, shape, off in net.param_info:
    used[off:off + int(np.prod(shape))] = True
  del net
  return n, np.flatnonzero(~used)


def _constants(hp, scale):
  b1, b2, eps, _ = HPARAMS[hp]
  return float(f32(1) - f32(b1)), float(f32(1) - f32(b2)), float(f32(eps)), float(f32(scale))


def reference(p, g, m, v, lr_t, hp, scale):
  """float64 Keras update of fp32 inputs -> (m', v', bar m', bar v', D(m', v') as a function)."""
  ob1, ob2, eps, s = _constants(hp, scale)
  p, g, m, v = (np.asarray(x, f64) for x in (p, g, m, v))
  sg = g * s
  m2 = m + (sg - m) * ob1
  v2 = v + (sg * sg - v) * ob2
  bm = K * U * (np.abs(m) + np.abs(sg) * ob1 + np.abs(m) * ob1) + K * TINY
  bv = K * U * (v + sg * sg * ob2 + v * ob2) + K * TINY
  delta = lambda mm, vv: (np.asarray(mm, f64) * lr_t) / (np.sqrt(np.asarray(vv, f64)) + eps)
  return m2, v2, bm, bv, delta


def check_step(before, after, lr_t, hp, scale, where=''):
  """Asserts the three bars for one step: before = fp32 (p, g, m, v), after = fp32 (p', m', v')."""
  p, g, m, v = before
  p2, m2, v2 = after
  rm, rv, bm, bv, delta = reference(p, g, m, v, lr_t, hp, scale)
  for nm, got, want, bar in (('m', m2, rm, bm), ('v', v2, rv, bv)):
    err = np.abs(got.astype(f64) - want)
    bad = np.flatnonzero(~(err <= bar))
    assert bad.size == 0, "%s%s': %d elements over the bar, first %d: gpu %r ref %r bar %r (g %r)" % (
        where, nm, bad.size, bad[0], got[bad[0]], want[bad[0]], bar[bad[0]], g[bad[0]])
  d = delta(m2, v2)
  want = p.astype(f64) - d
  bar = 0.5 * np.spacing(np.abs(p2)).astype(f64) + K * U * np.abs(d) + K * TINY
  err = np.abs(p2.astype(f64) - want)
  bad = np.flatnonzero(~(err <= bar))
  assert bad.size == 0, "%sp': %d elements over the bar, first %d: gpu %r ref %r bar %r (g %r m' %r v' %r)" % (
      where, bad.size, bad[0], p2[bad[0]], want[bad[0]], bar[bad[0]], g[bad[0]], m2[bad[0]], v2[bad[0]])


def _params(rng, n):
  return (rng.standard_normal(n) * 10.0 ** rng.uniform(-3, 1, n)).astype(f32)


def _grads(rng, n, zero):
  """Half N(0, 1e-3), half log-uniform from 1e-30 to 1e15 with random signs; exact zeros at `zero`."""
  g = rng.standard_normal(n) * 1e-3
  wide = rng.random(n) < 0.5
  g[wide] = 10.0 ** rng.uniform(-30, 15, int(wide.sum())) * rng.choice([-1.0, 1.0], int(wide.sum()))
  g = g.astype(f32)
  g[zero] = 0
  return g


def _zeros(n, gaps):
  return np.union1d(np.arange(3, n, 97), gaps).astype(np.int64)


def test_bars_hold_for_the_fp32_numpy_form():
  """CPU: the fp32 numpy form of the update (oracle/optim_oracle.py's arithmetic, one rounding per operation, no
  fused multiply-add) passes every bar on the same kind of inputs the GPU tests use, so the bars leave room for an
  honest fp32 implementation; and it fails them when 1 - b2 is replaced by the decimal 0.001."""
  rng = np.random.default_rng(7)
  n = 20011
  zero = _zeros(n, np.zeros(0, np.int64))
  for hp in HPARAMS:
    ob1, ob2, eps, _ = _constants(hp, 1.0)
    p, m, v = _params(rng, n), np.zeros(n, f32), np.zeros(n, f32)
    for it in range(STEPS):
      g = _grads(rng, n, zero)
      lr_t, s = _lr_t(hp, it), SCALES[it % 4]
      sg = g * f32(s)
      m2 = m + (sg - m) * f32(ob1)
      v2 = v + (sg * sg - v) * f32(ob2)
      p2 = p - (m2 * f32(lr_t)) / (np.sqrt(v2) + f32(eps))
      check_step((p, g, m, v), (p2, m2, v2), lr_t, hp, s, '%s step %d: ' % (hp, it))
      if it == 1:
        wrong = v + (sg * sg - v) * f32(0.001)
        with pytest.raises(AssertionError):
          check_step((p, g, m, v), (p2, m2, wrong), lr_t, hp, s)
      p, m, v = p2, m2, v2


# ---- on the GPU ------------------------------------------------------------------------------------------------
def _apply(p, g, m, v, lr_t, hp, scale, clamp_index=-1, clamp_lo=0.0, clamp_hi=0.0, n=None):
  """One seedrl_adam_apply on the CUDA tensors (or pointers offset into them); -> its return code."""
  from seed_rl_b200 import _lib
  b1, b2, eps, _ = HPARAMS[hp]
  ptr = lambda t: t if isinstance(t, ctypes.c_void_p) else _lib.ptr(t)
  return _lib.lib().seedrl_adam_apply(p.numel() if n is None else n, ptr(p), ptr(g), ptr(m), ptr(v), lr_t, b1, b2,
                                      eps, scale, clamp_index, clamp_lo, clamp_hi, _lib.stream_ptr())


def _cuda(*arrays):
  import torch
  return [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]


def _host(*tensors):
  return [t.cpu().numpy() for t in tensors]


@pytest.mark.gpu
@pytest.mark.parametrize('hp', sorted(HPARAMS))
@pytest.mark.parametrize('size', SIZES)
def test_adam_matches_float64(size, hp):
  """STEPS consecutive updates from m = v = 0, grad_scale cycling through 1, 1/2, 1/4, 1/8, the learning rate of
  each optimizer's schedule at iterations 0, 1, ...  Zero-gradient elements (every 97th and the arena's padding)
  keep p bit-identical and m = v = 0."""
  import torch
  n, gaps = _size(size)
  rng = np.random.default_rng(100 * SIZES.index(size) + sorted(HPARAMS).index(hp))
  zero = _zeros(n, gaps)
  p0 = _params(rng, n)
  p, g, m, v = _cuda(p0, np.zeros(n, f32), np.zeros(n, f32), np.zeros(n, f32))
  for it in range(STEPS):
    gh = _grads(rng, n, zero)
    g.copy_(torch.from_numpy(gh))
    before = _host(p, g, m, v)
    lr_t, s = _lr_t(hp, it), SCALES[it % 4]
    assert _apply(p, g, m, v, lr_t, hp, s) == 0
    after = _host(p, m, v)
    check_step(before, after, lr_t, hp, s, '%s %s step %d: ' % (size, hp, it))
  ph, mh, vh = _host(p, m, v)
  assert np.array_equal(ph[zero].view(np.uint32), p0[zero].view(np.uint32))
  assert not mh[zero].any() and not vh[zero].any()
  moved = np.setdiff1d(np.arange(n), zero)
  assert (ph[moved] != p0[moved]).mean() > 0.5     # the run really updates the arena


def _arena(rng, n):
  """A mid-run state: p, g, and m, v from a few earlier steps' worth of gradients."""
  p = _params(rng, n)
  g = _grads(rng, n, np.zeros(0, np.int64))
  m = (rng.standard_normal(n) * 1e-3).astype(f32)
  v = (m.astype(f64) ** 2 * rng.uniform(1, 4, n)).astype(f32)
  return p, g, m, v


@pytest.mark.gpu
@pytest.mark.parametrize('hp', sorted(HPARAMS))
def test_non_finite_gradients_poison_only_their_own_element(hp):
  """A NaN, a +Inf and a -Inf gradient (in the first pass, the second pass and the tail) make their own p, m and v
  non-finite, as Keras's elementwise update does; every other element is bit-identical to the run whose three
  gradients are finite."""
  n = 4 * (ONE_PASS + 1) + 3
  rng = np.random.default_rng(11)
  p, g, m, v = _arena(rng, n)
  bad = {5: np.nan, 4 * ONE_PASS + 1: np.inf, n - 1: -np.inf}
  gbad = g.copy()
  for i, x in bad.items():
    g[i] = 1.0
    gbad[i] = x
  fin, poi = _cuda(p, g, m, v), _cuda(p, gbad, m, v)
  lr_t = _lr_t(hp, 3)
  assert _apply(*fin, lr_t, hp, 0.5) == 0 and _apply(*poi, lr_t, hp, 0.5) == 0
  fin, poi = [_host(*x) for x in ((fin[0], fin[2], fin[3]), (poi[0], poi[2], poi[3]))]
  idx = np.array(sorted(bad))
  keep = np.setdiff1d(np.arange(n), idx)
  for a, b, nm in zip(fin, poi, 'pmv'):
    assert not np.isfinite(b[idx]).any(), nm
    assert np.array_equal(a[keep].view(np.uint32), b[keep].view(np.uint32)), nm
  check_step((p, g, m, v), tuple(fin), lr_t, hp, 0.5)


@pytest.mark.gpu
@pytest.mark.parametrize('index', [7, 4 * ONE_PASS + 2, 4 * (ONE_PASS + 1) + 1])
@pytest.mark.parametrize('case', ['lo', 'hi', 'neither'])
def test_clamp(case, index):
  """clamp_index takes p[index] to [clamp_lo, clamp_hi] after the update (the entropy_cost_param constraint):
  exactly the bound when it binds, the unclamped update when it does not; m, v and every other p are
  bit-identical to the unclamped call."""
  n = 4 * (ONE_PASS + 1) + 2
  rng = np.random.default_rng(13)
  p, g, m, v = _arena(rng, n)
  lo, hi = -2.0, 2.0
  p[index] = {'lo': -5.0, 'hi': 5.0, 'neither': 0.75}[case]
  free, clamped = _cuda(p, g, m, v), _cuda(p, g, m, v)
  lr_t = _lr_t('vtrace', 0)
  assert _apply(*free, lr_t, 'vtrace', 1.0) == 0
  assert _apply(*clamped, lr_t, 'vtrace', 1.0, clamp_index=index, clamp_lo=lo, clamp_hi=hi) == 0
  fp, fm, fv = _host(free[0], free[2], free[3])
  cp, cm, cv = _host(clamped[0], clamped[2], clamped[3])
  assert np.array_equal(fm.view(np.uint32), cm.view(np.uint32)) and np.array_equal(fv.view(np.uint32),
                                                                                    cv.view(np.uint32))
  others = np.setdiff1d(np.arange(n), [index])
  assert np.array_equal(fp[others].view(np.uint32), cp[others].view(np.uint32))
  if case == 'neither':
    assert lo < fp[index] < hi and cp[index] == fp[index]
  else:
    assert cp[index] == {'lo': f32(lo), 'hi': f32(hi)}[case]
    assert (fp[index] < lo) if case == 'lo' else (fp[index] > hi)
  check_step((p, g, m, v), (fp, fm, fv), lr_t, 'vtrace', 1.0)


@pytest.mark.gpu
def test_two_identical_calls_are_bit_identical():
  n = 4 * (ONE_PASS + 1) + 3
  p, g, m, v = _arena(np.random.default_rng(17), n)
  a, b = _cuda(p, g, m, v), _cuda(p, g, m, v)
  for x in (a, b):
    assert _apply(*x, _lr_t('r2d2', 0), 'r2d2', 0.25, clamp_index=n - 2, clamp_lo=-0.1, clamp_hi=0.1) == 0
  for x, y in zip(_host(*a), _host(*b)):
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.gpu
def test_empty_arena_launches_nothing():
  from seed_rl_b200 import _lib
  p, g, m, v = _cuda(*_arena(np.random.default_rng(19), 8))
  before = _lib.launch_count()
  assert _apply(p, g, m, v, 1e-3, 'vtrace', 1.0, clamp_index=0, clamp_lo=-1.0, clamp_hi=1.0, n=0) == 0
  assert _lib.launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize('bad', ['p', 'g', 'm', 'v', 'clamp=n', 'clamp>n'])
def test_refused_arguments_leave_the_arenas_untouched(bad):
  """A pointer 4 bytes off 16-byte alignment, or clamp_index >= n, returns SEEDRL_ERR_INVALID_ARGUMENT before any
  launch."""
  import torch
  from seed_rl_b200 import _lib
  n = 1027
  host = _arena(np.random.default_rng(23), n + 4)
  arenas = _cuda(*host)
  args = [a[:n] for a in arenas]
  clamp = -1
  if bad in 'pgmv':
    k = 'pgmv'.index(bad)
    args[k] = ctypes.c_void_p(arenas[k].data_ptr() + 4)
  else:
    clamp = n if bad == 'clamp=n' else n + 5
  before = _lib.launch_count()
  assert _apply(*args, 1e-3, 'vtrace', 1.0, clamp_index=clamp, clamp_lo=-1.0, clamp_hi=1.0, n=n) == \
      ERR_INVALID_ARGUMENT
  assert _lib.launch_count() == before
  torch.cuda.synchronize()
  for x, y in zip(_host(*arenas), host):
    assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
