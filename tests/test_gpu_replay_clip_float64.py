"""The R2D2 learner's steps around the network against float64: prioritized replay sampling
(seedrl_replay_sample, through learner.replay_sample and utils.PrioritizedReplay.sample) and the
global-norm clip (seedrl_clip_by_global_norm, through learner.clip_by_global_norm).  The float64
references are the numpy functions of this file; tests/test_r2d2_host_emulation.py runs the same
replay checks on the kernel's per-thread bodies compiled for the CPU.

Error and bar.  error = max_k |gpu_k - ref64_k| / |ref64_k| over the compared elements (where ref64
is 0 the GPU's value must be exactly 0); bar = max(FLOOR, C x m), m the same error of a float32
restatement in numpy of the same formula.  C = 4: the kernel and the restatement round the same
operations, in a different order (the norm) or with a different powf (CUDA's and numpy's differ in
the last bits), so neither should be more than a few times the other.  The floors are the roundings a
correct kernel makes where m happens to be near 0, in units u = 2^-24:
  * weights, W_FLOOR = 8u: each normalised weight is a quotient of two chains powf(alpha), two
    divisions, powf(beta); the common factors 1/limit and 1/total cancel.  Before the drawn item's
    probability came from its own mass, cdf[i] - cdf[i-1] had an absolute error ~ulp(total) that
    gave the rare items of a wide priority spread errors of 1e-5 to 1e-2.
  * probs_out, P_FLOOR = 8u: one powf and one division; m carries the serial fp32 sum in `total`.
  * clip, CLIP_FLOOR = 16u: the sum of squares is 4 * 132 per-CTA chains of up to 125 fma each,
    then a serial 528-term sum (random-walk error of a few u), and the scale adds two roundings.

The draw is checked against the float64 inverse CDF up to edge(limit) = (limit + 8) 2^-23 of the
total per bin edge: the fp32 prefix cdf[i] is within (i + 1 + 4) u cdf[i] of float64 (serial sum of
powf values), u_j * total within (limit + 2) u, and u >= 1 - 2^-24 is clamped below the total.
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
C = 4
W_FLOOR = 8 * U
P_FLOOR = 8 * U
CLIP_FLOOR = 16 * U
CLIP = 40.0
F = np.float32

LIMITS = (1, 2, 100, 1000, 4096, 8192)      # 100 = replay_buffer_size; 8192 = the sampler's cap
KINDS = ('uniform', 'lognormal2', 'lognormal3', 'equal', 'spike', 'zeros', 'loss')
EXPONENTS = ((0.9, 0.6), (1.0, 1.0), (0.9, 0.0))     # (priority_exp, importance_sampling_exponent)
NUM_SAMPLES = (4096, 1025, 1023, 64, 1)              # around the 1024-thread CTA of the max reduction;
                                                     # largest first, so wrong weights fail before probs_out
PINNED = np.array([0.0, 0.99999994, 1.0], F)         # first and last items with positive mass


# ---- replay sampling: float64 reference and checks ---------------------------------------------
def priorities(kind, limit, seed=0):
  """Host-side priority sets ('loss' comes from the loss kernel, see _loss_priorities)."""
  rng = np.random.default_rng(seed * 1000 + limit)
  if kind == 'uniform':
    p = rng.random(limit) + 0.01
  elif kind == 'lognormal2':
    p = np.exp(rng.normal(0.0, 2.0, limit))
  elif kind == 'lognormal3':
    p = np.exp(rng.normal(0.0, 3.0, limit))
  elif kind == 'equal':
    p = np.full(limit, 0.37)
  elif kind == 'spike':                       # one item 10^6 times the rest
    p = np.full(limit, 0.37)
    p[limit // 3] = 0.37e6
  elif kind == 'zeros':                       # ~10% exact zeros, leading and trailing runs of 3
    p = rng.random(limit) + 0.01
    zero = rng.random(limit) < 0.1
    zero[:3] = True
    zero[-3:] = True
    zero[limit // 2] = False                  # some item has mass
    p[zero] = 0.0
  else:
    raise ValueError(kind)
  return p.astype(F)


def rel_err(got, ref):
  """max |got - ref| / |ref| over ref != 0; got must be exactly 0 where ref is."""
  got = np.asarray(got, np.float64); ref = np.asarray(ref, np.float64)
  nz = ref != 0
  assert (got[~nz] == 0).all(), 'nonzero where the float64 reference is 0'
  return float((np.abs(got[nz] - ref[nz]) / np.abs(ref[nz])).max()) if nz.any() else 0.0


def mass64(prio, limit, alpha):
  """prio_i^alpha in float64, with alpha the float32 the kernel is given."""
  return np.power(np.asarray(prio[:limit], np.float64), float(F(alpha)))


def edge(limit):
  """Bound on how far an fp32 bin edge of the draw lies from float64, as a fraction of the total."""
  return (limit + 8) * 2.0 ** -23


def check_sample(prio, limit, alpha, beta, u, idx, w, probs=None):
  """Checks one draw of the sampler against float64.  Returns {'weights': (err, bar), 'probs': ...}."""
  m64 = mass64(prio, limit, alpha)
  cdf = np.cumsum(m64)
  total = cdf[-1]
  p64 = m64 / total
  idx = np.asarray(idx); w = np.asarray(w); u = np.asarray(u, np.float64)
  assert idx.shape == u.shape and w.shape == u.shape
  assert idx.min() >= 0 and idx.max() < limit
  # the draw: zero mass never, otherwise the float64 inverse CDF up to the fp32 prefix bound
  assert (m64[idx] > 0).all(), 'a zero-priority item was drawn'
  x = u * total
  lo = np.concatenate([[0.0], cdf[:-1]])[idx]
  e = edge(limit) * total
  bad = ~((x >= lo - e) & (x < cdf[idx] + e))
  assert not bad.any(), 'draws outside their float64 bin: u=%s idx=%s' % (u[bad][:4], idx[bad][:4])
  first, last = np.flatnonzero(m64 > 0)[[0, -1]]
  assert (idx[u == 0] == first).all()
  if m64[last] > 2 * e:                     # else the last item may be lost in the fp32 prefix
    assert (idx[u >= F(0.99999994)] == last).all()
  # weights: float64 over the GPU's own indices
  w64 = np.power((1.0 / limit) / p64[idx], float(F(beta)))
  w64 /= w64.max()
  m32 = np.power(np.asarray(prio[:limit], F), F(alpha))
  p32 = m32 / np.cumsum(m32, dtype=F)[-1]
  w32 = np.power((F(1) / F(limit)) / p32[idx], F(beta))
  w32 = w32 / w32.max()
  assert w.max() == 1.0, w.max()
  if beta == 0 or np.ptp(prio[:limit]) == 0:
    assert (w == 1.0).all(), 'weights must be exactly 1: %s' % w[w != 1.0][:4]
  out = {'weights': (rel_err(w, w64), max(W_FLOOR, C * rel_err(w32, w64)))}
  if probs is not None:
    out['probs'] = (rel_err(probs, p64), max(P_FLOOR, C * rel_err(p32, p64)))
  for k, (err, bar) in out.items():
    assert err <= bar, '%s: error %.3e > bar %.3e (limit %d, alpha %g, beta %g)' % (k, err, bar, limit, alpha, beta)
  return out


def check_grid(prio, limit, alpha, idx):
  """The dense grid u_j = (j + 1/2) / N: each item's count / N is its float64 probability, up to one
  grid point and the displacement of its two fp32 edges."""
  p64 = mass64(prio, limit, alpha)
  p64 = p64 / p64.sum()
  n = len(idx)
  freq = np.bincount(np.asarray(idx), minlength=limit) / n
  assert len(freq) == limit
  assert (freq[p64 == 0] == 0).all()
  dev = np.abs(freq - p64).max()
  assert dev <= 1.0 / n + 2 * edge(limit), (dev, 1.0 / n + 2 * edge(limit))
  return dev


def grid_uniforms(n=1 << 20):
  return ((np.arange(n) + 0.5) / n).astype(F)        # exact in float32


# ---- replay sampling on the GPU --------------------------------------------------------------
def _cuda(a):
  return torch.as_tensor(np.asarray(a)).cuda()


def _loss_priorities(limit):
  """Priorities as the learner writes them back: seedrl_r2d2_loss_fwd_bwd on random Q values."""
  from types import SimpleNamespace as NS
  from seed_rl_b200.agents.r2d2 import learner
  rng = np.random.default_rng(limit)
  T, A = 12, 18
  q, qt = (_cuda(rng.normal(size=(T, limit, A)).astype(F)) for _ in range(2))
  env = NS(reward=_cuda(rng.normal(size=(T, limit)).astype(F)), done=_cuda(rng.random((T, limit)) < 0.05))
  act = NS(action=_cuda(rng.integers(0, A, (T, limit))))
  _, prio, _ = learner.compute_loss_and_priorities_from_agent_outputs(NS(q_values=q), NS(q_values=qt), env, act,
                                                                      gamma=0.997)
  return prio.cpu().numpy()


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('limit', LIMITS)
def test_replay_sample_vs_float64(limit, kind):
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  prio = _loss_priorities(limit) if kind == 'loss' else priorities(kind, limit)
  assert (prio >= 0).all() and (prio > 0).any()
  rng = np.random.default_rng(limit + 7)
  u = np.concatenate([PINNED, rng.random(max(NUM_SAMPLES) - len(PINNED)).astype(F)])
  pr, uc = _cuda(prio), _cuda(u)
  worst = {}
  for alpha, beta in EXPONENTS:
    for n in NUM_SAMPLES:
      idx, w, probs = learner.replay_sample(pr, limit, n, alpha, beta, uniforms=uc[:n])
      res = check_sample(prio, limit, alpha, beta, u[:n], idx.cpu().numpy(), w.cpu().numpy(), probs.cpu().numpy())
      for k, v in res.items():
        worst[k] = max(worst.get(k, v), v)
    # PrioritizedReplay.sample runs the same kernel on its ring (values = slot numbers)
    rb = utils.PrioritizedReplay(limit, (utils.TensorSpec([], 'int32', 'slot'),), importance_sampling_exponent=beta)
    rb.insert((_cuda(np.arange(limit, dtype=np.int32)),), pr)
    i_rb, w_rb, (slots,) = rb.sample(1025, alpha, uniforms=uc[:1025])
    idx, w, _ = learner.replay_sample(pr, limit, 1025, alpha, beta, uniforms=uc[:1025])
    assert torch.equal(i_rb, idx) and torch.equal(w_rb, w)
    assert torch.equal(slots.long(), i_rb)
  # one call on a dense deterministic grid
  for alpha in (0.9, 1.0):
    ug = grid_uniforms()
    idx, _, _ = learner.replay_sample(pr, limit, len(ug), alpha, 0.6, uniforms=_cuda(ug))
    dev = check_grid(prio, limit, alpha, idx.cpu().numpy())
  print('replay limit %d %-10s  weights err %.2e bar %.2e  probs err %.2e bar %.2e  grid dev %.2e' %
        (limit, kind, *worst['weights'], *worst['probs'], dev))


def test_replay_limit_above_the_cap_is_refused():
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  prio = _cuda(priorities('uniform', 8193))
  n0 = _lib.launch_count()
  with pytest.raises(_lib.SeedrlError, match='8192'):
    learner.replay_sample(prio, 8193, 64, 0.9, 0.6)
  assert _lib.launch_count() == n0
  rb = utils.PrioritizedReplay(8200, (utils.TensorSpec([], 'int32', 'slot'),), importance_sampling_exponent=0.6)
  rb.insert((_cuda(np.arange(8193, dtype=np.int32)),), prio)
  with pytest.raises(_lib.SeedrlError, match='8192'):
    rb.sample(64, 0.9)
  assert _lib.launch_count() == n0
  # uniform sampling does not use the kernel and has no cap
  idx, w, (slots,) = rb.sample(4096, 0.0, generator=torch.Generator(device='cuda').manual_seed(3))
  i = idx.cpu().numpy()
  assert i.min() >= 0 and i.max() < 8193 and len(np.unique(i)) > 3000
  assert (w.cpu().numpy() == 1.0).all() and torch.equal(slots.long(), idx)


# ---- global-norm clip ------------------------------------------------------------------------
ARENA = 4357281                              # DuelingLSTMDQNNet's parameter arena at A = 18
SIZES = (1, 3, ARENA, (1 << 24) + 3)


def _gradients(kind, n, seed):
  rng = np.random.default_rng(seed)
  g = rng.normal(size=n)
  if kind == 'blocks':                       # blocks at scales 1e-8 .. 1e2, the largest last
    for s, part in zip(np.logspace(-8, 2, min(n, 11)), np.array_split(np.arange(n), min(n, 11))):
      g[part] *= s
  return g


def _exact_40(n, seed):
  """Norm exactly 40: 1600 ones (n >= 1600), else (40,) and (0, -24, 32)."""
  if n == 1:
    return np.array([40.0], F)
  if n == 3:
    return np.array([0.0, -24.0, 32.0], F)
  g = np.zeros(n, F)
  g[np.random.default_rng(seed).choice(n, 1600, replace=False)] = 1.0
  return g


def _clip_gpu(g):
  from seed_rl_b200.agents.r2d2 import learner
  gc = _cuda(g)
  norm = learner.clip_by_global_norm(gc, CLIP)
  return gc, norm


def _check_clip(g):
  """Clips g (float32) twice on the GPU; checks norm and elements against float64.  -> errors, bars."""
  g64 = g.astype(np.float64)
  n64 = np.sqrt(np.dot(g64, g64))
  ref = g64 * (CLIP / max(n64, CLIP))
  n32 = np.sqrt(np.sum(g * g, dtype=F))
  out32 = g * (F(CLIP) / np.maximum(n32, F(CLIP)))
  a, na = _clip_gpu(g)
  b, nb = _clip_gpu(g)
  assert torch.equal(a, b) and torch.equal(na, nb), 'two calls differ'
  out = a.cpu().numpy()
  err = {'norm': (rel_err([float(na)], [n64]), max(CLIP_FLOOR, C * rel_err([n32], [n64]))),
         'elements': (rel_err(out, ref), max(CLIP_FLOOR, C * rel_err(out32, ref)))}
  for k, (e, bar) in err.items():
    assert e <= bar, '%s: error %.3e > bar %.3e (n %d, norm %.6g)' % (k, e, bar, len(g), n64)
  if n64 <= CLIP:
    assert np.array_equal(out, g), 'a norm at or below the clip must leave the gradients bit-identical'
  return err


@pytest.mark.parametrize('level', ['below', 'above', 'far'])
@pytest.mark.parametrize('kind', ['normal', 'blocks'])
@pytest.mark.parametrize('n', SIZES)
def test_clip_by_global_norm_vs_float64(n, kind, level):
  target = {'below': 4.0, 'above': CLIP * (1 + 2.0 ** -16), 'far': 1e4 * CLIP}[level]
  g = _gradients(kind, n, seed=n % 1000 + len(kind))
  g = (g * (target / np.sqrt(np.dot(g, g)))).astype(F)
  n64 = np.sqrt(np.dot(g.astype(np.float64), g.astype(np.float64)))
  assert (n64 < CLIP) if level == 'below' else (n64 > CLIP)
  err = _check_clip(g)
  print('clip n %d %-6s %-5s  norm err %.2e bar %.2e  elements err %.2e bar %.2e' %
        (n, kind, level, *err['norm'], *err['elements']))


@pytest.mark.parametrize('n', SIZES)
def test_clip_norm_exactly_40_is_identity(n):
  g = _exact_40(n, seed=n)
  assert np.dot(g.astype(np.float64), g.astype(np.float64)) == CLIP ** 2
  _, norm = _clip_gpu(g)
  assert float(norm) == CLIP
  _check_clip(g)


@pytest.mark.parametrize('case', ['inf', 'nan', 'overflow'])
@pytest.mark.parametrize('n', SIZES)
def test_clip_non_finite_norm_makes_every_element_nan(n, case):
  """tf.clip_by_global_norm: a non-finite global norm turns every clipped tensor into NaN."""
  g = _gradients('normal', n, seed=n).astype(F)
  if case == 'overflow':
    g[:] = 1e20                                # finite elements whose squares overflow fp32
  else:
    g[np.random.default_rng(n).integers(n)] = np.inf if case == 'inf' else np.nan
  out, norm = _clip_gpu(g)
  assert not np.isfinite(float(norm))
  assert torch.isnan(out).all(), '%d of %d elements are not NaN' % (int((~torch.isnan(out)).sum()), n)


def test_clip_empty_arena_norm_is_zero():
  import ctypes
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.r2d2 import learner
  L = _lib.lib()
  g = torch.empty(0, dtype=torch.float32, device='cuda')
  norm = torch.full((), float('nan'), device='cuda')
  scratch = torch.empty(int(L.seedrl_clip_scratch_bytes()), dtype=torch.uint8, device='cuda')
  _lib.check(L.seedrl_clip_by_global_norm(0, None, ctypes.c_float(CLIP), _lib.ptr(norm), _lib.ptr(scratch),
                                          _lib.stream_ptr()))
  assert float(norm) == 0.0
  assert float(learner.clip_by_global_norm(g, CLIP)) == 0.0
