"""The R2D2 loss kernels against float64: r2d2_loss_kernel (the reference's n-step double-DQN targets) and
r2d2_retrace_loss_kernel (Retrace(lambda) targets), which run r2d2_loss_thread and r2d2_retrace_loss_thread of
seed_rl_b200/csrc/r2d2_thread.inl, one thread per sequence.  They produce the learner's per-sequence loss, its
gradient dq and the priorities the replay samples by; central inference takes its initial priorities from them.

Reference.  `restate` restates both bodies in numpy in a dtype F, in the bodies' order of operations, from the
float32 inputs and the float32 gamma, eta, eps and lambda the kernels are given, with h and h^-1 in one of the two
forms of tests/r2d2_float64_reference.py.  In float64 with the stable forms it is the float64 reference.  In float32
with the stable forms it is the bodies' own arithmetic: the CPU build of the bodies (tests/host_emulation, g++
without fp contraction) matches it bit for bit.  In float32 with the literal forms it is the reference's arithmetic,
oracle/r2d2_oracle.py's, whose h^-1 cancels: test_literal_forms_fail_the_bars_at_small_q shows these bars reject it.

Outputs and error.  targets (the raw Bellman targets the kernels leave in their scratch array, before h; rows
0..T-1 for n-step, 1..T-1 for Retrace), loss [B], priorities [B] and dq [T, B, A].  Per sequence b: for targets and
dq, max_t |got - ref64| / max_t |ref64|, and a sequence whose reference is all zero must be exactly zero; for loss
and priorities, |got - ref64| / |ref64|.  The error is the largest over b.  Per sequence, because the priorities of a
batch differ in scale by orders of magnitude (reward-free sequences next to rewarded ones) and the replay samples
each sequence by its own: against the batch's largest |td| the cancellation of the literal h^-1 is invisible.

Bar = max(FLOOR, C m), m the same error of the float32 stable restatement (the rule of the other float64 files).
C = 4: the GPU rounds the same operations in the same order, except that nvcc contracts a * b + c into one fma
(the Bellman passes, h, h^-1's argument, the sum of squares, the priority), which moves each rounding but does not
add any.  The floors, in units u = 2^-24, cover a case whose m happens to be near 0 (T = 2, B = 1: one TD error):
  * targets, 16u: a target is h^-1 of a Q value, within 8u of float64 (10 roundings: 4 in the sqrt argument, the
    sqrt, 2 in the denominator, the quotient, 2 in d (2 + d); test_host_rescaling_is_the_float32_stable_form), plus
    one multiply-add per Bellman pass or Retrace step;
  * loss and priorities, 16u: td = h(target) - q adds h, within 4u, and one subtraction to the target's error; then
    |td| is squared and summed (loss), or maximised, summed, averaged and blended with eta (priorities);
  * dq, 16u: -(w / B) td, two roundings on top of td.
Measured on an H100 80GB HBM3 at a 700 W power limit, the largest error of any run is 0.41 of its bar for dq, 0.34
for the priorities, 0.33 for the loss and 0.29 for the targets.

Every run also checks: all outputs NaN-poisoned before the call; every dq entry but the replayed action of rows
0..T-2 exactly 0; nothing written past the end of any output; on the GPU, two launches bit-identical and the call
through learner.compute_loss_and_priorities_from_agent_outputs bit-identical to the direct one.
"""
import collections
import ctypes
import functools
import os
import subprocess
import zlib

import numpy as np
import pytest

import r2d2_float64_reference as RF

HERE = os.path.dirname(os.path.abspath(__file__))
F32, F64 = np.float32, np.float64
U = 2.0 ** -24
C = 4
FLOOR = dict(targets=16 * U, loss=16 * U, priorities=16 * U, dq=16 * U)
OUTPUTS = tuple(FLOOR)
PAD = 64                                          # poisoned elements after the end of every output
POISON = np.array([0x7FC0DEAD], np.uint32).view(F32)[0]

# ---- cases ----------------------------------------------------------------------------------------------------------
Case = collections.namedtuple('Case', 'name T B A n gamma eta eps q rewards done weights actions greedy lams small '
                                       'seed')


def _case(name, small=False, **kw):
  """The bench.py --agent r2d2 loss (T = 101, B = 64, A = 18, n = 5, gamma = 0.997, eta = 0.9, eps = 1e-3) with
  the given changes.  q: the scale of the Q values; greedy: the fraction of replayed actions that are the online
  network's argmax; lams: the Retrace lambdas run besides the n-step kernel; small: the literal h^-1 must fail."""
  d = dict(T=101, B=64, A=18, n=5, gamma=0.997, eta=0.9, eps=1e-3, q=1.0, rewards='sparse', done='rare',
           weights='random', actions='random', greedy=0.5, lams=(0.95,))
  d.update(kw)
  return Case(name=name, small=small, seed=zlib.crc32(name.encode()), **d)


CASES = (
    # Q values of scale 1e-4 .. 300; sparse rewards, half of the sequences reward-free
    [_case('bench-q%g' % q, q=q, lams=(0.0, 0.5, 0.95, 1.0), small=q <= 0.1)
     for q in (1e-4, 1e-3, 1e-2, 0.1, 1, 10, 300)]
    + [_case('rewards-zero', rewards='zero'), _case('rewards-zero-q1e-3', rewards='zero', q=1e-3, small=True),
       _case('rewards-negative', rewards='negative'), _case('rewards-unclipped', rewards='unclipped'),
       _case('rewards-normal-q1e-2', rewards='normal', q=1e-2, small=True)]
    # episode ends at row 0, at the last row, on every row, and on each offset of the n-step window
    + [_case('done-' + k, done=k) for k in ('row0', 'last', 'every', 'window')]
    + [_case('done-window-n3', done='window', n=3), _case('done-window-n8', done='window', n=8)]
    # n_steps 1 .. 8, and T = 2, 3 with n >= T
    + [_case('n%d' % n, n=n) for n in (1, 2, 3, 4, 6, 7, 8)]
    + [_case('T2-n%d' % n, T=2, n=n, lams=(0.0, 1.0)) for n in (1, 2, 8)]
    + [_case('T3-n%d' % n, T=3, n=n, lams=(0.0, 0.5, 1.0)) for n in (1, 3, 8)]
    # gamma = 0 only at n = 1: the reference pads the targets with q / gamma^k, NaN for k >= 1 at gamma = 0
    + [_case('gamma0', gamma=0.0, n=1, lams=(0.0, 0.95, 1.0)), _case('gamma0.99', gamma=0.99),
       _case('gamma1', gamma=1.0, lams=(0.95, 1.0))]
    + [_case('eps1e-2', eps=1e-2), _case('eps1e-6', eps=1e-6), _case('eps1e-6-q1e-3', eps=1e-6, q=1e-3, small=True)]
    # one 64-thread CTA, a partial one, several
    + [_case('B%d' % B, B=B) for B in (1, 63, 65, 4096)]
    + [_case('A1', A=1, lams=(0.5, 1.0)), _case('B1-A1', B=1, A=1, lams=(1.0,))]
    # tied maxima (the first wins), replayed actions outside [0, A) (clamped), importance weights
    + [_case('ties', actions='ties', lams=(0.5, 1.0)), _case('outside', actions='outside', lams=(0.5, 1.0)),
       _case('weights-none', weights='none'), _case('weights-zero', weights='zero')]
    # Retrace with no, half and all replayed actions greedy
    + [_case('greedy0', greedy=0.0, lams=(0.5, 0.95, 1.0)), _case('greedy1', greedy=1.0, lams=(0.0, 0.5, 0.95, 1.0)),
       _case('greedy1-q1e-3', greedy=1.0, q=1e-3, lams=(0.95, 1.0), small=True)])
BY_NAME = {c.name: c for c in CASES}
assert len(BY_NAME) == len(CASES)

# a run: one kernel on one case; param is n_steps for 'n_step', lambda for 'retrace'
RUNS = [(c.name, 'n_step', c.n) for c in CASES] + [(c.name, 'retrace', lam) for c in CASES for lam in c.lams]


def run_id(run):
  name, rule, param = run
  return '%s-%s' % (name, 'n%d' % param if rule == 'n_step' else 'lambda%g' % param)


@functools.lru_cache(maxsize=4)
def inputs(name):
  """(q_train, q_target [T,B,A] float32, replay actions [T,B] int64, reward [T,B] float32, done [T,B] bool,
  importance weights [B] float32 or None)."""
  c = BY_NAME[name]
  rng = np.random.default_rng(c.seed)
  T, B, A = c.T, c.B, c.A
  z = rng.normal(size=(T, B, A))
  if c.actions == 'ties':                         # few distinct values: many tied maxima
    z = np.round(z * 2) / 2
  tq = (z * c.q).astype(F32)
  gq = ((z + 0.3 * rng.normal(size=z.shape)) * c.q).astype(F32)     # the target network near the online one
  greedy = tq.argmax(-1)
  other = (greedy + rng.integers(1, max(A, 2), (T, B))) % A          # a non-greedy action (A > 1)
  ra = np.where(rng.random((T, B)) < c.greedy, greedy, other if A > 1 else greedy).astype(np.int64)
  if c.actions == 'ties':                         # a tied maximum that is not the first one is not greedy
    for t, b in zip(*np.nonzero((tq == tq.max(-1, keepdims=True)).sum(-1) > 1)):
      if rng.random() < 0.5:
        ra[t, b] = np.nonzero(tq[t, b] == tq[t, b].max())[0][-1]
  elif c.actions == 'outside':
    pick = rng.random((T, B)) < 0.2
    ra[pick] = rng.choice(np.array([-1, -7, A, A + 5, 1 << 40, -(1 << 40)]), int(pick.sum()))
  if c.rewards == 'sparse':
    r = (rng.random((T, B)) < 0.02).astype(F32)
    r[:, :B // 2] = 0
  elif c.rewards == 'zero':
    r = np.zeros((T, B), F32)
  elif c.rewards == 'negative':
    r = -((rng.random((T, B)) < 0.1) * rng.random((T, B)) * 2)
  elif c.rewards == 'unclipped':                  # |r| in [0.1, 1e3] on a fifth of the rows
    r = (rng.random((T, B)) < 0.2) * rng.choice([-1., 1.], (T, B)) * 10 ** rng.uniform(-1, 3, (T, B))
  else:
    r = rng.normal(size=(T, B))
  done = rng.random((T, B)) < 0.01
  if c.done == 'row0':
    done[0] = True
  elif c.done == 'last':
    done[-1] = True
  elif c.done == 'every':
    done[:] = True
  elif c.done == 'window':
    # columns b < B/2: every n rows at offset b mod n; the others: one done k rows before the end, k = 0 .. n + 1
    # (the rows whose n-step windows reach into the padding)
    t, b = np.meshgrid(np.arange(T), np.arange(B), indexing='ij')
    done = np.where(b < B // 2, (t - b) % c.n == 0, t == T - 1 - b % (c.n + 2))
  w = {'random': (rng.random(B) * 2).astype(F32), 'zero': np.zeros(B, F32), 'none': None}[c.weights]
  return tq, gq, ra, np.asarray(r, F32), done, w


def restate(inp, rule, param, gamma, eta, eps, F, forms='stable'):
  """One launch restated in numpy in F (see the module docstring).  inp: as `inputs` returns; param: n_steps for
  'n_step', lambda for 'retrace'.  -> dict targets [T', B] (the rows of `target_rows`), loss [B], priorities [B],
  dq [T, B, A]."""
  tq, gq, ra, r, done, w = inp
  T, B, A = tq.shape
  h, hinv = ((RF.stable_value_function_rescaling, RF.stable_inverse_value_function_rescaling) if forms == 'stable'
             else (RF.literal_value_function_rescaling, RF.literal_inverse_value_function_rescaling))
  gamma32 = float(F32(gamma))                     # the kernels are given float32 values
  g, eta, eps = F(gamma32), F(F32(eta)), F(F32(eps))
  tt, bb = np.meshgrid(np.arange(T), np.arange(B), indexing='ij')
  greedy = tq.argmax(-1)                          # first maximum
  a = np.clip(ra, 0, A - 1)
  q_star = hinv(gq[tt, bb, greedy], eps, F)
  if rule == 'n_step':
    y = RF.n_step_bellman_target(r, done, q_star, gamma32, param, F)
  else:
    lam = F(F32(param))
    q_act = hinv(gq[tt, bb, a], eps, F)
    nd = np.where(done, F(0), F(1))
    y = np.zeros((T, B), F)
    for i in range(T - 1, 0, -1):                 # r2d2_retrace_loss_thread's backward walk
      v = q_star[i]
      if i + 1 < T:
        v = v + np.where(a[i] == greedy[i], lam, F(0)) * (y[i + 1] - q_act[i])
      y[i] = r[i].astype(F) + g * nd[i] * v
  td = h(y[1:], eps, F) - tq[:-1].astype(F)[tt[:-1], bb[:-1], a[:-1]]
  ad = np.abs(td)
  s = np.cumsum(ad, axis=0, dtype=F)[-1]          # serial sums, as one thread adds
  sq = np.cumsum(ad * ad, axis=0, dtype=F)[-1]
  prio = eta * ad.max(axis=0) + (F(1) - eta) * (s / F(T - 1))
  wb = (np.ones(B, F) if w is None else w.astype(F)) / F(B)
  dq = np.zeros((T, B, A), F)
  dq[tt[:-1], bb[:-1], a[:-1]] = -wb[None] * td
  return dict(targets=y[target_rows(rule, T)], loss=F(0.5) * sq, priorities=prio, dq=dq)


def target_rows(rule, T):
  return slice(0, T) if rule == 'n_step' else slice(1, T)


@functools.lru_cache(maxsize=16)
def reference(run, F, forms='stable'):
  name, rule, param = run
  c = BY_NAME[name]
  out = restate(inputs(name), rule, param, c.gamma, c.eta, c.eps, F, forms)
  for v in out.values():
    v.setflags(write=False)
  return out


def _seq_err(got, ref):
  """got, ref [B, K]: max over b of max_k |got - ref| / max_k |ref|; inf where got is not finite or a sequence
  whose reference is all zero is not."""
  got = np.asarray(got, F64); ref = np.asarray(ref, F64)
  if not np.isfinite(got).all():
    return float('inf')
  num, den = np.abs(got - ref).max(axis=1), np.abs(ref).max(axis=1)
  if (num[den == 0] != 0).any():
    return float('inf')
  return float((num[den > 0] / den[den > 0]).max()) if (den > 0).any() else 0.0


def errors(out, ref):
  """{output: error} for the outputs in `out` (any of OUTPUTS)."""
  B = ref['loss'].shape[0]
  per_seq = dict(targets=lambda x: np.asarray(x).T, loss=lambda x: np.asarray(x)[:, None],
                 priorities=lambda x: np.asarray(x)[:, None], dq=lambda x: np.swapaxes(x, 0, 1).reshape(B, -1))
  return {k: _seq_err(per_seq[k](out[k]), per_seq[k](ref[k])) for k in OUTPUTS if k in out}


def bars(ref32, ref64):
  m = errors(ref32, ref64)
  return {k: max(FLOOR[k], C * m[k]) for k in OUTPUTS}


def check_outputs(out, inp, rule, param, gamma, eta, eps, ref64=None, ref32=None, what=''):
  """Asserts that the outputs of one launch (a dict with any of OUTPUTS) are within the bars of the float64
  reference and, if dq is given, that it is 0 off the replayed actions of rows 0..T-2.  -> {output: (err, bar)}."""
  tq, _, ra, _, _, _ = inp
  T, B, A = tq.shape
  if 'dq' in out:
    tt, bb = np.meshgrid(np.arange(T - 1), np.arange(B), indexing='ij')
    replayed = np.zeros((T, B, A), bool)
    replayed[tt, bb, np.clip(ra[:-1], 0, A - 1)] = True
    dq = np.asarray(out['dq'])
    assert (dq[~replayed] == 0).all(), '%s: %d dq entries off the replayed actions are not 0' % (
        what, int((dq[~replayed] != 0).sum()))
  args = (inp, rule, param, gamma, eta, eps)
  ref64 = restate(*args, F64) if ref64 is None else ref64
  ref32 = restate(*args, F32) if ref32 is None else ref32
  err, bar = errors(out, ref64), bars(ref32, ref64)
  res = {k: (err[k], bar[k]) for k in err}
  bad = {k: v for k, v in res.items() if not v[0] <= v[1]}
  assert not bad, '%s: error > bar: %s' % (what, ', '.join('%s %.3e > %.3e' % (k, e, b) for k, (e, b) in bad.items()))
  return res


def check(run, out):
  name, rule, param = run
  c = BY_NAME[name]
  return check_outputs(out, inputs(name), rule, param, c.gamma, c.eta, c.eps, reference(run, F64),
                       reference(run, F32), run_id(run))


def report(run, res, tag):
  print('%s %-28s ' % (tag, run_id(run)) + '  '.join('%s %.2e/%.2e (%.2f)' % (k, e, b, e / b)
                                                     for k, (e, b) in res.items()))


# ---- output buffers: poisoned, with a poisoned tail ---------------------------------------------------------------
def scratch_floats(rule, param, T, B):
  return B * (T + param) if rule == 'n_step' else T * B


def poisoned_buffers(rule, param, T, B, A):
  n = dict(loss=B, priorities=B, dq=T * B * A, scratch=scratch_floats(rule, param, T, B))
  return {k: np.full(v + PAD, POISON, F32) for k, v in n.items()}


def unpack(bufs, rule, param, T, B, A):
  """The outputs of poisoned_buffers after a call; asserts that every tail is still poisoned."""
  for k, v in bufs.items():
    tail = np.asarray(v[-PAD:]).view(np.uint32)
    assert (tail == POISON.view(np.uint32)).all(), '%s: written past the end' % k
  s = bufs['scratch'][:-PAD]
  if rule == 'n_step':
    targets = s.reshape(B, T + param)[:, :T].T
  else:
    targets = s.reshape(T, B)[target_rows(rule, T)]
  return dict(targets=targets, loss=bufs['loss'][:B], priorities=bufs['priorities'][:B],
              dq=bufs['dq'][:-PAD].reshape(T, B, A))


# ---- the bodies on the CPU ----------------------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('emu') / '_r2d2_loss_host.so')
  subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', so,
                         os.path.join(HERE, 'host_emulation', 'r2d2_host.cpp'),
                         os.path.join(HERE, 'host_emulation', 'r2d2_retrace_host.cpp')])
  return ctypes.CDLL(so)


def run_host(emu, run):
  name, rule, param = run
  c = BY_NAME[name]
  tq, gq, ra, r, done, w = inputs(name)
  T, B, A = tq.shape
  bufs = poisoned_buffers(rule, param, T, B, A)
  p = lambda x: None if x is None else x.ctypes.data_as(ctypes.c_void_p)
  f = ctypes.c_float
  args = [p(tq), p(gq), p(ra), p(r), p(done.astype(np.uint8)), p(w)]
  outs = [p(bufs[k]) for k in ('loss', 'priorities', 'dq', 'scratch')]
  if rule == 'n_step':
    rc = emu.emu_r2d2_loss(T, B, A, *args, f(c.gamma), param, f(c.eta), f(c.eps), *outs)
  else:
    rc = emu.emu_r2d2_retrace_loss(T, B, A, *args, f(c.gamma), f(param), f(c.eta), f(c.eps), *outs)
  assert rc == 0
  return unpack(bufs, rule, param, T, B, A)


@pytest.mark.parametrize('run', RUNS, ids=run_id)
def test_host_bodies_meet_the_float64_bars(emu, run):
  """The kernels' bodies built for the CPU: within the float64 bars, and bit for bit the float32 restatement."""
  out = run_host(emu, run)
  report(run, check(run, out), 'HOST')
  ref32 = reference(run, F32)
  for k in OUTPUTS:
    np.testing.assert_array_equal(out[k], ref32[k], err_msg='%s: %s' % (run_id(run), k))


@pytest.mark.parametrize('run', [x for x in RUNS if BY_NAME[x[0]].small], ids=run_id)
def test_literal_forms_fail_the_bars_at_small_q(run):
  """The bars have teeth: the reference's literal h and h^-1 in float32 (oracle/r2d2_oracle.py's) miss them for
  small Q values, in the targets, the loss, the priorities and dq alike."""
  err = errors(reference(run, F32, 'literal'), reference(run, F64))
  b = bars(reference(run, F32), reference(run, F64))
  print('LITERAL %-28s ' % run_id(run) + '  '.join('%s %.2e (%.0f x bar)' % (k, err[k], err[k] / b[k])
                                                   for k in OUTPUTS))
  assert all(err[k] > b[k] for k in OUTPUTS), (err, b)


# ---- h and h^-1 ---------------------------------------------------------------------------------------------------
EPSILONS = (1e-3, 1e-2, 1e-6)


def _sweep():
  x = np.concatenate([np.logspace(-30, 30, 4001), np.logspace(-4, 4, 4001), np.linspace(0, 50, 2001)[1:]])
  return np.concatenate([x, -x]).astype(F32)


@pytest.mark.parametrize('eps', EPSILONS)
def test_float64_forms_are_the_literal_formula_in_longdouble(eps):
  """The stable forms in float64 against the reference's literal formula in np.longdouble, whose own rounding is
  bounded by its two cancellations: |sqrt(|x| + 1) - 1| to ~ulp(sqrt(|x| + 1)) for h, and inner - 1 to
  ~ulp(s) / (2 eps), then inner^2 - 1 to twice that times inner, for h^-1."""
  L = np.longdouble
  uL = float(np.finfo(L).eps)
  x = _sweep().astype(F64)
  x = x[np.abs(x) <= 1e15]
  e = float(F32(eps))
  xl, el = x.astype(L), L(e)
  h_lit = np.sign(xl) * (np.sqrt(np.abs(xl) + 1) - 1) + el * xl
  s_l = np.sqrt(1 + 4 * el * (np.abs(xl) + 1 + el))
  inner = (s_l - 1) / (2 * el)
  hinv_lit = np.sign(xl) * (inner * inner - 1)
  h64 = RF.value_function_rescaling(x, e, F64)
  hinv64 = RF.inverse_value_function_rescaling(x, e, F64)
  u64 = 2.0 ** -53
  bound_h = 8 * u64 * np.abs(h64) + 4 * uL * np.sqrt(np.abs(x) + 1)
  bound_hinv = 8 * u64 * np.abs(hinv64) + 4 * uL * (s_l.astype(F64) / e) * inner.astype(F64)
  assert (np.abs(h64 - h_lit.astype(F64)) <= bound_h).all()
  assert (np.abs(hinv64 - hinv_lit.astype(F64)) <= bound_hinv).all()
  # and the two are inverse to each other
  np.testing.assert_allclose(RF.inverse_value_function_rescaling(h64, e, F64), x, rtol=4e-15, atol=0)


@pytest.mark.parametrize('eps', EPSILONS)
def test_host_rescaling_is_the_float32_stable_form(emu, eps):
  """vf_rescale and vf_rescale_inv, built for the CPU, are the float32 stable forms bit for bit; they are within a
  few roundings of float64 wherever the result is a normal float32 (4u for h, 3.5u seen; 8u for h^-1, 7u seen; the
  literal forms lose every bit near 0), and keep the reference's values at 0, NaN and +-inf."""
  x = np.concatenate([_sweep(), np.array([0.0, -0.0, np.inf, -np.inf, np.nan, 1e-45, -1e-45,
                                          np.finfo(F32).max, -np.finfo(F32).max], F32)])
  e = F32(eps)
  got = {}
  for inverse, fn in ((0, RF.stable_value_function_rescaling), (1, RF.stable_inverse_value_function_rescaling)):
    out = np.zeros_like(x)
    assert emu.emu_vf_rescale(len(x), x.ctypes.data_as(ctypes.c_void_p), ctypes.c_float(e), inverse,
                              out.ctypes.data_as(ctypes.c_void_p)) == 0
    np.testing.assert_array_equal(out, fn(x, e, F32))
    got[inverse] = out
  for inverse, want in ((0, RF.value_function_rescaling), (1, RF.inverse_value_function_rescaling)):
    out, ref = got[inverse], want(x.astype(F64), float(e), F64)
    ok = np.isfinite(ref) & (np.abs(ref) < np.finfo(F32).max) & (np.abs(ref) > np.finfo(F32).tiny)
    rel = np.abs(out[ok] - ref[ok]) / np.abs(ref[ok])
    assert rel.max() <= (4 if inverse == 0 else 8) * U, (inverse, rel.max() / U)
  for inverse in (0, 1):
    out = got[inverse][-9:]
    assert out[0] == 0 and out[1] == 0
    assert out[2] == np.inf and out[3] == -np.inf and np.isnan(out[4])


# ---- the kernels on the GPU -----------------------------------------------------------------------------------------
def _launch(run, L, lib, dev):
  import torch
  name, rule, param = run
  c = BY_NAME[name]
  tq, gq, ra, r, done, w = (None if x is None else torch.as_tensor(x).to(dev) for x in inputs(name))
  T, B, A = tq.shape
  bufs = {k: torch.as_tensor(v).to(dev) for k, v in poisoned_buffers(rule, param, T, B, A).items()}
  args = [lib.ptr(x) for x in (tq, gq, ra, r, done, w)]
  outs = [lib.ptr(bufs[k]) for k in ('loss', 'priorities', 'dq', 'scratch')]
  assert L.seedrl_r2d2_loss_scratch_bytes(T, B, c.n) == 4 * scratch_floats('n_step', c.n, T, B)
  assert L.seedrl_r2d2_retrace_loss_scratch_bytes(T, B) == 4 * scratch_floats('retrace', 0.5, T, B)
  if rule == 'n_step':
    rc = L.seedrl_r2d2_loss_fwd_bwd(T, B, A, *args, c.gamma, param, c.eta, c.eps, *outs, lib.stream_ptr())
  else:
    rc = L.seedrl_r2d2_retrace_loss_fwd_bwd(T, B, A, *args, c.gamma, param, c.eta, c.eps, *outs, lib.stream_ptr())
  lib.check(rc)
  return {k: v.cpu().numpy() for k, v in bufs.items()}


@pytest.mark.gpu
@pytest.mark.parametrize('run', RUNS, ids=run_id)
def test_loss_kernels_vs_float64(run):
  import torch
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  L = _lib.lib()
  name, rule, param = run
  c = BY_NAME[name]
  dev = torch.device('cuda')
  first = _launch(run, L, _lib, dev)
  again = _launch(run, L, _lib, dev)
  for k in first:
    np.testing.assert_array_equal(first[k].view(np.uint32), again[k].view(np.uint32), err_msg='%s: repeat' % k)
  T, B, A = inputs(name)[0].shape
  out = unpack(first, rule, param, T, B, A)
  res = check(run, out)
  report(run, res, 'GPU')
  # the learner's entry point launches the same kernel
  tq, gq, ra, r, done, w = (None if x is None else torch.as_tensor(x).to(dev) for x in inputs(name))
  kw = dict(n_steps=param) if rule == 'n_step' else dict(bellman_target='retrace', retrace_lambda=param)
  got = learner.compute_loss_and_priorities_from_agent_outputs(
      learner.AgentOutput(None, tq), learner.AgentOutput(None, gq), utils.EnvOutput(r, done, None, None, None),
      learner.AgentOutput(ra, None), c.gamma, eta=c.eta, importance_weights=w, value_function_rescaling_epsilon=c.eps,
      **kw)
  for k, v in zip(('loss', 'priorities', 'dq'), got):
    np.testing.assert_array_equal(v.cpu().numpy().view(np.uint32), np.asarray(out[k]).view(np.uint32),
                                  err_msg='%s: learner entry point' % k)
