"""CPU: abandoned episodes (a time limit, not the task, ended them) in the V-trace and R2D2 losses.

* The float64 reference (tests/abandoned_float64_reference.py) reproduces the reference's own
  advantages.vtrace targets and advantages.NStep targets (tests/golden/abandoned_golden.npz, written by
  tests/golden/make_golden_abandoned.py from the unmodified reference code).
* The R2D2 n-step and Retrace thread bodies (seed_rl_b200/csrc/r2d2_thread.inl, the source the GPU kernels
  compile) run as host C++ with an abandoned mask against that reference, and are bit-identical to
  themselves without a mask when the mask is NULL or all zero.
* The setting is off by default in both learners, and the flags parse."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import abandoned_float64_reference as R

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, 'golden', 'abandoned_golden.npz')


# ---- the float64 reference against the reference's advantages.py -----------------------------------------------
@pytest.mark.parametrize('case', [0, 1])
@pytest.mark.parametrize('lam', [0.95, 1.0])
def test_vtrace_targets_match_reference_advantages_vtrace(case, lam):
  g = np.load(GOLD)
  p = 'c%d_' % case
  done, ab, V, r = g[p + 'done'], g[p + 'abandoned'], g[p + 'values'], g[p + 'reward']
  assert ab[1:].any() and (done & ~ab)[1:].any()
  gamma = float(g['gamma'])
  vs, pg = R.vtrace(g[p + 'log_rhos'], gamma * (1.0 - done[1:]), r[1:], V[:-1], V[-1], ab[1:], lambda_=lam)
  want = g[p + 'vtrace_l%g_targets' % lam]
  np.testing.assert_allclose(vs, want, rtol=1e-5, atol=1e-5 * np.abs(want).max())
  np.testing.assert_array_equal(vs[ab[1:]], V[:-1][ab[1:]])   # target = own value at a masked transition
  assert np.all(pg[ab[1:]] == 0)


@pytest.mark.parametrize('case', [0, 1])
@pytest.mark.parametrize('n', [1, 3, 5])
def test_nstep_targets_match_reference_nstep(case, n):
  g = np.load(GOLD)
  p = 'c%d_' % case
  want = g[p + 'nstep_n%d_targets' % n]
  got = R.n_step_targets(g[p + 'q_star'], g[p + 'reward'], g[p + 'done'], g[p + 'abandoned'], float(g['gamma']), n)
  np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5 * np.abs(want).max())


def test_golden_covers_the_unroll_ends():
  g = np.load(GOLD)
  for c in (0, 1):
    ab = g['c%d_abandoned' % c]
    assert ab[1].any() and ab[-1].any() and ab[2:-1].any()


# ---- the R2D2 thread bodies as host C++ --------------------------------------------------------------------------
@pytest.fixture(scope='module')
def emu(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('emu') / '_r2d2_abandoned_host.so')
  subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', so,
                         os.path.join(HERE, 'host_emulation', 'r2d2_abandoned_host.cpp')])
  return ctypes.CDLL(so)


P = ctypes.c_void_p
ptr = lambda a: None if a is None else a.ctypes.data_as(P)


def run_emu(emu, rule, param, q, qt, act, rew, done, ab, w, gamma=0.997, eta=0.9, eps=1e-3):
  T, B, A = q.shape
  loss, prio = np.full(B, np.nan, np.float32), np.full(B, np.nan, np.float32)
  dq = np.full((T, B, A), np.nan, np.float32)
  d8 = done.astype(np.uint8)
  a8 = None if ab is None else np.ascontiguousarray(ab.astype(np.uint8))
  if rule == 'n_step':
    scratch = np.zeros(B * (T + param), np.float32)
    emu.emu_r2d2_loss_abandoned(T, B, A, ptr(q), ptr(qt), ptr(act), ptr(rew), ptr(d8), ptr(a8), ptr(w),
                                ctypes.c_float(gamma), int(param), ctypes.c_float(eta), ctypes.c_float(eps),
                                ptr(loss), ptr(prio), ptr(dq), ptr(scratch))
  else:
    scratch = np.zeros(B * T, np.float32)
    emu.emu_r2d2_retrace_loss_abandoned(T, B, A, ptr(q), ptr(qt), ptr(act), ptr(rew), ptr(d8), ptr(a8), ptr(w),
                                        ctypes.c_float(gamma), ctypes.c_float(param), ctypes.c_float(eta),
                                        ctypes.c_float(eps), ptr(loss), ptr(prio), ptr(dq), ptr(scratch))
  return dict(loss=loss, priorities=prio, dq=dq)


RUNS = [('n_step', n) for n in (1, 2, 3, 5)] + [('retrace', lam) for lam in (0.0, 0.95, 1.0)]


@pytest.mark.parametrize('rule,param', RUNS)
@pytest.mark.parametrize('T,B,A', [(16, 6, 5), (101, 8, 18), (3, 4, 3)])
def test_host_bodies_with_abandoned_match_float64(emu, rule, param, T, B, A):
  q, qt, act, rew, done, ab, w = R.r2d2_inputs(T, B, A, seed=T + B)
  got = run_emu(emu, rule, param, q, qt, act, rew, done, ab, w)
  ref = R.r2d2_loss(q, qt, act, rew, done, ab, 0.997, rule, param, weights=w)
  for k in ('loss', 'priorities', 'dq'):
    scale = max(np.abs(ref[k]).max(), 1e-30)
    assert np.abs(got[k] - ref[k]).max() <= 1e-4 * scale, (k, np.abs(got[k] - ref[k]).max(), scale)
  masked = np.zeros((T, B), bool)
  masked[:-1] = ab[1:]
  assert np.all(got['dq'][masked] == 0)


@pytest.mark.parametrize('rule,param', RUNS)
def test_host_bodies_bit_identical_without_abandonment(emu, rule, param):
  T, B, A = 40, 6, 7
  q, qt, act, rew, done, ab, w = R.r2d2_inputs(T, B, A, seed=5)
  base = run_emu(emu, rule, param, q, qt, act, rew, done, None, w)
  zero = run_emu(emu, rule, param, q, qt, act, rew, done, np.zeros((T, B), bool), w)
  for k in base:
    np.testing.assert_array_equal(base[k].view(np.uint32), zero[k].view(np.uint32))
  assert not np.array_equal(run_emu(emu, rule, param, q, qt, act, rew, done, ab, w)['loss'], base['loss'])


# ---- settings and flags ------------------------------------------------------------------------------------------
def test_settings_default_off():
  from seed_rl_b200.agents.r2d2 import learner as r2d2_learner
  from seed_rl_b200.agents.vtrace import learner as vtrace_learner
  assert vtrace_learner.default_loss_settings().bootstrap_abandoned is False
  old = vtrace_learner.LossSettings(.99, 1., .5, 0.00025, 0., 0., None, 10., False, 1e-2)   # the fields of before
  assert old.bootstrap_abandoned is False
  assert vtrace_learner.default_loss_settings(bootstrap_abandoned=True).bootstrap_abandoned is True
  assert r2d2_learner.default_settings().bootstrap_abandoned is False
  fields = r2d2_learner.R2D2Settings._fields
  old = r2d2_learner.R2D2Settings(*[r2d2_learner.default_settings()._asdict()[k] for k in fields[:-1]])
  assert fields[-1] == 'bootstrap_abandoned' and old.bootstrap_abandoned is False


def test_flag_parses():
  from absl import flags
  from seed_rl_b200.agents.r2d2 import learner as r2d2_learner  # noqa: F401
  from seed_rl_b200.agents.vtrace import learner as vtrace_learner  # noqa: F401
  fl = flags.FLAGS['bootstrap_abandoned']
  assert fl.default is False
  fv = flags.FlagValues()
  fv[fl.name] = fl
  fv(['learner', '--bootstrap_abandoned'])
  assert fv.bootstrap_abandoned is True
  fv(['learner', '--nobootstrap_abandoned'])
  assert fv.bootstrap_abandoned is False
  fl.unparse()
