"""CPU: the opt-in Retrace(lambda) targets of the R2D2 learner (not in the reference).

  * tests/retrace_oracle.py (float64, the explicit sum) against the UNMODIFIED reference
    n_step_bellman_target (tests/golden/r2d2_retrace_golden.npz) in its two reductions: lambda = 0 is
    n_steps = 1; lambda = 1 with every replayed action greedy is n_steps >= T - 1.  Done flags inside
    the sequences, T = 2 to 101.
  * A hand-computed T = 4 case in which an off-policy action cuts the trace.
  * r2d2_retrace_loss_thread (seed_rl_b200/csrc/r2d2_thread.inl, the body the GPU kernel runs) compiled
    as host C++ against the oracle and the float64 bars: loss, priorities, dq, with ties in the argmax.
  * Validation of the flags, the Python arguments and the C entry point (no launch is reached).
"""
import ctypes
import math
import os
import subprocess

import numpy as np
import pytest

import retrace_oracle as RO
import test_gpu_r2d2_loss_float64 as LF
from oracle import r2d2_oracle as R

HERE = os.path.dirname(os.path.abspath(__file__))
P = ctypes.c_void_p
ptr = lambda a: a.ctypes.data_as(P)
f = ctypes.c_float


@pytest.fixture(scope='module')
def gold():
  return np.load(os.path.join(HERE, 'golden', 'r2d2_retrace_golden.npz'))


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('emu') / '_r2d2_retrace_host.so')
  subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', so,
                         os.path.join(HERE, 'host_emulation', 'r2d2_retrace_host.cpp')])
  return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def emu_nstep(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('emu_nstep') / '_r2d2_host.so')
  subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', so,
                         os.path.join(HERE, 'host_emulation', 'r2d2_host.cpp')])
  return ctypes.CDLL(so)


def _golden_case(gold, name):
  r, d, q = gold[name + '_in']
  n, gamma = gold[name + '_cfg']
  return r, d > 0, q, int(n), float(gamma), gold[name + '_out']


@pytest.mark.parametrize('name', ['l0_a', 'l0_b', 'l0_c', 'l0_d'])
def test_lambda0_is_reference_one_step_target(gold, name):
  r, d, q, n, gamma, want = _golden_case(gold, name)
  assert n == 1 and (r.shape[0] == 2 or d[1:-1].any())     # episode ends inside the sequences
  # with lambda = 0 neither the replayed action's value nor greediness may matter
  rng = np.random.default_rng(0)
  q_act = rng.normal(size=q.shape) * 10
  greedy = rng.random(q.shape) < 0.5
  y = RO.retrace_targets(r, d, q, q_act, greedy, gamma, 0.0)
  np.testing.assert_allclose(y[1:], want[1:], rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize('name', ['l1_a', 'l1_b', 'l1_c', 'l1_d', 'l1_e'])
def test_lambda1_greedy_is_reference_long_n_step_target(gold, name):
  r, d, q, n, gamma, want = _golden_case(gold, name)
  T = r.shape[0]
  assert n >= T - 1 and (T == 2 or d[1:-1].any())
  y = RO.retrace_targets(r, d, q, q, np.ones(q.shape, bool), gamma, 1.0)
  np.testing.assert_allclose(y[1:], want[1:], rtol=2e-6, atol=2e-5 * max(1., np.abs(want).max()))


def test_hand_computed_T4_trace_cut():
  """gamma 0.9, lambda 0.5, r = (0, 1, 2, 3), q* = (10, 20, 30, 40).
  Column 0: the action at row 2 is off-policy (qa = 7), so c_2 = 0 and the trace stops there:
    Y3 = 3 + .9*40 = 39;  Y2 = 2 + .9*30 = 29;  Y1 = 1 + .9*(20 + .5*(29 - 20)) = 23.05;
    Y0 = .9*(10 + .5*(23.05 - 10)) = 14.8725.
  Column 1: all greedy, episode ends into row 2 (done_2 = 1, g_2 = 0):
    Y3 = 39;  Y2 = 2;  Y1 = 1 + .9*(20 + .5*(2 - 20)) = 10.9;  Y0 = .9*(10 + .5*(10.9 - 10)) = 9.405."""
  r = np.array([[0., 0.], [1., 1.], [2., 2.], [3., 3.]])
  qs = np.array([[10., 10.], [20., 20.], [30., 30.], [40., 40.]])
  qa = np.array([[10., 10.], [20., 20.], [7., 30.], [40., 40.]])
  greedy = np.array([[1, 1], [1, 1], [0, 1], [1, 1]], bool)
  done = np.array([[0, 0], [0, 0], [0, 1], [0, 0]], bool)
  y = RO.retrace_targets(r, done, qs, qa, greedy, 0.9, 0.5)
  np.testing.assert_allclose(y[:, 0], [14.8725, 23.05, 29., 39.], rtol=1e-12)
  np.testing.assert_allclose(y[:, 1], [9.405, 10.9, 2., 39.], rtol=1e-12)
  # nothing after the cut reaches the rows before it
  r2 = r.copy(); r2[3] += 100.
  y2 = RO.retrace_targets(r2, done, qs, qa, greedy, 0.9, 0.5)
  np.testing.assert_array_equal(y2[:3], y[:3])


def _inputs(T, B, A, seed, ties=False, p_greedy=0.7, q=1.0):
  """q: the scale of the Q values."""
  rng = np.random.default_rng(seed)
  tq = rng.normal(size=(T, B, A))
  if ties:                                          # few distinct values: many tied maxima
    tq = np.round(tq * 2) / 2
  tq = (tq * q).astype(np.float32)
  gq = (rng.normal(size=(T, B, A)) * 3 * q).astype(np.float32)
  greedy = tq.argmax(-1)
  ra = np.where(rng.random((T, B)) < p_greedy, greedy, rng.integers(0, A, (T, B))).astype(np.int64)
  if ties:                                          # a tied maximum that is not the first one is off-policy
    for t, b in zip(*np.nonzero((tq == tq.max(-1, keepdims=True)).sum(-1) > 1)):
      ra[t, b] = np.nonzero(tq[t, b] == tq[t, b].max())[0][-1]
  r = rng.normal(size=(T, B)).astype(np.float32)
  d = rng.random((T, B)) < 0.1
  w = (rng.random(B) + 0.1).astype(np.float32)
  return tq, gq, ra, r, d, w


def _run_emu(emu, tq, gq, ra, r, d, w, gamma, lam, eta, eps):
  T, B, A = tq.shape
  loss = np.zeros(B, np.float32); prio = np.zeros(B, np.float32); dq = np.full((T, B, A), 9, np.float32)
  scratch = np.zeros((T, B), np.float32)
  assert emu.emu_r2d2_retrace_loss(T, B, A, ptr(tq), ptr(gq), ptr(ra), ptr(r), ptr(d.astype(np.uint8)), ptr(w),
                                   f(gamma), f(lam), f(eta), f(eps), ptr(loss), ptr(prio), ptr(dq), ptr(scratch)) == 0
  return loss, prio, dq


@pytest.mark.parametrize('q', [1.0, 1e-3])
@pytest.mark.parametrize('lam', [0.0, 0.95, 1.0])
@pytest.mark.parametrize('T,B,A,ties', [(16, 6, 18, False), (101, 8, 18, False), (4, 2, 3, False), (2, 3, 4, False),
                                        (20, 6, 4, True)])
def test_retrace_thread_body_vs_float64(emu, T, B, A, ties, lam, q):
  """r2d2_retrace_loss_thread against the float64 oracle (the explicit sum, h and h^-1 without cancellation) and
  within the per-sequence float64 bars of test_gpu_r2d2_loss_float64.py, at Q values of scale 1 and 1e-3."""
  tq, gq, ra, r, d, w = _inputs(T, B, A, seed=T + A, ties=ties, q=q)
  if ties:
    assert ((tq == tq.max(-1, keepdims=True)).sum(-1) > 1).any()
  gamma, eta, eps = 0.997, 0.9, 1e-3
  loss, prio, dq = _run_emu(emu, tq, gq, ra, r, d, w, gamma, lam, eta, eps)
  want_loss, want_prio, _, want_dq = RO.loss_and_priorities(tq, gq, ra, r, d, gamma, lam, eta, eps, w)
  np.testing.assert_allclose(loss, want_loss, rtol=2e-5, atol=1e-6 * q)
  np.testing.assert_allclose(prio, want_prio, rtol=2e-5, atol=1e-6 * q)
  np.testing.assert_allclose(dq, want_dq, rtol=2e-4, atol=1e-7 * q)
  LF.check_outputs(dict(loss=loss, priorities=prio, dq=dq), (tq, gq, ra, r, d, w), 'retrace', lam, gamma, eta, eps)


def test_retrace_thread_body_lambda0_is_nstep_body_n1(emu, emu_nstep):
  """lambda = 0: the same fp32 operations, in the same order, as the n-step body at n_steps = 1."""
  tq, gq, ra, r, d, w = _inputs(101, 8, 18, seed=3)
  loss, prio, dq = _run_emu(emu, tq, gq, ra, r, d, w, 0.997, 0.0, 0.9, 1e-3)
  T, B, A = tq.shape
  l1 = np.zeros(B, np.float32); p1 = np.zeros(B, np.float32); dq1 = np.zeros_like(tq)
  scratch = np.zeros((B, T + 1), np.float32)
  assert emu_nstep.emu_r2d2_loss(T, B, A, ptr(tq), ptr(gq), ptr(ra), ptr(r), ptr(d.astype(np.uint8)), ptr(w),
                                 f(0.997), 1, f(0.9), f(1e-3), ptr(l1), ptr(p1), ptr(dq1), ptr(scratch)) == 0
  np.testing.assert_array_equal(loss, l1)
  np.testing.assert_array_equal(prio, p1)
  np.testing.assert_array_equal(dq, dq1)
  # and the oracle's lambda = 0 loss is the reference restatement's 1-step loss
  want_loss, want_prio, _ = R.loss_and_priorities(tq, tq.argmax(-1), gq, ra, r, d, 0.997, n_steps=1)
  got_loss, got_prio, _, _ = RO.loss_and_priorities(tq, gq, ra, r, d, 0.997, 0.0)
  np.testing.assert_allclose(got_loss, want_loss, rtol=2e-5)
  np.testing.assert_allclose(got_prio, want_prio, rtol=2e-5)


def test_flags_and_settings():
  from absl import flags
  from seed_rl_b200.agents.r2d2 import learner
  assert flags.FLAGS['bellman_target'].default == 'n_step'
  assert flags.FLAGS['retrace_lambda'].default == 0.95
  s = learner.default_settings()
  assert (s.bellman_target, s.retrace_lambda) == ('n_step', 0.95)
  assert 'bellman_target' in learner.R2D2Settings._fields and 'retrace_lambda' in learner.R2D2Settings._fields
  assert learner.default_settings(bellman_target='retrace', retrace_lambda=0.5).bellman_target == 'retrace'


@pytest.mark.parametrize('kind,lam', [('retrce', 0.95), ('', 0.95), (None, 0.95), ('retrace', -0.01), ('retrace', 1.5),
                                      ('retrace', math.nan)])
def test_bad_target_arguments_raise(kind, lam):
  from seed_rl_b200.agents.r2d2 import learner, learner_loop
  with pytest.raises(ValueError):
    learner.check_bellman_target(kind, lam)
  # every entry point refuses them before it touches a tensor or the device
  with pytest.raises(ValueError):
    learner.compute_loss_and_priorities_from_agent_outputs(None, None, None, None, 0.997, bellman_target=kind,
                                                           retrace_lambda=lam)
  with pytest.raises(ValueError):
    learner.compute_loss_and_priorities(None, None, None, None, None, None, 0.997, 40, bellman_target=kind,
                                        retrace_lambda=lam)
  bad = learner.default_settings(bellman_target=kind, retrace_lambda=lam)
  with pytest.raises(ValueError):
    learner.R2D2LearnerStep(None, None, None, settings=bad)
  with pytest.raises(ValueError):
    learner_loop.R2D2InferenceHost(None, 4, 1, 2, (4, 4, 1), settings=bad)


def test_n_step_ignores_retrace_lambda():
  from seed_rl_b200.agents.r2d2 import learner
  learner.check_bellman_target('n_step', 7.0)
  learner.check_bellman_target('retrace', 0.0)
  learner.check_bellman_target('retrace', 1.0)


def test_c_entry_point_refuses_bad_arguments():
  from seed_rl_b200 import _lib
  L = _lib.lib()
  T, B, A = 4, 2, 3
  bufs = [np.zeros(n, np.float32) for n in (T * B * A, T * B * A, 2 * T * B, T * B, T * B, B, B, B, T * B * A, T * B)]
  p = [ptr(x) for x in bufs]
  args = lambda T=T, lam=0.5, **null: [T, B, A] + [None if i in null.get('nulls', ()) else p[i] for i in range(6)] + \
      [0.997, lam, 0.9, 1e-3] + [None if i in null.get('nulls', ()) else p[i] for i in range(6, 10)] + [None]
  for a in (args(T=1), args(T=0), args(lam=-0.5), args(lam=1.01), args(lam=math.nan), args(lam=math.inf),
            args(nulls=(0,)), args(nulls=(2,)), args(nulls=(4,)), args(nulls=(7,)), args(nulls=(9,))):
    assert L.seedrl_r2d2_retrace_loss_fwd_bwd(*a) == 3, a
  assert L.seedrl_r2d2_retrace_loss_scratch_bytes(101, 64) == 101 * 64 * 4


def test_cpu_learner_oracle_lambda0_is_n_step_1(monkeypatch):
  """The oracle learner's retrace rule at lambda = 0 is its n-step rule at n_steps = 1, gradients included.  The
  retrace rule takes h^-1 in float64; the n-step rule (oracle/r2d2_learner_oracle.py) takes the reference's float32
  formula, whose cancellation alone moves these priorities by 2e-5, so here it is given the float64 h^-1 too."""
  from oracle import r2d2_learner_oracle as RL
  monkeypatch.setattr(R, 'inverse_value_function_rescaling',
                      lambda x, eps=1e-3: RO.inverse_value_function_rescaling(x, eps).astype(np.float32))
  A, obs, S = 4, (36, 36, 1), 4
  b = RL.synthetic_replay_batch(9, 3, A, obs, seed=2, done_p=0.2)
  got = RO.CpuR2D2Learner(A, obs, S, burn_in=3, n_steps=1, bellman_target='retrace', retrace_lambda=0.0).grads(b)
  want = RO.CpuR2D2Learner(A, obs, S, burn_in=3, n_steps=1).grads(b)
  np.testing.assert_allclose(got[0], want[0], rtol=1e-5)
  np.testing.assert_allclose(got[2], want[2], rtol=1e-5)
  for k in want[3]:
    np.testing.assert_allclose(got[3][k], want[3][k], rtol=1e-4, atol=1e-6 * np.abs(want[3][k]).max(), err_msg=k)
