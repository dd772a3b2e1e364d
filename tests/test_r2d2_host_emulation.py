"""CPU: the per-thread bodies of the R2D2 CUDA kernels (seed_rl_b200/csrc/r2d2_thread.inl -- the
same source text the GPU executes) compiled as host C++ and run thread by thread against
oracle/r2d2_oracle.py (frame stacking) and float64 (the loss and the replay sampler).  This
validates the algorithm and indexing of those kernels where no GPU is present (their GPU parity
tests are tests/test_gpu_r2d2.py); it is a test harness, not a product path."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

from oracle import r2d2_oracle as R
import test_gpu_r2d2_loss_float64 as LF
import test_gpu_replay_clip_float64 as RC

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope='module')
def emu(tmp_path_factory):
  so = str(tmp_path_factory.mktemp('emu') / '_r2d2_host.so')
  subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-o', so,
                         os.path.join(HERE, 'host_emulation', 'r2d2_host.cpp')])
  return ctypes.CDLL(so)


P = ctypes.c_void_p
ptr = lambda a: a.ctypes.data_as(P)


@pytest.mark.parametrize('T,B,H,W,S', [(6, 2, 3, 4, 4), (9, 3, 5, 2, 3), (4, 1, 2, 2, 2), (25, 3, 7, 5, 4), (1, 2, 3, 3, 4),
                                       (0, 2, 2, 2, 4)])
def test_stack_frames_thread_body_bit_exact(emu, T, B, H, W, S):
  rng = np.random.default_rng(T * 7 + B)
  fr = rng.integers(0, 256, (T, B, H, W, 1), dtype=np.uint8)
  dn = (rng.random((T, B)) < 0.3)
  st = rng.integers(0, 1 << (8 * (S - 1)), (B, H * W)).astype(np.int32)
  out = np.full((T, B, H, W, S), 77, np.uint8); ns = np.zeros_like(st)
  assert emu.emu_stack_frames(T, B, H * W, S, ptr(fr), ptr(st), ptr(dn.astype(np.uint8)), ptr(out), ptr(ns)) == 0
  if T == 0:
    np.testing.assert_array_equal(ns, st)
    return
  want, want_state = R.stack_frames(fr.astype(np.float32), st, dn, S)
  np.testing.assert_array_equal(out, want.astype(np.uint8))
  np.testing.assert_array_equal(ns, want_state)


def test_stack_frames_thread_body_reference_sequence(emu):      # atari/networks_test.py:176-247
  def run(frames, state, done):
    fr = np.array(frames, np.uint8).reshape(len(frames), 1, 1, 1)
    dn = np.array(done, np.uint8).reshape(len(done), 1)
    out = np.zeros((len(frames), 1, 1, 4), np.uint8); ns = np.zeros_like(state)
    emu.emu_stack_frames(len(frames), 1, 1, 4, ptr(fr), ptr(state), ptr(dn), ptr(out), ptr(ns))
    return out.reshape(len(frames), 4), ns
  z = np.zeros((1, 1), np.int32)
  o, s = run([1], z, [0]); assert o.tolist() == [[1, 0, 0, 0]]
  o, s = run([2], s, [0]); assert o.tolist() == [[2, 1, 0, 0]]
  o, s = run([3, 4, 5, 6, 7, 8], s, [0] * 6); assert o[0].tolist() == [3, 2, 1, 0] and o[5].tolist() == [8, 7, 6, 5]
  o, s = run([1], z, [0]); o, s = run([2], s, [1]); assert o.tolist() == [[2, 0, 0, 0]]
  o, s = run([3, 4, 5, 6, 7, 8], s, [0, 0, 0, 0, 1, 0])
  assert o[0].tolist() == [3, 2, 0, 0] and o[5].tolist() == [8, 7, 0, 0]


@pytest.mark.parametrize('q', [1.0, 1e-3])
@pytest.mark.parametrize('T,B,A,n', [(16, 6, 18, 5), (101, 8, 18, 5), (4, 2, 3, 5), (12, 3, 4, 1), (2, 1, 2, 3)])
def test_loss_thread_body_vs_float64(emu, T, B, A, n, q):
  """r2d2_loss_thread against the float64 loss of test_gpu_r2d2_loss_float64.py, with its bars, at Q values of
  scale 1 and 1e-3: the raw n-step targets (the scratch array, scratch[b, :T] = targets before h), loss,
  priorities and dq.  Not against oracle/r2d2_oracle.py's float32 loss: its h^-1 cancels, the body's does not."""
  rng = np.random.default_rng(T + A)
  tq = (rng.normal(size=(T, B, A)) * q).astype(np.float32); gq = (rng.normal(size=(T, B, A)) * q).astype(np.float32)
  ra = rng.integers(0, A, (T, B)).astype(np.int64); r = rng.normal(size=(T, B)).astype(np.float32)
  d = rng.random((T, B)) < 0.1
  w = (rng.random(B) + 0.1).astype(np.float32)
  gamma, eta, eps = 0.997, 0.9, 1e-3
  loss = np.zeros(B, np.float32); prio = np.zeros(B, np.float32); dq = np.full((T, B, A), 9, np.float32)
  scratch = np.zeros((B, T + n), np.float32)
  f = ctypes.c_float
  assert emu.emu_r2d2_loss(T, B, A, ptr(tq), ptr(gq), ptr(ra), ptr(r), ptr(d.astype(np.uint8)), ptr(w), f(gamma), n,
                           f(eta), f(eps), ptr(loss), ptr(prio), ptr(dq), ptr(scratch)) == 0
  LF.check_outputs(dict(targets=scratch[:, :T].T, loss=loss, priorities=prio, dq=dq), (tq, gq, ra, r, d, w), 'n_step',
                   n, gamma, eta, eps)


def _emu_replay_sample(emu, prio, limit, alpha, beta, u):
  n = len(u)
  idx = np.zeros(n, np.int64); w = np.zeros(n, np.float32); probs = np.zeros(limit, np.float32)
  f = ctypes.c_float
  assert emu.emu_replay_sample(limit, ptr(prio), f(alpha), f(beta), n, ptr(u), ptr(idx), ptr(w), ptr(probs)) == 0
  return idx, w, probs


def test_replay_sample_phase_bodies(emu):                       # common/utils.py:327-352
  rng = np.random.default_rng(0)
  prio = (rng.random(100) + 0.01).astype(np.float32); limit = 70
  u = rng.random(4096).astype(np.float32)
  idx, w, probs = _emu_replay_sample(emu, prio, limit, 0.9, 0.6, u)
  p = R.replay_probabilities(prio, limit, 0.9)
  np.testing.assert_allclose(probs, p, rtol=2e-5)
  assert idx.min() >= 0 and idx.max() < limit and w.max() == 1.0
  RC.check_sample(prio, limit, 0.9, 0.6, u, idx, w, probs)     # weights and probs_out vs float64
  freq = np.bincount(idx, minlength=limit) / len(idx)
  assert np.abs(freq - p).max() < 0.02                         # statistical, like tests/utils_test.py:353-365
  # the draw is the inverse CDF of the given uniforms
  cdf = np.cumsum(np.power(prio[:limit], np.float32(0.9)).astype(np.float32), dtype=np.float32)
  want = np.minimum(np.searchsorted(cdf, u * cdf[-1], side='right'), limit - 1)
  assert (idx == want).mean() > 0.999                          # (equal up to fp32 prefix rounding at bin edges)


@pytest.mark.parametrize('kind', ['uniform', 'lognormal2', 'lognormal3', 'equal', 'spike', 'zeros'])
@pytest.mark.parametrize('limit', [100, 1000, 8192])
def test_replay_sample_phase_bodies_vs_float64(emu, limit, kind):
  """The replay sampler's bodies against float64 (the checks of test_gpu_replay_clip_float64.py): the
  weights of rare items with wide priority spreads, probs_out, and weights of exactly 1 for equal priorities."""
  prio = RC.priorities(kind, limit)
  u = np.concatenate([RC.PINNED, np.random.default_rng(limit).random(4093).astype(np.float32)])
  for alpha, beta in RC.EXPONENTS:
    idx, w, probs = _emu_replay_sample(emu, prio, limit, alpha, beta, u)
    RC.check_sample(prio, limit, alpha, beta, u, idx, w, probs)
  ug = RC.grid_uniforms()
  idx, _, _ = _emu_replay_sample(emu, prio, limit, 0.9, 0.6, ug)
  RC.check_grid(prio, limit, 0.9, idx)


@pytest.mark.parametrize('limit,kind', [(1000, 'lognormal2'), (1000, 'lognormal3'), (8192, 'lognormal2'),
                                        (8192, 'lognormal3')])
def test_replay_weight_bar_rejects_the_prefix_difference(emu, limit, kind):
  """The float64 weight bar is tight enough to see the error of p_i = (cdf[i] - cdf[i-1]) / total, the
  probability replay_sample_kernel does not use: at wide priority spreads it exceeds the bar."""
  prio = RC.priorities(kind, limit)
  u = np.random.default_rng(limit).random(4096).astype(np.float32)
  idx = np.zeros(len(u), np.int64); w = np.zeros(len(u), np.float32)
  f = ctypes.c_float
  assert emu.emu_replay_sample_prefix_only(limit, ptr(prio), f(0.9), f(0.6), len(u), ptr(u), ptr(idx), ptr(w)) == 0
  with pytest.raises(AssertionError, match='weights: error'):
    RC.check_sample(prio, limit, 0.9, 0.6, u, idx, w)
  mass_idx, mass_w, _ = _emu_replay_sample(emu, prio, limit, 0.9, 0.6, u)
  np.testing.assert_array_equal(mass_idx, idx)                 # the two forms draw the same items
  RC.check_sample(prio, limit, 0.9, 0.6, u, mass_idx, mass_w)
