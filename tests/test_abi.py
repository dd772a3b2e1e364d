"""CPU: the C-ABI shared library loads and exports every symbol include/seedrl_b200.h
declares; host-side logic (batcher, queues, config validation) that needs no GPU."""
import ctypes
import os
import re
import threading
import types

import numpy as np
import pytest
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.common import utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
  hdr = open(os.path.join(ROOT, 'include', 'seedrl_b200.h')).read()
  hdr = re.sub(r'/\*.*?\*/', '', hdr, flags=re.S)
  declared = set(re.findall(r'\b(seedrl_[a-z0-9_]+)\s*\(', hdr))
  assert len(declared) >= 30
  lib = ctypes.CDLL(_lib.LIB_PATH)
  for name in declared:
    assert hasattr(lib, name), name
  assert declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
  assert _lib.lib().seedrl_abi_version() == 1


def test_argument_errors_are_reported_not_crashed():
  L = _lib.lib()
  rc = L.seedrl_vtrace_from_importance_weights(4, 4, None, None, None, None, None, None,
                                               1.0, 1.0, 1.0, None, None, None)
  assert rc == 3
  assert b'null pointer' in L.seedrl_last_error()
  with pytest.raises(_lib.SeedrlError):
    _lib.check(rc)
  # the wgmma conv takes only the documented descriptor layout: any other `variant` is refused before
  # the weights are packed or the conv launched
  n0 = _lib.launch_count()
  for variant in (1, 2, 3):
    rc = L.seedrl_debug_conv3x3_tc(16, 16, 1, 0, 1, 8, 8, None, None, None, None, None, None, 0, variant,
                                   None, None, None)
    assert rc == 3
    assert b'variant' in L.seedrl_last_error()
  assert _lib.launch_count() == n0


def test_net_param_table_matches_reference_variable_count():
  """reference tests/agents_test.py:45: ImpalaDeep has 39 trainable tensors."""
  L = _lib.lib()
  h = ctypes.c_void_p()
  cfg = _lib.NetConfig(_lib.NET_DEEP, 18, 84, 84, 4)
  _lib.check(L.seedrl_net_create(ctypes.byref(cfg), ctypes.byref(h)))
  assert L.seedrl_net_num_param_tensors(h) == 39
  assert L.seedrl_net_num_params(h) == 1638883
  from oracle import net_oracle
  specs = net_oracle.param_specs('deep', 18, (84, 84, 4))
  for i, (name, shape) in enumerate(specs):
    buf = ctypes.create_string_buffer(128); dims = (ctypes.c_int64 * 4)(); off = ctypes.c_size_t()
    rank = L.seedrl_net_param_info(h, i, buf, 128, dims, ctypes.byref(off))
    assert buf.value.decode() == name
    assert tuple(dims[k] for k in range(rank)) == tuple(shape)
    assert off.value % 64 == 0
  assert L.seedrl_net_workspace_bytes(h, 21, 64) > 2 * 10**9
  L.seedrl_net_destroy(h)
  cfg = _lib.NetConfig(_lib.NET_SHALLOW, 18, 84, 84, 4)
  _lib.check(L.seedrl_net_create(ctypes.byref(cfg), ctypes.byref(h)))
  assert L.seedrl_net_num_param_tensors(h) == 13
  assert L.seedrl_net_num_params(h) == sum(
      int(np.prod(s)) for _, s in net_oracle.param_specs('shallow', 18, (84, 84, 4)))
  L.seedrl_net_destroy(h)


# ---- batcher (grpc/python/ops_test.py batching semantics) ---------------------------
class Batcher(object):
  def __init__(self, n, in_rows, out_rows, slabs=2):
    L = _lib.lib()
    self.L = L
    self.h = ctypes.c_void_p()
    a = (ctypes.c_size_t * len(in_rows))(*in_rows)
    b = (ctypes.c_size_t * len(out_rows))(*out_rows)
    _lib.check(L.seedrl_batcher_create(n, slabs, len(in_rows), a, len(out_rows), b, 0,
                                       ctypes.byref(self.h)))

  def call(self, values):
    """One client call contributing len(values) int32 rows; returns its outputs."""
    L, k = self.L, len(values)
    slab, row = ctypes.c_int(), ctypes.c_int()
    _lib.check(L.seedrl_batcher_claim(self.h, k, ctypes.byref(slab), ctypes.byref(row)))
    src = np.asarray(values, np.int32)
    ctypes.memmove(L.seedrl_batcher_input_ptr(self.h, slab, 0, row), src.ctypes.data, 4 * k)
    _lib.check(L.seedrl_batcher_commit(self.h, slab, k))
    st = ctypes.c_int()
    rc = L.seedrl_batcher_wait_outputs(self.h, slab, ctypes.byref(st))
    if rc != 0:
      L.seedrl_batcher_release(self.h, slab)
      _lib.check(rc)
    out = np.empty(k, np.int32)
    ctypes.memmove(out.ctypes.data, L.seedrl_batcher_output_ptr(self.h, slab, 0, row), 4 * k)
    L.seedrl_batcher_release(self.h, slab)
    return out, st.value

  def serve(self, n, fn, count):
    L = self.L
    for _ in range(count):
      slab = ctypes.c_int()
      rc = L.seedrl_batcher_next_full(self.h, -1, ctypes.byref(slab))
      if rc != 0:
        return
      x = np.ctypeslib.as_array(
          ctypes.cast(L.seedrl_batcher_input_ptr(self.h, slab, 0, 0), ctypes.POINTER(ctypes.c_int32)), (n,))
      y = np.ctypeslib.as_array(
          ctypes.cast(L.seedrl_batcher_output_ptr(self.h, slab, 0, 0), ctypes.POINTER(ctypes.c_int32)), (n,))
      y[:] = fn(x)
      L.seedrl_batcher_publish(self.h, slab, 0)


def test_batcher_stress_10_clients_100_calls_batch_5():
  """reference grpc/python/ops_test.py:632-664."""
  b = Batcher(5, [4], [4], slabs=3)
  server = threading.Thread(target=b.serve, args=(5, lambda x: x + 1, 10**9))
  server.start()
  errs, finished = [], []

  def client(cid):
    try:
      for i in range(100):
        out, st = b.call([cid * 1000 + i])
        if out[0] != cid * 1000 + i + 1 or st != 0:
          errs.append((cid, i, out))
      finished.append(cid)
    except _lib.SeedrlError as e:      # cancelled by the shutdown below
      if e.code != 1:
        errs.append((cid, str(e)))
  ts = [threading.Thread(target=client, args=(c,)) for c in range(10)]
  [t.start() for t in ts]
  import time
  deadline = time.time() + 60
  # Like the reference test: shut down once more than half the clients completed -- the
  # last batch may never fill up (a partially filled batch blocks forever).
  while len(finished) <= 5 and time.time() < deadline:
    time.sleep(0.01)
  b.L.seedrl_batcher_shutdown(b.h)
  [t.join(30) for t in ts]
  server.join(30)
  assert not errs and len(finished) > 5
  assert not any(t.is_alive() for t in ts) and not server.is_alive()


def test_batcher_prebatched_slices_2_plus_2():
  """reference grpc/python/ops_test.py:776-799: [2]+[2] -> one [4] batch."""
  b = Batcher(4, [4], [4])
  seen = []

  def fn(x):
    seen.append(x.copy())
    return x * 2
  server = threading.Thread(target=b.serve, args=(4, fn, 1))
  server.start()
  res = {}
  ts = [threading.Thread(target=lambda v=v: res.__setitem__(v[0], b.call(v)[0]))
        for v in ([1, 2], [3, 4])]
  [t.start() for t in ts]; [t.join() for t in ts]; server.join()
  assert len(seen) == 1 and sorted(seen[0].tolist()) == [1, 2, 3, 4]
  assert res[1].tolist() == [2, 4] and res[3].tolist() == [6, 8]
  b.L.seedrl_batcher_destroy(b.h)


def test_batcher_too_many_rows_and_shutdown_cancels_waiters():
  """overflow: grpc.cc:653 ; shutdown: grpc.cc:771-787 / ops_test.py:384-501."""
  b = Batcher(4, [4], [4])
  slab, row = ctypes.c_int(), ctypes.c_int()
  assert b.L.seedrl_batcher_claim(b.h, 5, ctypes.byref(slab), ctypes.byref(row)) == 11
  got = []

  def waiter():
    try:
      b.call([7])
    except _lib.SeedrlError as e:
      got.append(e)
  t = threading.Thread(target=waiter); t.start()
  import time; time.sleep(0.2)
  b.L.seedrl_batcher_shutdown(b.h)
  t.join(5)
  assert got and got[0].code == 1 and 'Server shutdown.' in str(got[0])


# ---- host logic in common/utils ------------------------------------------------------
def test_validate_learner_config():
  """reference common/utils.py:989-1002."""
  c = types.SimpleNamespace(num_envs=256, env_batch_size=4, inference_batch_size=-1)
  utils.validate_learner_config(c)
  assert c.inference_batch_size == 128
  c = types.SimpleNamespace(num_envs=4, env_batch_size=3, inference_batch_size=4)
  with pytest.raises(AssertionError):
    utils.validate_learner_config(c)


def test_batch_apply_and_make_time_major():
  """reference tests/utils_test.py:291-301, 587-606."""
  a = torch.tensor([[[0, 1], [2, 3]], [[4, 5], [6, 7]]])
  b = torch.tensor([[[8, 9], [10, 11]], [[12, 13], [14, 15]]])
  s, m = utils.batch_apply(lambda x, y: (x.sum(-1), y.max(-1).values), (a, b))
  assert s.tolist() == [[1, 5], [9, 13]] and m.tolist() == [[9, 11], [13, 15]]
  x = torch.arange(6).reshape(2, 3)
  assert utils.make_time_major(x).tolist() == [[0, 3], [1, 4], [2, 5]]
  assert utils.make_time_major((torch.arange(3),))[0].tolist() == [0, 1, 2]


def test_structured_fifo_queue_capacity_and_close():
  specs = (utils.TensorSpec([], 'int32', 'a'), utils.TensorSpec([2], 'float32', 'b'))
  q = utils.StructuredFIFOQueue(1, specs)
  q.enqueue((torch.tensor(1), torch.zeros(2)))
  blocked = []
  t = threading.Thread(target=lambda: (q.enqueue((torch.tensor(2), torch.ones(2))), blocked.append(1)))
  t.start()
  import time; time.sleep(0.1)
  assert not blocked and q.size() == 1          # capacity-1 back-pressure (learner.py:336)
  assert int(q.dequeue()[0]) == 1
  t.join(2); assert blocked
  q.enqueue_many  # exists
  assert int(q.dequeue()[0]) == 2
  q.close()
  with pytest.raises(utils.QueueClosedError):
    q.dequeue()


def test_conv_position_maps_on_host():
  """The conv kernels' tall-image geometry (N images stacked with one shared zero row between
  them, one zero column each side; positions flattened) and its multiply-high division,
  evaluated on the host through the C-ABI against a straightforward numpy statement."""
  import ctypes
  import numpy as np
  from seed_rl_b200 import _lib
  L = _lib.lib()
  for N, H, W in [(3, 84, 84), (5, 42, 42), (7, 21, 21), (9, 11, 11), (4, 9, 7), (2, 5, 3), (3, 1, 1),
                  (1344, 84, 84), (2, 126, 126)]:
    PW, RH = W + 2, H + 1
    Q = N * RH * PW
    for which in (0, 1):
      starts = [0] if Q < 400000 else [0, Q // 2 - 1000, Q - 100000]
      for start in starts:
        count = min(Q + 3 * PW - start, 200000)
        out = np.empty(count, np.int32)
        _lib.check(L.seedrl_debug_conv_pixels(N, H, W, which, start, count, out.ctypes.data_as(ctypes.c_void_p)))
        p = np.arange(start, start + count, dtype=np.int64)
        R, c = p // PW, p % PW
        n, r = R // RH, R % RH
        if which == 0:
          ok = (r != 0) & (c != 0) & (c <= W) & (n < N)
          want = np.where(ok, (n * H + (r - 1)) * W + (c - 1), -1)
        else:
          ok = (r < H) & (c < W) & (n < N)
          want = np.where(ok, (n * H + r) * W + c, -1)
        np.testing.assert_array_equal(out, want)


def test_batcher_native_thread_stress(tmp_path):
  """Native threads lap the slab ring while one caller sits between claim and commit
  (tests/host_emulation/batcher_stress.cc).  Regression test: seedrl_batcher_claim reported a
  spurious 'would straddle two batches' for a fully claimed, not yet fully committed slab,
  which killed callers (1 run in ~40 of the Python stress test above stalled)."""
  import subprocess
  exe = str(tmp_path / 'batcher_stress')
  libdir = os.path.join(ROOT, 'seed_rl_b200')
  subprocess.check_call(['g++', '-O2', '-std=c++17', '-o', exe,
                         os.path.join(ROOT, 'tests', 'host_emulation', 'batcher_stress.cc'),
                         '-L' + libdir, '-lseedrl_b200', '-Wl,-rpath,' + libdir, '-lpthread'])
  r = subprocess.run([exe, '300'], capture_output=True, text=True, timeout=300)
  assert r.returncode == 0, r.stdout + r.stderr
  assert r.stdout.strip() == 'stalls=0 bad=0 claim_errors=0'
