"""CPU: the entry points behind the R2D2 CUDA-graph inference path (device epsilon-greedy and the
eval-aware store append) reject bad arguments with SEEDRL_ERR_INVALID_ARGUMENT, without launching."""
import ctypes

from seed_rl_b200 import _lib

INVALID = 3
FAKE = ctypes.c_void_p(256)      # never dereferenced: every call below fails its argument check first


def test_epsilon_greedy_rejects_null_pointers_and_bad_sizes():
  L = _lib.lib()
  ok = (FAKE, FAKE, 7, FAKE, FAKE, None)
  assert L.seedrl_r2d2_epsilon_greedy(4, 0, *ok) == INVALID                       # A < 1
  assert b'A >= 1' in L.seedrl_last_error()
  assert L.seedrl_r2d2_epsilon_greedy(-1, 6, *ok) == INVALID                      # N < 0
  for k in (0, 1, 3, 4):                                                          # each pointer null
    args = list(ok)
    args[k] = None
    assert L.seedrl_r2d2_epsilon_greedy(4, 6, *args) == INVALID, k
    assert b'null pointer' in L.seedrl_last_error()


def test_rows_multi_limit_rejects_null_pointers_and_bad_sizes():
  L = _lib.lib()
  jobs = (_lib.RowJob * 17)(*[_lib.RowJob(256, 256, 4, _lib.ROW_APPEND, 8) for _ in range(17)])
  assert L.seedrl_rows_multi_limit(None, 1, FAKE, 4, FAKE, 10, None) == INVALID
  assert L.seedrl_rows_multi_limit(jobs, 1, None, 4, FAKE, 10, None) == INVALID
  assert L.seedrl_rows_multi_limit(jobs, 17, FAKE, 4, FAKE, 10, None) == INVALID   # > SEEDRL_MAX_ROW_JOBS
  assert L.seedrl_rows_multi_limit(jobs, 1, FAKE, -1, FAKE, 10, None) == INVALID
  assert L.seedrl_rows_multi_limit(jobs, 1, FAKE, 4, FAKE, -1, None) == INVALID    # id_limit < 0
  assert L.seedrl_rows_multi_limit(jobs, 1, FAKE, 4, None, 10, None) == INVALID    # append job without index
  assert b'append job needs index' in L.seedrl_last_error()


def test_store_advance_limit_rejects_null_pointers_and_bad_sizes():
  L = _lib.lib()
  ok = [FAKE, FAKE, 4, 10, FAKE, FAKE, 5, None]
  for k in (0, 1, 4, 5):
    args = list(ok)
    args[k] = None
    assert L.seedrl_store_advance_limit(*args) == INVALID, k
  args = list(ok)
  args[2] = -1
  assert L.seedrl_store_advance_limit(*args) == INVALID
  args = list(ok)
  args[6] = -1
  assert L.seedrl_store_advance_limit(*args) == INVALID
