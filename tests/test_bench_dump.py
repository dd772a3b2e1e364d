"""bench.py --dump-outputs: what the last timed step computed, as .npy files, for comparing two
builds output for output."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import bench

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dump_outputs_writes_float32_or_float64(tmp_path):
  out = str(tmp_path / 'd')
  bench.dump_outputs(out, {'idx': torch.arange(5, dtype=torch.int64), 'f64': np.linspace(0, 1, 3),
                           'loss': torch.tensor(1.5)})
  assert sorted(os.listdir(out)) == ['f64.npy', 'idx.npy', 'loss.npy']
  idx, f64, loss = (np.load(os.path.join(out, n + '.npy')) for n in ('idx', 'f64', 'loss'))
  assert idx.dtype == np.float32 and idx.tolist() == [0, 1, 2, 3, 4]
  assert f64.dtype == np.float64 and f64.tolist() == [0.0, 0.5, 1.0]
  assert loss.dtype == np.float32 and loss.shape == () and float(loss) == 1.5


def test_dump_outputs_over_the_limit_writes_nothing(tmp_path):
  out = str(tmp_path / 'd')
  small = np.zeros(4, np.float32)
  big = np.zeros(bench.DUMP_LIMIT_BYTES // 4, np.float32)       # with `small` one float over the limit
  with pytest.raises(SystemExit):
    bench.dump_outputs(out, {'small': small, 'big': big})
  assert not os.path.exists(out)


def test_dump_outputs_refused_for_the_reference_arm(tmp_path):
  out = str(tmp_path / 'd')
  p = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--impl', 'reference', '--steps', '1',
                      '--dump-outputs', out], capture_output=True, text=True, timeout=120)
  assert p.returncode != 0 and '--dump-outputs' in p.stderr
  assert not os.path.exists(out)


@pytest.mark.gpu
def test_bench_dump_outputs_are_reproducible(tmp_path):
  """Two runs with the same arguments time exactly --steps steps and dump identical outputs."""
  runs = []
  for k in range(2):
    out = str(tmp_path / ('d%d' % k))
    p = subprocess.run([sys.executable, os.path.join(ROOT, 'bench.py'), '--gpus', '1', '--steps', '3',
                        '--warmup', '1', '--no-extras', '--dump-outputs', out],
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stderr[-2000:]
    assert json.loads(p.stdout.strip().splitlines()[-1])['steps'] == 3
    runs.append({n: np.load(os.path.join(out, n)) for n in sorted(os.listdir(out))})
  assert sorted(runs[0]) == ['gradients.npy', 'loss.npy', 'loss_terms.npy', 'parameters.npy']
  for n, a in runs[0].items():
    assert a.dtype == np.float32 and np.isfinite(a).all(), n
    assert np.array_equal(a, runs[1][n]), n
