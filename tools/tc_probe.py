"""Bring-up probe for the wgmma kernels: one launch per case, error vs the CPU oracle
printed per case; each case runs in a fresh subprocess so a faulting case cannot poison the
others.  Usage: python tools/tc_probe.py [case_index]"""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

CASES = [  # kind, cin, cout, mode, N, H, W, flip
    ('conv', 32, 32, 0, 3, 21, 21, 0), ('conv', 16, 16, 1, 5, 42, 42, 0), ('conv', 32, 16, 0, 2, 42, 42, 1),
    ('wgrad', 32, 32, 1, 3, 21, 21, 0), ('wgrad', 32, 32, 0, 40, 11, 11, 0), ('wgrad', 16, 16, 1, 5, 42, 42, 0),
    ('wgrad', 16, 32, 0, 2, 42, 42, 0), ('wgrad', 32, 32, 1, 700, 21, 21, 0), ('wgrad', 32, 32, 0, 1, 4, 4, 0)]


def one(i):
  import numpy as np
  import torch
  from test_gpu_zz_tc import _ref, _relerr, _run, _run_wgrad
  from oracle import net_oracle
  kind, cin, cout, mode, N, H, W, flip = CASES[i]
  rng = np.random.default_rng(0)
  x = rng.normal(size=(N, H, W, cin)).astype(np.float32)
  if kind == 'wgrad':
    dy = rng.normal(size=(N, H, W, cout)).astype(np.float32)
    xin = torch.relu(torch.as_tensor(x)) if mode == 1 else torch.as_tensor(x)
    wt = torch.zeros(3, 3, cin, cout, requires_grad=True); bt = torch.zeros(cout, requires_grad=True)
    (net_oracle._conv_nhwc(xin, wt, bt, 1, True) * torch.as_tensor(dy)).sum().backward()
    dw, db, err = _run_wgrad(cin, cout, mode, N, H, W, x, dy)
    print('CASE', i, CASES[i], 'dw relerr %.4g' % _relerr(dw, wt.grad.numpy()),
          'db relerr %.4g' % _relerr(db, bt.grad.numpy()), 'timeout_flag', err, 'nan', int(np.isnan(dw).sum()),
          'dw[0,0,0,:3]', dw[0, 0, 0, :3], 'want', wt.grad.numpy()[0, 0, 0, :3], flush=True)
    return
  if flip:
    w = (rng.normal(size=(3, 3, cout, cin)) * 0.2).astype(np.float32)   # source layout [tap][cout'][cin']
    xt = torch.tensor(np.zeros((N, H, W, cout), np.float32), requires_grad=True)
    y = net_oracle._conv_nhwc(xt, torch.as_tensor(w), None, 1, True)
    (y * torch.as_tensor(x)).sum().backward()
    want = xt.grad.numpy(); b = None
  else:
    w = (rng.normal(size=(3, 3, cin, cout)) * 0.2).astype(np.float32)
    b = rng.normal(size=(cout,)).astype(np.float32)
    want = _ref(x, w, b, mode).numpy()
  got, err = _run(cin, cout, mode, N, H, W, x, w, b, None, None, flip)
  print('CASE', i, CASES[i], 'relerr %.4g' % _relerr(got, want), 'timeout_flag', err, 'nan',
        int(np.isnan(got).sum()), flush=True)


if __name__ == '__main__':
  if len(sys.argv) > 1:
    one(int(sys.argv[1]))
  else:
    for i in range(len(CASES)):
      p = subprocess.run([sys.executable, __file__, str(i)], capture_output=True, text=True,
                         env=dict(os.environ, CUDA_LAUNCH_BLOCKING='1'), timeout=300)
      out = [l for l in p.stdout.splitlines() if l.startswith('CASE')]
      print(out[0] if out else 'CASE %d %s FAILED rc=%d: %s' % (
          i, CASES[i], p.returncode, (p.stderr.strip().splitlines() or ['?'])[-1][:300]), flush=True)
