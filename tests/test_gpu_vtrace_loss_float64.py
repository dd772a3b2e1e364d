"""The fused V-trace loss kernels (vtrace_loss_kernel and vtrace_loss_stream_kernel<9|18|19|0>) against the float64
loss of tests/vtrace_float64_reference.py, at the benchmarked batch sizes, every scan width of the stream kernel,
the compiled and run-time action counts, and the inputs a trained agent produces; then vtrace_kernel<5> and the
categorical log-prob / entropy kernel against float64.

Each case calls learner.vtrace_loss_fwd_bwd(..., want_vtrace=True) once per kernel setting that applies to it:
seedrl_debug_set_loss_stream(0) (vtrace_loss_kernel), 1 (the default choice) and 2 / 4 / 8 / 16 (the stream kernel
pinned to that many columns per tile).  torch.profiler's kernel names show that each launch ran the kernel and
template instantiation the case names, so a shape the stream kernel refuses cannot quietly test the other kernel.
Every launch is made twice and must repeat bit for bit.

Bars, per stage (the 11 logged terms and the total, vs, pg_advantages, dlogits, dbaseline, d_entropy_cost_param,
and dlogits row by row: the largest over rows of max|diff| / max|ref row|, since the rows of a peaked policy differ
in scale by orders of magnitude): error = max|gpu - ref64| / max|ref64| (relative difference for scalars),
bar = max(FLOOR, C x m), m = the same error of the float32 reference, the rule of test_gpu_vtrace_float64.py.  The
loss has no discrete decisions to share: the rho clips are kinks, not jumps.  The bootstrap row of dlogits and
dbaseline must be exactly zero.
"""
import collections
import re

import numpy as np
import pytest
import torch

import vtrace_float64_reference as RF

pytestmark = pytest.mark.gpu

C = 8
FLOOR = 1e-6
CHUNK = 8192                 # columns per reference evaluation (B = 65536 in float64 within host memory)
_worst = collections.OrderedDict()      # group -> (error / bar, case, stage), printed by the last test


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _lpc(T):
  """Lanes per column of the stream kernel's reverse scan (vtrace_loss_stream_kernel)."""
  lpc = 32
  while lpc > 1 and T <= lpc * 4:
    lpc >>= 1
  return lpc


def _stream_bytes(T, A, BB):
  """stream_smem_bytes of vtrace_kernels.cu."""
  rows = T * BB
  stride = (T * BB * A + 31) & ~31
  return (3 * stride + 9 * rows + (T + 1) * BB + rows + 32) * 4 + 3 * 8 + 128


def _stream_bbs(T, B, A):
  """The columns per tile pick_stream accepts when pinned (16-byte aligned inputs)."""
  if T > 256 or (B * A) % 4:
    return []
  out = []
  for BB in (2, 4, 8, 16):
    if B % BB or (BB * A) % 4 or BB * A > 256 or B // BB < _sms():
      continue
    if _stream_bytes(T, A, BB) > 227 * 1024 - 2048:
      continue
    rows = T * BB
    rounds = -(-rows // 1024)
    per_round = -(-rows // rounds)
    th = max(128, -(-per_round // 32) * 32)
    if (T + 1) * BB > 4 * th:
      continue
    out.append(BB)
  return out


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _rel(a, w):
  return abs(float(a) - float(w)) / max(abs(float(w)), 1e-30)


def _rowmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  a = a.reshape(-1, a.shape[-1]); w = w.reshape(-1, w.shape[-1])
  return float((np.abs(a - w).max(1) / (np.abs(w).max(1) + 1e-30)).max())


# ---- cases ----------------------------------------------------------------------------------------------------------
STREAM, SMALL = 'vtrace_loss_stream_kernel<%d>', 'vtrace_loss_kernel'
Case = collections.namedtuple('Case', 'group name T make modes')   # modes: {debug setting: expected kernel}


def _stream_name(A):
  return STREAM % (A if A in (9, 18, 19) else 0)


def _normal_inputs(T1, B, A, seed):
  rng = np.random.default_rng(seed)
  return dict(ll=rng.normal(size=(T1, B, A)).astype(np.float32), lb=rng.normal(size=(T1, B)).astype(np.float32),
              bl=rng.normal(size=(T1, B, A)).astype(np.float32), act=rng.integers(0, A, (T1, B)),
              rew=(rng.normal(size=(T1, B)) * 2).astype(np.float32), done=rng.random((T1, B)) < 0.1), rng


def _plain(T1, B, A, seed, **kw):
  return lambda: (_normal_inputs(T1, B, A, seed)[0], kw)


def _bench(B):
  """bench.py's roofline_vtrace_loss inputs at batch B (T1 = 21, A = 18), built the same way on the GPU."""
  def make():
    T1, A = 21, 18
    g = torch.Generator(device='cuda').manual_seed(0)
    ll = torch.randn(T1, B, A, device='cuda', generator=g); lb = torch.randn(T1, B, device='cuda', generator=g)
    bl = torch.randn(T1, B, A, device='cuda', generator=g)
    act = torch.randint(0, A, (T1, B), device='cuda', generator=g)
    rew = torch.randn(T1, B, device='cuda', generator=g); dn = torch.rand(T1, B, device='cuda', generator=g) < 0.02
    return {k: v.cpu().numpy() for k, v in dict(ll=ll, lb=lb, bl=bl, act=act, rew=rew, done=dn).items()}, {}
  return make


def _regime(name, T1, B, A, seed):
  """Inputs of a trained agent's policy, or of unusual settings, around N(0, 1) logits."""
  def make():
    c, rng = _normal_inputs(T1, B, A, seed)
    kw = {}
    rows = (T1, B)
    if name.startswith('peaked'):          # peaked: most p_j below 1e-30 at s = 60; some actions the least likely
      s = float(name.split('-')[1])
      c['ll'] = (c['ll'] * s).astype(np.float32)
      c['bl'] = (c['ll'] + rng.normal(size=c['ll'].shape) * 0.5).astype(np.float32)
      least = rng.random(rows) < 0.5
      c['act'] = np.where(least, c['ll'].argmin(-1), c['act'])
    elif name == 'offset':                 # a large common offset per row, learner and behaviour alike
      c['ll'] = (c['ll'] + rng.choice([-1e3, 1e3], size=rows + (1,))).astype(np.float32)
      c['bl'] = (c['bl'] + rng.choice([-1e3, 1e3], size=rows + (1,))).astype(np.float32)
    elif name == 'on-policy':              # rho on the min(1, rho) kink
      c['bl'] = (c['ll'] + 1e-3 * rng.normal(size=c['ll'].shape)).astype(np.float32)
    elif name == 'off-policy':             # learner and behaviour peaked on different actions: |log rho| ~ 100
      k1 = rng.integers(0, A, rows)
      k2 = (k1 + rng.integers(1, A, rows)) % A
      c['ll'] = (c['ll'] + 100 * np.eye(A)[k1]).astype(np.float32)
      c['bl'] = (c['bl'] + 100 * np.eye(A)[k2]).astype(np.float32)
      u = rng.random(rows)
      c['act'] = np.where(u < 1 / 3, k1, np.where(u < 2 / 3, k2, c['act']))
    elif name.startswith('rewards'):       # |r| up to 1e3, unclipped and clipped
      c['rew'] = rng.uniform(-1e3, 1e3, rows).astype(np.float32)
      kw = dict(max_abs_reward=float(name.split('-')[1]))
    elif name == 'done-all':
      c['done'][:] = True
    elif name == 'done-none':
      c['done'][:] = False
    elif name == 'done-ends':
      c['done'][:] = False
      c['done'][0] = c['done'][-1] = True
    elif name == 'settings':
      kw = dict(kl_cost=0.3, entropy_cost=0.01, target_entropy=1.5, lambda_=0.9)
    else:
      raise ValueError(name)
    return c, kw
  return make


REGIMES = ('peaked-5', 'peaked-20', 'peaked-60', 'offset', 'on-policy', 'off-policy', 'rewards-0', 'rewards-1',
           'done-all', 'done-none', 'done-ends', 'settings')
WIDTH_TS = (1, 8, 9, 16, 17, 32, 33, 64, 65, 128, 129, 255, 256)


def _cases():
  n = _sms()
  out = []
  # the benchmarked sizes
  out.append(Case('bench', 'B=64', 20, _bench(64), {1: SMALL}))
  for B in (4096, 65536):
    out.append(Case('bench', 'B=%d' % B, 20, _bench(B), {0: SMALL, 1: STREAM % 18}))
  # every scan width, at BB = 2 and the largest BB that fits; T = 257 is past the stream kernel's limit
  for T in WIDTH_TS:
    bbs = _stream_bbs(T, 16 * n, 18)
    B = max(bbs) * n
    modes = {0: SMALL}
    for bb in sorted({2, max(bbs)}):
      modes[bb] = STREAM % 18
    out.append(Case('scan width', 'T=%d lpc=%d BB=%s' % (T, _lpc(T), '/'.join(str(b) for b in sorted({2, max(bbs)}))),
                    T, _plain(T + 1, B, 18, 100 + T), modes))
  out.append(Case('scan width', 'T=257', 257, _plain(258, 2 * n, 18, 357), {1: SMALL}))
  # action counts: the compiled instantiations and the run-time path, every BB the stream kernel takes
  for A in (9, 18, 19, 1, 2, 6, 15, 31):
    modes = {0: SMALL, 1: _stream_name(A)}
    for bb in _stream_bbs(20, 16 * n, A):
      modes[bb] = _stream_name(A)
    out.append(Case('actions', 'A=%d' % A, 20, _plain(21, 16 * n, A, 200 + A), modes))
  # the small kernel alone: one action, large and odd A (odd B * A: the scalar tile copy), ragged B
  for A, B in ((1, 64), (100, 7), (257, 7), (257, 65), (18, 1), (18, 7), (18, 129)):
    out.append(Case('small only', 'A=%d B=%d' % (A, B), 20, _plain(21, B, A, 300 + A + B), {1: SMALL}))
  # logits at a 4-byte offset: the stream kernel refuses them on alignment, the small kernel copies them by floats
  for which in ('ll', 'bl', 'll+bl'):
    out.append(Case('offset view', which, 20, _plain(21, 16 * n, 18, 400), {1: SMALL, 'view': which}))
  # policy regimes, at one stream shape and one small-kernel shape
  for r in REGIMES:
    out.append(Case('regime ' + r, 'stream', 20, _regime(r, 21, 16 * n, 18, 500), {0: SMALL, 1: STREAM % 18}))
    out.append(Case('regime ' + r, 'small', 20, _regime(r, 21, 64, 18, 501), {1: SMALL}))
  return out


def _case_ids():
  # ids without touching the GPU at collection time (the SM count enters only the shapes)
  ids = ['bench B=64', 'bench B=4096', 'bench B=65536']
  ids += ['width T=%d' % T for T in WIDTH_TS] + ['width T=257']
  ids += ['actions A=%d' % A for A in (9, 18, 19, 1, 2, 6, 15, 31)]
  ids += ['small A=%d B=%d' % ab for ab in ((1, 64), (100, 7), (257, 7), (257, 65), (18, 1), (18, 7), (18, 129))]
  ids += ['view ' + w for w in ('ll', 'bl', 'll+bl')]
  ids += ['%s %s' % (r, s) for r in REGIMES for s in ('stream', 'small')]
  return ids


# ---- the GPU side ---------------------------------------------------------------------------------------------------
def _kernels(prof):
  names = [e.name for e in prof.events() if 'vtrace' in e.name]
  out = []
  for nm in names:
    m = re.search(r'vtrace_loss_stream_kernel<(\d+)>', nm)
    if m:
      out.append(STREAM % int(m.group(1)))
    elif re.search(r'vtrace_loss_kernel\b', nm):
      out.append(SMALL)
  return out


def _cuda_view(x, offset):
  """x on the GPU, at a 4-byte offset from a 16-byte aligned allocation when `offset`."""
  t = torch.as_tensor(np.asarray(x)).cuda()
  if not offset:
    return t
  buf = torch.empty(t.numel() + 4, dtype=t.dtype, device='cuda')
  v = buf[1:1 + t.numel()].view(t.shape)
  v.copy_(t)
  assert v.data_ptr() % 16 == 4 and v.is_contiguous()
  return v


def _gpu(c, kw, setting, view=''):
  """Two launches at one loss-stream setting: -> (numpy results, kernels that ran); asserts the repeat is exact."""
  from seed_rl_b200 import _lib
  from seed_rl_b200.agents.vtrace import learner
  st = learner.default_loss_settings(**kw)
  ecp = torch.tensor(np.float32(np.log(st.entropy_cost) / st.entropy_cost_adjustment_speed)).cuda()
  args = [_cuda_view(c[k], k in view.split('+')) for k in ('ll', 'lb', 'bl', 'act', 'rew', 'done')]
  runs = []
  try:
    _lib.check(_lib.lib().seedrl_debug_set_loss_stream(setting))
    # a short profiler session now and then returns without some of its kernel records: profile again when
    # it has none (at most five sessions); the caller asserts on the kernels of the last one
    for _ in range(5):
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                              torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
          r = learner.vtrace_loss_fwd_bwd(st, *args, ecp, want_vtrace=True)
          torch.cuda.synchronize()
          runs.append({k: v.clone() for k, v in r.items() if torch.is_tensor(v)})
      ran = _kernels(prof)
      if ran:
        break
  finally:
    _lib.check(_lib.lib().seedrl_debug_set_loss_stream(1))
  for run in runs[1:]:
    for k in runs[0]:
      assert torch.equal(runs[0][k], run[k]), 'setting %s: %s differs between two launches' % (setting, k)
  r = {k: v.cpu().numpy() for k, v in runs[0].items()}
  lt = r['loss_terms']
  logs = {name: float(lt[_lib.LT[key]]) for name, key in learner._LOG_NAMES}
  return (float(lt[_lib.LT['total']]), logs, r['dlogits'], r['dbaseline'], float(r['d_entropy_cost_param']),
          r['vs'], r['pg_advantages']), ran


def _stages(x, ref):
  total, logs, dl, db, dep, vs, pg = x
  e = collections.OrderedDict(total=_rel(total, ref[0]))
  for k in ref[1]:
    e['log ' + k] = _rel(logs[k], ref[1][k])
  e['vs'] = _relmax(vs, ref[5])
  e['pg_advantages'] = _relmax(pg, ref[6])
  e['dlogits'] = _relmax(dl, ref[2])
  e['dlogits per row'] = _rowmax(dl[:-1], ref[2][:-1])
  e['dbaseline'] = _relmax(db, ref[3])
  e['d_entropy_cost_param'] = _rel(dep, ref[4])
  return e


def _check(group, name, errs, bars, bad):
  for k in errs:
    print('    %-44s %.2e / %.2e' % (k, errs[k], bars[k]))
    ratio = errs[k] / bars[k]
    if not errs[k] <= bars[k]:
      bad.append((name, k, errs[k], bars[k]))
    if group not in _worst or not ratio <= _worst[group][0]:
      _worst[group] = (ratio, name, k)


_CASES = None


@pytest.mark.parametrize('idx', range(len(_case_ids())), ids=_case_ids())
def test_vtrace_loss_matches_float64(idx):
  global _CASES
  if _CASES is None:
    _CASES = _cases()
  assert len(_CASES) == len(_case_ids())
  case = _CASES[idx]
  c, kw = case.make()
  from oracle import loss_oracle
  cfg = loss_oracle.default_config(**kw)
  ecp = np.float32(np.log(cfg.entropy_cost) / cfg.entropy_cost_adjustment_speed)
  args = [c[k] for k in ('ll', 'lb', 'bl', 'act', 'rew', 'done')]
  T1, B, A = c['ll'].shape
  with np.errstate(over='ignore', under='ignore'):
    ref = RF.loss_and_grads(cfg, *args, ecp, torch.float64, chunk=CHUNK)
    m = _stages(RF.loss_and_grads(cfg, *args, ecp, torch.float32, chunk=CHUNK), ref)
  bars = {k: max(FLOOR, C * v) for k, v in m.items()}
  modes = dict(case.modes)
  view = modes.pop('view', '')
  print('VTRACE LOSS FLOAT64 %s %s (T=%d B=%d A=%d %s): error / bar' % (case.group, case.name, T1 - 1, B, A, kw))
  bad = []
  for setting, want in modes.items():
    x, ran = _gpu(c, kw, setting, view)
    label = '%s, setting %d: %s' % (case.name, setting, want)
    print('  setting %d ran %s' % (setting, sorted(set(ran))))
    assert ran and set(ran) == {want}, (label, ran)
    assert float(np.abs(x[2][-1]).max()) == 0.0 and float(np.abs(x[3][-1]).max()) == 0.0, label
    _check(case.group, label, _stages(x, ref), bars, bad)
  assert not bad, bad


def test_cases_cover_every_kernel_instantiation_and_scan_width():
  """The case table, whose every launch the test above checks by kernel name, runs vtrace_loss_kernel, the four
  stream instantiations, the stream kernel at every scan width lpc = 1 .. 32 and with BB = 2, 4, 8 and 16 pinned,
  and T up to the stream kernel's limit of 256 (lpc = 32 with empty top-lane segments from T = 129)."""
  ran, widths, pinned, stream_ts = set(), set(), set(), set()
  for case in _cases():
    for setting, want in case.modes.items():
      if setting == 'view':
        continue
      ran.add(want)
      if want != SMALL:
        widths.add(_lpc(case.T))
        stream_ts.add(case.T)
        pinned.add(setting)
  assert ran == {SMALL} | {STREAM % a for a in (0, 9, 18, 19)}, ran
  assert widths == {1, 2, 4, 8, 16, 32}, widths
  assert {2, 4, 8, 16} <= pinned, pinned
  assert {129, 255, 256} <= stream_ts and 257 not in stream_ts
  # at T = 129 the lanes own ceil(129 / 32) = 5 steps each: lanes 26..31 start past the last step
  assert 26 * 5 >= 129


# ---- vtrace_kernel<5> and the categorical kernel ----------------------------------------------------------------------
def _vtrace_inputs(T, B, seed, regime='normal'):
  rng = np.random.default_rng(seed)
  a = dict(target_action_log_probs=rng.uniform(-2, 2, (T, B)), behaviour_action_log_probs=rng.uniform(-2, 2, (T, B)),
           discounts=0.99 * (rng.random((T, B)) < 0.9), rewards=rng.normal(size=(T, B)),
           values=rng.normal(size=(T, B)), bootstrap_value=rng.normal(size=(B,)))
  if regime == 'off-policy':
    a['target_action_log_probs'] = -rng.uniform(0, 100, (T, B))
    a['behaviour_action_log_probs'] = -rng.uniform(0, 100, (T, B))
  return {k: x.astype(np.float32) for k, x in a.items()}


@pytest.mark.parametrize('T,B,regime,kw', [
    (20, 1 << 18, 'normal', {}), (1, 300, 'normal', {}), (4, 300, 'normal', {}), (5, 300, 'normal', {}),
    (6, 300, 'normal', {}), (11, 300, 'normal', {}), (1000, 300, 'normal', dict(lambda_=0.95)),
    (20, 4096, 'off-policy', {}), (20, 4096, 'off-policy', dict(clip_rho_threshold=3.7, clip_pg_rho_threshold=2.2))])
def test_vtrace_from_importance_weights_matches_float64(T, B, regime, kw):
  """vtrace_kernel<5> (common/vtrace.py), whose loads run five steps ahead of the scan: the full-size batch, T on
  both sides of the prefetch chunk, and log rho spread over +-100."""
  from seed_rl_b200.common import vtrace
  a = _vtrace_inputs(T, B, 600 + T, regime)
  with np.errstate(over='ignore', under='ignore'):
    ref = RF.vtrace_from_importance_weights(*a.values(), np.float64, **kw)
    f32 = RF.vtrace_from_importance_weights(*a.values(), np.float32, **kw)
  got = vtrace.from_importance_weights(**{k: torch.as_tensor(x).cuda() for k, x in a.items()}, **kw)
  got = (got.vs.cpu().numpy(), got.pg_advantages.cpu().numpy())
  print('VTRACE FLOAT64 vtrace_kernel<5> T=%d B=%d %s %s: error / bar' % (T, B, regime, kw))
  bad = []
  errs = {'vs': _relmax(got[0], ref[0]), 'pg_advantages': _relmax(got[1], ref[1])}
  bars = {'vs': max(FLOOR, C * _relmax(f32[0], ref[0])), 'pg_advantages': max(FLOOR, C * _relmax(f32[1], ref[1]))}
  _check('vtrace_kernel<5>', 'T=%d B=%d %s' % (T, B, regime), errs, bars, bad)
  assert not bad, bad


def _categorical_inputs(N, A, regime, seed):
  rng = np.random.default_rng(seed)
  lg = rng.normal(size=(N, A))
  act = rng.integers(0, A, N)
  if regime.startswith('peaked'):
    lg = lg * float(regime.split('-')[1])
    act = np.where(rng.random(N) < 0.5, lg.argmin(-1), act)
  elif regime == 'offset':
    lg = lg + rng.choice([-1e3, 1e3], size=(N, 1))
  else:
    lg = lg * 3
  return lg.astype(np.float32), act


@pytest.mark.parametrize('N,A,regime', [
    (4096, 18, 'peaked-5'), (4096, 18, 'peaked-20'), (4096, 18, 'peaked-60'), (4096, 18, 'offset'),
    (1000, 33, 'normal'), (1000, 64, 'normal'), (300, 1000, 'normal'), (300, 1000, 'offset')])
def test_categorical_log_prob_and_entropy_match_float64(N, A, regime):
  """categorical_logprob_entropy_kernel (one warp per row, lanes striding A) against float64 log-softmax."""
  from seed_rl_b200.common import parametric_distribution as pd
  lg, act = _categorical_inputs(N, A, regime, 700 + A)
  d = pd.categorical_distribution(A, 'int64')
  got = (d.log_prob(torch.as_tensor(lg).cuda(), torch.as_tensor(act).cuda()).cpu().numpy(),
         d.entropy(torch.as_tensor(lg).cuda()).cpu().numpy())

  def ref(dtype):
    lsm = torch.log_softmax(torch.as_tensor(lg).to(dtype), -1)
    return (lsm.gather(-1, torch.as_tensor(act)[:, None])[:, 0].numpy(), (-(lsm.exp() * lsm).sum(-1)).numpy())

  r64, r32 = ref(torch.float64), ref(torch.float32)
  errs = {'log_prob': _relmax(got[0], r64[0]), 'entropy': _relmax(got[1], r64[1])}
  bars = {'log_prob': max(FLOOR, C * _relmax(r32[0], r64[0])), 'entropy': max(FLOOR, C * _relmax(r32[1], r64[1]))}
  print('VTRACE FLOAT64 categorical N=%d A=%d %s: error / bar' % (N, A, regime))
  bad = []
  _check('categorical', 'A=%d %s' % (A, regime), errs, bars, bad)
  assert not bad, bad


def test_zz_worst_error_per_group():
  """Prints the worst error / bar of every case group that ran in this session."""
  print('VTRACE LOSS FLOAT64 worst error / bar per group')
  for g, (ratio, name, stage) in _worst.items():
    print('  %-24s %.3f  (%s, %s)' % (g, ratio, name, stage))
