"""The PopArt, multi-task PopArt and abandoned-mask forms of the fused V-trace loss kernels against the float64
compositions of tests/popart_reference.py and tests/popart_tasks_reference.py, at the kernel instantiations, scan
widths, tile widths and shapes tests/test_gpu_vtrace_loss_float64.py holds the plain kernels to.

Every case runs in up to six configurations: PopArt (learner.popart_loss_fwd_bwd: vtrace_popart_loss_*kernel, then
vtrace_popart_update_kernel), multi-task PopArt with K tasks (learner.popart_tasks_loss_fwd_bwd:
vtrace_popart_tasks_loss_*kernel, vtrace_popart_task_moments_kernel, vtrace_popart_tasks_update_kernel) and the same
entry points with one task (which run the single-task kernels), each without and with an abandoned mask
(abandoned_float64_reference.masks: abandoned rows at the first, an interior and the last transition, each a
terminated row).  A configuration is launched at every loss-stream setting of its case
(seedrl_debug_set_loss_stream 0: the small kernel, 1: the launcher's choice, 2 / 4 / 8 / 16: the stream kernel pinned
to that many columns per tile).  The mask (T x BB bytes) and the task table ((kMaxTasks + 1) x 16 bytes) take
shared memory from the stream kernel's tile, so `_variant_bbs` restates the launcher's pick_stream for each
configuration: a pinned width it refuses must fall back to the small kernel.

Every launch: torch.profiler shows exactly the expected kernels; two launches repeat bit for bit; the bootstrap rows
of dlogits and dbaseline are exactly 0; a task without columns keeps its state bit for bit with +0 gradients and zero
sums; the row counts are exact; masked transitions have pg_advantages exactly 0 and vs = u.  Against float64: the
loss terms, vs, pg_advantages, dlogits (whole and row by row), dbaseline, d_entropy_cost_param, d(sigma, mu), the new
state and the moment sums, task by task in the multi-task form (each task on its own scale).  Bars as in
tests/test_gpu_vtrace_popart.py: error = max|gpu - ref64| / max|ref64| (relative difference for scalars),
bar = max(1e-5, 8 m), m = the same error of the float32 composition.  A quantity formed as a sum or difference of
larger terms (a dlogits row whose advantage r + d vs' - u or entropy gradient p_j (log p_j + H) cancels, d(sigma,
mu) as means of e V and e, the sum of vs, the new mu1 and mu) is measured relative to the magnitude of those terms
where that is larger than its own.
"""
import collections
import re

import numpy as np
import pytest
import torch

import abandoned_float64_reference as AR
import popart_reference as PR
import popart_tasks_reference as PT
from test_gpu_vtrace_loss_float64 import (WIDTH_TS, _bench, _cuda_view, _lpc, _normal_inputs, _plain, _regime, _rel,
                                          _relmax, _sms, _stream_bytes)

pytestmark = pytest.mark.gpu

C = 8
FLOOR = 1e-5
BETA = 0.05
CHUNK = 8192                 # columns per single-task reference evaluation (B = 65536 in float64 within host memory)
K_DEFAULT = 30               # DMLab-30
KEYS = ('ll', 'lb', 'bl', 'act', 'rew', 'done')
_worst = collections.OrderedDict()      # group -> (error / bar, case, stage), printed by the coverage test

# (mu1, mu2, sigma, mu): generic (s = 3); the initial state; mu2 - mu1^2 = 0 exactly (s clipped up to 1e-6); s
# clipped down to 1e6; returns around 1e4 with mu1 = 1e4 and s = 1e3 (the rewards of the case are 100 +- 10)
STATES = {'generic': (2.0, 13.0, 1.2, -0.1), 'initial': (0.0, 1.0, 1.0, 0.0), 'std-floor': (1000.0, 1.0e6, 0.9, 0.1),
          'std-ceiling': (0.0, 4.0e12, 1.1, -0.05), 'returns-1e4': (1.0e4, 1.01e8, 1.0, 0.0)}

# ---- kernels and configurations ---------------------------------------------------------------------------------
Config = collections.namedtuple('Config', 'mode masked')   # mode: 'popart' | 'tasks' | 'tasks1'
CONFIGS = tuple(Config(m, ab) for m in ('popart', 'tasks', 'tasks1') for ab in (False, True))
PLAIN = Config('plain', False)     # vtrace_loss_stream_kernel's own widths
SMALL = {'popart': 'vtrace_popart_loss_kernel', 'tasks': 'vtrace_popart_tasks_loss_kernel'}
STREAM = {'popart': 'vtrace_popart_loss_stream_kernel<%d>', 'tasks': 'vtrace_popart_tasks_loss_stream_kernel<%d>'}
PHASE2 = {'popart': ('vtrace_popart_update_kernel',),
          'tasks': ('vtrace_popart_task_moments_kernel', 'vtrace_popart_tasks_update_kernel')}


def _family(config):
  return 'tasks' if config.mode == 'tasks' else 'popart'


def _label(config):
  return '%s%s' % (config.mode, '+mask' if config.masked else '')


def _variant_bbs(T, B, A, config, sms):
  """The columns per tile pick_stream accepts when pinned, for the configuration (16-byte aligned inputs): the plain
  kernel's, less the mask's T x BB bytes and, with K > 1 tasks, the task table's (64 + 1) x 16 bytes."""
  if T > 256 or (B * A) % 4:
    return []
  limit = 227 * 1024 - 2048 - (65 * 16 if config.mode == 'tasks' else 0)
  out = []
  for BB in (2, 4, 8, 16):
    if B % BB or (BB * A) % 4 or BB * A > 256 or B // BB < sms:
      continue
    if _stream_bytes(T, A, BB) + (T * BB if config.masked else 0) > limit:
      continue
    rows = T * BB
    rounds = -(-rows // 1024)
    per_round = -(-rows // rounds)
    th = max(128, -(-per_round // 32) * 32)
    if (T + 1) * BB > 4 * th:
      continue
    out.append(BB)
  return out


def _expected(case, config, setting, sms):
  """The loss kernel the setting runs for the case and configuration."""
  bbs = [] if case.view else _variant_bbs(case.T, case.B, case.A, config, sms)
  stream = bool(bbs) if setting == 1 else setting in bbs
  fam = _family(config)
  return STREAM[fam] % (case.A if case.A in (9, 18, 19) else 0) if stream else SMALL[fam]


# ---- cases ------------------------------------------------------------------------------------------------------
Case = collections.namedtuple('Case', 'group name T B A make settings view K layout state modes')
ALL_MODES = ('popart', 'tasks', 'tasks1')


def _width_settings(bbs):
  return [0] + sorted({2, max(bbs)}) if bbs else [0, 2]


def _returns_1e4(T1, B, A, seed):
  def make():
    c, rng = _normal_inputs(T1, B, A, seed)
    c['rew'] = (100.0 + 10.0 * rng.normal(size=(T1, B))).astype(np.float32)
    return c, {}
  return make


TASK_BS = (1, 7, 33, 129)    # the small kernel; the moments and update kernels get a partial last warp
LAYOUTS = ('blocks', 'mod', 'one', 'descending')
EDGES = ('initial', 'std-floor', 'std-ceiling', 'returns-1e4')
REGIMES = ('peaked-60', 'offset', 'off-policy', 'rewards-0', 'done-all', 'done-ends', 'settings')
# (T, A, BB) at the shared-memory limit: the plain kernel takes them; the mask refuses the first, the task table the
# second, only the two together the third
LIMIT_SHAPES = ((94, 9, 16), (67, 32, 8), (110, 18, 8))


def _cases(n):
  """The case table for a GPU of n SMs (n enters the shapes only, never the names)."""
  out = []

  def add(group, name, T, B, A, make, settings, view='', K=K_DEFAULT, layout='uneven', state='generic',
          modes=ALL_MODES):
    out.append(Case(group, name, T, B, A, make, settings, view, K, layout, state, modes))
  # the benchmarked shape, once per configuration
  add('bench', 'B=65536', 20, 65536, 18, _bench(65536), lambda bbs: [1])
  # every scan width at BB = 2 and the largest BB the configuration takes; T = 257 is past the stream kernel
  for T in WIDTH_TS:
    B = max(_variant_bbs(T, 16 * n, 18, PLAIN, n)) * n
    add('scan width', 'T=%d lpc=%d' % (T, _lpc(T)), T, B, 18, _plain(T + 1, B, 18, 100 + T), _width_settings)
  add('scan width', 'T=257', 257, 2 * n, 18, _plain(258, 2 * n, 18, 357), lambda bbs: [1])
  # a pinned width the plain kernel takes and the mask and / or the task table leave no room for
  for T, A, BB in LIMIT_SHAPES:
    add('tile limit', 'T=%d A=%d BB=%d' % (T, A, BB), T, BB * n, A, _plain(T + 1, BB * n, A, 800 + T),
        lambda bbs, BB=BB: [0, BB])
  # the compiled instantiations and the run-time path, every BB the stream kernel takes
  for A in (9, 18, 19, 1, 2, 6, 15, 31):
    add('actions', 'A=%d' % A, 20, 16 * n, A, _plain(21, 16 * n, A, 200 + A), lambda bbs: [0, 1] + bbs)
  for A, B in ((1, 64), (100, 7), (257, 7), (257, 65), (18, 1), (18, 7), (18, 129)):
    add('small only', 'A=%d B=%d' % (A, B), 20, B, A, _plain(21, B, A, 300 + A + B), lambda bbs: [1])
  for which in ('ll', 'bl', 'll+bl'):
    add('offset view', which, 20, 16 * n, 18, _plain(21, 16 * n, 18, 400), lambda bbs: [1], view=which)
  for r in REGIMES:
    add('regime ' + r, 'stream', 20, 16 * n, 18, _regime(r, 21, 16 * n, 18, 500), lambda bbs: [0, 1])
    add('regime ' + r, 'small', 20, 64, 18, _regime(r, 21, 64, 18, 501), lambda bbs: [1])
  for s in EDGES:
    mk = _returns_1e4 if s == 'returns-1e4' else (lambda T1, B, A, seed: _plain(T1, B, A, seed))
    add('state ' + s, 'stream', 20, 16 * n, 18, mk(21, 16 * n, 18, 900), lambda bbs: [0, 1], state=s)
    add('state ' + s, 'small', 20, 64, 18, mk(21, 64, 18, 901), lambda bbs: [1], state=s)
  # task counts, ragged batches and task layouts (the multi-task form alone), at DMLab's nine actions
  for K in (2, 30, 64):
    for B in TASK_BS + (16 * n,):
      name = 'K=%d B=%s uneven' % (K, 'stream' if B == 16 * n else B)
      add('tasks K=%d' % K, name, 20, B, 9, _plain(21, B, 9, 1000 + K + B), lambda bbs: [0, 1] if bbs else [1],
          K=K, modes=('tasks',))
    for layout in LAYOUTS:
      for B in (129, 16 * n):
        name = 'K=%d B=%s %s' % (K, 'stream' if B == 16 * n else B, layout)
        add('tasks K=%d' % K, name, 20, B, 9, _plain(21, B, 9, 1100 + K + B), lambda bbs: [0, 1] if bbs else [1],
            K=K, layout=layout, modes=('tasks',))
  return out


def _case_ids():
  return ['%s %s' % (c.group, c.name) for c in _cases(132)]


def _task_ids(layout, B, K, seed):
  b = np.arange(B)
  if layout == 'uneven':                 # task k draws a share proportional to 1 / (k + 1)
    p = 1.0 / np.arange(1, K + 1)
    ids = np.random.default_rng(seed).choice(K, size=B, p=p / p.sum())
  elif layout == 'blocks':               # contiguous runs across warps and CTAs
    ids = b * K // B
  elif layout == 'mod':
    ids = b % K
  elif layout == 'one':                  # K - 1 tasks absent
    ids = np.full(B, K - 1)
  elif layout == 'descending':
    ids = (B - 1 - b) * K // B
  else:
    raise ValueError(layout)
  return ids.astype(np.int32)


def _task_states(K, seed, edge):
  """States of returns from ~0.1 to ~1e3 across the tasks; the even tasks take the edge state, if any."""
  rng = np.random.default_rng(seed)
  scale = 10.0 ** rng.uniform(-1, 3, K)
  mu1 = scale * rng.normal(size=K)
  s = scale * rng.uniform(0.5, 2.0, K)
  st = np.stack([mu1, mu1 * mu1 + s * s, rng.uniform(0.7, 1.3, K), rng.normal(size=K) * 0.2], 1).astype(np.float32)
  if edge != 'generic':
    st[::2] = STATES[edge]
  return st


def _setup(case, config):
  """-> (inputs, settings kwargs, mask or None, state [K,4], task ids [B], K) of the case in the configuration."""
  c, kw = case.make()
  T1, B = c['lb'].shape
  ab = None
  if config.masked:
    done, ab = AR.masks(T1, B, 77 + T1 + B, p_done=0.0)
    c = dict(c, done=c['done'] | done)
  if config.mode == 'tasks':
    K = case.K
    return c, kw, ab, _task_states(K, 5 + K, case.state), _task_ids(case.layout, B, K, 3 + B + K), K
  return c, kw, ab, np.array(STATES[case.state], np.float32)[None], np.zeros(B, np.int32), 1


def _loss_settings(config, K, kw):
  from seed_rl_b200.agents.vtrace import learner
  return learner.default_loss_settings(popart=True, popart_beta=BETA, popart_tasks=K if config.mode == 'tasks' else 1,
                                       **kw)


def _ecp(st):
  return np.float32(np.log(st.entropy_cost) / st.entropy_cost_adjustment_speed)


# ---- the float64 and float32 compositions -------------------------------------------------------------------------
def _reference(config, st, c, ab, state, ids, FT):
  """The composition in dtype FT, with state [K,4], dcomp [K,2] and sums [K,3] in every configuration."""
  args = [c[k] for k in KEYS]
  ecp = _ecp(st)
  B = c['lb'].shape[1]
  if config.mode == 'tasks':
    return PT.loss_and_grads(st, *args, ecp, state, ids, BETA, FT, abandoned=ab)
  if B <= CHUNK:
    r = PR.loss_and_grads(st, *args, ecp, state[0], BETA, FT, abandoned=ab)
    return dict(r, state=r['state'][None], dcomp=r['dcomp'][None], sums=r['sums'][None])
  # column chunks as tasks that share the state and the moment sums of the whole batch
  chunks = (np.arange(B) // CHUNK).astype(np.int32)
  states = np.repeat(state, chunks[-1] + 1, 0)
  total = PT.task_sums(st, *args, states, chunks, FT, ab).sum(0)
  r = PT.loss_and_grads(st, *args, ecp, states, chunks, BETA, FT, global_sums=np.tile(total, (len(states), 1)),
                        abandoned=ab)
  new = r['state'][0]
  terms = dict(r['terms'], popart_mean=new[0], popart_std=FT(np.clip(np.sqrt(FT(new[1] - new[0] * new[0])), 1e-6, 1e6)))
  return dict(r, terms=terms, state=new[None], dcomp=r['dcomp'].sum(0, dtype=FT)[None], sums=total[None])


# ---- the GPU side -------------------------------------------------------------------------------------------------
def _kernels(prof):
  out = []
  for e in prof.events():
    m = re.search(r'\b(vtrace_\w+_kernel)(<\d+>)?', e.name)
    if m:
      out.append(m.group(1) + (m.group(2) or ''))
  return out


def _launch(config, st, args, ab, state, ids, K):
  """Both phases once, from `state`: -> dict of tensors."""
  from seed_rl_b200.agents.vtrace import learner
  ecp = torch.tensor(_ecp(st)).cuda()
  mom = torch.as_tensor(state[:, :2]).contiguous().cuda()
  comp = torch.as_tensor(state[:, 2:]).contiguous().cuda()
  dcomp = torch.zeros(K, 2, device='cuda')
  if config.mode == 'popart':
    mom, comp, dcomp = mom[0].contiguous(), comp[0].contiguous(), dcomp[0].contiguous()
    seen = {}
    out = learner.popart_loss_fwd_bwd(st, *args, ecp, mom, comp, dcomp,
                                      reduce_moment_sums=lambda s: seen.setdefault('sums', s.clone()),
                                      want_vtrace=True, abandoned=ab)
    out['moment_sums'] = seen['sums']
  else:
    err = torch.zeros(1, dtype=torch.int32, device='cuda')
    out = learner.popart_tasks_loss_fwd_bwd(st, *args, ecp, mom, comp, dcomp, torch.as_tensor(ids).cuda(), err,
                                            want_vtrace=True, abandoned=ab)
    out['task_error'] = err
  out.update(mom=mom, comp=comp, dcomp=dcomp)
  return out


def _gpu(config, st, c, ab, state, ids, K, setting, view, want):
  """Two launches at one loss-stream setting: -> (numpy results in the reference's layout, kernels that ran);
  asserts that the two repeat bit for bit."""
  from seed_rl_b200 import _lib
  args = [_cuda_view(c[k], k in view.split('+')) for k in KEYS]
  abt = None if ab is None else torch.as_tensor(ab).cuda()
  try:
    _lib.check(_lib.lib().seedrl_debug_set_loss_stream(setting))
    # a short profiler session now and then returns without some of its kernel records: profile again while one
    # of the expected kernels is missing (at most five sessions); the caller asserts on the last one
    for _ in range(5):
      runs = []
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU,
                                              torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(2):
          r = _launch(config, st, args, abt, state, ids, K)
          torch.cuda.synchronize()
          runs.append({k: v.detach().cpu().numpy().copy() for k, v in r.items() if torch.is_tensor(v)})
      ran = _kernels(prof)
      if set(want) <= set(ran):
        break
  finally:
    _lib.check(_lib.lib().seedrl_debug_set_loss_stream(1))
  for k in runs[0]:
    a, b = np.ascontiguousarray(runs[0][k]), np.ascontiguousarray(runs[1][k])
    assert a.tobytes() == b.tobytes(), 'setting %s: %s differs between two launches' % (setting, k)
  r = runs[0]
  lt = r['loss_terms']
  x = dict(terms={k: float(lt[i]) for k, i in _lib.LT.items()}, vs=r['vs'], pg_adv=r['pg_advantages'],
           dlogits=r['dlogits'], dbaseline=r['dbaseline'], d_entropy_cost_param=float(r['d_entropy_cost_param']),
           state=np.concatenate([r['mom'].reshape(-1, 2), r['comp'].reshape(-1, 2)], 1),
           dcomp=r['dcomp'].reshape(-1, 2), sums=r['moment_sums'].reshape(K, -1),
           task_error=int(r['task_error'][0]) if 'task_error' in r else 0)
  return x, ran


TERMS = ('total', 'policy', 'V', 'entropy', 'kl', 'entropy_adj', 'v_mean', 'v_l2_error', 'mean_entropy',
         'entropy_cost', 'mean_kl', 'max_action_abs')


def _rel_to(a, w, scale):
  """|a - w| relative to |w|, or to `scale` where that is larger: the magnitude of the terms w is a sum of."""
  return abs(float(a) - float(w)) / max(abs(float(w)), float(scale), 1e-30)


def _scales(c, ref, state, ids, K, st):
  """Magnitudes of what each compared quantity is a sum or difference of, from the float64 composition (PopArt's
  return-sized differences cancel: pg_adv = r + d vs' - u, mean e, m - m' + s mu).  -> dict of arrays / [K]."""
  T1, B, A = c['ll'].shape
  T, N = T1 - 1, float((T1 - 1) * B)
  st64 = state.astype(np.float64)
  s = np.clip(np.sqrt(st64[:, 1] - st64[:, 0] ** 2), 1e-6, 1e6)[ids]                  # [B]
  u, vs = ref['u'], ref['vs']
  r = np.abs(np.asarray(c['rew'], np.float64)[1:])
  if st.max_abs_reward:
    r = np.minimum(r, st.max_abs_reward)
  d = st.discounting * ~np.asarray(c['done'], bool)[1:]
  vs_next = np.concatenate([vs[1:], u[-1:]], 0)
  kappa = (r + d * np.abs(vs_next) + np.abs(u[:-1])) / s / N                         # bound of |d adv| / eps / N
  ll = np.asarray(c['ll'], np.float64)[:-1]
  z = ll - ll.max(-1, keepdims=True)
  lsm = z - np.log(np.exp(z).sum(-1, keepdims=True))
  p = np.exp(lsm)
  onehot = np.zeros_like(p)
  np.put_along_axis(onehot, np.asarray(c['act'])[:-1, :, None].astype(np.int64), 1.0, -1)
  H = -(p * lsm).sum(-1, keepdims=True)
  ec = np.exp(st.entropy_cost_adjustment_speed * np.float64(_ecp(st)))
  # the advantage term's and the entropy term's (p_j (log p_j + H), which cancels near a uniform row) magnitudes
  row = kappa * np.abs(onehot - p).max(-1) + ec / N * (p * (np.abs(lsm) + H)).max(-1)   # [T,B]
  e, V = ref['e'], np.asarray(c['lb'], np.float64)[:-1]
  bc = st.baseline_cost
  out = dict(row=row, ev=np.zeros(K), e=np.zeros(K), vs=np.zeros(K), mu1=np.zeros(K), mu=np.zeros(K))
  for k in range(K):
    cols = ids == k
    if not cols.any():
      continue
    mu1, mu2, sigma, mu = st64[k]
    new = np.asarray(ref['state'][k], np.float64)
    sk = s[cols][0]
    sn = np.clip(np.sqrt(max(new[1] - new[0] ** 2, 0.0)), 1e-6, 1e6)
    out['ev'][k] = bc * np.abs(e[:, cols] * V[:, cols]).sum() / N
    out['e'][k] = bc * np.abs(e[:, cols]).sum() / N
    out['vs'][k] = np.abs(vs[:, cols]).sum()
    out['mu1'][k] = abs(mu1) + BETA * (np.abs(vs[:, cols]).mean() + abs(mu1))
    out['mu'][k] = (abs(mu1) + abs(new[0]) + sk * abs(mu)) / sn
  return out


def _stages(config, x, ref, ids, K, sc):
  """error of every compared quantity, by stage name; per task in the multi-task form.  Quantities that are sums
  or differences of larger terms are taken relative to the magnitude of those terms (`_scales`)."""
  e = collections.OrderedDict()
  tasks = config.mode == 'tasks'
  for k in TERMS + (() if tasks else ('popart_mean', 'popart_std')):
    e['term ' + k] = _rel(x['terms'][k], ref['terms'][k])
  e['d_entropy_cost_param'] = _rel(x['d_entropy_cost_param'], ref['d_entropy_cost_param'])
  # row by row (rows differ in scale by orders of magnitude), each row relative to its own largest entry or to the
  # magnitude of the terms its advantage and entropy gradient are differences of, whichever is larger
  dl, w = np.asarray(x['dlogits'][:-1], np.float64), np.asarray(ref['dlogits'][:-1], np.float64)
  e['dlogits per row'] = float((np.abs(dl - w).max(-1) / np.maximum(np.abs(w).max(-1), sc['row']).clip(1e-30)).max())
  present = [k for k in range(K) if (ids == k).any()]
  for k in present:
    tag = ' task %d' % k if tasks else ''
    cols = ids == k
    for key in ('vs', 'pg_adv', 'dlogits', 'dbaseline'):
      e[key + tag] = _relmax(x[key][:, cols], ref[key][:, cols])
    for j, nm in enumerate(('mu1', 'mu2', 'sigma', 'mu')):
      scale = sc['mu1'][k] if nm == 'mu1' else sc['mu'][k] if nm == 'mu' else 0.0
      e['state %s%s' % (nm, tag)] = _rel_to(x['state'][k, j], ref['state'][k, j], scale)
    e['d sigma' + tag] = _rel_to(x['dcomp'][k, 0], ref['dcomp'][k, 0], sc['ev'][k])
    e['d mu' + tag] = _rel_to(x['dcomp'][k, 1], ref['dcomp'][k, 1], sc['e'][k])
    e['sum vs' + tag] = _rel_to(x['sums'][k, 0], ref['sums'][k, 0], sc['vs'][k])
    e['sum vs^2' + tag] = _rel(x['sums'][k, 1], ref['sums'][k, 1])
  return e


def _exact_checks(config, x, ref64, c, ab, state, ids, K, label):
  T = c['lb'].shape[0] - 1
  assert not x['dlogits'][-1].any() and not x['dbaseline'][-1].any(), label + ': bootstrap row'
  assert x['task_error'] == 0, label
  if config.mode == 'tasks':
    assert x['terms']['popart_mean'] == 0 and x['terms']['popart_std'] == 0, label
  for k in range(K):
    n = int((ids == k).sum())
    if config.mode != 'popart':
      assert x['sums'][k, 2] == T * n, (label, k, x['sums'][k])
    if n == 0:   # an absent task: its state bit for bit, +0 gradients, no sums
      assert x['state'][k].tobytes() == state[k].tobytes(), (label, k, x['state'][k], state[k])
      assert np.all(x['dcomp'][k] == 0) and not np.signbit(x['dcomp'][k]).any(), (label, k, x['dcomp'][k])
      assert np.all(x['sums'][k] == 0), (label, k)
  if ab is not None:   # a masked transition: target = the value u, no policy gradient
    m = ab[1:]
    assert m.any()
    assert np.all(x['pg_adv'][m] == 0), label + ': masked pg_advantages'
    u = ref64['u'][:-1]
    for k in range(K):
      mk = m & (ids == k)[None]
      if mk.any():
        scale = np.abs(u[:, ids == k]).max()
        err = np.abs(x['vs'][mk] - u[mk]).max()
        assert err <= 2e-6 * scale, (label, 'masked vs - u', k, err, scale)


def _check(group, name, errs, bars, bad):
  ranked = sorted(errs, key=lambda k: -errs[k] / bars[k])
  for k in ranked[:3]:
    print('    %-36s %.2e / %.2e' % (k, errs[k], bars[k]))
  for k in errs:
    if not errs[k] <= bars[k]:
      bad.append((name, k, errs[k], bars[k]))
  k = ranked[0]
  ratio = errs[k] / bars[k]
  if group not in _worst or not ratio <= _worst[group][0]:
    _worst[group] = (ratio, name, k)


_CASES = None


@pytest.mark.parametrize('idx', range(len(_case_ids())), ids=_case_ids())
def test_vtrace_loss_variants_match_float64(idx):
  global _CASES
  n = _sms()
  if _CASES is None:
    _CASES = _cases(n)
  assert ['%s %s' % (c.group, c.name) for c in _CASES] == _case_ids()
  case = _CASES[idx]
  bad = []
  for config in CONFIGS:
    if config.mode not in case.modes:
      continue
    c, kw, ab, state, ids, K = _setup(case, config)
    st = _loss_settings(config, K, kw)
    T1, B, A = c['ll'].shape
    with np.errstate(all='ignore'):
      ref = _reference(config, st, c, ab, state, ids, np.float64)
      sc = _scales(c, ref, state, ids, K, st)
      m = _stages(config, _reference(config, st, c, ab, state, ids, np.float32), ref, ids, K, sc)
    bars = {k: max(FLOOR, C * v) for k, v in m.items()}
    bbs = [] if case.view else _variant_bbs(case.T, case.B, case.A, config, n)
    group = '%s / %s' % (case.group, _label(config))
    print('VTRACE LOSS VARIANTS FLOAT64 %s %s %s (T=%d B=%d A=%d K=%d %s, BB taken %s): worst error / bar'
          % (case.group, case.name, _label(config), T1 - 1, B, A, K, kw, bbs))
    for setting in case.settings(bbs):
      loss = _expected(case, config, setting, n)
      want = (loss,) + PHASE2[_family(config)]
      x, ran = _gpu(config, st, c, ab, state, ids, K, setting, case.view, want)
      label = '%s %s, setting %d: %s' % (case.name, _label(config), setting, loss)
      print('  setting %d ran %s' % (setting, sorted(set(ran))))
      assert ran and set(ran) == set(want), (label, ran)
      _exact_checks(config, x, ref, c, ab, state, ids, K, label)
      _check(group, label, _stages(config, x, ref, ids, K, sc), bars, bad)
  assert not bad, bad


def test_cases_cover_every_instantiation_scan_width_and_mask():
  """The case table runs, in each of the six configurations, the small kernel and the four stream instantiations,
  and the stream kernel at every scan width lpc = 1 .. 32; some pinned width the plain kernel takes falls back to
  the small kernel for a configuration with the mask or the task table; the multi-task form runs K = 2, 30 and 64,
  batches with a partial last warp, and every task layout.  Then prints the worst error / bar of every group that
  ran in this session."""
  n = _sms()
  ran = collections.defaultdict(set)
  widths = collections.defaultdict(set)
  fallbacks = set()
  for case in _cases(n):
    for config in CONFIGS:
      if config.mode not in case.modes:
        continue
      bbs = [] if case.view else _variant_bbs(case.T, case.B, case.A, config, n)
      for setting in case.settings(bbs):
        k = _expected(case, config, setting, n)
        ran[config].add(k)
        if k != SMALL[_family(config)]:
          widths[config].add(_lpc(case.T))
        elif setting > 1 and setting in _variant_bbs(case.T, case.B, case.A, PLAIN, n):
          fallbacks.add(config)
  for config in CONFIGS:
    fam = _family(config)
    assert ran[config] == {SMALL[fam]} | {STREAM[fam] % a for a in (0, 9, 18, 19)}, (config, ran[config])
    assert widths[config] == {1, 2, 4, 8, 16, 32}, (config, widths[config])
  assert Config('popart', True) in fallbacks and Config('tasks', False) in fallbacks and Config('tasks', True) in fallbacks
  assert Config('popart', False) not in fallbacks and Config('tasks1', False) not in fallbacks
  tasks = [c for c in _cases(n) if c.modes == ('tasks',)]
  assert {c.K for c in tasks} == {2, 30, 64}
  assert {c.layout for c in tasks} == {'uneven'} | set(LAYOUTS)
  assert {c.B % 32 for c in tasks} - {0} and {c.B for c in tasks} >= set(TASK_BS) | {16 * n}
  print('VTRACE LOSS VARIANTS FLOAT64 worst error / bar per group')
  for g, (ratio, name, stage) in _worst.items():
    print('  %-40s %.3f  (%s, %s)' % (g, ratio, name, stage))
