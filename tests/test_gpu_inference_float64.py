"""Central inference against a float64 reference at the batch sizes it serves: the V-trace InferenceHost (ImpalaDeep
in conv_mode 'tc3p', 'tc3p' with the 'tc3' recurrence, 'tc3' and 'simt'; ImpalaShallow in 'tc3'; A = 18, 84x84x4)
and the R2D2InferenceHost (DuelingLSTMDQNNet in gemm_mode 'tc3', 'tc3' with the 'tc3' recurrence and 'simt';
A = 18, 84x84x1 stacked 4), each on its CUDA-graph host and its eager host, at inference batch N = 64 and 256.

Why these sizes.  A T=1 batch of n envs is n frames: every GEMM with M = n (conv_to_linear, the LSTM input
projection, the heads) runs on sgemm below 64 rows and on wgmma from 64, the recurrence runs with B = n and the
plane convs get small-N tails.  N = 64 sits on that boundary; partial batches of 1, 63, 65 (where below N) and N-1
rows run eagerly on both hosts.  The learner float64 tests never reach these shapes.

The script.  num_envs = 2N (R2D2: plus 8 eval envs); 14 batches (R2D2: 16) from a seeded rng: full batches of
permuted, duplicate-free ids (every other one the same N-id core, so that unrolls complete), the partial batches
interleaved, done at 10%, new run ids for a few envs at batch 7, and one core env sitting out batches 3..9.
episode_step carries the env id, so that a completed unroll names its env.  V-trace unroll_length 4; R2D2
burn_in 2, unroll_length 5.  Every env's first batch is a run-id reset.

Per batch:
  1. arithmetic: the GPU's logits and baseline (R2D2: q), the new h and c read back from the tables, and every
     activation seedrl_debug_net_views / seedrl_debug_r2d2_net_views locate in the (1, n) workspace (the graph's
     own on a replay) against the float64 reference (tests/vtrace_float64_reference.py / r2d2_float64_reference.py
     `forward`) fed the table rows read before the call and conditioned on the GPU's ReLU masks and pool taps.
     error = max|gpu - ref| / max|ref|, bar = max(FLOOR, C m), the rule of test_gpu_vtrace_float64.py: m is the
     float32 reference's distance under the same decisions, measured on every batch and the run's largest taken;
     for bf16x3 modes the larger of that and the float64 reference's response to a 2^-16 perturbation of the parameters and the input state,
     measured once per run (configuration, host, N) on its fifth batch (a full batch with non-zero states).
     Decisions the GPU made otherwise than float64 must be near-ties within the layer's bar.
  2. actions: V-trace, the served action is categorical_sample_np of the GPU logits at the Philox offset read before
     the call (agent._rng_offset eager, host._g_counter on a replay) wherever its Gumbel gap exceeds 1e-4, and that
     of the float64 logits where their gap exceeds 1e-4 too.  R2D2, the GPU's greedy action (first max of its q)
     is the float64 argmax except at near-ties within the q bar; the served action is epsilon_greedy_np of it on a
     replay, and learner.apply_epsilon_greedy from a clone of the host generator's state on the eager path.
  3. bookkeeping, bit for bit: the forward was fed the table rows (zero state, previous action 0 after a run-id
     reset); afterwards the rows at the ids hold the forward's new state and the served actions, every other row is
     unchanged, and R2D2's frame-stacking rows are r2d2_oracle.stack_frames chained through the script.
  4. completed unrolls, bit for bit: the completing envs are those the append count predicts, and each unroll (a
     queue item, or the BatchAssembler's columns) is row by row what the env was fed and served over its last
     T+1 (R2D2: burn_in + unroll_length + 1) steps; an R2D2 env's first unroll after a reset completes burn_in
     steps early, behind burn_in zero rows.  Its first agent state is the state fed at row burn_in (V-trace: row
     0): the reference's rule (agents/r2d2/learner.py:826), which records the state before the step that completed
     the previous unroll, the last of the burn_in + 1 rows the next unroll repeats; after a reset, the zero state.  R2D2's initial priorities
     equal the float64 n-step priorities of the GPU's q within the same bar rule (m: the float32 restatement).
     Eval envs never reach the store.
  5. the bounded-wait error flag of the (1, n) workspace is clear.
"""
import ctypes

import numpy as np
import pytest
import torch

import r2d2_float64_reference as R2
import vtrace_float64_reference as RV
from test_gpu_r2d2_graph_inference import categorical_sample_np, epsilon_greedy_np
from test_gpu_vtrace_float64 import _read_views, _view_names

pytestmark = pytest.mark.gpu

C = 8
FLOOR = 1e-6
DELTA = 2.0 ** -16
A = 18
VT_OBS, VT_T = (84, 84, 4), 4
R_OBS, S, R_EVAL, BURN_IN, R_UNROLL = (84, 84, 1), 4, 8, 2, 5
VTRACE = {'deep-tc3p': ('deep', 'tc3p', 'tiled'), 'deep-tc3p-lstm-tc3': ('deep', 'tc3p', 'tc3'),
          'deep-tc3': ('deep', 'tc3', 'tiled'), 'deep-simt': ('deep', 'simt', 'tiled'),
          'shallow-tc3': ('shallow', 'tc3', 'tiled')}
R2D2 = {'tc3': ('tc3', 'tiled'), 'tc3-lstm-tc3': ('tc3', 'tc3'), 'simt': ('simt', 'tiled')}
RESP_BATCH = 4
_cache = {}


def _relmax(a, w):
  a = np.asarray(a, np.float64); w = np.asarray(w, np.float64)
  return float(np.abs(a - w).max() / (np.abs(w).max() + 1e-30))


def _params(kind, net=None):
  key = ('params', kind, net)
  if key not in _cache:
    torch.set_num_threads(max(1, min(32, torch.get_num_threads())))
    if kind == 'vtrace':
      from oracle import net_oracle
      _cache[key] = net_oracle.init_params(net, A, VT_OBS, seed=1)      # test_gpu_vtrace_float64.py's
    else:
      from oracle import r2d2_net_oracle
      _cache[key] = r2d2_net_oracle.init_params(A, R_OBS, S, seed=5)   # test_gpu_r2d2_float64.py's
  return _cache[key]


def _script(N, num_envs, obs, calls, seed):
  """[(ids int32, run ids, EnvOutput of numpy arrays, raw rewards)]."""
  from seed_rl_b200.common import utils
  rng = np.random.default_rng(seed)
  run_ids = rng.integers(1, 2 ** 40, num_envs)
  core = rng.permutation(num_envs)[:N]
  sitter, spare = core[0], np.setdiff1d(np.arange(num_envs), core)[0]
  partial = iter(sorted({n for n in (1, 63, 65, N - 1) if n < N}))
  seq = []
  for i in range(calls):
    sitting = 3 <= i <= 9
    pool = np.setdiff1d(np.arange(num_envs), [sitter]) if sitting else np.arange(num_envs)
    n = next(partial, N) if i % 3 == 2 else N
    if n == N and i % 2 == 0:
      ids = rng.permutation(np.where(core == sitter, spare, core) if sitting else core)
    else:
      ids = rng.permutation(pool)[:n]
    if i == 7:
      run_ids[ids[:3]] += 1
    env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), rng.random(n) < 0.1,
                          rng.integers(0, 256, (n,) + obs, dtype=np.uint8), np.zeros(n, bool), ids.astype(np.int32))
    seq.append((ids.astype(np.int32), run_ids[ids].copy(), env, rng.normal(size=n).astype(np.float32)))
  assert all(i != sitter for b in seq[3:10] for i in b[0])
  return seq


def _recording(base, vtrace):
  class Recorded(base):
    """Keeps what its last eager call was fed and returned, and what the call a CUDA graph captured was."""

    def __call__(self, *args, **kw):
      out = super().__call__(*args, **kw)
      fed = (args[0], args[2]) if vtrace else (args[0][0], args[1])
      if torch.cuda.is_current_stream_capturing():
        self.captured = (fed, out)
      else:
        self.last = (fed, out)
      return out
  return Recorded


def _flat_state(state):
  from seed_rl_b200.common import utils
  return [t for t in utils.flatten(state)]


class _Run(object):
  """One script through one host; collects per-batch stage errors and measures, and asserts the exact checks."""

  def __init__(self, kind, mode, host_kind, N, calls=None, mutate=None):
    from seed_rl_b200.agents.r2d2 import learner as r2d2_learner, learner_loop as r2d2_loop
    from seed_rl_b200.agents.vtrace import learner_loop as vtrace_loop
    from seed_rl_b200.atari import networks as atari_networks
    from seed_rl_b200.common import utils
    from seed_rl_b200.dmlab import networks as dmlab_networks
    self.kind, self.mode, self.host_kind, self.N = kind, mode, host_kind, N
    self.vtrace = vt = kind == 'vtrace'
    graph = host_kind == 'graph'
    if vt:
      self.net, conv_mode, lstm_mode = VTRACE[mode]
      self.params = _params(kind, self.net)
      base = dmlab_networks.ImpalaDeep if self.net == 'deep' else dmlab_networks.ImpalaShallow
      self.agent = _recording(base, True)(A, VT_OBS, seed=11, conv_mode=conv_mode, lstm_mode=lstm_mode)
      self.num_envs, self.ntr, self.L, self.unroll, self.overlap = 2 * N, 2 * N, VT_T + 1, VT_T, 0
      self.obs = VT_OBS
      if graph:
        self.host = vtrace_loop.InferenceHost(self.agent, self.num_envs, VT_T, N, VT_OBS, training_batch_size=N)
        assert self.host.use_graph
      else:
        self.host = vtrace_loop.InferenceHost(self.agent, self.num_envs, VT_T, N, VT_OBS)
        self.host.unroll_queue = utils.StructuredFIFOQueue(-1, self.host.unroll_specs)   # nobody trains here
    else:
      gemm_mode, lstm_mode = R2D2[mode]
      self.params = _params(kind)
      self.agent = _recording(atari_networks.DuelingLSTMDQNNet, False)(A, R_OBS, S, seed=11, gemm_mode=gemm_mode,
                                                                       lstm_mode=lstm_mode)
      self.num_envs, self.ntr = 2 * N + R_EVAL, 2 * N
      self.L, self.unroll, self.overlap, self.obs = BURN_IN + R_UNROLL + 1, R_UNROLL, BURN_IN, R_OBS
      self.settings = r2d2_learner.default_settings(burn_in=BURN_IN, unroll_length=R_UNROLL)
      self.generator = torch.Generator(device='cuda').manual_seed(17)
      self.host = r2d2_loop.R2D2InferenceHost(self.agent, self.num_envs, R_EVAL, N, R_OBS, settings=self.settings,
                                              unroll_queue_max_size=-1, generator=self.generator, cuda_graph=graph,
                                              epsilon_seed=0x0123456789ABCDEF)
      self.st = R2.settings(A, S, self.settings, 0.00048, 1e-3)
    gpu_params = dict(self.params)
    if mutate:
      gpu_params[mutate] = np.asarray(gpu_params[mutate], np.float64) * (1 + 2.0 ** -12)
    self.agent.load_named_parameters(gpu_params)
    calls = calls or (14 if vt else 16)
    self.script = _script(N, self.num_envs, self.obs, calls, seed=1000 * N + (7 if vt else 8))
    self.run_ids = np.zeros(self.num_envs, np.int64)
    self.fs = np.zeros((self.num_envs, int(np.prod(self.obs))), np.int32)     # R2D2 frame-stacking mirror
    self.history = [[] for _ in range(self.num_envs)]
    self.appends = np.zeros(self.num_envs, np.int64)
    self.batches = []        # per batch: n, errs, m32, ties, prio (errs, m32)
    self.completed = 0
    self.sizes = set()
    self._assembled = []
    if vt and graph:
      orig = self.host.store.complete_into

      def complete_into(nc, into, on_placed=None):
        ids, placed = orig(nc, into, on_placed)
        self._assembled.append((ids, placed))
        return ids, placed
      self.host.store.complete_into = complete_into

  # ---- the run ----------------------------------------------------------------------------------------------
  def run(self):
    self.resp = None
    for i, batch in enumerate(self.script):
      self._batch(i, *batch)
    if not self.vtrace:
      # the store has rows for the training envs only (eval ids never complete: `expect` in _batch)
      assert all(t.shape[0] == self.ntr for t in self.host.store._state + [self.host.store._index])
    assert self.completed > 0 or len(self.script) <= RESP_BATCH + 1
    return self

  def _tables(self):
    return [t.cpu().numpy().copy() for t in self.host.agent_states._state], self.host.actions._state[0].cpu().numpy()

  def _batch(self, i, ids, run_ids, env, raw):
    from seed_rl_b200 import _lib
    from seed_rl_b200.agents.r2d2 import learner as r2d2_learner
    host, agent, n, vt = self.host, self.agent, len(ids), self.vtrace
    on_graph = host.use_graph and n == self.N
    states0, actions0 = self._tables()
    reset = run_ids != self.run_ids[ids]
    self.run_ids[ids] = run_ids
    # what the forward must be fed: the table rows, or after a run-id reset zero state and previous action 0
    fed = [np.where(reset.reshape((-1,) + (1,) * (t.ndim - 1)), 0, t[ids]) for t in states0]
    fed_prev = np.where(reset, 0, actions0[ids])
    if not vt:
      self.fs[ids[reset]] = 0
      np.testing.assert_array_equal(fed[2], self.fs[ids])
    offset = (int(host._g_counter) if host._graph is not None else 0) if on_graph else (
        agent._rng_offset if vt else None)
    gen_state = None if vt or on_graph else self.generator.get_state()
    served = host.inference(ids, run_ids, env, raw)
    torch.cuda.synchronize()
    self.sizes.add(n)
    if on_graph:
      (fed_actions, fed_state), (_, new_state) = agent.captured
      outputs, ws = host._g_out, host._g_workspace
    else:
      (fed_actions, fed_state), (outputs, new_state) = agent.last
      ws = agent.workspace(1, n)
    # 5. the error flag of this workspace
    check = _lib.lib().seedrl_net_check_error if vt else _lib.lib().seedrl_r2d2_net_check_error
    assert check(agent._h, 1, n, _lib.ptr(ws), ws.numel(), _lib.stream_ptr()) == 0, 'batch %d: error flag' % i
    # 3. bookkeeping
    np.testing.assert_array_equal(fed_actions.cpu().numpy().reshape(-1), fed_prev)
    for got, want in zip(_flat_state(fed_state), fed):
      np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg='batch %d: fed state' % i)
    new = [t.cpu().numpy() for t in _flat_state(new_state)]
    states1, actions1 = self._tables()
    others = np.setdiff1d(np.arange(self.num_envs), ids)
    for t0, t1, nw in zip(states0, states1, new):
      np.testing.assert_array_equal(t1[ids], nw, err_msg='batch %d: state rows' % i)
      np.testing.assert_array_equal(t1[others], t0[others], err_msg='batch %d: other rows' % i)
    np.testing.assert_array_equal(actions1[ids], served)
    np.testing.assert_array_equal(actions1[others], actions0[others])
    np.testing.assert_array_equal(outputs.action.cpu().numpy().reshape(-1) if on_graph or vt else served, served)
    if not vt:
      from oracle import r2d2_oracle
      _, fs1 = r2d2_oracle.stack_frames(env.observation[None].astype(np.float32), self.fs[ids], env.done[None], S)
      self.fs[ids] = fs1
      np.testing.assert_array_equal(states1[2][ids], fs1, err_msg='batch %d: frame-stacking rows' % i)
    # 1. arithmetic against float64 under the GPU's decisions
    inputs = dict(prev_actions=fed_prev[None], reward=env.reward[None], done=env.done[None],
                  observation=env.observation[None], h0=fed[0], c0=fed[1])
    if vt:
      gpu_views = _read_views(agent, self.net, 1, n, ws)
      post = {name: p for _, name, p in _view_names(self.net, agent.conv_mode)}
      views = {k: v for k, v in gpu_views.items() if not k.endswith('/pool')}
      cond = dict(masks={k: v > 0 for k, v in views.items()},
                  taps={k: v for k, v in gpu_views.items() if k.endswith('/pool')})
      fwd = lambda p, x, dt: RV.forward(self.net, p, x, dt, **cond)
      gpu = dict(logits=outputs.policy_logits.cpu().numpy()[None], baseline=outputs.baseline.cpu().numpy()[None],
                 h=new[0], c=new[1])
    else:
      inputs['frame_state'] = fed[2]
      views = self._r2d2_views(ws, n)
      post = {k: True for k in views}
      cond = dict(masks={k: v > 0 for k, v in views.items()})
      fwd = lambda p, x, dt: R2.forward(p, x, A, S, dt, **cond)
      gpu = dict(q=outputs.q_values.cpu().numpy()[None], h=new[0], c=new[1])
    masks, outs = cond['masks'], tuple(gpu)
    shape = lambda r: {k: r['acts'][k] * masks[k] if post[k] else r['acts'][k] for k in views}

    def stages(x, ref):
      e = {k: _relmax(x[k], ref[k]) for k in outs}
      xv, rv = (x['views'] if 'views' in x else shape(x)), shape(ref)
      e.update({'act ' + k: _relmax(xv[k], rv[k]) for k in rv})
      return e
    ref = fwd(self.params, inputs, torch.float64)
    gpu['views'] = views
    errs = stages(gpu, ref)
    m32 = stages(fwd(self.params, inputs, torch.float32), ref)
    if i == RESP_BATCH:
      assert n == self.N
      if (agent.conv_mode if vt else agent.gemm_mode) != 'simt' or agent.lstm_mode == 'tc3':
        pert = (RV.perturbed(self.params, inputs, DELTA) if vt else
                (lambda p, _, b: (p, b))(*R2.perturbed(self.params, {}, inputs, DELTA)))
        self.resp = stages(fwd(pert[0], pert[1], torch.float64), ref)
    rv = shape(ref)
    ties = {k: (v, float(np.abs(rv[k.replace('pool', 'p')]).max())) for k, v in ref['ties'].items()}
    rec = dict(i=i, n=n, errs=errs, m32=m32, ties=ties, prio=None)
    # 2. actions
    if vt:
      want, gap = categorical_sample_np(gpu['logits'][0].astype(np.float64), agent._seed, offset)
      clear = gap > 1e-4
      np.testing.assert_array_equal(served[clear], want[clear], err_msg='batch %d: sampled actions' % i)
      # a score moves by at most the logits' error times their max-abs, a gap by twice that
      want64, gap64 = categorical_sample_np(ref['logits'][0], agent._seed, offset)
      clear64 = clear & (gap64 > 1e-4 + 2 * errs['logits'] * np.abs(ref['logits']).max())
      np.testing.assert_array_equal(served[clear64], want64[clear64], err_msg='batch %d: float64 actions' % i)
      assert n < 16 or clear64.mean() > 0.9
      if not on_graph:
        assert agent._rng_offset == offset + 1
    else:
      q = gpu['q'][0]
      greedy = q.argmax(-1).astype(np.int32)
      rec['greedy'] = (greedy, ref['q'][0])
      if on_graph:
        want = epsilon_greedy_np(greedy, ids, host.envs_epsilon.cpu().numpy(), A, host.epsilon_seed, offset)
      else:
        np.testing.assert_array_equal(outputs.action.cpu().numpy(), greedy)     # the kernel's greedy action
        g = torch.Generator(device='cuda')
        g.set_state(gen_state)
        want = r2d2_learner.apply_epsilon_greedy(torch.as_tensor(greedy).cuda(), torch.as_tensor(ids).cuda(),
                                                 self.ntr, self.num_envs - self.ntr, self.settings.eval_epsilon, A,
                                                 generator=g).cpu().numpy()
      np.testing.assert_array_equal(served, want, err_msg='batch %d: epsilon-greedy actions' % i)
    # 4. completed unrolls
    for k, e in enumerate(ids):
      if reset[k]:
        self.history[e], self.appends[e] = [], 0
      step = dict(prev=fed_prev[k], reward=env.reward[k], done=env.done[k], observation=env.observation[k],
                  episode_step=env.episode_step[k], action=served[k], state=[f[k] for f in fed])
      step.update({key: gpu[key][0][k] for key in (('logits', 'baseline') if vt else ('q',))})
      self.history[e].append(step)
      self.history[e] = self.history[e][-self.L:]
      self.appends[e] += 1
    a = self.appends[ids]
    first = self.L - self.overlap        # a reset store starts an unroll after its `overlap` zero rows
    expect = ids[(ids < self.ntr) & (a >= first) & ((a - first) % self.unroll == 0)]
    got_ids, unrolls = self._completed()
    np.testing.assert_array_equal(got_ids, expect, err_msg='batch %d: completing envs' % i)
    self.completed += len(got_ids)
    prio = []
    for e, u in zip(got_ids, unrolls):
      h = self.history[e]
      pad = self.L - len(h)
      assert pad in (0, self.overlap)
      for key, fld in (('prev', u['prev']), ('reward', u['reward']), ('done', u['done']),
                       ('observation', u['observation']), ('episode_step', u['episode_step']),
                       ('action', u['action'])) + tuple((key, u[key]) for key in
                                                        (('logits', 'baseline') if vt else ('q',))):
        want = np.stack([s[key] for s in h])
        want = np.concatenate([np.zeros((pad,) + want.shape[1:], want.dtype), want])
        np.testing.assert_array_equal(fld, want, err_msg='batch %d env %d %s' % (i, e, key))
      assert not u['abandoned'].any()
      for got, want in zip(u['state'], h[self.overlap - pad]['state']):
        np.testing.assert_array_equal(got, want, err_msg='batch %d env %d: first state' % (i, e))
      if not vt:
        prio.append((u['priority'], u['q'], u['action'], u['reward'], u['done']))
    if prio:
      sl = slice(BURN_IN, None)
      q, act, rew, dn = (np.stack([p[j][sl] for p in prio], axis=1) for j in (1, 2, 3, 4))
      greedy = q.argmax(-1)
      p64, p32 = (R2.priorities(q.astype(F), q.astype(F), act, rew, dn, greedy, self.st, F)
                  for F in (np.float64, np.float32))
      rec['prio'] = (_relmax([p[0] for p in prio], p64), _relmax(p32, p64))
    self.batches.append(rec)

  def _r2d2_views(self, ws, n):
    from seed_rl_b200 import _lib
    shapes = dict(conv0=(n, 20, 20, 32), conv1=(n, 9, 9, 64), conv2=(n, 7, 7, 64), dense=(n, 512 + 1 + A),
                  value=(n, 512), advantage=(n, 512))
    out = {}
    for index, name in enumerate(R2.MASKS):
      off, nb = ctypes.c_size_t(), ctypes.c_size_t()
      _lib.check(_lib.lib().seedrl_debug_r2d2_net_views(self.agent._h, 1, n, index, ctypes.byref(off),
                                                        ctypes.byref(nb)))
      assert nb.value == 4 * int(np.prod(shapes[name]))
      y = ws[off.value:off.value + nb.value].view(torch.float32).reshape(shapes[name])
      out[name] = (y[:, :512] if name == 'dense' else y).cpu().numpy()
    return out

  def _completed(self):
    """(env ids, [{field: numpy [L, ...]}]) of the unrolls the last batch completed."""
    from seed_rl_b200.common import utils
    names = ['prev', 'reward', 'done', 'observation', 'abandoned', 'episode_step', 'action']
    names += ['logits', 'baseline'] if self.vtrace else ['q']
    out = []
    if self.vtrace and self.host.assembler is not None:
      asm = self.host.assembler
      for ids, placed in self._assembled:
        ids = ids.cpu().numpy()
        start = 0
        for slot, col0, room in placed:
          for j in range(room):
            u = {k: asm.field(slot, f)[:, col0 + j].cpu().numpy() for f, k in enumerate(names)}
            u['state'] = [t[col0 + j].cpu().numpy() for t in asm._states[slot]]
            u['id'] = ids[start + j]
            out.append(u)
          start += room
      self._assembled = []
      while asm._ready:                              # hand full batches back, as the learner would
        slot, _, _ = asm.get()
        asm.release(slot)
    else:
      q = self.host.unroll_queue
      for _ in range(q.size()):
        item = q.dequeue()
        flat = [t.cpu().numpy() for t in utils.flatten(item)]
        ns = 2 if self.vtrace else 3
        u = {'state': flat[:ns]}
        if not self.vtrace:
          u['priority'] = flat[ns]
          ns += 1
        u.update(zip(names, flat[ns:]))
        u['id'] = int(u['episode_step'][-1])
        out.append(u)
    return np.array([u['id'] for u in out], np.int64), out

  # ---- bars -------------------------------------------------------------------------------------------------
  def report(self, title):
    """Prints the error / bar table per stage and batch size; -> the failures and the worst error / bar."""
    bad, worst = [], (0.0, None)
    sizes = sorted({b['n'] for b in self.batches})
    table = {}
    # m: the run's largest float32 distance per stage.  One batch's is a poor sample where a stage has few
    # elements: at n = 1 the baseline is one number, and on an H100 deep-simt's float32 distance there was below
    # FLOOR / C while the GPU's error was 1.05e-6 (1.7 fp32 ulps of the largest logit-sized value).
    m = {k: max(b['m32'][k] for b in self.batches) for k in self.batches[0]['m32']}
    if self.resp is not None:
      m = {k: max(m[k], self.resp[k]) for k in m}
    bars = {k: max(FLOOR, C * m[k]) for k in m}
    prio_m = max([b['prio'][1] for b in self.batches if b['prio'] is not None] or [0.0])
    for b in self.batches:
      entries = dict((k, (b['errs'][k], bars[k])) for k in b['errs'])
      if b['prio'] is not None:
        entries['priorities'] = (b['prio'][0], max(FLOOR, C * prio_m))
      for k, (e, bar) in entries.items():
        cur = table.setdefault(k, {}).get(b['n'])
        if cur is None or e / bar > cur[0] / cur[1]:
          table[k][b['n']] = (e, bar)
        if not e <= bar:
          bad.append((b['i'], b['n'], k, e, bar))
        if e / bar > worst[0]:
          worst = (e / bar, (b['n'], k))
      for k, (v, scale) in b['ties'].items():
        stage = 'act ' + k.replace('pool', 'p')
        if v.size and not v.max() / scale <= bars[stage]:
          bad.append((b['i'], b['n'], 'decision ' + k, v.size, float(v.max() / scale), bars[stage]))
      if 'greedy' in b:
        greedy, q64 = b['greedy']
        own = q64.argmax(-1)
        off = np.nonzero(own != greedy)[0]
        gap = (q64[off, own[off]] - q64[off, greedy[off]]) / np.abs(q64).max()
        if off.size and not gap.max() <= bars['q']:
          bad.append((b['i'], b['n'], 'greedy', off.size, float(gap.max()), bars['q']))
    print('%s: error / bar, worst per batch size, C = %g, floor %.0e, m = %s' % (
        title, C, FLOOR, 'float32 reference' if self.resp is None else 'max(float32 reference, 2^-16 response)'))
    print('  %-28s' % 'stage' + ''.join('%22s' % ('n = %d' % n) for n in sizes))
    for k, row in table.items():
      print('  %-28s' % k + ''.join('%22s' % ('%.2e / %.2e' % row[n] if n in row else '-') for n in sizes))
    print('  worst error / bar %.2f (n = %s, %s); %d unrolls completed' % (worst[0], worst[1][0], worst[1][1],
                                                                          self.completed))
    return bad, worst


def _check(kind, mode, host_kind, N):
  r = _Run(kind, mode, host_kind, N).run()
  assert {1, 63}.issubset(r.sizes) and N in r.sizes and (N < 256 or 65 in r.sizes)
  bad, _ = r.report('%s INFERENCE FLOAT64 %s %s host N=%d' % (kind.upper(), mode, host_kind, N))
  del r
  torch.cuda.empty_cache()
  assert not bad, bad


@pytest.mark.parametrize('N', [64, 256])
@pytest.mark.parametrize('host_kind', ['graph', 'eager'])
@pytest.mark.parametrize('mode', list(VTRACE))
def test_vtrace_inference_matches_float64(mode, host_kind, N):
  _check('vtrace', mode, host_kind, N)


@pytest.mark.parametrize('N', [64, 256])
@pytest.mark.parametrize('host_kind', ['graph', 'eager'])
@pytest.mark.parametrize('mode', list(R2D2))
def test_r2d2_inference_matches_float64(mode, host_kind, N):
  _check('r2d2', mode, host_kind, N)


@pytest.mark.parametrize('kind,mode,name', [('vtrace', 'deep-simt', 'policy_logits/kernel'),
                                            ('r2d2', 'simt', 'advantage/head/kernel')])
def test_a_head_scaled_by_one_part_in_4096_fails_its_bar(kind, mode, name):
  """The comparison can fail: the GPU agent's policy-logits (R2D2: advantage-head) kernel scaled by 1 + 2^-12, the
  reference's unchanged, over the first five batches of the eager host at N = 64, in the fp32 modes.  (The
  parameters' biases are zero, so a bias would not do.)  The output stage exceeds its bar on every batch; the
  activations before the head do not."""
  r = _Run(kind, mode, 'eager', 64, calls=RESP_BATCH + 1, mutate=name).run()
  bad, _ = r.report('%s INFERENCE FLOAT64 %s, %s scaled by 1 + 2^-12' % (kind.upper(), mode, name))
  out = 'logits' if kind == 'vtrace' else 'q'
  assert {b[0] for b in bad if b[2] == out} == set(range(RESP_BATCH + 1)), bad
  assert not [b for b in bad if b[2].startswith('act ')], bad
