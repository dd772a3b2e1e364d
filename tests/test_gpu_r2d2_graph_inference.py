"""GPU: R2D2 central inference as one CUDA-graph replay per batch (R2D2InferenceHost(cuda_graph=True)):
the device epsilon-greedy kernel against a numpy restatement of its Philox draw, the eval-aware store
append, bit-for-bit parity with the eager host in greedy mode (also with partial batches of two other
sizes, through which the graph host keeps the workspace it captured), exploration statistics,
reproducibility, two hosts sharing one agent, and the hand-off to the replay and the learner."""
import threading

import numpy as np
import pytest
import torch

from seed_rl_b200 import _lib
from seed_rl_b200.agents.r2d2 import learner, learner_loop
from seed_rl_b200.atari import networks
from seed_rl_b200.common import optimizers, utils

pytestmark = pytest.mark.gpu

MASK32 = np.uint64(0xFFFFFFFF)


def philox4x32_10(c0, c1, c2, c3, k0, k1):
  """Philox4x32-10 on uint64 arrays holding 32-bit words (common.cuh)."""
  c0, c1, c2, c3, k0, k1 = (np.asarray(x, np.uint64) & MASK32 for x in (c0, c1, c2, c3, k0, k1))
  M0, M1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57)
  W0, W1 = np.uint64(0x9E3779B9), np.uint64(0xBB67AE85)
  for _ in range(10):
    p0, p1 = M0 * c0, M1 * c2
    c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & MASK32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & MASK32)
    k0, k1 = (k0 + W0) & MASK32, (k1 + W1) & MASK32
  return c0, c1, c2, c3


def epsilon_greedy_np(greedy, env_ids, envs_epsilon, A, seed, counter):
  """seedrl_r2d2_epsilon_greedy: row n draws r = philox((counter lo, counter hi, n, 0), seed)."""
  n = np.arange(len(greedy), dtype=np.uint64)
  c, s = np.uint64(counter), np.uint64(seed)
  x, y, _, _ = philox4x32_10(c & MASK32, c >> np.uint64(32), n, 0, s & MASK32, s >> np.uint64(32))
  u = (x >> np.uint64(8)).astype(np.float32) * np.float32(2.0 ** -24)
  explore = u < np.asarray(envs_epsilon, np.float32)[env_ids]
  rand = ((y * np.uint64(A)) >> np.uint64(32)).astype(np.int32)
  return np.where(explore, rand, greedy).astype(np.int32)


def categorical_sample_np(logits, seed, offset):
  """seedrl_categorical_sample (Gumbel-max, Philox counter = (offset lo, offset hi, row, j // 4)) in
  float64; returns (actions, gap between the two best scores)."""
  N, A = logits.shape
  scores = np.empty((N, A))
  o, s = np.uint64(offset), np.uint64(seed)
  for j0 in range(0, A, 4):
    r = philox4x32_10(o & MASK32, o >> np.uint64(32), np.arange(N, dtype=np.uint64), j0 // 4, s & MASK32,
                      s >> np.uint64(32))
    for k in range(4):
      if j0 + k < A:
        u = (r[k].astype(np.float32) + np.float32(0.5)) * np.float32(2.3283064365386963e-10)
        u = np.minimum(np.maximum(u, np.float32(1e-10)), np.float32(0.99999994)).astype(np.float64)
        scores[:, j0 + k] = logits[:, j0 + k] - np.log(-np.log(u))
  top2 = np.sort(scores, axis=1)[:, -2:]
  return scores.argmax(1), top2[:, 1] - top2[:, 0]


# ---- 1. kernel ---------------------------------------------------------------------------------
@pytest.mark.parametrize('N', [3, 64, 300])
@pytest.mark.parametrize('A', [6, 18])
def test_epsilon_greedy_kernel_matches_philox_restatement(N, A):
  rng = np.random.default_rng(N * 31 + A)
  num_training, num_eval = 320, 80
  table = learner.get_envs_epsilon(torch.arange(num_training + num_eval).cuda(), num_training, num_eval, 0.5)
  table_np = table.cpu().numpy()
  ids = rng.permutation(num_training + num_eval)[:N].astype(np.int32)          # training and eval ids mixed
  assert (ids < num_training).any() and (ids >= num_training).any() or N == 3
  greedy = rng.integers(0, A, N).astype(np.int32)
  ids_dev = torch.as_tensor(ids).cuda()
  seed, c0 = 0x0123456789ABCDEF, (1 << 32) + 5                                 # both words of seed and counter
  counter = torch.tensor(c0, dtype=torch.int64).cuda()
  outs = []
  for k in range(3):
    act = torch.as_tensor(greedy).cuda()
    learner.device_epsilon_greedy(act, ids_dev, table, A, seed, counter)
    assert int(counter) == c0 + k + 1                                          # advanced by exactly one
    want = epsilon_greedy_np(greedy, ids, table_np, A, seed, c0 + k)
    np.testing.assert_array_equal(act.cpu().numpy(), want)
    outs.append(want)
  assert not np.array_equal(outs[0], outs[1]) or N == 3
  # the same counter value gives the same actions
  counter.fill_(c0)
  act = torch.as_tensor(greedy).cuda()
  learner.device_epsilon_greedy(act, ids_dev, table, A, seed, counter)
  np.testing.assert_array_equal(act.cpu().numpy(), outs[0])
  # all-explore and never-explore tables
  act = torch.as_tensor(greedy).cuda()
  learner.device_epsilon_greedy(act, ids_dev, torch.ones_like(table), A, seed, counter)
  np.testing.assert_array_equal(act.cpu().numpy(), epsilon_greedy_np(greedy, ids, np.ones_like(table_np), A, seed,
                                                                     c0 + 1))
  act = torch.as_tensor(greedy).cuda()
  learner.device_epsilon_greedy(act, ids_dev, torch.zeros_like(table), A, seed, counter)
  np.testing.assert_array_equal(act.cpu().numpy(), greedy)


def test_categorical_sampler_bits_against_philox_restatement():
  """The Gumbel-max sampler draws from the same (shared) Philox: its actions on fixed (seed, offset)
  are those of the float64 restatement wherever the two best scores are apart by more than the
  float32 rounding of the scores."""
  rng = np.random.default_rng(5)
  N, A = 512, 18
  logits = rng.normal(size=(N, A)).astype(np.float32)
  lg = torch.as_tensor(logits).cuda()
  for seed, offset in ((0, 0), (0x0123456789ABCDEF, (1 << 32) + 7), (42, 3)):
    act = torch.empty(N, dtype=torch.int64).cuda()
    _lib.check(_lib.lib().seedrl_categorical_sample(N, A, _lib.ptr(lg), None, seed, offset, _lib.ptr(act),
                                                    _lib.stream_ptr()))
    want, gap = categorical_sample_np(logits.astype(np.float64), seed, offset)
    clear = gap > 1e-4
    assert clear.mean() > 0.98
    np.testing.assert_array_equal(act.cpu().numpy()[clear], want[clear])
    counter = torch.tensor(offset, dtype=torch.int64).cuda()
    act2 = torch.empty(N, dtype=torch.int64).cuda()
    _lib.check(_lib.lib().seedrl_categorical_sample_counter(N, A, _lib.ptr(lg), None, seed, _lib.ptr(counter),
                                                            _lib.ptr(act2), _lib.stream_ptr()))
    assert torch.equal(act, act2) and int(counter) == offset + 1


# ---- 2. eval-aware store append ----------------------------------------------------------------
def test_device_append_with_id_limit_equals_append_of_training_subset():
  k, num_envs, unroll, overlap = 5, 8, 3, 2
  specs = (utils.TensorSpec([], 'int32', 'a'), utils.TensorSpec([3], 'float32', 'b'),
           utils.TensorSpec([5], 'uint8', 'c'))
  masked = utils.UnrollStore(num_envs, unroll, specs, num_overlapping_steps=overlap)   # has rows for eval ids too
  eager = utils.UnrollStore(k, unroll, specs, num_overlapping_steps=overlap)
  rng = np.random.default_rng(0)
  for step in range(17):
    ids = rng.permutation(num_envs)[:6].astype(np.int32)
    vals = (rng.integers(0, 100, 6).astype(np.int32), rng.normal(size=(6, 3)).astype(np.float32),
            rng.integers(0, 256, (6, 5)).astype(np.uint8))
    if step == 9:
      masked.reset([1]); eager.reset([1])
    masked.device_append(torch.as_tensor(ids).cuda(), [torch.as_tensor(v).cuda() for v in vals], id_limit=k)
    tr = np.nonzero(ids < k)[0]
    done_host, pos = masked.host_advance(ids[tr])
    got_ids, got = masked.complete(int(done_host.size))
    want_ids, want = eager.append(ids[tr], tuple(torch.as_tensor(v[tr]).cuda() for v in vals))
    assert got_ids.tolist() == want_ids.tolist() == done_host.tolist()          # batch order of the kept rows
    np.testing.assert_array_equal(ids[tr][pos], done_host)
    for a, b in zip(utils.flatten(got), utils.flatten(want)):
      assert torch.equal(a, b)
    for a, b in zip(masked._state, eager._state):
      assert torch.equal(a[:k], b)
      assert int(a[k:].abs().max()) == 0                                          # eval rows never touched
    assert torch.equal(masked._index[:k], eager._index)
    assert masked._index[k:].tolist() == [overlap] * (num_envs - k)


# ---- shared driver -----------------------------------------------------------------------------
def make_host(agent, obs, N, num_envs, num_eval, st, **kw):
  return learner_loop.R2D2InferenceHost(agent, num_envs=num_envs, num_eval_envs=num_eval, inference_batch_size=N,
                                        observation_shape=obs, settings=st, unroll_queue_max_size=-1, **kw)


def call_sequence(obs, num_envs, batches, calls, seed, done_p=0.05, partial_at=None, reset_at=None):
  """The inputs of `calls` inference calls cycling over `batches` (arrays of env ids).  episode_step
  carries the env id, so that a stored unroll can be attributed to its env."""
  rng = np.random.default_rng(seed)
  run_ids = rng.integers(1, 2**40, num_envs)
  seq = []
  for i in range(calls):
    ids = batches[i % len(batches)]
    if i == partial_at:
      ids = ids[:len(ids) // 2 + 1]
    if i == reset_at:                          # actors restarted: new run ids (for training and eval envs)
      run_ids[ids[::max(1, len(ids) // 2)]] += 1
    n = len(ids)
    env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), rng.random(n) < done_p,
                          rng.integers(0, 256, (n,) + obs, dtype=np.uint8), np.zeros(n, bool), ids.astype(np.int32))
    seq.append((ids, run_ids[ids].copy(), env, rng.normal(size=n).astype(np.float32)))
  return seq


def drain(host):
  return [host.unroll_queue.dequeue() for _ in range(host.unroll_queue.size())]


# ---- 3. greedy parity, graph vs eager ----------------------------------------------------------
TOY = dict(A=6, obs=(36, 36, 1), S=4, N=4, num_envs=7, num_eval=2, unroll=4, burn_in=2, calls=60)
CFG5 = dict(A=18, obs=(84, 84, 1), S=4, N=64, num_envs=80, num_eval=16, unroll=100, burn_in=40, calls=206)


@pytest.mark.parametrize('gemm_mode', ['tc3', 'simt'])
@pytest.mark.parametrize('shape', ['toy', 'cfg5'])
def test_graph_host_equals_eager_host_in_greedy_mode(shape, gemm_mode, monkeypatch):
  c = TOY if shape == 'toy' else CFG5
  st = learner.default_settings(unroll_length=c['unroll'], burn_in=c['burn_in'])
  agent = networks.DuelingLSTMDQNNet(c['A'], c['obs'], c['S'], seed=1, gemm_mode=gemm_mode)
  monkeypatch.setattr(learner, 'apply_epsilon_greedy', lambda actions, *a, **k: actions)
  eager = make_host(agent, c['obs'], c['N'], c['num_envs'], c['num_eval'], st)
  graph = make_host(agent, c['obs'], c['N'], c['num_envs'], c['num_eval'], st, cuda_graph=True)
  graph.envs_epsilon.zero_()
  if shape == 'toy':
    rng = np.random.default_rng(3)
    batches = [rng.permutation(c['num_envs'])[:c['N']].astype(np.int32) for _ in range(5)]
  else:      # ids 0..15 are only in the first batch: 206 calls give each of them 103 steps (> 101)
    batches = [np.arange(0, 64, dtype=np.int32), np.arange(16, 80, dtype=np.int32)[::-1].copy()]
  seq = call_sequence(c['obs'], c['num_envs'], batches, c['calls'], seed=11, partial_at=c['calls'] // 3,
                      reset_at=c['calls'] // 2)
  for i, (ids, run_ids, env, raw) in enumerate(seq):
    a = eager.inference(ids, run_ids, env, raw)
    b = graph.inference(ids, run_ids, env, raw)
    assert a.dtype == b.dtype == np.int32
    np.testing.assert_array_equal(a, b, err_msg='call %d' % i)
  assert graph._graph is not None
  for x, y in ((eager.first_agent_states, graph.first_agent_states), (eager.agent_states, graph.agent_states),
               (eager.actions, graph.actions)):
    for t, u in zip(x._state, y._state):
      assert torch.equal(t, u), x.name
  for t, u in zip(eager.store._state + [eager.store._index], graph.store._state + [graph.store._index]):
    assert torch.equal(t, u)
  assert np.array_equal(eager.store._host_index, graph.store._host_index)
  for t, u in zip(eager.env_infos, graph.env_infos):
    assert np.array_equal(t, u)
  qa, qb = drain(eager), drain(graph)
  assert len(qa) == len(qb) > 0
  if shape == 'cfg5':                                                         # every training env completed one
    assert {int(u.env_outputs.episode_step[-1]) for u in qa} == set(range(c['num_envs'] - c['num_eval']))
  for u, v in zip(qa, qb):
    for t1, t2 in zip(utils.flatten(u), utils.flatten(v)):
      assert torch.equal(t1, t2)
  assert eager.info_queue.size() == graph.info_queue.size() > 0
  agent.check_errors()


def test_graph_host_keeps_its_workspace_through_partial_batches_of_two_sizes(monkeypatch):
  """Eager partial batches of two other sizes between full batches evict the (1, N) workspace the graph
  captured from the agent's cache (each thread keeps two shapes).  The host holds that workspace itself, so
  every replay still writes into memory it owns: actions, tables and unrolls equal an eager host's."""
  c = TOY
  st = learner.default_settings(unroll_length=c['unroll'], burn_in=c['burn_in'])
  monkeypatch.setattr(learner, 'apply_epsilon_greedy', lambda actions, *a, **k: actions)
  eager = make_host(networks.DuelingLSTMDQNNet(c['A'], c['obs'], c['S'], seed=1), c['obs'], c['N'], c['num_envs'],
                    c['num_eval'], st)
  agent = networks.DuelingLSTMDQNNet(c['A'], c['obs'], c['S'], seed=1)
  captured, workspace = [], agent.workspace

  def recording_workspace(T1, B):
    ws = workspace(T1, B)
    if torch.cuda.is_current_stream_capturing():
      captured.append(ws)
    return ws
  monkeypatch.setattr(agent, 'workspace', recording_workspace)
  graph = make_host(agent, c['obs'], c['N'], c['num_envs'], c['num_eval'], st, cuda_graph=True)
  graph.envs_epsilon.zero_()
  rng = np.random.default_rng(5)
  batches = [rng.permutation(c['num_envs'])[:n].astype(np.int32) for n in (c['N'], 2, c['N'], 3)]
  evicted = False
  for i, (ids, run_ids, env, raw) in enumerate(call_sequence(c['obs'], c['num_envs'], batches, 40, seed=6)):
    np.testing.assert_array_equal(eager.inference(ids, run_ids, env, raw), graph.inference(ids, run_ids, env, raw),
                                  err_msg='call %d' % i)
    if captured:
      cached = agent._workspaces[threading.get_ident()].values()
      evicted |= not any(ws is captured[0] for ws in cached)
  assert len(captured) == 1 and graph._g_workspace is captured[0]
  assert evicted                                                   # the case this test is about happened
  for x, y in ((eager.first_agent_states, graph.first_agent_states), (eager.agent_states, graph.agent_states),
               (eager.actions, graph.actions)):
    for t, u in zip(x._state, y._state):
      assert torch.equal(t, u), x.name
  for t, u in zip(eager.store._state + [eager.store._index], graph.store._state + [graph.store._index]):
    assert torch.equal(t, u)
  qa, qb = drain(eager), drain(graph)
  assert len(qa) == len(qb) > 0
  for u, v in zip(qa, qb):
    for t1, t2 in zip(utils.flatten(u), utils.flatten(v)):
      assert torch.equal(t1, t2)
  agent.check_errors()


# ---- 4. exploration statistics -----------------------------------------------------------------
def test_exploration_rate_per_env_matches_schedule():
  """With the reference schedule (0.4 ** linspace(1, 8) for the training envs, eval_epsilon for the
  eval envs), the rate at which the recorded action differs from the argmax of the q-values is
  eps * (A - 1) / A per env.  Fixed seed; tolerance 5 binomial standard deviations + 2 / n."""
  A, obs, S, num_envs, num_eval, calls = 6, (36, 36, 1), 4, 10, 2, 3000
  st = learner.default_settings(unroll_length=20, burn_in=4, eval_epsilon=0.25)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=2)
  host = make_host(agent, obs, num_envs, num_envs, num_eval, st, cuda_graph=True, epsilon_seed=12345)
  ntr = num_envs - num_eval
  ids = np.arange(num_envs, dtype=np.int32)
  rng = np.random.default_rng(4)
  run_ids = rng.integers(1, 2**40, num_envs)
  frames = [rng.integers(0, 256, (num_envs,) + obs, dtype=np.uint8) for _ in range(16)]
  diff, cnt = np.zeros(num_envs), np.zeros(num_envs)
  for i in range(calls):
    env = utils.EnvOutput(rng.normal(size=num_envs).astype(np.float32), rng.random(num_envs) < 0.02, frames[i % 16],
                          np.zeros(num_envs, bool), ids.copy())       # episode_step = env id
    act = host.inference(ids, run_ids, env, np.zeros(num_envs, np.float32))
    # eval envs have no store rows: their q-values are the graph's output of this call
    greedy = host._g_out.q_values.argmax(1).cpu().numpy()
    diff[ntr:] += (act != greedy)[ntr:]
    cnt[ntr:] += 1
  # training envs: the recorded actions and q-values of the stored unrolls; the rows after the
  # overlap are new in every unroll
  for u in drain(host):
    e = int(u.env_outputs.episode_step[-1])
    a = u.agent_outputs.action[st.burn_in + 1:].cpu().numpy()
    q = u.agent_outputs.q_values[st.burn_in + 1:].cpu().numpy()
    diff[e] += (a != q.argmax(1)).sum()
    cnt[e] += len(a)
  eps = host.envs_epsilon.cpu().numpy().astype(np.float64)
  np.testing.assert_allclose(eps[:ntr], 0.4 ** np.linspace(1, 8, ntr), rtol=1e-5)
  assert (eps[ntr:] == np.float32(0.25)).all()
  p = eps * (A - 1) / A
  assert cnt[:ntr].min() > 2500 and (cnt[ntr:] == calls).all()
  rate = diff / cnt
  tol = 5 * np.sqrt(p * (1 - p) / cnt) + 2 / cnt
  assert (np.abs(rate - p) <= tol).all(), (rate, p, tol)


# ---- 5. reproducibility ------------------------------------------------------------------------
def test_same_epsilon_seed_same_actions():
  A, obs, S, N, num_envs = 6, (36, 36, 1), 4, 8, 12
  st = learner.default_settings(unroll_length=5, burn_in=2)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=3)
  batches = [np.arange(0, 8, dtype=np.int32), np.arange(4, 12, dtype=np.int32)]
  seq = call_sequence(obs, num_envs, batches, 40, seed=5)
  streams = []
  for seed in (7, 7, 8):
    host = make_host(agent, obs, N, num_envs, 2, st, cuda_graph=True, epsilon_seed=seed)
    streams.append(np.stack([host.inference(*x) for x in seq]))
  assert np.array_equal(streams[0], streams[1])
  assert not np.array_equal(streams[0], streams[2])


# ---- 6. two hosts sharing one agent ------------------------------------------------------------
def test_two_graph_hosts_on_two_threads_equal_each_host_alone():
  A, obs, S, N, num_envs = 6, (36, 36, 1), 4, 8, 16
  st = learner.default_settings(unroll_length=5, burn_in=2)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=4)
  batches = [np.arange(0, 8, dtype=np.int32), np.arange(8, 16, dtype=np.int32)]
  seqs = [call_sequence(obs, num_envs, batches, 50, seed=20 + k, reset_at=25) for k in range(2)]

  def new_host():
    h = make_host(agent, obs, N, num_envs, 3, st, cuda_graph=True)
    h.envs_epsilon.zero_()
    return h
  alone = []
  for k in range(2):
    h = new_host()
    alone.append(([h.inference(*x) for x in seqs[k]], drain(h)))
  capture_lock = threading.Lock()
  gate = threading.Barrier(2)
  together, errors = [None, None], []

  def lane(k):
    try:
      h = new_host()
      with capture_lock:                      # one host captures its graph at a time
        out = [h.inference(*seqs[k][0])]
      gate.wait(120)
      out += [h.inference(*x) for x in seqs[k][1:]]
      together[k] = (out, drain(h))
    except Exception as exc:                  # pylint: disable=broad-except
      errors.append(exc)
      gate.abort()
  threads = [threading.Thread(target=lane, args=(k,)) for k in range(2)]
  for th in threads:
    th.start()
  for th in threads:
    th.join(300)
  assert not errors, errors
  for k in range(2):
    assert len(together[k][0]) == len(alone[k][0])
    for a, b in zip(alone[k][0], together[k][0]):
      np.testing.assert_array_equal(a, b)
    assert len(alone[k][1]) == len(together[k][1]) > 0
    for u, v in zip(alone[k][1], together[k][1]):
      for t1, t2 in zip(utils.flatten(u), utils.flatten(v)):
        assert torch.equal(t1, t2)


# ---- 7. end to end -----------------------------------------------------------------------------
def test_graph_host_feeds_replay_and_learner():
  """As test_gpu_r2d2.py's host test, with the graph host: its unrolls go through the replay to one
  learner step."""
  A, obs, S = 6, (36, 36, 1), 4
  st = learner.default_settings(batch_size=6, replay_ratio=1.5, unroll_length=4, burn_in=2, replay_buffer_size=16,
                                replay_buffer_min_size=4, update_target_every_n_step=10**9)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=1, gemm_mode='simt')
  target = networks.DuelingLSTMDQNNet(A, obs, S, seed=1, gemm_mode='simt')
  host = learner_loop.R2D2InferenceHost(agent, num_envs=6, num_eval_envs=1, inference_batch_size=3,
                                        observation_shape=obs, settings=st, cuda_graph=True, epsilon_seed=9)
  seq = call_sequence(obs, 6, [np.array([0, 1, 2], np.int32), np.array([5, 3, 4], np.int32)], 26, seed=0, done_p=0.1)
  for x in seq:
    act = host.inference(*x)
    assert act.shape == (3,) and act.dtype == np.int32 and (0 <= act).all() and (act < A).all()
  assert host.unroll_queue.size() == 15          # as the eager host: 3 unrolls for each of 5 training envs
  replay = utils.PrioritizedReplay(st.replay_buffer_size, host.unroll_specs, st.importance_sampling_exponent)
  feeder = learner.ReplayFeeder(replay, st, generator=torch.Generator(device='cuda').manual_seed(1))
  assert learner_loop.fill_replay(host, feeder) and feeder.ready() and replay.num_inserted == 4
  assert learner_loop.fill_replay(host, feeder) and replay.num_inserted == 8
  assert float(replay._priorities[:8].min()) > 0
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(1e-3, epsilon=1e-3), settings=st)
  sampled = feeder.sample()
  loss, priorities, indices, norm = step.minimize(sampled)
  feeder.update_priorities(indices, priorities)
  agent.check_errors()
  assert np.isfinite(float(loss)) and np.isfinite(float(norm)) and bool((priorities >= 0).all())
  assert torch.equal(replay._priorities[indices], priorities) or len(set(indices.tolist())) < len(indices)
