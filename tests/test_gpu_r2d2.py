"""GPU: R2D2 post-network kernels (SURVEY 8(a) row a11) against oracle/r2d2_oracle.py."""
import numpy as np
import pytest
import torch

import test_gpu_r2d2_loss_float64 as LF
from oracle import r2d2_oracle as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize('T,B,H,W,S', [(6, 2, 3, 4, 4), (9, 3, 5, 2, 3), (4, 1, 2, 2, 2), (20, 4, 84, 84, 4), (1, 2, 3, 3, 4)])
def test_stack_frames_bit_exact(T, B, H, W, S):
  from seed_rl_b200.atari import networks
  rng = np.random.default_rng(T + B)
  fr = rng.integers(0, 256, (T, B, H, W, 1), dtype=np.uint8)
  dn = rng.random((T, B)) < 0.3
  st = rng.integers(0, 1 << (8 * (S - 1)), (B, H * W)).astype(np.int32)
  want, want_state = R.stack_frames(fr.astype(np.float32), st, dn, S)
  got, got_state = networks.stack_frames(torch.as_tensor(fr).cuda(), torch.as_tensor(st).cuda(),
                                         torch.as_tensor(dn).cuda(), S)
  np.testing.assert_array_equal(got.cpu().numpy(), want.astype(np.uint8))
  np.testing.assert_array_equal(got_state.cpu().numpy(), want_state)
  # the reference's known-answer sequence (atari/networks_test.py:176-247) chained through the state
  z = networks.initial_frame_stacking_state(4, 1, [1])
  f = lambda v: torch.tensor(v, dtype=torch.uint8).reshape(len(v), 1, 1).cuda()
  d = lambda v: torch.tensor(v).reshape(len(v), 1).cuda()
  o, s = networks.stack_frames(f([1]), z, d([False]), 4)
  o, s = networks.stack_frames(f([2]), s, d([True]), 4)
  assert o.flatten().tolist() == [2, 0, 0, 0]
  o, s = networks.stack_frames(f([3, 4, 5, 6, 7, 8]), s, d([False, False, False, False, True, False]), 4)
  assert o[0].flatten().tolist() == [3, 2, 0, 0] and o[5].flatten().tolist() == [8, 7, 0, 0]


@pytest.mark.parametrize('q', [1.0, 1e-3])
@pytest.mark.parametrize('T,B,A,n', [(16, 6, 18, 5), (101, 64, 18, 5), (4, 2, 3, 5), (12, 3, 4, 1)])
def test_loss_and_priorities_vs_float64(T, B, A, n, q):
  """Loss, priorities and dq against the float64 loss of test_gpu_r2d2_loss_float64.py, with its bars (not against
  oracle/r2d2_oracle.py's float32 loss, whose h^-1 cancels), at Q values of scale 1 and 1e-3; dq is the gradient
  of mean_b(w_b loss_b): -(w_b / B) * td on the replayed action, zero elsewhere and on the last row."""
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  rng = np.random.default_rng(T + A)
  tq = (rng.normal(size=(T, B, A)) * q).astype(np.float32); gq = (rng.normal(size=(T, B, A)) * q).astype(np.float32)
  ra = rng.integers(0, A, (T, B)); r = rng.normal(size=(T, B)).astype(np.float32); d = rng.random((T, B)) < 0.1
  w = rng.random(B).astype(np.float32) + 0.1
  c = lambda a: torch.as_tensor(a).cuda()
  env = utils.EnvOutput(c(r), c(d), None, None, None)
  got_loss, got_prio, dq = learner.compute_loss_and_priorities_from_agent_outputs(
      learner.AgentOutput(None, c(tq)), learner.AgentOutput(None, c(gq)), env, learner.AgentOutput(c(ra), None),
      0.997, n_steps=n, importance_weights=c(w))
  LF.check_outputs(dict(loss=got_loss.cpu().numpy(), priorities=got_prio.cpu().numpy(), dq=dq.cpu().numpy()),
                   (tq, gq, ra, r, d, w), 'n_step', n, 0.997, 0.9, 1e-3)


def test_replay_sample_and_clip():
  from seed_rl_b200.agents.r2d2 import learner
  rng = np.random.default_rng(0)
  prio = rng.random(100).astype(np.float32) + 0.01
  u = rng.random(4096).astype(np.float32)
  idx, wts, probs = learner.replay_sample(torch.as_tensor(prio).cuda(), 70, 4096, 0.9, 0.6, uniforms=torch.as_tensor(u).cuda())
  p = R.replay_probabilities(prio, 70, 0.9)
  np.testing.assert_allclose(probs.cpu().numpy(), p, rtol=5e-5)   # powf vs numpy power: 1.3e-5 seen
  i = idx.cpu().numpy()
  assert i.min() >= 0 and i.max() < 70
  np.testing.assert_allclose(wts.cpu().numpy(), R.replay_importance_weights(p, i, 0.6), rtol=5e-5)
  # inverse-CDF draw: index = first i with cdf_i > u * total
  cdf = np.cumsum(np.power(prio[:70], np.float32(0.9), dtype=np.float32), dtype=np.float32)
  np.testing.assert_array_equal(i, np.minimum(np.searchsorted(cdf, u * cdf[-1], side='right'), 69))
  freq = np.bincount(i, minlength=70) / len(i)
  assert np.abs(freq - p).max() < 0.02                                   # statistical, like utils_test.py
  g = rng.normal(size=1 << 20).astype(np.float32)
  gc = torch.as_tensor(g).cuda()
  norm = learner.clip_by_global_norm(gc, 40.0)
  n64 = np.sqrt((g.astype(np.float64) ** 2).sum())
  np.testing.assert_allclose(float(norm), n64, rtol=1e-5)
  np.testing.assert_allclose(gc.cpu().numpy(), g * np.float32(40.0 / max(n64, 40.0)), rtol=1e-5)


# ---- DuelingLSTMDQNNet (csrc/r2d2_net.cu) and the cfg-5 learner step vs the CPU oracle -----------
def _net_case(T, B, A, obs, S, seed, done_p=0.15):
  from oracle import r2d2_learner_oracle as RL, r2d2_net_oracle as NO
  params = NO.init_params(A, obs, S, seed=seed)
  b = RL.synthetic_replay_batch(T, B, A, obs, seed=seed + 1, done_p=done_p)
  return params, b


def _to_cuda_inputs(b, S):
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import utils
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  T, B = b['reward'].shape
  env = utils.EnvOutput(c(b['reward']), c(b['done']), c(b['observation']),
                        torch.zeros(T, B, dtype=torch.bool).cuda(), torch.zeros(T, B, dtype=torch.int32).cuda())
  state = networks.AgentState((c(b['h0']), c(b['c0'])), c(b['frame_state']) if S > 1 else ())
  return c(b['prev_actions']), env, state


@pytest.mark.parametrize('mode,tol', [('simt', 2e-4), ('tc3', 5e-4)])
@pytest.mark.parametrize('T,B,A,obs,S', [(5, 3, 6, (36, 36, 1), 4), (3, 2, 18, (84, 84, 1), 4), (4, 2, 4, (44, 40, 4), 1)])
def test_dueling_net_forward_backward_vs_oracle(mode, tol, T, B, A, obs, S):
  from oracle import r2d2_net_oracle as NO
  from seed_rl_b200.atari import networks
  params, b = _net_case(T, B, A, obs, S, seed=T + A)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, gemm_mode=mode)
  assert len(agent.trainable_variables) == 18          # 3 advantage + 8 body + 3 core + 4 value (head has no bias)
  agent.load_named_parameters(params)
  pa, env, state = _to_cuda_inputs(b, S)
  out, new_state = agent((pa, env), state, unroll=True, is_training=True)
  agent.check_errors()
  pt = {k: torch.tensor(v, requires_grad=True) for k, v in params.items()}
  fs = b['frame_state'] if S > 1 else ()
  want, want_state = NO.unroll(pt, b['prev_actions'], b['reward'], b['done'], b['observation'],
                               NO.AgentState((torch.as_tensor(b['h0']), torch.as_tensor(b['c0'])), fs), A, S)
  q, wq = out.q_values.cpu().numpy(), want.q_values.detach().numpy()
  scale = np.abs(wq).max()
  assert np.abs(q - wq).max() <= tol * scale + 1e-6, np.abs(q - wq).max() / scale
  # greedy action: bit-exact wherever the top-2 gap of the oracle exceeds the forward tolerance
  srt = np.sort(wq, axis=-1)
  clear = (srt[..., -1] - srt[..., -2]) > 4 * tol * scale
  np.testing.assert_array_equal(out.action.cpu().numpy()[clear], want.action.numpy()[clear])
  np.testing.assert_array_equal(out.action.cpu().numpy(), q.argmax(-1))       # argmax of its own Q, first max
  np.testing.assert_allclose(new_state.core_state[0].cpu().numpy(), want_state.core_state[0].detach().numpy(),
                             atol=tol)
  np.testing.assert_allclose(new_state.core_state[1].cpu().numpy(), want_state.core_state[1].detach().numpy(),
                             atol=2 * tol)
  if S > 1:
    np.testing.assert_array_equal(new_state.frame_stacking_state.cpu().numpy(), want_state.frame_stacking_state)
  # backward: random dq
  rng = np.random.default_rng(3)
  dq = rng.normal(size=wq.shape).astype(np.float32)
  (want.q_values * torch.as_tensor(dq)).sum().backward()
  agent.backward(torch.as_tensor(dq).cuda())
  agent.check_errors()
  mine = agent.named_gradients()
  # tolerance: per tensor max|a-w|/max|w| <= gtol, or 4x the oracle's own sensitivity to relative
  # parameter perturbations of the size of the mode's arithmetic (1e-6 for fp32 SIMT, 2^-15 for
  # bf16x3).  A tiny random batch sits on ReLU kinks: a pre-activation within rounding of zero
  # flips its mask and moves a whole gradient column by percents (this seed has
  # a value/hidden unit on the kink -- the fp32 oracle itself moves 4e-2 there under a 1e-7
  # perturbation), so several probes are taken and the largest response bounds the comparison.
  gtol = {'simt': 2e-3, 'tc3': 5e-3}[mode]
  sens = {k: 0.0 for k in pt}
  for seed_, eps_ in ((0, 1e-6), (1, 1e-6), (2, 1e-6), (3, {'simt': 1e-6, 'tc3': 3e-5}[mode])):
    prng = np.random.default_rng(seed_)
    pt2 = {k: torch.tensor((v * (1 + eps_ * prng.normal(size=v.shape))).astype(np.float32), requires_grad=True)
           for k, v in params.items()}
    want2, _ = NO.unroll(pt2, b['prev_actions'], b['reward'], b['done'], b['observation'],
                         NO.AgentState((torch.as_tensor(b['h0']), torch.as_tensor(b['c0'])), fs), A, S)
    (want2.q_values * torch.as_tensor(dq)).sum().backward()
    for k, v in pt.items():
      w = v.grad.numpy()
      sens[k] = max(sens[k], float(np.abs(pt2[k].grad.numpy() - w).max() / (np.abs(w).max() + 1e-30)))
  errs = {}
  for k, v in pt.items():
    w = v.grad.numpy()
    e = np.abs(mine[k].cpu().numpy() - w) / (np.abs(w).max() + 1e-30)
    if w.shape[-1] >= 16 and e.max() < 0.2:
      # one flipped ReLU unit of the producing layer moves exactly one output-channel slice of its
      # kernel / bias gradient: the two worst output channels are left out of the bound, everything
      # else must hold
      per_ch = e.reshape(-1, w.shape[-1]).max(axis=0)
      e = np.sort(per_ch)[:-2]
    errs[k] = float(e.max())
  bad = {k: (errs[k], sens[k]) for k in errs if not errs[k] < max(gtol, 4 * sens[k])}
  print('R2D2_NET %s T=%d B=%d: worst grad err %.2e (max probe response %.2e)' % (mode, T, B, max(errs.values()),
                                                                              max(sens.values())))
  assert not bad, bad


@pytest.mark.parametrize('mode', ['simt', 'tc3'])
def test_r2d2_learner_step_vs_oracle(mode):
  """compute_loss_and_priorities with burn-in + minimize (clip, Adam) + target sync, 2 steps."""
  from oracle import r2d2_learner_oracle as RL, r2d2_net_oracle as NO
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers
  A, obs, S, T, B, burn = 6, (36, 36, 1), 4, 12, 4, 4
  params = NO.init_params(A, obs, S, seed=5)
  tparams = NO.init_params(A, obs, S, seed=6)
  cpu = RL.CpuR2D2Learner(A, obs, S, burn_in=burn, params=params, target_params=tparams, lr=1e-3)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, gemm_mode=mode); agent.load_named_parameters(params)
  target = networks.DuelingLSTMDQNNet(A, obs, S, gemm_mode=mode); target.load_named_parameters(tparams)
  st = learner.default_settings(burn_in=burn, update_target_every_n_step=10**9)
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(1e-3, epsilon=1e-3), settings=st)
  tol = {'simt': 2e-3, 'tc3': 6e-3}[mode]
  for it in range(2):
    b = RL.synthetic_replay_batch(T, B, A, obs, seed=20 + it, done_p=0.1)
    pa, env, state = _to_cuda_inputs(b, S)
    c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
    unrolls = learner.Unroll(state, None, pa, env, learner.AgentOutput(c(b['action']), None))
    sampled = learner.SampledUnrolls(unrolls, c(b['indices']), c(b['importance_weights']))
    total, loss_b, prio, g, norm, _ = cpu.grads(b)
    loss, priorities, indices, gnorm = step.compute_gradients(sampled)
    agent.check_errors()
    assert abs(float(loss) - total) < 1e-3 * max(1.0, abs(total)), (float(loss), total)
    np.testing.assert_allclose(priorities.cpu().numpy(), prio, rtol=2e-3, atol=1e-4)
    np.testing.assert_allclose(float(gnorm), norm, rtol=5e-3)
    scale = np.float32(st.clip_norm / max(norm, st.clip_norm))
    mine = agent.named_gradients()
    # the oracle's own sensitivity to a 1e-6 relative parameter perturbation bounds what any fp32
    # implementation can agree to on this tiny batch
    prng = np.random.default_rng(it)
    pert = RL.CpuR2D2Learner(A, obs, S, burn_in=burn, lr=1e-3,
                             params={k: v.detach().numpy() * (1 + 1e-6 * prng.normal(size=tuple(v.shape))).astype(np.float32)
                                     for k, v in cpu.params.items()},
                             target_params={k: v.numpy() for k, v in cpu.target.items()})
    g2 = pert.grads(b)[3]
    for k in g:
      w = g[k] * scale
      sens = np.abs(g2[k] - g[k]).max() / (np.abs(g[k]).max() + 1e-30)
      err = np.abs(mine[k].cpu().numpy() - w).max() / (np.abs(w).max() + 1e-30)
      assert err < max(tol, 4 * sens), (it, k, err, sens)
    step.apply_gradients()
    cpu.step(b)
    for k, v in agent.named_parameters().items():
      np.testing.assert_allclose(v.cpu().numpy(), cpu.params[k].detach().numpy(), atol=3e-4, rtol=0)
  # update_target_agent: target_var.assign(source_var)
  step.update_target_agent()
  assert torch.equal(target.params, agent.params)


def test_prioritized_replay_and_feeder():
  """insert wrap-around / sample / update_priorities (common/utils.py:260-370; sequences of
  tests/utils_test.py:304-365) on the GPU-resident buffer, and the ReplayFeeder hand-off."""
  from seed_rl_b200.agents.r2d2 import learner
  from seed_rl_b200.common import utils
  spec = (utils.TensorSpec([2], 'float32', 'a'), utils.TensorSpec([], 'int32', 'b'))
  rb = utils.PrioritizedReplay(4, spec, importance_sampling_exponent=0.6)
  with pytest.raises(ValueError, match='Cannot sample if replay buffer is empty'):
    rb.sample(1, 1.0)
  c = lambda a: torch.as_tensor(np.asarray(a)).cuda()
  idx = rb.insert((c(np.arange(6, dtype=np.float32).reshape(3, 2)), c(np.array([10, 11, 12], np.int32))),
                  c(np.array([1., 2., 3.], np.float32)))
  assert idx.tolist() == [0, 1, 2] and rb.num_inserted == 3
  idx = rb.insert((c(np.arange(6, 10, dtype=np.float32).reshape(2, 2)), c(np.array([13, 14], np.int32))),
                  c(np.array([4., 5.], np.float32)))
  assert idx.tolist() == [3, 0] and rb.num_inserted == 5              # FIFO wrap-around
  u = np.linspace(0.01, 0.99, 512).astype(np.float32)
  i, w, (a, bvals) = rb.sample(512, 1.0, uniforms=c(u))
  prio = np.array([5., 2., 3., 4.], np.float32)
  p = R.replay_probabilities(prio, 5, 1.0)
  np.testing.assert_allclose(w.cpu().numpy(), R.replay_importance_weights(p, i.cpu().numpy(), 0.6), rtol=5e-5)
  np.testing.assert_array_equal(bvals.cpu().numpy(), np.array([14, 11, 12, 13])[i.cpu().numpy()])
  freq = np.bincount(i.cpu().numpy(), minlength=4) / 512
  assert np.abs(freq - p).max() < 0.01
  rb.update_priorities(c(np.array([1, 2], np.int64)), c(np.array([0., 0.], np.float32)))
  i, _, _ = rb.sample(256, 1.0)
  assert set(i.cpu().numpy().tolist()) <= {0, 3}                       # zero-priority items are never drawn
  i, w, _ = rb.sample(64, 0)                                           # uniform branch (:335-337)
  assert float(w.min()) == 1.0 and i.max() < 4
  # epsilon schedule (agents/r2d2/learner_test.py:60-70) and greedy override
  eps = learner.get_envs_epsilon(torch.arange(5), 3, 2, 0.001).cpu().numpy()
  np.testing.assert_allclose(eps, R.get_envs_epsilon(np.arange(5), 3, 2, 0.001), rtol=1e-6)
  acts = learner.apply_epsilon_greedy(torch.full([4096], 7, dtype=torch.int32).cuda(), torch.zeros(4096, dtype=torch.int64),
                                      2, 1, 0.0, 18)
  frac = float((acts != 7).float().mean())
  assert abs(frac - 0.4 * 17 / 18) < 0.05


def test_r2d2_inference_host_feeds_replay_and_learner():
  """R2D2InferenceHost._inference == reference agents/r2d2/learner.py:711-790 (run-id resets, T=1
  forward with frame stacking, epsilon-greedy, store with burn_in overlapping steps for training
  environments only, initial priorities from the behaviour Q values, first-state bookkeeping), then
  the replay feed + one learner step (create_dataset :410-461, minimize, priority write-back)."""
  from seed_rl_b200.agents.r2d2 import learner, learner_loop
  from seed_rl_b200.atari import networks
  from seed_rl_b200.common import optimizers, utils
  A, obs, S = 6, (36, 36, 1), 4
  st = learner.default_settings(batch_size=6, replay_ratio=1.5, unroll_length=4, burn_in=2, replay_buffer_size=16,
                                replay_buffer_min_size=4, update_target_every_n_step=10**9)
  agent = networks.DuelingLSTMDQNNet(A, obs, S, seed=1, gemm_mode='simt')
  target = networks.DuelingLSTMDQNNet(A, obs, S, seed=1, gemm_mode='simt')
  host = learner_loop.R2D2InferenceHost(agent, num_envs=6, num_eval_envs=1, inference_batch_size=3,
                                        observation_shape=obs, settings=st,
                                        generator=torch.Generator(device='cuda').manual_seed(0))
  rng = np.random.default_rng(0)
  run_ids = rng.integers(1, 2**40, 6)
  returned = {e: [] for e in range(6)}
  for step_i in range(13):
    for ids in (np.array([0, 1, 2], np.int32), np.array([5, 3, 4], np.int32)):
      n = len(ids)
      env = utils.EnvOutput(rng.normal(size=n).astype(np.float32), rng.random(n) < 0.1,
                            rng.integers(0, 256, (n,) + obs, dtype=np.uint8), np.zeros(n, bool), np.full(n, step_i, np.int32))
      act = host.inference(ids, run_ids[ids], env, np.zeros(n, np.float32))
      assert act.shape == (3,) and act.dtype == np.int32 and (0 <= act).all() and (act < A).all()
      for e, a in zip(ids, act):
        returned[int(e)].append(int(a))
  torch.cuda.synchronize()
  # full_length = burn_in + unroll_length + 1 = 7 and the index starts at burn_in (the first unroll's
  # first burn_in rows are zero padding, UnrollStore :142-145): unrolls complete at steps 4, 8 and 12
  # for each of the 5 training environments; the eval environment (id 5) never reaches the store
  assert host.unroll_queue.size() == 15
  items = [host.unroll_queue.dequeue() for _ in range(15)]
  for k, u in enumerate(items):
    assert tuple(u.prev_actions.shape) == (7,) and tuple(u.env_outputs.observation.shape) == (7,) + obs
    lo = st.burn_in if k < 5 else 0
    assert torch.equal(u.agent_outputs.action[lo:-1], u.prev_actions[lo + 1:])  # :829-830
    assert float(u.priority) > 0
    # initial priority (:807-821) against the float64 loss on the suffix, q = target q = the behaviour q
    q = u.agent_outputs.q_values[st.burn_in:].cpu().numpy()[:, None]
    suf = lambda x: x[st.burn_in:].cpu().numpy()[:, None]
    LF.check_outputs(dict(priorities=np.array([float(u.priority)])),
                     (q, q, suf(u.agent_outputs.action).astype(np.int64), suf(u.env_outputs.reward),
                      suf(u.env_outputs.done), None),
                     'n_step', st.n_steps, st.discounting, 0.9, st.value_function_rescaling_epsilon)
  for k, u in enumerate(items[:5]):
    # first unroll of environment k: zero padding, then the behaviour Q values == a training-mode
    # unroll of the real steps from the initial state (the state the environment was reset to)
    assert float(u.agent_outputs.q_values[:st.burn_in].abs().max()) == 0.0
    assert float(u.agent_state.core_state[0].abs().max()) == 0.0
    tm = lambda t: t[st.burn_in:].unsqueeze(1)
    env = utils.EnvOutput(*(tm(x) for x in u.env_outputs))
    out, _ = agent((tm(u.prev_actions), env), agent.initial_state(1), unroll=True)
    np.testing.assert_allclose(out.q_values[:, 0].cpu().numpy(), u.agent_outputs.q_values[st.burn_in:].cpu().numpy(),
                               rtol=2e-4, atol=2e-5)
    # the actions handed back to the actors are the ones recorded (after epsilon-greedy)
    assert returned[k][:5] == u.agent_outputs.action[st.burn_in:].cpu().tolist()
  # consecutive unrolls of an environment overlap on burn_in + 1 rows (UnrollStore :234-252)
  for k in range(5):
    a, b = items[k], items[k + 5]
    for x, y in zip(utils.flatten(tuple(a[2:])), utils.flatten(tuple(b[2:]))):
      assert torch.equal(x[-(st.burn_in + 1):], y[:st.burn_in + 1])
  for u in items:
    host.unroll_queue.enqueue(u)
  replay = utils.PrioritizedReplay(st.replay_buffer_size, host.unroll_specs, st.importance_sampling_exponent)
  feeder = learner.ReplayFeeder(replay, st, generator=torch.Generator(device='cuda').manual_seed(1))
  assert learner.get_replay_insertion_batch_size(st) == 4
  assert learner_loop.fill_replay(host, feeder) and feeder.ready() and replay.num_inserted == 4
  assert learner_loop.fill_replay(host, feeder) and replay.num_inserted == 8
  step = learner.R2D2LearnerStep(agent, target, optimizers.Adam(1e-3, epsilon=1e-3), settings=st)
  sampled = feeder.sample()
  assert tuple(sampled.unrolls.env_outputs.observation.shape) == (7, 6) + obs      # time-major
  loss, priorities, indices, norm = step.minimize(sampled)
  feeder.update_priorities(indices, priorities)
  agent.check_errors()
  assert np.isfinite(float(loss)) and np.isfinite(float(norm)) and bool((priorities >= 0).all())
  assert torch.equal(replay._priorities[indices], priorities) or len(set(indices.tolist())) < len(indices)
