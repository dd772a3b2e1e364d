"""CPU: the Python side of the agent networks (common/cuda_net.py and its two subclasses), built with
device='cpu' -- parameter tables and arena views, the Keras initialisation, the checkpoint format and the
per-thread workspace cache.  Nothing here launches a kernel."""
import math
import threading

import numpy as np
import pytest
import torch

from oracle import net_oracle, r2d2_net_oracle
from seed_rl_b200.atari import networks as atari_networks
from seed_rl_b200.dmlab import networks

A = 9
CONFIGS = {
    'deep84': (lambda seed=0: networks.ImpalaDeep(A, (84, 84, 4), seed=seed, device='cpu'),
               lambda: net_oracle.param_specs('deep', A, (84, 84, 4)), 256),
    'deep72': (lambda seed=0: networks.ImpalaDeep(A, (72, 96, 3), seed=seed, device='cpu'),
               lambda: net_oracle.param_specs('deep', A, (72, 96, 3)), 256),
    'shallow': (lambda seed=0: networks.ImpalaShallow(A, (84, 84, 4), seed=seed, device='cpu'),
                lambda: net_oracle.param_specs('shallow', A, (84, 84, 4)), 256),
    'r2d2': (lambda seed=0: atari_networks.DuelingLSTMDQNNet(A, (84, 84, 1), 4, seed=seed, device='cpu'),
             lambda: r2d2_net_oracle.param_specs(A, (84, 84, 1), 4), 512),
}


@pytest.mark.parametrize('config', sorted(CONFIGS))
def test_parameter_table_names_and_arena_views(config):
  make, specs, _ = CONFIGS[config]
  agent = make()
  want = specs()
  impala = config != 'r2d2'
  assert len(agent.param_info) == len(want) + (1 if impala else 0)
  if impala:          # the library's table is the reference's variable order, then the scalar
    assert [(n, s) for n, s, _ in agent.param_info[:-1]] == [(n, tuple(s)) for n, s in want]
    assert agent.param_info[-1][:2] == ('entropy_cost_param', ())
    assert agent.entropy_cost_param_index == agent.param_info[-1][2]
    assert agent.entropy_cost_param.shape == ()
  else:               # tf.Module attribute order: _advantage, _body, _core, _value
    assert dict((n, s) for n, s, _ in agent.param_info) == dict((n, tuple(s)) for n, s in want)
    names = agent.variable_names
    assert names[0].startswith('advantage/') and names[-1].startswith('value/')
  tensors = [s for _, s, _ in agent.param_info[:len(want)]]
  assert agent.num_params == sum(int(np.prod(s)) for s in tensors)
  assert agent.variable_names == [n for n, _ in agent.named_parameters().items()]
  assert len(agent.trainable_variables) == len(want)
  assert list(agent.named_gradients()) == [n for n, _, _ in agent.param_info]
  end = 0
  views = agent.trainable_variables + ([agent.entropy_cost_param] if impala else [])
  for (name, shape, off), v, g in zip(agent.param_info, views, agent.named_gradients().values()):
    assert off % 64 == 0 and off >= end, name
    assert tuple(v.shape) == tuple(g.shape) == shape
    assert v.data_ptr() == agent.params.data_ptr() + 4 * off          # views into the arenas
    assert g.data_ptr() == agent.grads.data_ptr() + 4 * off
    end = off + int(np.prod(shape))
  assert end <= agent.arena_floats == agent.params.numel() == agent.grads.numel()


@pytest.mark.parametrize('config', sorted(CONFIGS))
def test_keras_initialisation(config):
  make, _, units = CONFIGS[config]
  agent = make(seed=1)
  arena = agent.params.numpy()
  covered = np.zeros(arena.size, bool)
  for (name, _, off), p in zip(agent.param_info, agent.trainable_variables):
    a = p.numpy()
    covered[off:off + a.size] = True
    if name.endswith('bias'):
      want = np.zeros_like(a)
      if name == 'core/bias':
        want[units:2 * units] = 1.0                                    # unit_forget_bias
      np.testing.assert_array_equal(a, want, err_msg=name)
    elif name == 'core/recurrent_kernel':                                # orthogonal [H, 4H]: rows orthonormal
      assert a.shape == (units, 4 * units)
      np.testing.assert_allclose(a @ a.T, np.eye(units), atol=2e-5, err_msg=name)
    else:                                                                # glorot_uniform
      rf = int(np.prod(a.shape[:-2])) if a.ndim > 2 else 1
      lim = math.sqrt(6.0 / (a.shape[-2] * rf + a.shape[-1] * rf))
      assert np.abs(a).max() <= lim, name
      assert np.abs(a).max() > 0.9 * lim and abs(float(a.mean())) < 0.05 * lim, name
  assert not arena[~covered].any()                                       # padding and the scalar stay zero
  other = make(seed=2).params.numpy()
  assert not np.array_equal(arena, other) and np.array_equal(arena, make(seed=1).params.numpy())


@pytest.mark.parametrize('config', ['deep72', 'r2d2'])
def test_state_dict_round_trip(config):
  make, _, _ = CONFIGS[config]
  a, b = make(seed=3), make(seed=4)
  if config != 'r2d2':
    a.init_entropy_cost(0.01, 10.0)
  d = a.state_dict()
  assert d['param_info'] == a.param_info and d['params'].device.type == 'cpu'
  b.load_state_dict(d)
  assert torch.equal(a.params, b.params)
  # every entry of the table, the scalar included, by name
  b.load_named_parameters({n: np.full(s, i, np.float32) for i, (n, s, _) in enumerate(b.param_info)})
  for i, (n, s, off) in enumerate(b.param_info):
    assert (b.params[off:off + int(np.prod(s))] == i).all(), n
  with pytest.raises(ValueError):
    b.load_named_parameters({'core/bias': np.zeros(3, np.float32)})
  with pytest.raises(KeyError):
    b.load_named_parameters({'no/such/variable': np.zeros(3, np.float32)})


# ---- the workspace cache -------------------------------------------------------------------------
def _shallow():
  return CONFIGS['shallow'][0]()


def test_workspace_two_alternating_shapes_are_reused():
  agent = _shallow()
  a, b = agent.workspace(1, 3), agent.workspace(2, 5)
  assert a.dtype == torch.uint8 and a.device.type == 'cpu' and a is not b
  for _ in range(3):
    assert agent.workspace(1, 3) is a
    assert agent.workspace(2, 5) is b


def test_workspace_third_shape_evicts_least_recently_used():
  agent = _shallow()
  a, b = agent.workspace(1, 3), agent.workspace(2, 5)
  assert agent.workspace(1, 3) is a               # b is now the least recently used
  c = agent.workspace(4, 1)
  assert agent.workspace(1, 3) is a and agent.workspace(4, 1) is c
  assert agent.workspace(2, 5) is not b           # evicted: a new buffer
  assert agent.workspace(4, 1) is c               # ... which evicted a, the older of a and c
  assert agent.workspace(1, 3) is not a


def test_workspace_threads_do_not_interact():
  agent = _shallow()
  mine = agent.workspace(1, 3)
  got = {}

  def other():
    got['same'] = agent.workspace(1, 3)
    got['more'] = [agent.workspace(1, n) for n in (4, 5, 6)]
  th = threading.Thread(target=other)
  th.start()
  th.join()
  assert got['same'] is not mine                   # never shared across threads
  assert agent.workspace(1, 3) is mine             # the other thread's evictions left this one alone


def test_workspace_held_reference_survives_eviction():
  agent = _shallow()
  held = agent.workspace(1, 3)
  held[:16] = torch.arange(16, dtype=torch.uint8)
  agent.workspace(1, 4)
  agent.workspace(1, 5)                            # evicts (1, 3) from the cache
  assert agent.workspace(1, 3) is not held
  assert held[:16].tolist() == list(range(16))     # the holder's buffer is still its own


def test_r2d2_workspace_keeps_burn_in_and_suffix():
  agent = CONFIGS['r2d2'][0]()
  burn, suffix = agent.workspace(2, 3), agent.workspace(5, 3)
  for _ in range(2):
    assert agent.workspace(2, 3) is burn and agent.workspace(5, 3) is suffix
