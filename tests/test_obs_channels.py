"""CPU: ImpalaDeep on frames of 1 to 16 channels -- the oracle against the reference run on such
frames (tests/golden/net_channels_golden.npz), and the library's observation contract: which
channel counts seedrl_net_create takes, the parameter table it builds for them, and the conv modes
it refuses for them (with messages that name the modes that do run)."""
import ctypes
import os
import sys

import numpy as np
import pytest
import torch

from oracle import net_oracle
from seed_rl_b200 import _lib

HERE = os.path.dirname(os.path.abspath(__file__))


def _create(C, H=84, W=84, A=6):
  L = _lib.lib()
  h = ctypes.c_void_p()
  cfg = _lib.NetConfig(_lib.NET_DEEP, A, H, W, C)
  return L.seedrl_net_create(ctypes.byref(cfg), ctypes.byref(h)), h


def test_oracle_matches_reference_on_other_channel_counts():
  sys.path.insert(0, os.path.join(HERE, 'golden'))
  import make_golden_net_channels as G
  g = np.load(os.path.join(HERE, 'golden', 'net_channels_golden.npz'))
  t = torch.as_tensor
  for tag, obs in G.SHAPES.items():
    p, i = G.make_params(obs), G.make_inputs(obs)
    assert tuple(g[tag + '_first_kernel_shape']) == (3, 3, obs[2], 16)
    assert int(g[tag + '_num_variables']) == len(p) == 39
    with torch.no_grad():
      logits, baseline, (h, c) = net_oracle.unroll('deep', p, t(i['prev']), t(i['rew']), t(i['done']), t(i['obs']),
                                                   (t(i['h0']), t(i['c0'])), G.A)
    for got, want in ((logits, 'logits'), (baseline, 'baseline'), (h, 'h'), (c, 'c')):
      np.testing.assert_allclose(got.numpy(), g[tag + '_' + want], rtol=1e-5, atol=1e-5, err_msg=tag + want)
    assert i['done'].any() and not i['done'].all()


@pytest.mark.parametrize('C', list(range(1, 17)))
def test_create_accepts_1_to_16_channels_with_reference_parameter_table(C):
  L = _lib.lib()
  rc, h = _create(C, 72, 90)
  assert rc == 0, L.seedrl_last_error()
  try:
    specs = net_oracle.param_specs('deep', 6, (72, 90, C))
    assert L.seedrl_net_num_param_tensors(h) == 39 == len(specs)
    end = 0
    for i, (name, shape) in enumerate(specs):
      buf = ctypes.create_string_buffer(128); dims = (ctypes.c_int64 * 4)(); off = ctypes.c_size_t()
      rank = L.seedrl_net_param_info(h, i, buf, 128, dims, ctypes.byref(off))
      assert buf.value.decode() == name
      assert tuple(dims[k] for k in range(rank)) == tuple(shape)
      assert off.value % 64 == 0
      end = off.value + (int(np.prod(shape)) + 63) // 64 * 64
    assert tuple(dict(specs)['stack0/conv/kernel']) == (3, 3, C, 16)
    assert L.seedrl_net_arena_floats(h) == end + 64          # + the entropy_cost_param slot
    assert L.seedrl_net_num_params(h) == sum(int(np.prod(s)) for _, s in specs)
    assert L.seedrl_net_workspace_bytes(h, 5, 3) > 0
  finally:
    L.seedrl_net_destroy(h)


@pytest.mark.parametrize('C', [0, 17, -1])
def test_create_refuses_other_channel_counts(C):
  L = _lib.lib()
  rc, _ = _create(C)
  assert rc == 3
  assert b'1 to 16 channels' in L.seedrl_last_error()


@pytest.mark.parametrize('C', [1, 2, 5, 8, 12, 16])
def test_tc_modes_refused_for_new_channel_counts(C):
  L = _lib.lib()
  rc, h = _create(C)
  assert rc == 0
  try:
    for mode in (1, 2):
      assert L.seedrl_net_set_conv_mode(h, mode) == 3
      msg = L.seedrl_last_error()
      assert b'simt' in msg and b'tc3p' in msg, msg
    assert L.seedrl_net_set_conv_mode(h, 3) == 0
    assert L.seedrl_net_set_conv_mode(h, 0) == 0
  finally:
    L.seedrl_net_destroy(h)


@pytest.mark.parametrize('C', [3, 4])
def test_dmlab_and_4_channel_frames_keep_every_mode(C):
  L = _lib.lib()
  rc, h = _create(C, 72, 96)
  assert rc == 0
  try:
    for mode in (0, 1, 2, 3):
      assert L.seedrl_net_set_conv_mode(h, mode) == 0
  finally:
    L.seedrl_net_destroy(h)


@pytest.mark.parametrize('C,W,ok', [(1, 107, True), (12, 107, True), (1, 108, False), (16, 160, False)])
def test_tc3p_width_limit_for_new_channel_counts(C, W, ok):
  L = _lib.lib()
  rc, h = _create(C, 84, W)
  assert rc == 0
  try:
    rc = L.seedrl_net_set_conv_mode(h, 3)
    if ok:
      assert rc == 0
    else:
      assert rc == 3
      msg = L.seedrl_last_error()
      assert b'107' in msg and b'simt' in msg, msg
      assert L.seedrl_net_set_conv_mode(h, 0) == 0
  finally:
    L.seedrl_net_destroy(h)


def test_python_agent_rejects_channel_counts_before_the_library():
  from seed_rl_b200.dmlab import networks
  for C in (0, 17):
    with pytest.raises(ValueError, match='1 to 16'):
      networks.ImpalaDeep(6, (84, 84, C))
