"""Generates tests/golden/net_channels_golden.npz.  Run ONLY in the build container (where
/root/reference exists):   python tests/golden/make_golden_net_channels.py

The UNMODIFIED reference dmlab/networks.py (ImpalaDeep, which takes whatever frame shape it is
given) over the Keras-layer shim of make_golden_net.py, on frame shapes other than DMLab's: one
grayscale channel on an odd width and twelve channels (four stacked RGB frames).  Pins the same
wiring as net_golden.npz for the channel counts the deep net accepts beyond 3 and 4.  Parameters
and inputs come from seeds (make_params / make_inputs), so only the outputs are committed."""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE); sys.path.insert(0, ROOT)
import make_golden_net as M  # noqa: E402
from oracle import net_oracle  # noqa: E402

A, T1, B = 5, 5, 3
SHAPES = {'c1': (16, 18, 1), 'c12': (12, 20, 12)}


def make_params(obs):
  p = net_oracle.to_torch(net_oracle.init_params('deep', A, obs, seed=4 + obs[2]))
  rng = np.random.default_rng(9 + obs[2])
  for k in p:                                   # non-zero biases so that bias wiring is visible
    if k.endswith('bias'):
      p[k] = p[k] + torch.as_tensor(rng.normal(size=tuple(p[k].shape)).astype(np.float32)) * 0.1
  return p


def make_inputs(obs):
  rng = np.random.default_rng(10 + obs[2])
  done = rng.random((T1, B)) < 0.3
  done[1, 0], done[2, 1] = True, False           # at least one reset, never all
  return dict(obs=rng.integers(0, 256, (T1, B) + tuple(obs), dtype=np.uint8),
              rew=(rng.normal(size=(T1, B)) * 2).astype(np.float32), done=done,
              prev=rng.integers(0, A, (T1, B)), h0=rng.normal(size=(B, 256)).astype(np.float32),
              c0=rng.normal(size=(B, 256)).astype(np.float32))


def run_reference(obs):
  T = M.T
  p = make_params(obs)
  tf, order = M.build_tf(p, lambda logits: logits.argmax(-1))
  for s in range(3):                            # creation order, dmlab/networks.py:29-44, 74-89
    order['conv'] += ['stack%d/conv' % s, 'stack%d/res_0/conv2d_0' % s, 'stack%d/res_1/conv2d_0' % s,
                      'stack%d/res_0/conv2d_1' % s, 'stack%d/res_1/conv2d_1' % s]
  order['dense'] += ['conv_to_linear', 'policy_logits', 'baseline']
  sys.modules['tensorflow'] = tf
  seed_rl = types.ModuleType('seed_rl'); common = types.ModuleType('seed_rl.common')
  utils = types.ModuleType('seed_rl.common.utils')
  utils.batch_apply = M._extract_function(os.path.join(M.REF, 'common/utils.py'), 'batch_apply', {'tf': tf})
  seed_rl.common = common; common.utils = utils
  sys.modules.update({'seed_rl': seed_rl, 'seed_rl.common': common, 'seed_rl.common.utils': utils})
  ref = M._load(os.path.join(M.REF, 'dmlab/networks.py'), 'ref_networks_c%d' % obs[2])
  agent = ref.ImpalaDeep(A)
  i = make_inputs(obs)
  env = M.EnvOutput(T(i['rew']), T(i['done']), T(i['obs']), T(np.zeros((T1, B), bool)),
                    T(np.zeros((T1, B), np.int32)))
  with torch.no_grad():
    out, state = agent(T(i['prev']), env, [T(i['h0']), T(i['c0'])], unroll=True)
  return {'logits': M.raw(out.policy_logits).numpy(), 'baseline': M.raw(out.baseline).numpy(),
          'h': M.raw(state[0]).numpy(), 'c': M.raw(state[1]).numpy(),
          'first_kernel_shape': np.asarray(p['stack0/conv/kernel'].shape, np.int64),
          'num_variables': np.asarray(len(p), np.int64)}


def main():
  arrays = {}
  for tag, obs in SHAPES.items():
    for k, v in run_reference(obs).items():
      arrays['%s_%s' % (tag, k)] = v
    print(tag, obs, 'logits', arrays[tag + '_logits'].shape)
  np.savez_compressed(os.path.join(HERE, 'net_channels_golden.npz'), **arrays)
  print('wrote net_channels_golden.npz')


if __name__ == '__main__':
  main()
