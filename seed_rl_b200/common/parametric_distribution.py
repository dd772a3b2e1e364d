"""Categorical action distribution -- mirror of the reference's
`common/parametric_distribution.py` for the discrete case
(ParametricDistribution :30-80, categorical_distribution :83-97,
get_parametric_distribution_for_action_space :293-330).  Continuous / joint
distributions (mujoco) are out of scope (SURVEY 2, row 3).
"""
import torch

from seed_rl_b200 import _lib

_DTYPES = {'int32': torch.int32, 'int64': torch.int64}


class _Categorical(object):
  """What `tfd.Categorical(logits=parameters, dtype=dtype)` offers on this path."""

  def __init__(self, logits, dtype):
    self.logits = _lib.require_cuda(logits, torch.float32, 'logits')
    self.dtype = dtype
    self._generator_offset = 0

  def _flat(self):
    A = self.logits.shape[-1]
    return self.logits.reshape(-1, A), A

  def log_prob(self, actions):
    flat, A = self._flat()
    a = _lib.require_cuda(actions, torch.int64, 'actions').reshape(-1)
    if a.numel() != flat.shape[0]:
      raise ValueError('actions shape %s does not match logits %s' %
                       (tuple(actions.shape), tuple(self.logits.shape)))
    out = torch.empty(flat.shape[0], dtype=torch.float32, device=flat.device)
    _lib.check(_lib.lib().seedrl_categorical_log_prob(
        flat.shape[0], A, _lib.ptr(flat), _lib.ptr(a), _lib.ptr(out), _lib.stream_ptr()))
    return out.reshape(self.logits.shape[:-1])

  def entropy(self):
    flat, A = self._flat()
    out = torch.empty(flat.shape[0], dtype=torch.float32, device=flat.device)
    _lib.check(_lib.lib().seedrl_categorical_entropy(
        flat.shape[0], A, _lib.ptr(flat), _lib.ptr(out), _lib.stream_ptr()))
    return out.reshape(self.logits.shape[:-1])

  def sample(self, seed=0, offset=0, gumbel_noise=None):
    """Gumbel-max sample.  `gumbel_noise` [.., A] makes it bit-reproducible."""
    flat, A = self._flat()
    noise = None
    if gumbel_noise is not None:
      noise = _lib.require_cuda(gumbel_noise, torch.float32, 'gumbel_noise').reshape(-1, A)
    out = torch.empty(flat.shape[0], dtype=torch.int64, device=flat.device)
    _lib.check(_lib.lib().seedrl_categorical_sample(
        flat.shape[0], A, _lib.ptr(flat), _lib.ptr(noise), int(seed), int(offset),
        _lib.ptr(out), _lib.stream_ptr()))
    return out.reshape(self.logits.shape[:-1]).to(self.dtype)


class ParametricDistribution(object):
  """reference parametric_distribution.py:30-80."""

  def __init__(self, param_size, create_dist):
    self._param_size = param_size
    self._create_dist = create_dist

  @property
  def create_dist(self):
    return self._create_dist

  def __call__(self, params):
    return self.create_dist(params)

  @property
  def param_size(self):
    return self._param_size

  @property
  def reparametrizable(self):
    return False   # Categorical is not reparameterizable

  def sample(self, parameters, **kw):
    return self._create_dist(parameters).sample(**kw)

  def log_prob(self, parameters, actions):
    return self._create_dist(parameters).log_prob(actions)

  def entropy(self, parameters):
    return self._create_dist(parameters).entropy()


def categorical_distribution(n_actions, dtype):
  """reference parametric_distribution.py:83-97."""
  if not isinstance(dtype, torch.dtype):
    dtype = _DTYPES[getattr(dtype, 'name', str(dtype))]

  def create_dist(parameters):
    return _Categorical(parameters, dtype)

  return ParametricDistribution(n_actions, create_dist)


def get_parametric_distribution_for_action_space(action_space, continuous_config=None):
  """reference parametric_distribution.py:293-330, Discrete spaces only (anything with
  an integer `.n`, e.g. gym.spaces.Discrete)."""
  if hasattr(action_space, 'n') and not hasattr(action_space, 'nvec'):
    return categorical_distribution(int(action_space.n),
                                    dtype=getattr(action_space, 'dtype', 'int64'))
  raise ValueError('Only Discrete action spaces are on the GPU hot path; got %r '
                   '(continuous / multi-discrete / tuple spaces are out of scope).' %
                   (action_space,))
