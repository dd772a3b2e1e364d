"""V-trace targets -- drop-in for the reference's `common/vtrace.py`
(from_importance_weights, VTraceReturns; reference common/vtrace.py:31-148).

Same name, argument meaning and error behaviour; tensors are torch CUDA tensors
and the arithmetic is ONE sm_90a kernel behind the C-ABI
(seedrl_vtrace_from_importance_weights).  No CPU fallback.
"""
import collections
import math

import torch

from seed_rl_b200 import _lib

VTraceReturns = collections.namedtuple('VTraceReturns', 'vs pg_advantages')


def _assert_rank(t, rank, name):
  if t.dim() != rank:   # tf: shape.assert_has_rank, vtrace.py:99-107
    raise ValueError('Shape %s of %s must have rank %d' % (tuple(t.shape), name, rank))


def from_importance_weights(
    target_action_log_probs, behaviour_action_log_probs,
    discounts, rewards, values, bootstrap_value,
    clip_rho_threshold=1.0, clip_pg_rho_threshold=1.0, lambda_=1.0,
    name='vtrace_from_importance_weights'):
  """See reference common/vtrace.py:34-82 for the contract.  [T, B(, ...)] inputs,
  [B(, ...)] bootstrap; thresholds may be None (no clipping)."""
  f32 = torch.float32
  tlp = _lib.require_cuda(target_action_log_probs, f32, 'target_action_log_probs')
  blp = _lib.require_cuda(behaviour_action_log_probs, f32, 'behaviour_action_log_probs')
  discounts = _lib.require_cuda(discounts, f32, 'discounts')
  rewards = _lib.require_cuda(rewards, f32, 'rewards')
  values = _lib.require_cuda(values, f32, 'values')
  bootstrap_value = _lib.require_cuda(bootstrap_value, f32, 'bootstrap_value')
  rho_rank = tlp.dim()
  _assert_rank(blp, rho_rank, 'behaviour_action_log_probs')
  _assert_rank(values, rho_rank, 'values')
  _assert_rank(bootstrap_value, rho_rank - 1, 'bootstrap_value')
  _assert_rank(discounts, rho_rank, 'discounts')
  _assert_rank(rewards, rho_rank, 'rewards')
  for thr, nm in ((clip_rho_threshold, 'clip_rho_threshold'),
                  (clip_pg_rho_threshold, 'clip_pg_rho_threshold')):
    if thr is not None and isinstance(thr, torch.Tensor) and thr.dim() != 0:
      raise ValueError('%s must have rank 0' % nm)
  for t, nm in ((blp, 'behaviour_action_log_probs'), (discounts, 'discounts'),
                (rewards, 'rewards'), (values, 'values')):
    if t.shape != tlp.shape:
      raise ValueError('%s has shape %s, expected %s' % (nm, tuple(t.shape), tuple(tlp.shape)))
  if bootstrap_value.shape != tlp.shape[1:]:
    raise ValueError('bootstrap_value has shape %s, expected %s' %
                     (tuple(bootstrap_value.shape), tuple(tlp.shape[1:])))
  T = tlp.shape[0]
  B = int(bootstrap_value.numel())
  vs = torch.empty_like(tlp)
  pg = torch.empty_like(tlp)
  nan = float('nan')
  _lib.check(_lib.lib().seedrl_vtrace_from_importance_weights(
      T, B, _lib.ptr(tlp), _lib.ptr(blp), _lib.ptr(discounts), _lib.ptr(rewards),
      _lib.ptr(values), _lib.ptr(bootstrap_value),
      nan if clip_rho_threshold is None else float(clip_rho_threshold),
      nan if clip_pg_rho_threshold is None else float(clip_pg_rho_threshold),
      float(lambda_), _lib.ptr(vs), _lib.ptr(pg), _lib.stream_ptr()))
  # outputs never carry gradient (tf.stop_gradient, vtrace.py:147-148)
  return VTraceReturns(vs=vs, pg_advantages=pg)
