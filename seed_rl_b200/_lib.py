"""ctypes binding of libseedrl_b200.so (the C-ABI declared in include/seedrl_b200.h).

There is NO fallback: if the shared library is missing or a call fails, this
module raises.  PyTorch is used by callers only for device memory and streams;
nothing here imports torch types into the ABI (raw pointers + sizes only).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libseedrl_b200.so')

c_void_p, c_int, c_float, c_size_t = ctypes.c_void_p, ctypes.c_int, ctypes.c_float, ctypes.c_size_t
c_i64, c_u64 = ctypes.c_int64, ctypes.c_uint64
P = c_void_p


class SeedrlError(RuntimeError):

  def __init__(self, code, msg):
    super().__init__('libseedrl_b200 error %d: %s' % (code, msg))
    self.code = code


class LossConfig(ctypes.Structure):
  """struct seedrl_loss_config."""
  _fields_ = [('discounting', c_float), ('lambda_', c_float), ('baseline_cost', c_float),
              ('kl_cost', c_float), ('max_abs_reward', c_float),
              ('clip_rho_threshold', c_float), ('clip_pg_rho_threshold', c_float),
              ('target_entropy', c_float), ('has_target_entropy', ctypes.c_int32),
              ('entropy_cost_adjustment_speed', c_float)]


class RowJob(ctypes.Structure):
  _fields_ = [('table', ctypes.c_void_p), ('rows', ctypes.c_void_p), ('row_bytes', ctypes.c_size_t),
              ('mode', ctypes.c_int32), ('full_length', ctypes.c_int32)]


ROW_GATHER, ROW_SCATTER, ROW_APPEND = 0, 1, 2


def rows_multi(jobs, env_ids_i32, index=None, id_limit=None):
  """jobs: list of (table tensor, rows tensor, mode).  One launch (seedrl_rows_multi; with
  id_limit, seedrl_rows_multi_limit: append jobs skip the rows whose env id is >= id_limit)."""
  n = int(env_ids_i32.numel())
  arr = (RowJob * len(jobs))()
  for k, (table, rows, mode) in enumerate(jobs):
    rb = (table[0, 0] if mode == ROW_APPEND else table[0]).numel() * table.element_size()
    if rows.numel() * rows.element_size() != n * rb or rows.dtype != table.dtype or not rows.is_contiguous():
      raise ValueError('rows_multi: rows do not match the table (job %d)' % k)
    arr[k] = RowJob(table.data_ptr(), rows.data_ptr(), rb, mode, table.shape[1] if mode == ROW_APPEND else 0)
  if id_limit is None:
    check(lib().seedrl_rows_multi(arr, len(jobs), ptr(env_ids_i32), n, ptr(index), stream_ptr()))
  else:
    check(lib().seedrl_rows_multi_limit(arr, len(jobs), ptr(env_ids_i32), n, ptr(index), int(id_limit),
                                        stream_ptr()))


class NetConfig(ctypes.Structure):
  """struct seedrl_net_config."""
  _fields_ = [('net', ctypes.c_int32), ('num_actions', ctypes.c_int32),
              ('obs_h', ctypes.c_int32), ('obs_w', ctypes.c_int32), ('obs_c', ctypes.c_int32)]


NET_DEEP, NET_SHALLOW = 0, 1
LOSS_TERMS = 16
LT = dict(total=0, policy=1, V=2, entropy=3, kl=4, entropy_adj=5, v_mean=6, v_l2_error=7,
          mean_entropy=8, entropy_cost=9, mean_kl=10, max_action_abs=11, popart_mean=12, popart_std=13)

# name -> (restype, argtypes); every symbol of include/seedrl_b200.h
SIGNATURES = {
    'seedrl_last_error': (ctypes.c_char_p, []),
    'seedrl_abi_version': (c_int, []),
    'seedrl_kernel_launch_count': (c_u64, []),
    'seedrl_vtrace_from_importance_weights':
        (c_int, [c_int, c_int, P, P, P, P, P, P, c_float, c_float, c_float, P, P, P]),
    'seedrl_categorical_log_prob': (c_int, [c_int, c_int, P, P, P, P]),
    'seedrl_categorical_entropy': (c_int, [c_int, c_int, P, P, P]),
    'seedrl_categorical_sample': (c_int, [c_int, c_int, P, P, c_u64, c_u64, P, P]),
    'seedrl_categorical_sample_counter': (c_int, [c_int, c_int, P, P, c_u64, P, P, P]),
    'seedrl_vtrace_loss_scratch_bytes': (c_size_t, [c_int, c_int, c_int]),
    'seedrl_vtrace_loss_fwd_bwd':
        (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, ctypes.POINTER(LossConfig), P,
                 P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_popart_loss_fwd':
        (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, ctypes.POINTER(LossConfig), P, P, P,
                 P, P, P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_loss_fwd_bwd_abandoned':
        (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, ctypes.POINTER(LossConfig), P,
                 P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_popart_loss_fwd_abandoned':
        (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, ctypes.POINTER(LossConfig), P, P, P,
                 P, P, P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_popart_update':
        (c_int, [c_int, c_int, c_int, c_float, c_float, P, P, P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_popart_tasks_scratch_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'seedrl_vtrace_popart_tasks_loss_fwd':
        (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P, c_int, ctypes.POINTER(LossConfig), P, P, P,
                 P, P, P, P, P, P, P, P, P, P, P]),
    'seedrl_vtrace_popart_tasks_update':
        (c_int, [c_int, c_int, c_int, c_float, c_float, P, P, P, P, P, P, P, P, P, P, P]),
    'seedrl_adam_apply':
        (c_int, [c_size_t, P, P, P, P, c_float, c_float, c_float, c_float, c_float, c_i64,
                 c_float, c_float, P]),
    'seedrl_net_create': (c_int, [ctypes.POINTER(NetConfig), ctypes.POINTER(P)]),
    'seedrl_net_destroy': (None, [P]),
    'seedrl_net_num_param_tensors': (c_int, [P]),
    'seedrl_net_num_params': (c_size_t, [P]),
    'seedrl_net_arena_floats': (c_size_t, [P]),
    'seedrl_net_set_conv_mode': (c_int, [P, c_int]),
    'seedrl_net_set_lstm_mode': (c_int, [P, c_int]),
    'seedrl_net_param_info':
        (c_int, [P, c_int, ctypes.c_char_p, c_size_t, ctypes.POINTER(c_i64),
                 ctypes.POINTER(c_size_t)]),
    'seedrl_net_workspace_bytes': (c_size_t, [P, c_int, c_int]),
    'seedrl_net_forward':
        (c_int, [P, P, c_int, c_int, P, P, P, P, P, P, P, P, P, P, P, c_size_t, P]),
    'seedrl_net_backward':
        (c_int, [P, P, c_int, c_int, P, P, P, P, P, P, P, P, c_size_t, P]),
    'seedrl_net_backward_overlap':
        (c_int, [P, P, c_int, c_int, P, P, P, P, P, P, P, P, c_size_t, P, P]),
    'seedrl_net_grad_split': (c_size_t, [P]),
    'seedrl_net_check_error': (c_int, [P, c_int, c_int, P, c_size_t, P]),
    'seedrl_store_append_field': (c_int, [P, P, P, c_int, c_int, c_size_t, P, P]),
    'seedrl_store_advance': (c_int, [P, P, c_int, c_int, P, P, P]),
    'seedrl_store_advance_limit': (c_int, [P, P, c_int, c_int, P, P, ctypes.c_int32, P]),
    'seedrl_store_gather_field': (c_int, [P, P, c_int, c_int, c_size_t, c_int, c_int, P, P]),
    'seedrl_rows_multi': (c_int, [P, c_int, P, c_int, P, P]),
    'seedrl_rows_multi_limit': (c_int, [P, c_int, P, c_int, P, ctypes.c_int32, P]),
    'seedrl_store_gather_field_into': (c_int, [P, P, c_int, c_int, c_size_t, c_int, P, c_int, c_int, P]),
    'seedrl_store_finish': (c_int, [P, P, c_int, c_int, P]),
    'seedrl_store_reset': (c_int, [P, P, P, c_int, c_int, c_size_t, c_int, P]),
    'seedrl_batcher_create':
        (c_int, [c_int, c_int, c_int, ctypes.POINTER(c_size_t), c_int, ctypes.POINTER(c_size_t),
                 c_int, ctypes.POINTER(P)]),
    'seedrl_batcher_destroy': (None, [P]),
    'seedrl_batcher_claim': (c_int, [P, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    'seedrl_batcher_input_ptr': (P, [P, c_int, c_int, c_int]),
    'seedrl_batcher_output_ptr': (P, [P, c_int, c_int, c_int]),
    'seedrl_batcher_commit': (c_int, [P, c_int, c_int]),
    'seedrl_batcher_wait_outputs': (c_int, [P, c_int, ctypes.POINTER(c_int)]),
    'seedrl_batcher_release': (c_int, [P, c_int]),
    'seedrl_batcher_next_full': (c_int, [P, c_int, ctypes.POINTER(c_int)]),
    'seedrl_batcher_publish': (c_int, [P, c_int, c_int]),
    'seedrl_batcher_shutdown': (c_int, [P]),
    'seedrl_r2d2_net_create': (c_int, [c_int, c_int, c_int, c_int, ctypes.POINTER(P)]),
    'seedrl_r2d2_net_destroy': (None, [P]),
    'seedrl_r2d2_net_num_param_tensors': (c_int, [P]),
    'seedrl_r2d2_net_num_params': (c_size_t, [P]),
    'seedrl_r2d2_net_arena_floats': (c_size_t, [P]),
    'seedrl_r2d2_net_set_mode': (c_int, [P, c_int]),
    'seedrl_r2d2_net_set_lstm_mode': (c_int, [P, c_int]),
    'seedrl_r2d2_net_param_info':
        (c_int, [P, c_int, ctypes.c_char_p, c_size_t, ctypes.POINTER(c_i64), ctypes.POINTER(c_int),
                 ctypes.POINTER(c_size_t)]),
    'seedrl_r2d2_net_workspace_bytes': (c_size_t, [P, c_int, c_int]),
    'seedrl_r2d2_net_forward':
        (c_int, [P, P, c_int, c_int, P, P, P, P, P, P, P, P, P, P, P, c_size_t, P]),
    'seedrl_r2d2_net_backward': (c_int, [P, P, c_int, c_int, P, P, P, P, P, c_size_t, P]),
    'seedrl_r2d2_net_check_error': (c_int, [P, c_int, c_int, P, c_size_t, P]),
    'seedrl_r2d2_stack_frames': (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P]),
    'seedrl_r2d2_loss_scratch_bytes': (c_size_t, [c_int, c_int, c_int]),
    'seedrl_r2d2_loss_fwd_bwd': (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, c_float, c_int, c_float, c_float,
                                         P, P, P, P, P]),
    'seedrl_r2d2_retrace_loss_scratch_bytes': (c_size_t, [c_int, c_int]),
    'seedrl_r2d2_retrace_loss_fwd_bwd': (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, c_float, c_float, c_float,
                                                 c_float, P, P, P, P, P]),
    'seedrl_r2d2_loss_fwd_bwd_abandoned': (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, c_float, c_int,
                                                   c_float, c_float, P, P, P, P, P]),
    'seedrl_r2d2_retrace_loss_fwd_bwd_abandoned': (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, c_float,
                                                           c_float, c_float, c_float, P, P, P, P, P]),
    'seedrl_r2d2_epsilon_greedy': (c_int, [c_int, c_int, P, P, c_u64, P, P, P]),
    'seedrl_replay_sample': (c_int, [c_int, P, c_float, c_float, c_int, P, P, P, P, P]),
    'seedrl_clip_scratch_bytes': (c_size_t, []),
    'seedrl_clip_by_global_norm': (c_int, [c_size_t, P, c_float, P, P, P]),
    'seedrl_profile_num_categories': (c_int, []),
    'seedrl_profile_category_name': (ctypes.c_char_p, [c_int]),
    'seedrl_profile_begin': (c_int, [P]),
    'seedrl_profile_end': (c_int, [ctypes.POINTER(ctypes.c_double), ctypes.POINTER(c_u64)]),
    'seedrl_debug_planes_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'seedrl_debug_to_planes': (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P]),
    'seedrl_debug_from_planes': (c_int, [c_int, c_int, c_int, c_int, P, P, P]),
    'seedrl_debug_convp': (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, c_int, P, P, P, P, P, P]),
    'seedrl_debug_wgradp': (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, c_size_t, P, P]),
    'seedrl_debug_poolp': (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, P]),
    'seedrl_debug_conv3x3': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, P, P]),
    'seedrl_debug_conv3x3_flip': (c_int, [c_int, c_int, P, P, P]),
    'seedrl_debug_conv3x3_tc':
        (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, P, c_int, c_int, P, P, P]),
    'seedrl_debug_wgrad_partial_bytes': (c_size_t, []),
    'seedrl_debug_conv_pixels': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P]),
    'seedrl_debug_set_loss_stream': (c_int, [c_int]),
    'seedrl_debug_set_wgrad_chunk': (c_int, [c_int]),
    'seedrl_debug_set_conv_tile': (c_int, [c_int]),
    'seedrl_debug_set_first_layer_dense': (c_int, [c_int]),
    'seedrl_debug_conv0pool': (c_int, [c_int, c_int, c_int, P, P, P, P, P, P, P, P]),
    'seedrl_debug_conv0pool_c': (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P, P]),
    'seedrl_debug_first_wgrad_pooled_c': (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, c_size_t, P]),
    'seedrl_debug_conv3x3_wgrad_tc':
        (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, c_size_t, P, P]),
    'seedrl_debug_conv3x3_wgrad':
        (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, c_size_t, P]),
    'seedrl_debug_maxpool': (c_int, [c_int, c_int, c_int, c_int, c_int, P, P, P, P]),
    'seedrl_debug_gemm_tc':
        (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, P, c_int, P, c_int, P, c_int, P, P, c_int, c_int, c_int,
                 c_int, P, c_size_t, P, P]),
    'seedrl_debug_set_gemm_gather': (c_int, [c_int]),
    'seedrl_debug_colsum': (c_int, [c_int, c_int, P, c_int, P, P, c_size_t, P]),
    'seedrl_debug_sgemm':
        (c_int, [c_int, c_int, c_int, c_int, c_int, P, c_int, P, c_int, P, c_int, P, P, c_int,
                 c_int, c_int, c_int, P]),
    'seedrl_debug_strided_conv':
        (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P, P, P,
                 c_int, P, P, c_size_t, P, c_size_t, P, ctypes.POINTER(c_int), P]),
    'seedrl_debug_lstm_workspace_bytes': (c_size_t, [c_int, c_int, c_int, c_int]),
    'seedrl_debug_lstm_forward':
        (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P, P, P, c_size_t, P, P]),
    'seedrl_debug_lstm_backward':
        (c_int, [c_int, c_int, c_int, c_int, P, P, P, P, P, P, P, P, c_size_t, P, P]),
    'seedrl_debug_r2d2_net_views':
        (c_int, [P, c_int, c_int, c_int, ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t)]),
    'seedrl_debug_net_views':
        (c_int, [P, c_int, c_int, c_int, ctypes.POINTER(c_size_t), ctypes.POINTER(c_size_t),
                 ctypes.POINTER(c_int)]),
}

_lib = None


def lib():
  """Loads the shared library (once).  Raises if it is not built."""
  global _lib
  if _lib is None:
    if not os.path.exists(LIB_PATH):
      raise ImportError(
          'seed_rl_b200: %s is missing -- build it with `python -c "import '
          '__graft_entry__ as g; g.build()"` (seed_rl_b200/csrc/build.sh). There is no '
          'CPU or PyTorch fallback.' % LIB_PATH)
    l = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
      fn = getattr(l, name)     # AttributeError if the .so lacks a declared symbol
      fn.restype = res
      fn.argtypes = args
    _lib = l
  return _lib


def check(rc):
  if rc != 0:
    raise SeedrlError(rc, (lib().seedrl_last_error() or b'').decode('utf-8', 'replace'))


def launch_count():
  return int(lib().seedrl_kernel_launch_count())


# ---- torch plumbing (device memory + streams only) ---------------------------
def ptr(t):
  return None if t is None else ctypes.c_void_p(t.data_ptr())


def stream_ptr():
  import torch
  return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(t, dtype, name):
  """Returns a contiguous CUDA tensor of `dtype` (copying if it has to)."""
  import torch
  if not isinstance(t, torch.Tensor):
    t = torch.as_tensor(t)
  if not torch.cuda.is_available():
    raise RuntimeError('seed_rl_b200 needs a CUDA device (H100); there is no CPU path '
                       '(argument %r).' % name)
  if t.device.type != 'cuda':
    t = t.cuda()
  if t.dtype != dtype:
    t = t.to(dtype)
  return t.contiguous()
