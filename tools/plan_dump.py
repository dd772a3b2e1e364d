"""Prints the workspace sizes and parameter tables of the network schedules (no GPU needed).

Two builds of libseedrl_b200.so that plan the same workspaces and parameter arenas print the same text:
  python tools/plan_dump.py [path/to/libseedrl_b200.so] > plan.txt
Covers ImpalaDeep on 84x84x4 and 72x96x3 frames and the shallow net in every conv mode they take, at
(T+1, B) = (21, 64), (21, 256), (1, 64), and DuelingLSTMDQNNet (84x84x4) at (T, B) = (141, 64).
"""
import ctypes
import os
import sys

V, I, SZ = ctypes.c_void_p, ctypes.c_int, ctypes.c_size_t


class NetConfig(ctypes.Structure):
  _fields_ = [('net', ctypes.c_int32), ('num_actions', ctypes.c_int32),
              ('obs_h', ctypes.c_int32), ('obs_w', ctypes.c_int32), ('obs_c', ctypes.c_int32)]


def main():
  path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(__file__), '..', 'seed_rl_b200',
                                                             'libseedrl_b200.so')
  L = ctypes.CDLL(path)
  L.seedrl_net_workspace_bytes.restype = SZ
  L.seedrl_net_workspace_bytes.argtypes = [V, I, I]
  L.seedrl_r2d2_net_workspace_bytes.restype = SZ
  L.seedrl_r2d2_net_workspace_bytes.argtypes = [V, I, I]
  L.seedrl_net_param_info.argtypes = [V, I, ctypes.c_char_p, SZ, ctypes.POINTER(ctypes.c_int64),
                                      ctypes.POINTER(SZ)]
  L.seedrl_r2d2_net_param_info.argtypes = [V, I, ctypes.c_char_p, SZ, ctypes.POINTER(ctypes.c_int64),
                                           ctypes.POINTER(I), ctypes.POINTER(SZ)]
  name, dims, off, rank = ctypes.create_string_buffer(128), (ctypes.c_int64 * 4)(), SZ(), I()

  for label, net, h, w, c, modes in (('deep 84x84x4', 0, 84, 84, 4, (0, 1, 2, 3)),
                                     ('deep 72x96x3', 0, 72, 96, 3, (0, 1, 2, 3)),
                                     ('shallow 84x84x4', 1, 84, 84, 4, (0, 1, 2))):
    n = V()
    assert L.seedrl_net_create(ctypes.byref(NetConfig(net, 9, h, w, c)), ctypes.byref(n)) == 0
    for mode in modes:
      assert L.seedrl_net_set_conv_mode(n, mode) == 0
      for t1, b in ((21, 64), (21, 256), (1, 64)):
        print('%s conv_mode %d (%d, %d): workspace %d' % (label, mode, t1, b, L.seedrl_net_workspace_bytes(n, t1, b)))
    i = 0
    while True:
      r = L.seedrl_net_param_info(n, i, name, 128, dims, ctypes.byref(off))
      if r < 0:
        break
      print('%s param %d %s rank %d dims %s offset %d' % (label, i, name.value.decode(), r, list(dims), off.value))
      i += 1
    L.seedrl_net_destroy(n)

  n = V()
  assert L.seedrl_r2d2_net_create(9, 84, 84, 4, ctypes.byref(n)) == 0
  for mode in (0, 2):
    assert L.seedrl_r2d2_net_set_mode(n, mode) == 0
    print('r2d2 84x84x4 mode %d (141, 64): workspace %d' % (mode, L.seedrl_r2d2_net_workspace_bytes(n, 141, 64)))
  for i in range(L.seedrl_r2d2_net_num_param_tensors(n)):
    assert L.seedrl_r2d2_net_param_info(n, i, name, 128, dims, ctypes.byref(rank), ctypes.byref(off)) == 0
    print('r2d2 param %d %s rank %d dims %s offset %d' % (i, name.value.decode(), rank.value, list(dims), off.value))
  L.seedrl_r2d2_net_destroy(n)


if __name__ == '__main__':
  main()
