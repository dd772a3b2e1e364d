"""RPC layer -- mirror of the reference's `grpc/python/ops.py` (`Server.bind/start/shutdown`
:37-115, `Client` with dynamic methods :118-166) on top of

  * the C++ pinned-slab batcher of libseedrl_b200 (seedrl_batcher_*, replacing
    `DynamicFn`, grpc/ops/grpc.cc:591-861), and
  * `grpcio` generic handlers speaking the reference's service definition
    (`seed_rl.TensorService{Init, Call}`, grpc/service.proto:28-57) with tensors encoded as
    `tensorflow.TensorProto` bytes (dtype=1, tensor_shape=2{dim=2{size=1}},
    tensor_content=4 -- the form `AsProtoTensorContent` emits, grpc.cc:160-163) and output
    specs as `tensorflow.StructuredValue` (tensor_spec_value=33{name=1,shape=2,dtype=3},
    list_value=51, tuple_value=52, none_value=1).

The wire encodings are restated from TensorFlow's published .proto files with a
hand-written protobuf codec (no protoc / TF here).  NOT yet verified against a live TF 2.4.1
actor -- SURVEY 8(f) rank 1.  Error strings follow grpc.cc:513-549,187-190.
"""
import collections
import ctypes
import threading
from concurrent import futures

import numpy as np

from seed_rl_b200 import _lib
from seed_rl_b200.common import utils

TensorSpec = utils.TensorSpec

# tensorflow.DataType enum values [3P types.proto]
_DT = {np.dtype('float32'): 1, np.dtype('float64'): 2, np.dtype('int32'): 3, np.dtype('uint8'): 4,
       np.dtype('int64'): 9, np.dtype('bool'): 10, np.dtype('int8'): 6}
_DT_INV = {v: k for k, v in _DT.items()}
_DT_NAMES = {1: 'float', 2: 'double', 3: 'int32', 4: 'uint8', 9: 'int64', 10: 'bool', 6: 'int8'}

INVALID_ARGUMENT, INTERNAL, CANCELLED, UNAVAILABLE = 3, 13, 1, 14


class RpcError(RuntimeError):
  def __init__(self, code, message):
    super().__init__(message)
    self.code = code
    self.message = message


class InvalidArgumentError(RpcError):
  pass


class UnavailableError(RpcError):
  pass


# ---- protobuf wire format (varint / length-delimited only) ---------------------------
def _varint(n):
  n &= (1 << 64) - 1
  out = bytearray()
  while True:
    b = n & 0x7F
    n >>= 7
    if n:
      out.append(b | 0x80)
    else:
      out.append(b)
      return bytes(out)


def _key(field, wt):
  return _varint((field << 3) | wt)


def _ld(field, payload):
  return _key(field, 2) + _varint(len(payload)) + payload


class MalformedProto(ValueError):
  """A byte string that is not a well-formed protobuf message of the expected schema."""


def _read_varint(buf, i, n):
  v = 0; shift = 0
  while True:
    if i >= n or shift > 63:
      raise MalformedProto('truncated or over-long varint')
    b = buf[i]; i += 1
    v |= (b & 0x7F) << shift; shift += 7
    if not b & 0x80:
      return v & ((1 << 64) - 1), i


def _parse(buf):
  """Yields (field, wire_type, value) -- value is int for varint, bytes for len-delimited.
  Malformed input raises MalformedProto (a ValueError), never anything else."""
  i, n = 0, len(buf)
  while i < n:
    k, i = _read_varint(buf, i, n)
    field, wt = k >> 3, k & 7
    if field == 0:
      raise MalformedProto('field number 0')
    if wt == 0:
      v, i = _read_varint(buf, i, n)
      yield field, wt, v
    elif wt == 2:
      ln, i = _read_varint(buf, i, n)
      if ln > n - i:
        raise MalformedProto('length-delimited field runs past the end of the message')
      yield field, wt, bytes(buf[i:i + ln]); i += ln
    elif wt in (5, 1):
      w = 4 if wt == 5 else 8
      if w > n - i:
        raise MalformedProto('fixed-width field runs past the end of the message')
      yield field, wt, bytes(buf[i:i + w]); i += w
    else:
      raise MalformedProto('unsupported wire type %d' % wt)


def _expect(wt, want, what):
  if wt != want:
    raise MalformedProto('%s has wire type %d, expected %d' % (what, wt, want))


def _shape_proto(shape):
  # proto3: a zero size is the default and is not written
  return b''.join(_ld(2, (_key(1, 0) + _varint(int(d))) if int(d) else b'') for d in shape)


def _parse_shape(buf):
  dims = []
  for f, wt, v in _parse(buf):
    if f == 2:
      _expect(wt, 2, 'TensorShapeProto.dim')
      size = 0
      for f2, wt2, v2 in _parse(v):
        if f2 == 1:
          _expect(wt2, 0, 'Dim.size')
          size = v2 if v2 < (1 << 63) else v2 - (1 << 64)
      dims.append(size)
  return dims


def _utf8(v):
  try:
    return v.decode('utf-8')
  except UnicodeDecodeError:
    raise MalformedProto('string field is not valid UTF-8')


def _contig(a):
  a = np.asarray(a)          # (np.ascontiguousarray would turn 0-d into 1-d)
  return a if a.flags.c_contiguous else a.copy()


def encode_tensor(a):
  a = _contig(a)
  content = a.tobytes()
  return (_key(1, 0) + _varint(_DT[a.dtype]) + _ld(2, _shape_proto(a.shape)) +
          (_ld(4, content) if content else b''))


def decode_tensor(buf):
  dtype, shape, content = None, [], b''
  for f, wt, v in _parse(buf):
    if f == 1:
      _expect(wt, 0, 'TensorProto.dtype')
      if v not in _DT_INV:
        raise MalformedProto('unsupported TensorProto dtype %d' % v)
      dtype = _DT_INV[v]
    elif f == 2:
      _expect(wt, 2, 'TensorProto.tensor_shape')
      shape = _parse_shape(v)
    elif f == 4:
      _expect(wt, 2, 'TensorProto.tensor_content')
      content = v
  if dtype is None:
    raise MalformedProto('TensorProto without dtype')
  n = 1
  for d in shape:
    if d < 0:
      raise MalformedProto('negative dimension')
    n *= d
  if n * np.dtype(dtype).itemsize != len(content):
    raise MalformedProto('tensor_content has %d bytes, shape %s of %s needs %d' %
                         (len(content), shape, np.dtype(dtype).name, n * np.dtype(dtype).itemsize))
  return np.frombuffer(content, dtype=dtype).reshape(shape)


def encode_structure(specs):
  """nest of TensorSpec -> tensorflow.StructuredValue bytes."""
  if specs is None:
    return _ld(1, b'')
  if isinstance(specs, TensorSpec):
    body = b''
    if specs.name:
      body += _ld(1, specs.name.encode())
    body += _ld(2, _shape_proto(specs.shape))
    body += _key(3, 0) + _varint(_DT[np.dtype(specs.dtype)])
    return _ld(33, body)
  vals = b''.join(_ld(1, encode_structure(s)) for s in specs)
  return _ld(52 if isinstance(specs, tuple) else 51, vals)


def decode_structure(buf):
  for f, wt, v in _parse(buf):
    if f == 1:
      return None
    if f == 33:
      _expect(wt, 2, 'StructuredValue.tensor_spec_value')
      name, shape, dt = None, [], 1
      for f2, wt2, v2 in _parse(v):
        if f2 == 1:
          _expect(wt2, 2, 'TensorSpecProto.name'); name = _utf8(v2)
        elif f2 == 2:
          _expect(wt2, 2, 'TensorSpecProto.shape'); shape = _parse_shape(v2)
        elif f2 == 3:
          _expect(wt2, 0, 'TensorSpecProto.dtype'); dt = v2
      if dt not in _DT_INV:
        raise MalformedProto('unsupported TensorSpecProto dtype %d' % dt)
      return TensorSpec(shape, _DT_INV[dt].name, name)
    if f in (51, 52):
      _expect(wt, 2, 'StructuredValue.list_value / tuple_value')
      items = []
      for f2, wt2, v2 in _parse(v):
        if f2 == 1:
          _expect(wt2, 2, 'ListValue.values')
          items.append(decode_structure(v2))
      return tuple(items) if f == 52 else items
  return None


# ---- seed_rl.TensorService envelope (grpc/service.proto:28-57) ---------------------------
# The *_raw functions work on already-serialised payloads (TensorProto / StructuredValue
# bytes) and are pinned against the reference's compiled descriptor (tests/test_rpc.py,
# tests/golden/rpc_golden.json).  proto3: default values (0, '') are not emitted.
def _encode_call_request_raw(fn_name, tensor_bytes):
  out = _ld(1, fn_name.encode('utf-8')) if fn_name else b''
  return out + b''.join(_ld(2, t) for t in tensor_bytes)


def _decode_call_request_raw(buf):
  name, tensors = '', []
  for f, wt, v in _parse(buf):
    if f == 1:
      _expect(wt, 2, 'CallRequest.function'); name = _utf8(v)
    elif f == 2:
      _expect(wt, 2, 'CallRequest.tensor'); tensors.append(bytes(v))
  return name, tensors


def _encode_call_response_raw(tensor_bytes, code=0, msg=''):
  out = b''.join(_ld(1, t) for t in tensor_bytes)
  if code:
    out += _key(2, 0) + _varint(code)
  if msg:
    out += _ld(3, msg.encode('utf-8'))
  return out


def _decode_call_response_raw(buf):
  tensors, code, msg = [], 0, ''
  for f, wt, v in _parse(buf):
    if f == 1:
      _expect(wt, 2, 'CallResponse.tensor'); tensors.append(bytes(v))
    elif f == 2:
      _expect(wt, 0, 'CallResponse.status_code'); code = v if v < (1 << 31) else v - (1 << 64)
    elif f == 3:
      _expect(wt, 2, 'CallResponse.status_error_message'); msg = _utf8(v)
  return tensors, code, msg


def _encode_init_response_raw(signatures):
  """signatures: [(name, output_specs bytes)] -> InitResponse."""
  body = b''
  for name, spec in signatures:
    sig = (_ld(1, name.encode('utf-8')) if name else b'') + (_ld(2, spec) if spec else b'')
    body += _ld(1, sig)
  return body


def _decode_init_response_raw(buf):
  sigs = []
  for f, wt, v in _parse(buf):
    if f == 1:
      _expect(wt, 2, 'InitResponse.method_output_signature')
      name, spec = '', b''
      for f2, wt2, v2 in _parse(v):
        if f2 == 1:
          _expect(wt2, 2, 'MethodOutputSignature.name'); name = _utf8(v2)
        elif f2 == 2:
          _expect(wt2, 2, 'MethodOutputSignature.output_specs'); spec = bytes(v2)
      sigs.append((name, spec))
  return sigs


def _encode_call_request(fn_name, tensors):
  return _encode_call_request_raw(fn_name, [encode_tensor(t) for t in tensors])


def _decode_call_request(buf):
  name, raw = _decode_call_request_raw(buf)
  return name, [decode_tensor(t) for t in raw]


def _encode_call_response(tensors, code=0, msg=''):
  return _encode_call_response_raw([encode_tensor(t) for t in tensors], code, msg)


def _decode_call_response(buf):
  raw, code, msg = _decode_call_response_raw(buf)
  return [decode_tensor(t) for t in raw], code, msg


# ---- tf.function stand-in -------------------------------------------------------------
def function(input_signature, output_signature=None):
  """Decorator giving a python callable what `Server.bind` needs from a tf.function:
  `input_signature` (nest of batched TensorSpec [N, ...]) and `output_signature`."""
  def deco(fn):
    fn.input_signature = input_signature
    fn.output_signature = output_signature
    return fn
  return deco


_Bound = collections.namedtuple('_Bound', 'name fn in_specs out_specs out_structure batch_size '
                                          'batcher in_structure')


class Server(object):
  """reference grpc/python/ops.py:37-115."""

  def __init__(self, server_addresses, pinned=None, num_slabs=2, max_workers=64):
    import grpc
    self._grpc = grpc
    self._addresses = list(server_addresses)
    self._fns = {}
    self._threads = []
    self._started = False
    self._shutdown = False
    self._num_slabs = num_slabs
    if pinned is None:
      import torch
      pinned = torch.cuda.is_available()
    self._pinned = 1 if pinned else 0
    self._server = grpc.server(
        futures.ThreadPoolExecutor(max_workers=max_workers),
        options=[('grpc.max_send_message_length', -1), ('grpc.max_receive_message_length', -1)])
    handler = grpc.method_handlers_generic_handler('seed_rl.TensorService', {
        'Init': grpc.unary_unary_rpc_method_handler(self._init_rpc),
        'Call': grpc.stream_stream_rpc_method_handler(self._call_rpc)})
    self._server.add_generic_rpc_handlers((handler,))

  # -- binding ---------------------------------------------------------------------------
  def bind(self, fn):
    fns = fn if isinstance(fn, (list, tuple)) else [fn]
    for f in fns:
      if getattr(f, 'input_signature', None) is None:
        raise ValueError('function must have input_signature set.')
      name = f.__name__
      in_specs = utils.flatten(f.input_signature)
      out_specs = utils.flatten(f.output_signature) if f.output_signature is not None else []
      n = in_specs[0].shape[0] if in_specs and len(in_specs[0].shape) else -1
      for s in in_specs:       # batching only if every arg shares dim 0 (ops.py:64-71)
        if not len(s.shape) or s.shape[0] != n:
          n = -1
      if n <= 0:
        raise ValueError('seed_rl_b200 binds batched functions only (first dimension of all '
                         'arguments equal).')
      for s in out_specs:      # grpc.cc:696-710
        if not len(s.shape) or s.shape[0] != n:
          raise ValueError('Output must be at least rank 1 with first dimension %d' % n)
      L = _lib.lib()
      in_rows = [int(np.prod(s.shape[1:], dtype=np.int64)) * np.dtype(s.dtype).itemsize for s in in_specs]
      out_rows = [int(np.prod(s.shape[1:], dtype=np.int64)) * np.dtype(s.dtype).itemsize for s in out_specs]
      h = ctypes.c_void_p()
      _lib.check(L.seedrl_batcher_create(
          n, self._num_slabs, len(in_rows), (ctypes.c_size_t * len(in_rows))(*in_rows),
          len(out_rows), (ctypes.c_size_t * max(len(out_rows), 1))(*out_rows), self._pinned,
          ctypes.byref(h)))
      if name in self._fns:
        raise ValueError('seed_rl_b200: one function per name (round-robin over devices is the '
                         'multi-process launcher\'s job).')
      self._fns[name] = _Bound(name, f, in_specs, out_specs, f.output_signature, n, h,
                               f.input_signature)

  def start(self):
    for b in self._fns.values():
      t = threading.Thread(target=self._compute_loop, args=(b,), daemon=True)
      t.start()
      self._threads.append(t)
    for a in self._addresses:
      self._server.add_insecure_port(a)
    self._server.start()
    self._started = True

  def shutdown(self):
    self._shutdown = True
    L = _lib.lib()
    for b in self._fns.values():
      L.seedrl_batcher_shutdown(b.batcher)     # cancels waiters: "Server shutdown."
    self._server.stop(grace=0.5)
    for t in self._threads:
      t.join(5)

  # -- compute side ------------------------------------------------------------------------
  def _slab_array(self, b, slab, spec, field, out):
    L = _lib.lib()
    p = (L.seedrl_batcher_output_ptr if out else L.seedrl_batcher_input_ptr)(b.batcher, slab, field, 0)
    n = int(np.prod(spec.shape, dtype=np.int64))
    dt = np.dtype(spec.dtype)
    buf = (ctypes.c_uint8 * (n * dt.itemsize)).from_address(p)
    return np.frombuffer(buf, dtype=dt).reshape(spec.shape)

  def _compute_loop(self, b):
    L = _lib.lib()
    while True:
      slab = ctypes.c_int()
      rc = L.seedrl_batcher_next_full(b.batcher, -1, ctypes.byref(slab))
      if rc != 0:
        return
      status = 0
      try:
        args = [self._slab_array(b, slab.value, s, i, False) for i, s in enumerate(b.in_specs)]
        outs = b.fn(*utils.pack_sequence_as(b.in_structure, args))
        flat = utils.flatten(outs) if b.out_specs else []
        for i, (s, o) in enumerate(zip(b.out_specs, flat)):
          dst = self._slab_array(b, slab.value, s, i, True)
          if hasattr(o, 'detach'):
            o = o.detach().cpu().numpy()
          np.copyto(dst, np.asarray(o).reshape(s.shape).astype(s.dtype, copy=False))
      except Exception as e:   # propagate to every caller of this batch
        import traceback
        traceback.print_exc()
        self._last_error = str(e)
        status = INTERNAL
      L.seedrl_batcher_publish(b.batcher, slab.value, status)

  # -- request side ------------------------------------------------------------------------
  def _verify_args(self, b, args):
    """grpc.cc:513-549 + GetArgBatchSize.  Returns k (rows contributed)."""
    if len(args) != len(b.in_specs):
      raise InvalidArgumentError(INVALID_ARGUMENT, 'Expects %d arguments, but %d is provided' %
                                 (len(b.in_specs), len(args)))
    k = None
    for i, (a, s) in enumerate(zip(args, b.in_specs)):
      suffix = list(s.shape[1:])
      if a.ndim == len(suffix):
        bd, kk = 0, 1
      elif a.ndim == len(suffix) + 1:
        bd, kk = 1, a.shape[0]
      else:
        raise InvalidArgumentError(
            INVALID_ARGUMENT, 'Expects arg[%d] to have shape with %d dimension(s), but had shape %s' %
            (i, len(suffix), list(a.shape)))
      if list(a.shape[bd:]) != suffix:
        raise InvalidArgumentError(
            INVALID_ARGUMENT, 'Expects arg[%d] to have shape with suffix %s, but had shape %s' %
            (i, suffix, list(a.shape)))
      if a.dtype != np.dtype(s.dtype):
        raise InvalidArgumentError(
            INVALID_ARGUMENT, 'Expects arg[%d] to be %s but %s is provided' %
            (i, _DT_NAMES[_DT[np.dtype(s.dtype)]], _DT_NAMES.get(_DT.get(a.dtype), str(a.dtype))))
      if k is None:
        k, batched = kk, bd
      elif bd != batched or kk != k:
        raise InvalidArgumentError(INVALID_ARGUMENT, 'All arguments must agree on the batch dimension')
    return k or 1, bool(batched)

  def call_local(self, name, args):
    """One caller's contribution (k rows) -> its k output rows.  Used by the gRPC handler and
    directly by in-process callers (tests, local actors)."""
    L = _lib.lib()
    if name not in self._fns:
      raise RpcError(INTERNAL, 'Function %s not found' % name)        # grpc.cc:187-190
    b = self._fns[name]
    args = [_contig(a) for a in args]
    k, batched = self._verify_args(b, args)
    slab, row = ctypes.c_int(), ctypes.c_int()
    rc = L.seedrl_batcher_claim(b.batcher, k, ctypes.byref(slab), ctypes.byref(row))
    if rc != 0:
      msg = L.seedrl_last_error().decode()
      raise (UnavailableError if rc == CANCELLED else RpcError)(rc, msg)
    for i, a in enumerate(args):     # payload goes straight into the pinned slab
      ctypes.memmove(L.seedrl_batcher_input_ptr(b.batcher, slab, i, row), a.ctypes.data, a.nbytes)
    L.seedrl_batcher_commit(b.batcher, slab, k)
    st = ctypes.c_int()
    rc = L.seedrl_batcher_wait_outputs(b.batcher, slab, ctypes.byref(st))
    try:
      if rc != 0:
        raise UnavailableError(CANCELLED, 'Server shutdown.')
      if st.value != 0:
        raise RpcError(st.value, getattr(self, '_last_error', 'inference function failed'))
      outs = []
      for i, s in enumerate(b.out_specs):
        dt = np.dtype(s.dtype)
        shape = ([k] if batched else []) + list(s.shape[1:])
        o = np.empty(shape, dt)
        ctypes.memmove(o.ctypes.data, L.seedrl_batcher_output_ptr(b.batcher, slab, i, row), o.nbytes)
        outs.append(o)
      return outs
    finally:
      L.seedrl_batcher_release(b.batcher, slab)

  def _init_rpc(self, request, context):
    sigs = []
    for b in self._fns.values():
      unbatched = None
      if b.out_structure is not None:
        unbatched = utils.map_structure(lambda s: TensorSpec(list(s.shape[1:]), s.dtype, s.name),
                                        b.out_structure)
      sigs.append((b.name, encode_structure(unbatched)))
    return _encode_init_response_raw(sigs)

  def _call_rpc(self, request_iterator, context):
    for req in request_iterator:
      try:
        try:
          name, tensors = _decode_call_request(req)
        except MalformedProto as e:       # what a failed ParseFromString is in grpc.cc
          raise InvalidArgumentError(INVALID_ARGUMENT, 'Malformed CallRequest: %s' % e)
        outs = self.call_local(name, tensors)
        yield _encode_call_response(outs)
      except RpcError as e:
        if e.code == CANCELLED:
          return          # stream closed => client sees Unavailable (grpc.cc:1065-1071)
        yield _encode_call_response([], e.code, e.message)


class Client(object):
  """reference grpc/python/ops.py:118-166: methods appear from the server's Init reply."""

  def __init__(self, server_address, timeout=60):
    import grpc
    self._grpc = grpc
    self._channel = grpc.insecure_channel(
        server_address, options=[('grpc.max_send_message_length', -1),
                                 ('grpc.max_receive_message_length', -1)])
    grpc.channel_ready_future(self._channel).result(timeout=timeout)      # wait_for_ready
    ident = lambda x: x
    init = self._channel.unary_unary('/seed_rl.TensorService/Init', request_serializer=ident,
                                     response_deserializer=ident)
    self._call = self._channel.stream_stream('/seed_rl.TensorService/Call',
                                             request_serializer=ident, response_deserializer=ident)
    self._lock = threading.Lock()        # one in-flight call per stream (grpc.cc:1064)
    self._requests = _Feeder()
    self._responses = None
    for name, spec in _decode_init_response_raw(init(b'', wait_for_ready=True)):
      self._add_method(name, decode_structure(spec) if spec else None)

  def _add_method(self, name, output_specs):
    def call(*inputs):
      flat = [np.asarray(x) for x in utils.flatten(inputs)]
      with self._lock:
        if self._responses is None:
          self._responses = self._call(iter(self._requests))
        self._requests.put(_encode_call_request(name, flat))
        try:
          resp = next(self._responses)
        except (StopIteration, self._grpc.RpcError):
          raise UnavailableError(UNAVAILABLE, 'Read failed, is the server closed?')
      tensors, code, msg = _decode_call_response(resp)
      if code:
        raise (InvalidArgumentError if code == INVALID_ARGUMENT else RpcError)(code, msg)
      if output_specs is None:
        return None
      return utils.pack_sequence_as(output_specs, tensors)
    setattr(self, name, call)

  def close(self):
    self._requests.close()
    self._channel.close()


class _Feeder(object):
  """Blocking iterator feeding the request stream."""

  def __init__(self):
    self._q = collections.deque()
    self._cv = threading.Condition()
    self._closed = False

  def put(self, x):
    with self._cv:
      self._q.append(x)
      self._cv.notify()

  def close(self):
    with self._cv:
      self._closed = True
      self._cv.notify_all()

  def __iter__(self):
    return self

  def __next__(self):
    with self._cv:
      while not self._q and not self._closed:
        self._cv.wait()
      if self._q:
        return self._q.popleft()
      raise StopIteration
