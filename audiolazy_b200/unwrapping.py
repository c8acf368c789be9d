"""Phase unwrapping and clipping: reference ``audiolazy/lazy_analysis.py:619-683`` (``clip``, ``unwrap``), on the GPU.

``unwrap(sig, max_delta, step)`` and ``clip(sig, low, high)`` are the reference's lazy Streams.  :class:`Unwrap` and
:class:`Clip` are their batched forms on CUDA tensors ``[S, T]``: an :class:`Unwrap` continues many streams block by
block through an :class:`UnwrapState`, which is how a table of STFT phases is unwrapped along its frames.  Both run the
kernels of ``include/alz_b200_unwrap.h``.  Unlike the package's float32 lazy APIs, ``unwrap`` and ``clip`` read their
samples as float64 (phases come from complex128 spectra), and their values are the reference's bit for bit.
"""
from __future__ import annotations

import ctypes
import itertools as it
import math
from numbers import Real

from . import _build, _capi, _engine
from .stream import Stream

__all__ = ["unwrap", "Unwrap", "UnwrapState", "clip", "Clip"]

_i32, _i64, _f64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["unwrap"].path, "unwrap", {
  "alz_unwrap_last_error": (ctypes.c_char_p, []),
  "alz_unwrap_state_bytes": (_i64, [_i64]),
  "alz_unwrap_state_init": (_i32, [_vp, _i64, _vp]),
  "alz_unwrap_scratch_bytes": (_i64, [_i64, _i64]),
  "alz_unwrap_apply": (_i32, [_vp, _i32, _i64, _vp, _i32, _i64, _vp, _i64, _i64, _f64, _f64, _vp, _i64, _vp]),
  "alz_clip_apply": (_i32, [_vp, _i32, _i64, _vp, _i32, _i64, _i64, _i64, _f64, _i32, _f64, _i32, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})
#: every function include/alz_b200_unwrap.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check

FLOAT32, FLOAT64 = 0, 1


def _real(name, value):
  if not isinstance(value, Real):
    raise TypeError("%s must be a real number, not %s" % (name, type(value).__name__))
  return float(value)


def _same(a, b):
  return a == b or (math.isnan(a) and math.isnan(b))


def _dtype_code(torch, dtype, what):
  if dtype == torch.float32:
    return FLOAT32
  if dtype == torch.float64:
    return FLOAT64
  raise ValueError("%s must be torch.float32 or torch.float64" % what)


def _output(torch, x, out_dtype):
  S, T = x.shape
  return torch.empty((S, T), dtype=out_dtype, device=x.device)


class UnwrapState(object):
  """Device state of :class:`Unwrap` calls over ``n_streams`` streams: per stream the samples consumed, the previous
  sample, the running ``delta`` and the index of the first jump met with ``step == 0`` (see :meth:`failures`).  It is
  made for one ``max_delta`` and ``step``, stream count and device."""

  def __init__(self, uw, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.max_delta, self.step = uw.max_delta, uw.step
    self.consumed = 0
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_unwrap_state_bytes(self.n_streams))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_unwrap_state_init(self.tensor.data_ptr(), self.n_streams,
                                         torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device

  def failures(self):
    """CUDA int64 tensor ``[n_streams]``: per stream, the sample index (counted from the stream's start) of the first
    jump taken with ``step == 0``, where the reference raises ``ZeroDivisionError``, or -1.  The outputs from that
    sample on are NaN."""
    torch = _engine.torch_mod()
    return torch.bitwise_not(self.tensor[:32 * self.n_streams].view(torch.int64).view(self.n_streams, 4)[:, 3])


class Unwrap(object):
  """Unwrapping of many streams with one ``max_delta`` and ``step`` (reference ``unwrap``).

  * ``uw.apply(x, state=None, out_dtype=torch.float64)`` -> CUDA tensor ``[S, T]`` for a CUDA float32 or float64
    ``x[S, T]``: the reference's values (float64) or their rounding (float32).
  * ``uw.new_state(S)`` -> :class:`UnwrapState`, to continue streams block by block; blocks of any lengths give the
    bits of one call."""

  def __init__(self, max_delta=math.pi, step=2 * math.pi):
    self.max_delta = _real("max_delta", max_delta)
    self.step = _real("step", step)

  def new_state(self, n_streams):
    return UnwrapState(self, n_streams)

  def apply(self, x, state=None, out_dtype=None):
    torch = _engine.torch_mod()
    out_dtype = torch.float64 if out_dtype is None else out_dtype
    x, S, T, xs = _engine.stream_input64(x)
    oc = _dtype_code(torch, out_dtype, "out_dtype")
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      _engine.check_state(state, UnwrapState, "Unwrap", S, x.device)
      if not (_same(state.max_delta, self.max_delta) and _same(state.step, self.step)):
        raise ValueError("state belongs to an Unwrap with another max_delta or step")
      out = _output(torch, x, out_dtype)
      stream = torch.cuda.current_stream(x.device).cuda_stream
      nbytes = _check(lib().alz_unwrap_scratch_bytes(S, T))
      scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)   # on this stream: torch's allocator orders reuse
      _check(lib().alz_unwrap_apply(x.data_ptr(), _dtype_code(torch, x.dtype, "x"), xs, out.data_ptr(), oc, max(T, 1),
                                    state.tensor.data_ptr(), S, T, self.max_delta, self.step, scratch.data_ptr(),
                                    nbytes, stream))
    state.consumed += T
    return out


def unwrap(sig, max_delta=math.pi, step=2 * math.pi):
  """Parametrized signal unwrapping (reference ``unwrap``): when a step between adjacent samples is larger than
  ``max_delta`` in magnitude, the output is shifted by the multiple of ``step`` that makes the step smallest.

  Samples are read as float64 and the values are Python floats, the reference's bit for bit for float inputs.  With
  ``step == 0`` the Stream yields the values before the first jump, then raises ``ZeroDivisionError``, as the
  reference does; an empty input raises ``RuntimeError`` when iterated (PEP 479), as the reference's generator does.
  A non-real ``max_delta`` or ``step`` raises ``TypeError`` here, where the reference raises it at the first jump."""
  uw = Unwrap(max_delta, step)
  torch = _engine.torch_mod()
  state = uw.new_state(1)                          # no device: raises at call time
  device = state.device

  def pump():
    empty = True
    for xb in _engine._blocks64(sig):
      if len(xb) == 0:
        continue
      empty = False
      before = state.consumed
      y = uw.apply(torch.from_numpy(xb).to(device), state=state)[0]
      if uw.step == 0:
        bad = int(state.failures()[0])
        if bad >= 0:
          yield y[:bad - before].cpu().numpy().tolist()
          raise ZeroDivisionError("float modulo")
      yield y.cpu().numpy().tolist()
    if empty:
      raise RuntimeError("generator raised StopIteration")

  return Stream(it.chain.from_iterable(pump()))


class Clip(object):
  """Clipping of many streams (reference ``clip``): ``Clip(low, high).apply(x, out_dtype=None)`` -> CUDA tensor
  ``[S, T]`` for a CUDA float32 or float64 ``x[S, T]``, of ``x``'s dtype unless ``out_dtype`` says otherwise.  A limit
  of ``None`` is no limit; the comparisons and the limits are float64."""

  def __init__(self, low=-1., high=1.):
    self.low = None if low is None else _real("low", low)
    self.high = None if high is None else _real("high", high)
    if self.low is not None and self.high is not None and self.high < self.low:
      raise ValueError("Higher clipping limit is smaller than lower one")

  def apply(self, x, out_dtype=None):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input64(x)
    out_dtype = x.dtype if out_dtype is None else out_dtype
    oc = _dtype_code(torch, out_dtype, "out_dtype")
    with torch.cuda.device(x.device):
      out = _output(torch, x, out_dtype)
      _check(lib().alz_clip_apply(x.data_ptr(), _dtype_code(torch, x.dtype, "x"), xs, out.data_ptr(), oc, max(T, 1),
                                  S, T, 0. if self.low is None else self.low, int(self.low is not None),
                                  0. if self.high is None else self.high, int(self.high is not None),
                                  torch.cuda.current_stream(x.device).cuda_stream))
    return out


def clip(sig, low=-1., high=1.):
  """Clips the signal to ``low`` and ``high`` (reference ``clip``); a limit of ``None`` leaves that side unclipped,
  and with both ``None`` the result is ``Stream(sig)``.  ``high < low`` raises ``ValueError`` at the call, as in the
  reference.  Samples are read as float64 and the values are Python floats (a clipped value is the limit as a float,
  where the reference yields the limit object itself; an int limit therefore comes out as an equal float).  A non-real
  limit raises ``TypeError`` at the call."""
  if low is None and high is None:
    return Stream(sig)
  cl = Clip(low, high)
  torch = _engine.torch_mod()
  device = torch.device("cuda", torch.cuda.current_device())

  def pump():
    for xb in _engine._blocks64(sig):
      yield cl.apply(torch.from_numpy(xb).to(device))[0].cpu().numpy().tolist()

  return Stream(it.chain.from_iterable(pump()))
