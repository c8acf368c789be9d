"""Zero crossings: reference ``audiolazy/lazy_analysis.py:389-434`` (``zcross``), on the GPU.

``zcross(seq, hysteresis, first_sign)`` is the reference's lazy Stream of 0 / 1 crossing flags.  :class:`Zcross` is the
shape a batched pitch estimator needs: many streams, the flags of every sample or only the crossings per block of
``zcross(...).blocks(size, hop)``, continued block by block through a :class:`ZcrossState`.  Both run one kernel
(``include/alz_b200_zcross.h``); samples are float32 at the device boundary, compared against the float64
``hysteresis`` exactly.
"""
from __future__ import annotations

import ctypes
import itertools as it
import math
from numbers import Integral, Real

from . import _build, _capi, _engine
from ._engine import n_blocks
from .stream import Stream

__all__ = ["zcross", "Zcross", "ZcrossState"]

_i32, _i64, _f64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["zcross"].path, "zero-crossing", {
  "alz_zcross_last_error": (ctypes.c_char_p, []),
  "alz_zcross_state_bytes": (_i64, [_i64, _i32, _i32]),
  "alz_zcross_state_init": (_i32, [_vp, _i64, _f64, _i32, _i32, _vp]),
  "alz_zcross_scratch_bytes": (_i64, [_i64, _i64, _i32, _i32]),
  "alz_zcross_apply_f32": (_i32, [_vp, _i64, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _f64, _i32, _vp, _i64,
                                  _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})
#: every function include/alz_b200_zcross.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


def _real(name, value):
  if not isinstance(value, Real):
    raise TypeError("%s must be a real number, not %s" % (name, type(value).__name__))
  return float(value)


def _sign(first_sign):
  """The reference's starting sign: 0 ("search") for first_sign == 0 (-0. too), else -1 / +1 (NaN: +1)."""
  return 0 if first_sign == 0 else (-1 if first_sign < 0 else 1)


def _block_arg(name, value):
  if not isinstance(value, Integral) or isinstance(value, bool):
    raise TypeError("%s must be an integer" % name)
  if value < 1:
    raise ValueError("%s must be >= 1 (got %d)" % (name, value))
  return int(value)


class ZcrossState(object):
  """Device state of :class:`Zcross` calls over ``n_streams`` streams: per stream the carried sign, the samples
  consumed and, for :meth:`Zcross.counts`, the partial counts of the open blocks.  It is made for one hysteresis,
  starting sign, stream count, device and (``size``, ``hop``); a call with ``final=True`` ends it."""

  def __init__(self, zc, n_streams, size=None, hop=None):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.size = None if size is None else _block_arg("size", size)
    self.hop = None if size is None else (self.size if hop is None else _block_arg("hop", hop))
    if size is None and hop is not None:
      raise ValueError("hop needs a size")
    self.hysteresis = zc.hysteresis
    self.sign = zc.sign
    self.consumed = 0
    self.ended = False
    s, h = self.size or 0, self.hop or 1
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_zcross_state_bytes(self.n_streams, s, h))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_zcross_state_init(self.tensor.data_ptr(), self.n_streams, float(self.sign), s, h,
                                         torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


class Zcross(object):
  """Zero crossings of many streams with one ``hysteresis`` and starting sign (reference ``zcross``).

  * ``zc.apply(x, state=None)`` -> CUDA uint8 tensor ``[S, T]`` of crossing flags for a CUDA float32 ``x[S, T]``.
  * ``zc.counts(x, size, hop=None, state=None, final=False)`` -> CUDA int32 ``[S, n_blocks]``: the crossings of every
    block of ``zcross(...).blocks(size, hop)`` (``hop`` defaults to ``size``) that this call completes, plus, with
    ``final=True``, the reference's padded last block when it emits one.
  * ``zc.new_state(S, size=None, hop=None)`` -> :class:`ZcrossState`, to continue streams block by block; blocks of
    any lengths give the same flags and counts as one call."""

  def __init__(self, hysteresis=0., first_sign=0):
    self.hysteresis = _real("hysteresis", hysteresis)
    self.sign = _sign(_real("first_sign", first_sign))

  def new_state(self, n_streams, size=None, hop=None):
    return ZcrossState(self, n_streams, size=size, hop=hop)

  def _check_state(self, state, S, size, hop, device):
    _engine.check_state(state, ZcrossState, "Zcross", S, device)
    same_h = state.hysteresis == self.hysteresis or (math.isnan(state.hysteresis) and math.isnan(self.hysteresis))
    if not same_h or state.sign != self.sign:
      raise ValueError("state belongs to a Zcross with another hysteresis or first_sign")
    if (state.size, state.hop) != (size, hop):
      raise ValueError("state was created for size=%r, hop=%r; the call asks for size=%r, hop=%r"
                       % (state.size, state.hop, size, hop))
    if state.ended:
      raise ValueError("state was ended by a call with final=True")

  def _run(self, x, state, size, hop, final, flags):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input(x)
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S, size=size, hop=hop)
      self._check_state(state, S, size, hop, x.device)
      out = torch.empty((S, T), dtype=torch.uint8, device=x.device) if flags else None
      nb = n_blocks(state.consumed, T, size, hop, final) if size else 0
      counts = torch.empty((S, nb), dtype=torch.int32, device=x.device) if size else None
      s, h = size or 0, hop or 1
      stream = torch.cuda.current_stream(x.device).cuda_stream
      nbytes = _check(lib().alz_zcross_scratch_bytes(S, T, s, h))
      scratch = torch.empty(nbytes, dtype=torch.uint8, device=x.device)   # on this stream: torch's allocator orders reuse
      _check(lib().alz_zcross_apply_f32(x.data_ptr(), xs, out.data_ptr() if flags else None, max(T, 1),
                                        counts.data_ptr() if size else None, max(nb, 1), state.tensor.data_ptr(), S, T,
                                        s, h, self.hysteresis, int(bool(final)), scratch.data_ptr(), nbytes, stream))
    state.consumed += T
    state.ended = bool(final)
    return out if flags else counts

  def apply(self, x, state=None):
    """Crossing flags (uint8 0 / 1) of every sample of ``x[S, T]``."""
    return self._run(x, state, None, None, False, True)

  def counts(self, x, size, hop=None, state=None, final=False):
    """Crossings per block of ``size`` samples every ``hop`` samples (int32 ``[S, n_blocks]``)."""
    size = _block_arg("size", size)
    hop = size if hop is None else _block_arg("hop", hop)
    return self._run(x, state, size, hop, final, False)


def zcross(seq, hysteresis=0, first_sign=0):
  """Zero-crossing stream: 1 for each crossing detected, 0 otherwise (reference ``zcross``).  ``hysteresis`` makes
  two thresholds, ``hysteresis`` and ``-hysteresis``; ``first_sign`` is the sign memory from the past (0: the first
  sign is the first one found in the data).  A non-real ``hysteresis`` or ``first_sign`` raises ``TypeError`` here,
  where the reference raises it at the first value."""
  zc = Zcross(hysteresis, first_sign)
  torch = _engine.torch_mod()
  state = zc.new_state(1)                          # no device: raises at call time
  device = state.device

  def pump():
    for xb in _engine._blocks(seq):
      yield zc.apply(torch.from_numpy(xb).to(device), state=state)[0].cpu().numpy().tolist()

  return Stream(it.chain.from_iterable(pump()))
