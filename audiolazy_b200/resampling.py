"""Lagrange interpolation and sample-rate conversion: reference ``audiolazy/lazy_poly.py:493-603``, on the GPU.

* ``lagrange`` (strategies ``func`` and ``poly``) is the Waring-Lagrange interpolator, restated on the host with the
  reference's operation order, so its values and :class:`~audiolazy_b200.poly.Poly` coefficients are the reference's.
* ``resample(sig, old=1, new=1, order=3, zero=0.)`` is the reference's resampler with a constant step ``old / new``:
  a lazy Stream of float64 values equal to the reference's bit for bit, its errors raised where the reference raises
  them.  A time-varying step (a Stream ``old`` or ``new``) and a step that is not finite and positive (the reference's
  endless stream that never consumes its input) raise ``NotImplementedError``.
* :class:`Resampler` is the batched form: many streams of one rate pair through ``include/alz_b200_resample.h``,
  continued block by block through a :class:`ResampleState`.

The output schedule (how many outputs a block yields, and where) depends on the step only; the library walks it on
the host, the kernels compute the interpolation weights once per call and the compensated sums of every stream.
Input samples are read as float32, as everywhere in this package; ``zero`` is kept in float64.
"""
from __future__ import annotations

import ctypes
import math
import operator
from collections import deque
from collections.abc import Iterable
from functools import reduce
from numbers import Integral

import numpy as np

from . import _build, _capi, _engine
from .core import StrategyDict
from .poly import x as _x
from .stream import Stream, tostream

__all__ = ["lagrange", "resample", "Resampler", "ResampleState"]

MAX_ORDER = 64
ERR_UNSUPPORTED = _capi.ALZ_ERR_UNSUPPORTED
ERR_CAPACITY = -7

_i32, _i64, _f64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["resample"].path, "resampling", {
  "alz_resample_last_error": (ctypes.c_char_p, []),
  "alz_resample_state_doubles": (_i64, [_i32, _i64]),
  "alz_resample_state_init": (_i32, [_vp, _i64, _i32, _f64, _vp]),
  "alz_resample_schedule": (_i64, [_i32, _f64, _f64, _i64, _i64, _vp, _vp, ctypes.POINTER(_f64)]),
  "alz_resample_apply": (_i32, [_vp, _vp, _i32, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _i32, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError, ERR_UNSUPPORTED: NotImplementedError})
#: every function include/alz_b200_resample.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


# --------------------------------------------------------------------------------------
# lagrange (reference lazy_poly.py:493-535)
# --------------------------------------------------------------------------------------
lagrange = StrategyDict("lagrange")


@lagrange.strategy("func")
def lagrange(pairs):
  """Waring-Lagrange interpolator through the points ``pairs`` (``(x, y)`` tuples): a function of ``k`` returning
  ``sum(y_j * w_j(k))``, where ``w_j(k)`` is the left-to-right product of ``(k - x_r) / (x_j - x_r)`` over the other
  points and ``sum`` is Python's (compensated for floats)."""
  xs, ys = zip(*pairs)      # no points: ValueError, as in the reference

  def interpolate(k):
    terms = []
    for j, xj in enumerate(xs):
      factors = [(k - xr) / (xj - xr) for xr in xs if xr != xj]
      terms.append(ys[j] * reduce(operator.mul, factors))    # one point: TypeError, as in the reference
    return sum(terms)

  return interpolate


@lagrange.strategy("poly")
def lagrange(pairs):
  """Waring-Lagrange interpolator polynomial: the ``func`` strategy evaluated at the :class:`Poly` ``x``."""
  return lagrange.func(pairs)(_x)


# --------------------------------------------------------------------------------------
# the native library
# --------------------------------------------------------------------------------------
def _rint(v):
  """The reference's ``rint`` of a non-negative number: the nearest integer, halves away from zero."""
  return int(math.floor(v + .5))


def start_index(order):
  """The pending position a stream starts from: ``int(threshold) + rint(threshold)``, so that consuming the
  ``rint(threshold)`` samples the reference takes up front leaves the first output at ``int(threshold)``."""
  threshold = .5 * (order + 1)
  return float(int(threshold) + _rint(threshold))


def schedule(order, step, idx, n_samples):
  """``(pos, idx_out, idx_next)`` of a block of ``n_samples`` samples (``alz_resample_schedule``): int64 and float64
  numpy arrays, one entry per output, and the position to carry.  Runs on the host; needs no device."""
  # at most (n_samples + 1) / step outputs, up to the rounding of the idx += step additions, whose relative error
  # stays below 1e-6 for steps above 1e-6; below that (or for a step the library refuses) grow on demand
  ok = math.isfinite(step) and step > 0
  cap = int((n_samples + 1) / step * (1 + 1e-6)) + 4 if ok and step >= 1e-6 else 1 << 16
  while True:
    pos = np.empty(cap, dtype=np.int64)
    idxs = np.empty(cap, dtype=np.float64)
    nxt = ctypes.c_double()
    n = lib().alz_resample_schedule(int(order), float(step), float(idx), int(n_samples), cap, pos.ctypes.data,
                                    idxs.ctypes.data, ctypes.byref(nxt))
    if n != ERR_CAPACITY:
      _check(n)
      return pos[:n], idxs[:n], nxt.value
    cap *= 2


def _check_step(old, new):
  """``old / new`` (ZeroDivisionError for ``new == 0``, as the reference) as a float, refusing what the library does
  not evaluate."""
  step = old / new
  if isinstance(step, Iterable):
    raise NotImplementedError("resample with a time-varying step (a Stream old or new) is not supported")
  step = float(step)
  if not (math.isfinite(step) and step > 0):
    raise NotImplementedError("resample with a step old / new = %r is not supported: the reference's output never "
                              "consumes its input (the step must be finite and positive)" % step)
  return step


class ResampleState(object):
  """Device state of :meth:`Resampler.apply` over ``n_streams`` endless streams: the last ``order + 1`` samples of each
  (float64, ``zero`` before the streams start) and the pending position ``idx`` they share (host float).  It is made
  for one resampler and device."""

  def __init__(self, resampler, n_streams):
    torch = _engine.torch_mod()
    self.resampler = resampler
    self.n_streams = int(n_streams)
    self.idx = start_index(resampler.order)
    device = torch.device("cuda", torch.cuda.current_device())
    n = _check(lib().alz_resample_state_doubles(resampler.order, self.n_streams))
    self.tensor = torch.empty(max(1, n), dtype=torch.float64, device=device)
    _check(lib().alz_resample_state_init(self.tensor.data_ptr(), self.n_streams, resampler.order, resampler.zero,
                                         torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


class Resampler(object):
  """Lagrange resampling by the constant step ``old / new`` with ``order + 1`` neighbouring samples (1 <= order <= 64).

  * ``r.apply(x, state=None, dtype=torch.float32)`` -> CUDA tensor ``[S, n_out]`` (float32: the rounding of the float64
    value; or float64) for a CUDA float32 tensor ``x[S, T]`` of ``S`` streams.  Pass ``state=r.new_state(S)`` to
    continue streams across calls: a stream cut into blocks of any lengths gives the values of one call.
  * ``r(seq)`` -> the lazy Stream ``resample(seq, old, new, order, zero)``.

  Every call takes its tables from torch's allocator on the current CUDA stream, so one resampler may be used on
  several CUDA streams and host threads at once (each with its own state)."""

  def __init__(self, old, new, order=3, zero=0.):
    self.step = _check_step(old, new)
    if not isinstance(order, Integral):
      raise TypeError("order must be an integer")
    if order < 1:
      raise ValueError("order must be >= 1 (the reference fails on order %d)" % order)
    if order > MAX_ORDER:
      raise NotImplementedError("resample of order %d: orders above %d are not supported" % (order, MAX_ORDER))
    self.order = int(order)
    self.zero = float(zero)

  def new_state(self, n_streams):
    """State for :meth:`apply` calls that continue ``n_streams`` streams block by block."""
    return ResampleState(self, n_streams)

  def _check_state(self, state, n_streams, device):
    _engine.check_state(state, ResampleState, "Resampler", n_streams, device)
    other = state.resampler
    if other is not self and (other.order, other.step) != (self.order, self.step):
      raise ValueError("state belongs to another resampler")

  def schedule(self, idx, n_samples):
    """:func:`schedule` of this resampler's order and step."""
    return schedule(self.order, self.step, idx, n_samples)

  def apply(self, x, state=None, dtype=None):
    torch = _engine.torch_mod()
    dtype = torch.float32 if dtype is None else dtype
    if dtype not in (torch.float32, torch.float64):
      raise ValueError("dtype must be torch.float32 or torch.float64")
    x, S, T, xs = _engine.stream_input(x)
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      self._check_state(state, S, x.device)
      pos, idxs, idx_next = self.schedule(state.idx, T)
      n = len(pos)
      out = torch.empty((S, n), dtype=dtype, device=x.device)
      pos_d = torch.from_numpy(pos).to(x.device)
      idx_d = torch.from_numpy(idxs).to(x.device)
      w = torch.empty((n, self.order + 1), dtype=torch.float64, device=x.device)
      _check(lib().alz_resample_apply(x.data_ptr(), out.data_ptr(), int(dtype == torch.float64), state.tensor.data_ptr(),
                                      pos_d.data_ptr(), idx_d.data_ptr(), w.data_ptr(), n, S, T, xs, max(n, 1),
                                      self.order, torch.cuda.current_stream(x.device).cuda_stream))
    state.idx = idx_next
    return out

  def __call__(self, seq):
    return Stream(self._outputs(seq))

  def _outputs(self, seq):
    torch = _engine.torch_mod()
    state = self.new_state(1)
    for xb in _engine._blocks(seq):
      yield from self.apply(torch.from_numpy(xb).to(state.device), state=state, dtype=torch.float64)[0].tolist()
    # the reference's next() on the exhausted input, turned into RuntimeError by PEP 479
    raise RuntimeError("generator raised StopIteration")


@tostream
def resample(sig, old=1, new=1, order=3, zero=0.):
  """Generic resampler based on Waring-Lagrange interpolators (reference ``lazy_poly.py:538-603``).

  ``old / new`` is the time step: ``old=1, new=2`` yields two samples per input sample.  ``order + 1`` neighbouring
  samples enter each output, and the input is thought of as padded on the left with ``zero``.  The first output is
  the first input sample; the last is the last one whose samples exist, after which a finite input raises
  ``RuntimeError`` as in the reference (so take as many values as you need).  The reference's errors for a bad
  ``order`` or ``new == 0`` raise at the first value, as there; a time-varying step, a step that is not finite and
  positive, and an order above 64 raise ``NotImplementedError`` there."""
  threshold = .5 * (order + 1)
  step = old / new
  data = deque([zero] * (order + 1), maxlen=order + 1)
  if isinstance(step, Iterable):
    _check_step(old, new)
  sig = iter(sig)
  if order < 1:
    # what the reference meets next: its take of rint(threshold) samples, then an interpolator with no factors
    want = _rint(threshold)
    head = [v for _, v in zip(range(want), sig)]
    if len(head) < want:
      raise RuntimeError("generator raised StopIteration")
    data.extend(head)
    lagrange.func(enumerate(data))(int(threshold))
  yield from Resampler(old, new, order, zero)(sig)
