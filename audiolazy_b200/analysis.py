"""Average magnitude difference function (AMDF): reference ``audiolazy/lazy_analysis.py:686-718``, on the GPU.

``amdf(lag, size)(sig, zero)`` is the reference's ``maverage(size)(abs((1 - z ** -lag).linearize()(sig, zero=zero)),
zero=zero)`` with the deque moving average; its float64 value sequence is reproduced bit for bit and handed out as
float32-rounded Python floats, like every filter output of this package.  :class:`AmdfBank` is the shape a pitch
detector needs: many lags over many streams, evaluated by one kernel (``include/alz_b200_amdf.h``), decimated on the
device and continued block by block through an :class:`AmdfState`.  ``amdf`` is the one-lag case of the bank.
"""
from __future__ import annotations

import ctypes
from numbers import Integral

import numpy as np

from . import _build, _capi, _engine
from .filters import z

__all__ = ["amdf", "AmdfBank", "AmdfState"]

PLAN_SEQUENTIAL = 8

_i32, _i64, _f64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["amdf"].path, "AMDF", {
  "alz_amdf_last_error": (ctypes.c_char_p, []),
  "alz_amdf_plan_create": (_i32, [_vp, _vp, _vp, _i32, _i32, _i32, ctypes.POINTER(_vp)]),
  "alz_amdf_plan_destroy": (None, [_vp]),
  "alz_amdf_state_doubles": (_i64, [_vp, _i64]),
  "alz_amdf_state_init": (_i32, [_vp, _vp, _i64, _f64, _vp]),
  "alz_amdf_plan_chunks": (_i64, [_vp, _i64, _i64]),
  "alz_amdf_apply_f32": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError, _capi.ALZ_ERR_NONCAUSAL: ValueError})
#: every function include/alz_b200_amdf.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


def lag_taps(lag):
  """``[(delay, coeff), ...]``: the terms of ``(1 - z ** -lag).linearize()`` by ascending delay (at most 3, no zero
  coefficient), the difference filter of the reference's ``amdf``.  A term with a negative delay raises
  ``ValueError("Non-causal filter")``, as calling that filter does (a lag in (-1, 0) lands on delays 0 and 1 and is
  causal there too)."""
  terms = [(int(k), float(v)) for k, v in (1 - z ** -lag).linearize().numdict.items() if v != 0]
  if any(k < 0 for k, _ in terms):
    raise ValueError("Non-causal filter")
  return sorted(terms)


def _check_size(size):
  """The reference's errors for a bad ``size``, raised at call time: ``1. / size`` (ZeroDivisionError), then the
  deque of ``size`` items (TypeError for a non-integer, ValueError for a negative one)."""
  if size == 0:
    raise ZeroDivisionError("float division by zero")
  if not isinstance(size, Integral):
    raise TypeError("'%s' object cannot be interpreted as an integer" % type(size).__name__)
  if size < 0:
    raise ValueError("size must be a positive integer")
  return int(size)


class _Plan(object):
  """A compiled AMDF plan on the current CUDA device."""

  def __init__(self, taps, size, sequential=False):
    L = len(taps)
    n_taps = np.array([len(t) for t in taps], dtype=np.int32)
    delays = np.zeros((L, 3), dtype=np.int32)
    coefs = np.zeros((L, 3), dtype=np.float64)
    for l, t in enumerate(taps):
      for j, (k, c) in enumerate(t):
        delays[l, j], coefs[l, j] = k, c
    handle = ctypes.c_void_p()
    _check(lib().alz_amdf_plan_create(n_taps.ctypes.data, delays.ctypes.data, coefs.ctypes.data, L, int(size),
                                      PLAN_SEQUENTIAL if sequential else 0, ctypes.byref(handle)))
    self._h = handle
    self.n_lags = L

  def __del__(self):
    h, self._h = getattr(self, "_h", None), None
    if h and LIB.cdll is not None:
      LIB.cdll.alz_amdf_plan_destroy(h)

  def state_doubles(self, n_streams):
    return _check(lib().alz_amdf_state_doubles(self._h, int(n_streams)))

  def state_init(self, state_ptr, n_streams, zero, stream=0):
    _check(lib().alz_amdf_state_init(self._h, state_ptr, int(n_streams), float(zero), stream))

  def chunks(self, n_streams, n_samples):
    return _check(lib().alz_amdf_plan_chunks(self._h, int(n_streams), int(n_samples)))

  def apply(self, x_ptr, out_ptr, state_ptr, n_streams, n_samples, x_stride, out_stride, decim, phase, stream=0):
    _check(lib().alz_amdf_apply_f32(self._h, x_ptr, out_ptr, state_ptr, int(n_streams), int(n_samples), int(x_stride),
                                    int(out_stride), int(decim), int(phase), stream))


class AmdfState(object):
  """Device state of :meth:`AmdfBank.apply` over ``n_streams`` endless streams: per stream the last ``size + K``
  samples (float64), the running mean of every lag and the samples consumed, plus the decimation ``phase`` (samples of
  the current decimation window already consumed).  It is made for one bank, device and ``decim``."""

  def __init__(self, bank, n_streams, decim=1, zero=0.):
    if int(decim) < 1:
      raise ValueError("decim must be >= 1")
    torch = _engine.torch_mod()
    self.bank = bank
    self.n_streams = int(n_streams)
    self.decim = int(decim)
    self.zero = float(zero)
    self.phase = 0
    plan = bank._plan()
    self.tensor = torch.empty(max(1, plan.state_doubles(self.n_streams)), dtype=torch.float64, device=bank._device())
    plan.state_init(self.tensor.data_ptr(), self.n_streams, self.zero, torch.cuda.current_stream(self.device).cuda_stream)

  @property
  def device(self):
    return self.tensor.device


class AmdfBank(object):
  """The AMDF at many lags sharing one moving-average ``size``.

  * ``bank.apply(x, decim=1, state=None)`` -> CUDA float32 tensor ``[S, L, n_out]`` for a CUDA float32 tensor ``x[S, T]``
    of ``S`` independent streams: every ``decim``-th value of ``amdf(lags[l], size)`` of every stream.  Pass
    ``state=bank.new_state(S, decim)`` to continue streams across calls; then ``n_out = (state.phase + T) // decim``.
  * ``bank(seq, zero=0.)`` -> one lazy Stream per lag, ``[amdf(lag, size)(seq, zero) for lag in lags]``.

  ``sequential=True`` never evaluates few long streams time-parallel (nor does ``ALZ_NO_TIME_PARALLEL=1``); the
  time-parallel evaluation differs from the sequential one by its float64 rounding drift only."""

  def __init__(self, lags, size, sequential=False):
    self.size = _check_size(size)
    self.lags = tuple(v.item() if isinstance(v, np.generic) else v for v in lags)   # numpy scalars: Python numbers
    if not self.lags:
      raise ValueError("an AmdfBank needs at least one lag")
    self.taps = [lag_taps(lag) for lag in self.lags]
    self.sequential = bool(sequential)
    self._plans = {}

  def __len__(self):
    return len(self.lags)

  def _device(self):
    torch = _engine.torch_mod()
    return torch.device("cuda", torch.cuda.current_device())

  def _plan(self):
    dev = self._device()
    plan = self._plans.get(dev.index)
    if plan is None:
      _capi.set_device(dev.index)
      plan = self._plans[dev.index] = _Plan(self.taps, self.size, sequential=self.sequential)
    return plan

  def _same(self, other):
    return other is self or (other.taps == self.taps and other.size == self.size)

  def new_state(self, n_streams, decim=1, zero=0.):
    """State for :meth:`apply` calls that continue ``n_streams`` streams block by block; ``zero`` is the input before
    each stream starts (and seeds the moving average, as in the reference)."""
    return AmdfState(self, n_streams, decim=decim, zero=zero)

  def chunks(self, n_streams, n_samples):
    """Chunks per stream a block of this shape is cut into (1: sequential evaluation)."""
    return self._plan().chunks(n_streams, n_samples)

  def _check_state(self, state, n_streams, decim, device):
    _engine.check_state(state, AmdfState, "AmdfBank", n_streams, device)
    if not self._same(state.bank):
      raise ValueError("state belongs to another bank")
    if state.decim != int(decim):
      raise ValueError("state was created for decim=%d, the call asks for decim=%r" % (state.decim, decim))

  def apply(self, x, decim=1, state=None):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input(x)
    if int(decim) < 1:
      raise ValueError("decim must be >= 1")
    with torch.cuda.device(x.device):
      plan = self._plan()
      if state is None:
        state = self.new_state(S, decim=decim)
      self._check_state(state, S, decim, x.device)
      n_out = (state.phase + T) // state.decim
      out = torch.empty((S, len(self), n_out), dtype=torch.float32, device=x.device)
      plan.apply(x.data_ptr(), out.data_ptr(), state.tensor.data_ptr(), S, T, xs, max(n_out, 1), state.decim, state.phase,
                 torch.cuda.current_stream(x.device).cuda_stream)
    state.phase = (state.phase + T) % state.decim
    return out

  def __call__(self, seq, zero=0.):
    torch = _engine.torch_mod()
    state = self.new_state(1, decim=1, zero=zero)   # errors (no device, too long a lag) raise at call time
    device = state.device

    def pump():
      for xb in _engine._blocks(seq):
        yield self.apply(torch.from_numpy(xb).to(device), state=state)[0].cpu().numpy()

    return _engine.tee_streams(pump(), len(self))


def amdf(lag, size):
  """Average Magnitude Difference Function non-linear filter for a given size and a fixed lag (samples; see
  :func:`~audiolazy_b200.misc.freq2lag` to convert from a frequency).  Returns a callable ``amdf_filter(sig, zero=0.)``
  whose output is a lazy Stream with no decimation, as in the reference; errors (``size == 0``, a non-causal lag, a
  size that is not a positive integer) raise when it is called."""

  def amdf_filter(sig, zero=0.):
    stream, = AmdfBank([lag], size)(sig, zero=zero)
    return stream

  return amdf_filter
