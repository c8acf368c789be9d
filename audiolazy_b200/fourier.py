"""The discrete Fourier transform at arbitrary frequencies: the reference's ``dft(blk, freqs, normalize=True)``
(``audiolazy/lazy_analysis.py``), its batched form :class:`Dft` over every frame of many streams, and the lazy
:func:`dft_frames`, evaluated by the sm_90a kernel behind ``include/alz_b200_dft.h``.

The spectrum is evaluated at the frequencies the caller lists (rad/sample), with no bin grid and no zero padding: a
semitone grid for pitch tracking, a tone detector's frequencies, log-spaced analysis.  The results equal the
reference's bit for bit (a NaN part is any NaN): the twiddles ``cmath.exp(-1j * n * f)`` are made on the host (the
library restates CPython's arithmetic with the host's libm, and ``cmath`` itself fills the columns it cannot), and the
kernel adds the terms in the reference's order without fused multiply-adds.  Samples are read as float32, as at every
entry point of this package.
"""
from __future__ import annotations

import cmath
import ctypes
import itertools as it
import math
from numbers import Complex, Integral, Real

import numpy as np

from . import _build, _capi, _engine
from .spectral import _window_values
from .stream import Stream

__all__ = ["dft", "Dft", "DftState", "dft_frames"]

MAX_SIZE = 8192
MAX_FREQS = 4096

_i32, _i64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["dft"].path, "DFT", {
  "alz_dft_last_error": (ctypes.c_char_p, []),
  "alz_dft_frames": (_i64, [_i64, _i64, _i32, _i32, _i32]),
  "alz_dft_state_bytes": (_i64, [_i64, _i32]),
  "alz_dft_state_init": (_i32, [_vp, _i64, _i32, _vp]),
  "alz_dft_twiddles": (_i64, [_vp, _i32, _i32, _vp, _vp]),
  "alz_dft_apply_f32": (_i32, [_vp, _i64, _vp, _vp, _i32, _i32, _vp, _i32, _i64, _vp, _i64, _i64, _i32, _i32, _i32,
                               _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError, _capi.ALZ_ERR_UNSUPPORTED: NotImplementedError})
#: every function include/alz_b200_dft.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


def _freq_values(freqs):
  """``freqs`` as a list of floats (an int frequency is the float the reference's complex product makes of it)."""
  out = []
  for f in freqs:
    if isinstance(f, Complex) and not isinstance(f, Real):
      raise NotImplementedError("complex frequencies are not supported")
    out.append(float(f))
  return out


def twiddles(freqs, size):
  """The table ``[size][len(freqs)]`` complex128 (host) of ``cmath.exp(-1j * n * f)``: the library's host restatement,
  and ``cmath`` itself for the columns it leaves (frequencies that are not finite or whose ``n * f`` overflows), so
  that those give the reference's NaNs or raise its ``ValueError("math domain error")``."""
  freqs = np.ascontiguousarray(_freq_values(freqs), dtype=np.float64)
  nf = len(freqs)
  table = np.zeros((size, nf), dtype=np.complex128)
  unfilled = np.zeros(nf, dtype=np.uint8)
  _check(lib().alz_dft_twiddles(freqs.ctypes.data, nf, size, table.ctypes.data, unfilled.ctypes.data))
  for j in np.flatnonzero(unfilled):
    f = float(freqs[j])
    col = [cmath.exp(-1j * n * f) for n in range(size)]       # raises the reference's ValueError
    for v in col:
      # the kernel's term b * w equals the reference's complex(b, 0.0) * w in NaN-ness only when a twiddle that is
      # not finite is NaN in both parts, which is what cmath.exp gives for every such frequency
      if not (math.isfinite(v.real) and math.isfinite(v.imag)) and not (math.isnan(v.real) and math.isnan(v.imag)):
        raise NotImplementedError("twiddle %r of frequency %r is not supported" % (v, f))
    table[:, j] = col
  return table


class DftState(object):
  """Device state of :class:`Dft` calls over ``n_streams`` streams: per stream the samples consumed and the last
  ``size`` samples, which hold what the open frames still need.  It is made for one :class:`Dft` (frequencies, size,
  hop, window, normalization), stream count and device; a call with ``final=True`` ends it."""

  def __init__(self, owner, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.key = owner._key()
    self.consumed = 0
    self.ended = False
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_dft_state_bytes(self.n_streams, owner.size))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_dft_state_init(self.tensor.data_ptr(), self.n_streams, owner.size,
                                      torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


def _int_arg(name, value, lo, hi):
  if not isinstance(value, Integral) or isinstance(value, bool):
    raise TypeError("%s must be an integer, not %s" % (name, type(value).__name__))
  if not lo <= value <= hi:
    raise ValueError("%s must be in %d .. %d (got %d)" % (name, lo, hi, value))
  return int(value)


class Dft(object):
  """The reference's ``dft(block, freqs, normalize)`` of every frame of many streams: frame ``k`` is the block
  ``[k hop, k hop + size)`` of ``Stream(x).blocks(size, hop)`` (``hop`` defaults to ``size``; any hop >= 1), times
  ``wnd`` when given (``None``, a callable ``wnd(size)`` or ``size`` reals, one float64 rounding per sample).

  * ``d.apply(x, state=None, final=False)`` -> ``[S, F, n_freqs]`` of ``dtype`` (complex128, the reference's values
    bit for bit; or complex64, each part their float32 rounding) for a CUDA float32 ``x[S, T]``: the F frames this
    call completes, plus, with ``final=True``, the reference's padded last block when it emits one.
  * ``d.new_state(S)`` -> :class:`DftState`, to continue streams block by block; blocks of any lengths give the same
    bits as one call.  ``d.n_frames(consumed, T, final)``.

  The twiddle table is built on the host once, at construction (which raises the reference's ``ValueError`` when a
  twiddle overflows), and uploaded once per device."""

  def __init__(self, freqs, size, hop=None, wnd=None, normalize=True, dtype=None):
    torch = _engine.torch_mod()
    self.size = _int_arg("size", size, 1, MAX_SIZE)
    self.hop = self.size if hop is None else _int_arg("hop", hop, 1, 2 ** 31 - 1)
    self.freqs = tuple(_freq_values(freqs))
    if not 1 <= len(self.freqs) <= MAX_FREQS:
      raise ValueError("Dft needs 1 .. %d frequencies (got %d)" % (MAX_FREQS, len(self.freqs)))
    values = _window_values(wnd, self.size)
    self.window = None if values is None else np.array([float(v) for v in values], dtype=np.float64)
    self.normalize = bool(normalize)
    dtype = torch.complex128 if dtype is None else dtype
    if dtype not in (torch.complex64, torch.complex128):
      raise ValueError("dtype must be torch.complex64 or torch.complex128")
    self.dtype = dtype
    self.table = twiddles(self.freqs, self.size)
    self._dev = {}

  @property
  def n_freqs(self):
    return len(self.freqs)

  def _key(self):
    return (self.freqs, self.size, self.hop, None if self.window is None else self.window.tobytes(), self.normalize)

  def new_state(self, n_streams):
    return DftState(self, n_streams)

  def n_frames(self, consumed, T, final):
    """Frames a call on ``T`` samples emits after ``consumed`` samples."""
    return _engine.n_blocks(consumed, T, self.size, self.hop, final)

  def _tensors(self, device):
    got = self._dev.get(device)
    if got is None:
      torch = _engine.torch_mod()
      got = self._dev[device] = (torch.from_numpy(self.table).to(device),
                                 None if self.window is None else torch.from_numpy(self.window).to(device))
    return got

  def _check_state(self, state, S, device):
    _engine.check_state(state, DftState, "Dft", S, device)
    if state.key != self._key():
      raise ValueError("state belongs to a Dft with other frequencies, size, hop, window or normalization")
    if state.ended:
      raise ValueError("state was ended by a call with final=True")

  def apply(self, x, state=None, final=False):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input(x)
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      self._check_state(state, S, x.device)
      F = self.n_frames(state.consumed, T, final)
      dev = x.device
      tw, w = self._tensors(dev)
      out = torch.empty((S, F, self.n_freqs), dtype=self.dtype, device=dev)
      _check(lib().alz_dft_apply_f32(x.data_ptr(), xs, None if w is None else w.data_ptr(), tw.data_ptr(),
                                     self.n_freqs, int(self.normalize), out.data_ptr(),
                                     int(self.dtype == torch.complex128), F, state.tensor.data_ptr(), S, T, self.size,
                                     self.hop, int(bool(final)), torch.cuda.current_stream(dev).cuda_stream))
    state.consumed += T
    state.ended = bool(final)
    return out


def _block_values(blk):
  values = list(blk)
  for v in values:
    if isinstance(v, Complex) and not isinstance(v, Real):
      raise NotImplementedError("complex-valued blocks are not supported")
  return values


def dft(blk, freqs, normalize=True):
  """Complex DFT of the block ``blk`` at each frequency of ``freqs`` (rad/sample), in order: ``sum(blk[n] * exp(-1j *
  n * f))``, divided by ``len(blk)`` when ``normalize`` (reference ``lazy_analysis.py``).  Returns a list of Python
  complex values equal to the reference's bit for bit, from one frame of the sm_90a kernel; the samples are read as
  float32.  Raises the reference's errors: ``ValueError("math domain error")`` when ``n * f`` overflows for a sample
  ``n`` of the block, ``ZeroDivisionError`` for an empty block with ``normalize`` (without it, ``0`` per frequency).
  Complex samples or frequencies raise ``NotImplementedError``."""
  values = _block_values(blk)
  freqs = _freq_values(freqs)
  if not freqs:
    return []
  if not values:
    if normalize:
      raise ZeroDivisionError("division by zero")
    return [0] * len(freqs)
  torch = _engine.torch_mod()
  x = torch.from_numpy(_engine._to_f32(values)).to(torch.device("cuda", torch.cuda.current_device()))
  out = []
  for j in range(0, len(freqs), MAX_FREQS):
    d = Dft(freqs[j:j + MAX_FREQS], len(values), normalize=normalize)
    out.extend(d.apply(x, final=True)[0, 0].tolist())
  return out


def dft_frames(seq, freqs, size, hop=None, window=None, normalize=True):
  """Lazy Stream whose element ``k`` is the reference's ``dft(block k, freqs, normalize)`` (a list of complex) of
  ``Stream(seq).blocks(size, hop)``, each block times ``window`` when given (``None``, a callable or ``size`` reals),
  bit for bit.  The twiddles are made when the first frame is taken, which raises the reference's ``ValueError`` for
  a frequency whose ``n * f`` overflows."""
  freqs = _freq_values(freqs)

  def gen():
    if not freqs:                                  # every frame is [], one per block
      d = Dft([0.], size, hop, window, normalize)
      frames = (lambda res: [[] for _ in range(res.shape[1])])
    else:
      d = Dft(freqs, size, hop, window, normalize)
      frames = (lambda res: res[0].cpu().numpy().tolist())
    torch = _engine.torch_mod()
    state = d.new_state(1)
    device = state.device
    for xb in _engine._blocks(seq):
      yield frames(d.apply(torch.from_numpy(xb).to(device), state=state))
    yield frames(d.apply(torch.empty((1, 0), dtype=torch.float32, device=device), state=state, final=True))

  return Stream(it.chain.from_iterable(gen()))
