"""Linear predictive coding: block statistics -> analysis filter ``A(z)`` (a FIR ZFilter).

A caller of the filter hot path (SURVEY.md section 8f item 2): ``lpc(blk, order)`` returns the
whitening FIR filter, ``1 / lpc(blk, order)`` the all-pole synthesis filter, and applying either
to a signal goes through the CUDA kernels like any other ZFilter (orders above a biquad use the
generic ring kernel). Mirrors reference ``audiolazy/lazy_lpc.py`` (strategy names, ``error``
attribute, exceptions) and ``acorr`` / ``lag_matrix`` of ``lazy_analysis.py:277-342``; the
recursions here work on coefficient lists, not on filter algebra, so results agree with the
reference to rounding (tests: 1e-9 relative), not bit for bit.

Frame-wise analysis runs on the GPU (``include/alz_b200_lpc.h``): :class:`LpcFrames` evaluates
``lpc.kautocor`` or ``lpc.kcovar`` of every block of ``Stream(x).blocks(size, hop)`` of many
streams, continued block by block through an :class:`LpcState`, and :func:`lpc_frames` is its lazy
form.  :class:`LpcFilter` filters many streams with those rows, switched frame by frame: the residual through
the analysis filters, or an excitation through the all-pole synthesis filters (``include/alz_b200_lpcfilt.h``), the
synthesis of few long streams optionally cut into chunks evaluated in parallel (``include/alz_b200_lpcscan.h``).
Those follow the reference's arithmetic operation for operation (CPython 3.12's compensated
``sum()`` and, for ``kcovar``, its ZFilter algebra included), so they equal the reference's
``lpc.kautocor`` / ``lpc.kcovar`` bit for bit -- not the host strategies of this module, which agree
with it only to rounding.
"""
from __future__ import annotations

import cmath
import collections
import ctypes
import itertools as it
from numbers import Integral, Real

from . import _build, _capi, _engine
from .core import StrategyDict
from .filters import ZFilter
from .stream import Stream

__all__ = ["ParCorError", "acorr", "lag_matrix", "toeplitz", "levinson_durbin", "lpc", "parcor",
           "parcor_stable", "lsf", "lsf_stable", "LpcFrames", "LpcState", "lpc_frames", "parcor_batch", "ParcorResult",
           "LpcFilter", "LpcFilterState"]


class ParCorError(ZeroDivisionError):
  """A reflection (partial correlation) coefficient cannot be found (``lazy_lpc.py:37-41``)."""


def acorr(blk, max_lag=None):
  """Autocorrelation ``[sum_n blk[n] * blk[n + lag] for lag in 0..max_lag]`` of a block with
  a length; lags past the block give zeros (reference ``lazy_analysis.py:277-312``)."""
  blk = list(blk)
  if max_lag is None:
    max_lag = len(blk) - 1
  return [sum(blk[n] * blk[n + lag] for n in range(len(blk) - lag)) for lag in range(max_lag + 1)]


def lag_matrix(blk, max_lag=None):
  """Covariance-method lag matrix: cell ``[i][j] = sum_n blk[n - i] * blk[n - j]`` over the
  ``n`` that need no padding (reference ``lazy_analysis.py:315-342``)."""
  blk = list(blk)
  if max_lag is None:
    max_lag = len(blk) - 1
  elif max_lag >= len(blk):
    raise ValueError("Block length should be higher than order")
  span = range(max_lag, len(blk))
  return [[sum(blk[n - i] * blk[n - j] for n in span) for i in range(max_lag + 1)] for j in range(max_lag + 1)]


def toeplitz(vect):
  """Symmetric Toeplitz matrix (list of lists) from its first row (``lazy_lpc.py:44-49``)."""
  vect = list(vect)
  return [[vect[abs(i - j)] for i in range(len(vect))] for j in range(len(vect))]


def _quadratic_form(matrix, coefs):
  return sum(matrix(i, j) * ai * aj for i, ai in enumerate(coefs) for j, aj in enumerate(coefs))


def _fir(coefs, error):
  filt = ZFilter(list(coefs))
  filt.error = error
  return filt


def levinson_durbin(acdata, order=None):
  """Solve the Yule-Walker equations ``R a = -r`` for the predictor of the given order from
  autocorrelation lags; returns the analysis filter ``1 + a1 z^-1 + ...`` with the squared
  prediction error in ``.error`` (reference ``lazy_lpc.py:52-136``). O(order**2)."""
  acdata = list(acdata)
  if order is None:
    order = len(acdata) - 1
  elif order >= len(acdata):
    acdata = acdata + [0] * (order + 1 - len(acdata))
  a = [1]
  for m in range(1, order + 1):
    # prediction error of the order m-1 predictor, as the quadratic form a' R a
    err = _quadratic_form(lambda i, j: acdata[abs(i - j)], a)
    acc = sum(ai * acdata[m - i] for i, ai in enumerate(a))
    try:
      k = -acc / err
    except ZeroDivisionError:
      raise ParCorError("Can't find next PARCOR coefficient")
    padded = a + [0]
    a = [x + k * y for x, y in zip(padded, reversed(padded))]
  return _fir(a, _quadratic_form(lambda i, j: acdata[abs(i - j)], a))


lpc = StrategyDict("lpc")


@lpc.strategy("autocor", "acorr", "autocorrelation", "auto_correlation")
def lpc(blk, order=None):
  """Autocorrelation-method LPC: the least-squares solver for small orders, Levinson-Durbin
  above 100 (falling back when a reflection coefficient is undefined), ``lazy_lpc.py:142-183``."""
  blk = list(blk)
  if order is None:
    order = len(blk) - 1
  if order < 100:
    return lpc.nautocor(blk, order)
  try:
    return lpc.kautocor(blk, order)
  except ParCorError:
    return lpc.nautocor(blk, order)


def _least_squares(matrix, rhs):
  import numpy as np
  return (np.linalg.pinv(np.asarray(matrix, dtype=np.float64)) @ -np.asarray(rhs, dtype=np.float64)).tolist()


@lpc.strategy("nautocor", "nacorr", "nautocorrelation", "nauto_correlation")
def lpc(blk, order=None):
  """Autocorrelation method, normal equations solved with the pseudo-inverse (``lazy_lpc.py:186-225``)."""
  blk = list(blk)
  if order is None:
    order = len(blk) - 1
  acdata = acorr(blk, order)
  coeffs = _least_squares(toeplitz(acdata[:-1]), acdata[1:])
  return _fir([1] + coeffs, acdata[0] + sum(r * c for r, c in zip(acdata[1:], coeffs)))


@lpc.strategy("kautocor", "kacorr", "kautocorrelation", "kauto_correlation")
def lpc(blk, order=None):
  """Autocorrelation method through Levinson-Durbin (``lazy_lpc.py:228-272``).

  >>> filt = lpc.kautocor([-1, 0, 1, 0] * 4, 2)
  >>> filt.numerator, filt.error
  ([1.0, 0.0, 0.875], 1.875)
  """
  blk = list(blk)
  if order is None:
    order = len(blk) - 1
  return levinson_durbin(acorr(blk, order), order)


@lpc.strategy("covar", "cov", "covariance", "ncovar", "ncov", "ncovariance")
def lpc(blk, order=None):
  """Covariance method (no windowing assumption), pseudo-inverse solver (``lazy_lpc.py:275-294``)."""
  phi = lag_matrix(blk, order)
  coeffs = _least_squares([row[1:] for row in phi[1:]], [row[0] for row in phi[1:]])
  return _fir([1] + coeffs, phi[0][0] + sum(r * c for r, c in zip(phi[0][1:], coeffs)))


@lpc.strategy("kcovar", "kcov", "kcovariance")
def lpc(blk, order=None):
  """Covariance method solved greedily, one lattice-like stage per order, without NumPy: stage
  ``m`` adds ``k_m`` times the part of ``z^-m`` that is orthogonal (under the lag matrix) to
  the earlier stages' directions. Raises ``ValueError("Unstable filter")`` when a ``|k| >= 1``
  (reference ``lazy_lpc.py:297-340``)."""
  phi = lag_matrix(blk, order)
  order = len(phi) - 1
  size = order + 1

  def inner(a, b):
    return sum(phi[i][j] * ai * bj for i, ai in enumerate(a) if ai for j, bj in enumerate(b) if bj)

  def delay(m):
    return [1 if i == m else 0 for i in range(size)]

  a = delay(0)
  basis = [delay(1)]
  beta = [inner(basis[0], basis[0])]
  m = 1
  while True:
    try:
      k = -inner(a, delay(m)) / beta[m - 1]
    except ZeroDivisionError:
      raise ZeroDivisionError("Can't find next coefficient")
    if k >= 1 or k <= -1:
      raise ValueError("Unstable filter")
    a = [x + k * y for x, y in zip(a, basis[m - 1])]
    if m >= order:
      return _fir(a, inner(a, a))
    nxt = delay(m + 1)
    gamma = [inner(nxt, basis[q]) / beta[q] for q in range(m)]
    for q in range(m):
      nxt = [x - gamma[q] * y for x, y in zip(nxt, basis[q])]
    basis.append(nxt)
    beta.append(inner(nxt, nxt))
    m += 1


def _monic_fir(fir_filt):
  den = fir_filt.denominator
  if len(den) != 1:
    raise ValueError("Filter has feedback")
  num = list(fir_filt.numerator)
  if den[0] != 1:
    num = [c / den[0] for c in num]
  return num


def _scaled(terms, c):
  """``Poly(terms) * c`` of the reference: a zero scalar is the zero polynomial, and zero products are dropped."""
  if c == 0:
    return {}
  return {p: v * c for p, v in terms.items() if v * c != 0}


def parcor(fir_filt):
  """Generator of the reflection coefficients of a FIR filter, highest order first (step-down
  recursion; reference ``lazy_lpc.py:343-395``).

  It restates the reference's filter algebra, bit for bit: the polynomial keeps only its nonzero terms, each step is
  ``(A - k zB) * (1 / (1 - k ** 2))`` (a ZFilter divides by a number through its reciprocal, and ``k ** 2`` is
  CPython's float pow), so a finite ``k`` whose square overflows raises ``OverflowError``, and a zero ``1 - k ** 2``
  raises :class:`ParCorError`, both after that ``k`` was yielded.  ``parcor_batch`` evaluates the same on the GPU for
  many rows whose constant term is 1."""
  den = fir_filt.denominator
  if len(den) != 1:
    raise ValueError("Filter has feedback")
  num = list(fir_filt.numerator)
  a = {p: v for p, v in enumerate(num) if v != 0}
  if den[0] != 1:
    a = _scaled(a, 1 / den[0])
  for m in range(len(num) - 1, 0, -1):
    k = a.get(m, 0.0)
    yield k
    zb = {m - p: v for p, v in a.items()}                       # fir_filt(1 / z) * z ** -m
    for p, v in _scaled(zb, k).items():                         # minus k zB
      s = a[p] + -v if p in a else -v
      if s != 0:
        a[p] = s
      else:
        a.pop(p, None)
    try:
      r = 1 / (1 - k ** 2)
    except ZeroDivisionError:
      raise ParCorError("Can't find next PARCOR coefficient")
    a = _scaled(a, r)
    c0 = a.get(0, 0)                                            # (fir_filt - fir_filt.numpoly[0]) + 1
    if c0 != 0:
      s = a[0] + -c0
      if s != 0:
        a[0] = s
      else:
        del a[0]
    s = a[0] + 1 if 0 in a else 1
    if s != 0:
      a[0] = s
    else:
      a.pop(0, None)


def parcor_stable(filt):
  """True when every reflection coefficient of the denominator is inside the unit circle
  (``lazy_lpc.py:398-425``)."""
  try:
    return all(abs(k) < 1 for k in parcor(ZFilter(filt.denpoly)))
  except ParCorError:
    return False


def lsf(fir_filt):
  """Line spectral frequencies (rad/sample) of a FIR filter: the angles of the roots of the
  palindromic / antipalindromic pair, interleaved starting from the lowest (``lazy_lpc.py:428-457``)."""
  import numpy as np
  a = _monic_fir(fir_filt) + [0]
  rev = a[::-1]
  angles = []
  for sign in (1, -1):
    poly = [x + sign * y for x, y in zip(a, rev)]
    angles.append(sorted(cmath.phase(r) for r in np.roots(poly[::-1])))
  return tuple(it.chain.from_iterable(zip(*sorted(angles))))


def lsf_stable(filt):
  """True when the LSFs of the two polynomials strictly alternate (``lazy_lpc.py:460-487``)."""
  data = lsf(ZFilter(filt.denpoly))
  return all(x < y for x, y in zip(data, data[1:]))


# ---------------------------------------------------------------------------------------------------------------------
# Frame-wise LPC on the GPU (include/alz_b200_lpc.h)
# ---------------------------------------------------------------------------------------------------------------------

MAX_ORDER = 64
MAX_SIZE = 8192

_i32, _i64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["lpc"].path, "LPC", {
  "alz_lpc_last_error": (ctypes.c_char_p, []),
  "alz_lpc_frames": (_i64, [_i64, _i64, _i32, _i32, _i32]),
  "alz_lpc_state_bytes": (_i64, [_i64, _i32]),
  "alz_lpc_state_init": (_i32, [_vp, _i64, _i32, _vp]),
  "alz_lpc_scratch_bytes": (_i64, [_i64, _i64, _i32]),
  "alz_lpc_apply_f32": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp,
                               _i64, _vp]),
  "alz_lpc_covar_scratch_bytes": (_i64, [_i64, _i64, _i32]),
  "alz_lpc_covar_apply_f32": (_i32, [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _i32,
                                     _vp, _i64, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})
#: every function include/alz_b200_lpc.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


def _int_arg(name, value, lo, hi):
  if not isinstance(value, Integral) or isinstance(value, bool):
    raise TypeError("%s must be an integer, not %s" % (name, type(value).__name__))
  if not lo <= value <= hi:
    raise ValueError("%s must be in %d .. %d (got %d)" % (name, lo, hi, value))
  return int(value)


LpcResult = collections.namedtuple("LpcResult", ["coef", "error", "failed"])

#: the strategies of :data:`lpc` the GPU evaluates; the others solve with ``numpy.linalg.pinv``, whose SVD no kernel
#: can reproduce bit for bit
GPU_METHODS = ("kautocor", "kcovar")


def _method(name):
  """The canonical name of the :data:`lpc` strategy ``name`` (any of its aliases), which must be one the GPU runs."""
  if not isinstance(name, str):
    raise TypeError("method must be a string, not %s" % type(name).__name__)
  for canon in GPU_METHODS:
    if name in lpc and lpc[name] is lpc[canon]:
      return canon
  names = sorted(n for n in lpc._names if any(lpc[n] is lpc[c] for c in GPU_METHODS))
  raise ValueError("method %r is not evaluated on the GPU; the supported ones are %s" % (name, ", ".join(names)))


class LpcState(object):
  """Device state of :class:`LpcFrames` calls over ``n_streams`` streams: per stream the samples consumed and the last
  ``size`` samples, which hold what the open frames still need.  It is made for one :class:`LpcFrames` (order, size,
  hop, window), stream count and device; a call with ``final=True`` ends it."""

  def __init__(self, frames, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.key = frames._key()
    self.consumed = 0
    self.ended = False
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_lpc_state_bytes(self.n_streams, frames.size))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_lpc_state_init(self.tensor.data_ptr(), self.n_streams, frames.size,
                                      torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


class LpcFrames(object):
  """Linear prediction of every frame of many streams: frame ``k`` is the block ``[k hop, k hop + size)`` of
  ``Stream(x).blocks(size, hop)`` (``hop`` defaults to ``size``), times ``window`` when one is given (``size`` reals),
  and its result equals the reference's ``lpc.<method>(block, order)`` bit for bit.  ``method`` is ``"kautocor"``
  (autocorrelation method, Levinson-Durbin) or ``"kcovar"`` (covariance method, a Gram-Schmidt lattice on the lag
  matrix; it needs ``1 <= order < size``), or any alias :data:`lpc` gives them (``"kacorr"``, ``"kcov"``, ...).

  * ``lp.apply(x, state=None, final=False)`` -> :class:`LpcResult` ``(coef [S, F, order + 1] float64, error [S, F]
    float64, failed [S, F] uint8)`` for a CUDA float32 ``x[S, T]``: the F frames this call completes, plus, with
    ``final=True``, the reference's padded last block when it emits one.  ``coef[..., 0]`` is 1 and coefficients the
    reference drops as zero are 0.0; ``failed`` marks the frames where the reference raises (their coef and error are
    NaN): 1 for kautocor's :class:`ParCorError` and kcovar's ``ZeroDivisionError``, 2 for kcovar's
    ``ValueError("Unstable filter")``.
  * ``lp.acorr(x, state=None, final=False)`` -> the lags ``[S, F, order + 1]`` float64 of the same frames.
  * ``lp.lag_matrix(x, state=None, final=False)`` -> the reference's ``lag_matrix(block, order)`` ``[S, F, order + 1,
    order + 1]`` float64 of the same frames (``order < size``), the statistics of the covariance methods.
  * ``lp.new_state(S)`` -> :class:`LpcState`, to continue streams block by block; blocks of any lengths give the same
    bits as one call."""

  def __init__(self, order, size, hop=None, window=None, method="kautocor"):
    self.method = _method(method)
    self.order = _int_arg("order", order, 0, MAX_ORDER)
    self.size = _int_arg("size", size, 1, MAX_SIZE)
    if self.method == "kcovar":
      if self.order < 1:
        raise ValueError("kcovar needs order >= 1 (the reference raises IndexError at order 0)")
      if self.order >= self.size:
        raise ValueError("Block length should be higher than order")
    self.hop = self.size if hop is None else _int_arg("hop", hop, 1, 2 ** 31 - 1)
    if window is None:
      self.window = None
    else:
      try:
        values = list(window)
      except TypeError:
        raise TypeError("window must be a sequence of %d reals" % self.size)
      if not all(isinstance(v, Real) for v in values):
        raise TypeError("window must be a sequence of reals")
      if len(values) != self.size:
        raise ValueError("window has %d values, size is %d" % (len(values), self.size))
      self.window = tuple(float(v) for v in values)
    self._windows = {}

  def _key(self):
    return (self.order, self.size, self.hop, self.window, self.method)

  def new_state(self, n_streams):
    return LpcState(self, n_streams)

  def n_frames(self, consumed, T, final):
    """Frames a call on ``T`` samples emits after ``consumed`` samples (the block count of ``zcross``'s counts)."""
    return _engine.n_blocks(consumed, T, self.size, self.hop, final)

  def _window(self, device):
    if self.window is None:
      return None
    w = self._windows.get(device)
    if w is None:
      torch = _engine.torch_mod()
      w = self._windows[device] = torch.tensor(self.window, dtype=torch.float64, device=device)
    return w

  def _check_state(self, state, S, device):
    _engine.check_state(state, LpcState, "LpcFrames", S, device)
    if state.key != self._key():
      raise ValueError("state belongs to an LpcFrames with another order, size, hop or window, or another method")
    if state.ended:
      raise ValueError("state was ended by a call with final=True")

  def _run(self, x, state, final, solve, covar):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input(x)
    L = self.order + 1
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      self._check_state(state, S, x.device)
      F = self.n_frames(state.consumed, T, final)
      dev = x.device
      w = self._window(dev)
      wp = None if w is None else w.data_ptr()
      stream = torch.cuda.current_stream(dev).cuda_stream
      apply, scratch_bytes = ((lib().alz_lpc_covar_apply_f32, lib().alz_lpc_covar_scratch_bytes) if covar else
                              (lib().alz_lpc_apply_f32, lib().alz_lpc_scratch_bytes))
      if solve:
        coef = torch.empty((S, F, L), dtype=torch.float64, device=dev)
        err = torch.empty((S, F), dtype=torch.float64, device=dev)
        failed = torch.empty((S, F), dtype=torch.uint8, device=dev)
        nbytes = _check(scratch_bytes(S, F, self.order))
        scratch = torch.empty(max(8, nbytes), dtype=torch.uint8, device=dev)   # on this stream: torch's allocator orders reuse
        _check(apply(x.data_ptr(), xs, wp, None, coef.data_ptr(), err.data_ptr(), failed.data_ptr(), F,
                     state.tensor.data_ptr(), S, T, self.order, self.size, self.hop, int(bool(final)), scratch.data_ptr(),
                     nbytes, stream))
        out = LpcResult(coef, err, failed)
      else:
        out = torch.empty((S, F, L, L) if covar else (S, F, L), dtype=torch.float64, device=dev)
        _check(apply(x.data_ptr(), xs, wp, out.data_ptr(), None, None, None, F, state.tensor.data_ptr(), S, T,
                     self.order, self.size, self.hop, int(bool(final)), None, 0, stream))
    state.consumed += T
    state.ended = bool(final)
    return out

  def apply(self, x, state=None, final=False):
    """Coefficients, squared prediction errors and failure codes of every frame this call emits."""
    return self._run(x, state, final, True, self.method == "kcovar")

  def acorr(self, x, state=None, final=False):
    """Autocorrelation lags 0 .. order of every frame this call emits."""
    return self._run(x, state, final, False, False)

  def lag_matrix(self, x, state=None, final=False):
    """The covariance-method lag matrix of every frame this call emits: ``[S, F, order + 1, order + 1]`` float64,
    cell ``[j][i] = sum(b[n - i] * b[n - j] for n in order .. size - 1)`` (symmetric)."""
    if self.order >= self.size:
      raise ValueError("Block length should be higher than order")
    return self._run(x, state, final, False, True)


def lpc_frames(seq, order, size, hop=None, window=None, method="kautocor"):
  """Lazy Stream of the analysis filters of every block of ``Stream(seq).blocks(size, hop)`` (times ``window``, when
  given): element ``k`` is the reference's ``lpc.<method>(block k, order)`` (``"kautocor"`` or ``"kcovar"``, or an
  alias), a FIR :class:`ZFilter` with the squared prediction error in ``.error``, bit for bit.  Reaching a frame where
  the reference raises raises the same, after the frames before it: :class:`ParCorError` for kautocor,
  ``ZeroDivisionError("Can't find next coefficient")`` or ``ValueError("Unstable filter")`` for kcovar, and kcovar of
  order 0 raises ``IndexError`` at the first frame."""
  method = _method(method)
  covar0 = method == "kcovar" and isinstance(order, Integral) and order == 0
  lp = LpcFrames(order, size, hop, window, "kautocor" if covar0 else method)
  torch = _engine.torch_mod()
  state = lp.new_state(1)                          # no device: raises at call time
  device = state.device

  def frames(res):
    coef, err, failed = (t[0].cpu().numpy() for t in res)
    for c, e, f in zip(coef, err, failed):
      if covar0:
        raise IndexError("list index out of range")
      if f:
        if method == "kautocor":
          raise ParCorError("Can't find next PARCOR coefficient")
        if f == 1:
          raise ZeroDivisionError("Can't find next coefficient")
        raise ValueError("Unstable filter")
      filt = ZFilter([1] + c[1:].tolist())
      filt.error = float(e)
      yield filt

  def pump():
    for xb in _engine._blocks(seq):
      yield frames(lp.apply(torch.from_numpy(xb).to(device), state=state))
    yield frames(lp.apply(torch.empty((1, 0), dtype=torch.float32, device=device), state=state, final=True))

  return Stream(it.chain.from_iterable(pump()))


# ---------------------------------------------------------------------------------------------------------------------
# Batched PARCOR on the GPU (include/alz_b200_parcor.h)
# ---------------------------------------------------------------------------------------------------------------------

PARCOR_MAX_LEN = 65
PARCOR_LIB = _capi.NativeLib(_build.LIBRARIES["parcor"].path, "PARCOR", {
  "alz_parcor_last_error": (ctypes.c_char_p, []),
  "alz_parcor_f64": (_i32, [_vp, _i64, _i64, _i32, _vp, _vp, _vp, _vp, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})

ParcorResult = collections.namedtuple("ParcorResult", ["k", "count", "failed", "stable"])


def parcor_batch(coef):
  """The reflection coefficients of many FIR rows at once: for a CUDA float64 tensor ``coef[..., L]`` (any leading
  shape, ``1 <= L <= 65``, the last dimension contiguous; ``LpcFrames(...).apply(x).coef`` as it comes), a
  :class:`ParcorResult` of

  * ``k [..., L - 1]`` float64: what ``parcor(ZFilter(row))`` yields, in order (highest order first), NaN past count;
  * ``count [...]`` int32: how many values it yields;
  * ``failed [...]`` uint8: 0, 1 where it then raises :class:`ParCorError`, 2 where ``k ** 2`` raises
    ``OverflowError``, 3 for a row whose constant term is not 1 (not evaluated: NaN k, count 0; :func:`parcor` takes
    those);
  * ``stable [...]`` bool: ``parcor_stable(1 / ZFilter(row))``.

  The values equal the reference's bit for bit (a NaN by NaN-ness), ``k ** 2`` included (see
  ``include/alz_b200_parcor.h``)."""
  import torch
  if not isinstance(coef, torch.Tensor):
    raise TypeError("coef must be a torch tensor, not %s" % type(coef).__name__)
  if coef.dtype != torch.float64:
    raise TypeError("coef must be float64 (got %s)" % coef.dtype)
  if coef.dim() < 1:
    raise ValueError("coef needs a last dimension of coefficients")
  L = coef.shape[-1]
  if not 1 <= L <= PARCOR_MAX_LEN:
    raise ValueError("rows must have 1 .. %d coefficients (got %d)" % (PARCOR_MAX_LEN, L))
  if not coef.is_cuda:
    raise ValueError("coef must be a CUDA tensor")
  _engine.torch_mod()                                           # a usable CUDA device
  lead = tuple(coef.shape[:-1])
  with torch.cuda.device(coef.device):
    if coef.stride(-1) != 1:
      coef = coef.contiguous()
    rows = coef.reshape(-1, L) if coef.numel() else coef.new_empty((0, L))
    if rows.dim() != 2 or rows.stride(-1) != 1 or (rows.shape[0] > 1 and rows.stride(0) < L):
      rows = rows.contiguous()
    n = rows.shape[0]
    dev = coef.device
    k = torch.empty((n, L - 1), dtype=torch.float64, device=dev)
    count = torch.empty((n,), dtype=torch.int32, device=dev)
    failed = torch.empty((n,), dtype=torch.uint8, device=dev)
    stable = torch.empty((n,), dtype=torch.uint8, device=dev)
    if n:
      PARCOR_LIB.check(PARCOR_LIB.load().alz_parcor_f64(
        rows.data_ptr(), rows.stride(0), n, L, k.data_ptr(), count.data_ptr(), failed.data_ptr(), stable.data_ptr(),
        torch.cuda.current_stream(dev).cuda_stream))
  return ParcorResult(k.reshape(lead + (L - 1,)), count.reshape(lead), failed.reshape(lead),
                      stable.reshape(lead).bool())


# ---------------------------------------------------------------------------------------------------------------------
# Frame-wise LPC analysis and synthesis filtering on the GPU (include/alz_b200_lpcfilt.h)
# ---------------------------------------------------------------------------------------------------------------------

LPCFILT_LIB = _capi.NativeLib(_build.LIBRARIES["lpcfilt"].path, "LPC filter", {
  "alz_lpcfilt_last_error": (ctypes.c_char_p, []),
  "alz_lpcfilt_state_bytes": (_i64, [_i64, _i32]),
  "alz_lpcfilt_state_init": (_i32, [_vp, _i64, _i32, _vp]),
  "alz_lpcfilt_rows": (_i64, [_i64, _i64, _i64]),
  "alz_lpcfilt_apply": (_i32, [_vp, _i32, _i64, _vp, _i32, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _i32,
                               _i64, _i32, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})

LPCFILT_KINDS = {"analysis": 0, "synthesis": 1}

LPCSCAN_LIB = _capi.NativeLib(_build.LIBRARIES["lpcscan"].path, "time-parallel LPC synthesis", {
  "alz_lpcscan_last_error": (ctypes.c_char_p, []),
  "alz_lpcscan_chunks": (_i64, [_i64, _i64, _i32, _i64]),
  "alz_lpcscan_scratch_bytes": (_i64, [_i64, _i64, _i32]),
  "alz_lpcscan_apply": (_i32, [_vp, _i32, _i64, _vp, _i32, _i64, _vp, _i64, _i64, _i64, _vp, _i64, _i64, _i64, _i32,
                               _i64, _i64, _vp, _i64, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})


def _sample_dtype(torch, dtype, what):
  if dtype == torch.float32:
    return 0
  if dtype == torch.float64:
    return 1
  raise ValueError("%s must be torch.float32 or torch.float64" % what)


class LpcFilterState(object):
  """Device state of :class:`LpcFilter` calls over ``n_streams`` streams: the samples consumed (counted here, the
  same for every stream) and per stream the last ``order`` inputs (analysis) or outputs (synthesis) as float64.  It is
  made for one (order, hop, kind), stream count and device; a new state is zero, the reference's default ``memory``
  and ``zero``."""

  def __init__(self, filt, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.key = filt._key()
    self.consumed = 0
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      L = LPCFILT_LIB.load()
      nbytes = LPCFILT_LIB.check(L.alz_lpcfilt_state_bytes(self.n_streams, filt.order))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      LPCFILT_LIB.check(L.alz_lpcfilt_state_init(self.tensor.data_ptr(), self.n_streams, filt.order,
                                                 torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


class LpcFilter(object):
  """Frame-wise LPC filtering of many streams: row ``r`` of a stream's coefficient table (``1, c_1 .. c_order``, as
  :class:`LpcFrames` gives them) filters that stream's samples ``[r hop, (r + 1) hop)``.  ``kind="analysis"`` is the
  residual through ``A(z) = 1 + sum(c_k z^-k)``, ``kind="synthesis"`` the all-pole ``1 / A(z)``: the reference's
  ``1 + sum(held(k) * z ** -k)`` and ``1 / (1 + sum(held(k) * z ** -k))``, ``held(k)`` being each row's ``c_k``
  repeated ``hop`` times, with their default (zero) memory.

  * ``f.apply(x, coef, state=None)`` -> CUDA tensor ``[S, T]`` of ``dtype`` for a CUDA float32 or float64 ``x[S, T]``
    and a CUDA float64 ``coef[S, F, order + 1]`` (``LpcFrames(...).apply(x).coef`` as it comes: any strides but along
    the taps, and a stream stride of 0, from ``expand``, shares one table).  Column 0 is not read.  Row 0 of a call is
    the row that covers its first sample; ``F`` must be at least ``f.n_rows(state.consumed, T)`` (fewer raise
    ``ValueError``, where the reference raises when a coefficient Stream ends before its input) and rows past it are
    not read.  The values are the reference's bit for bit (float64) or their rounding (float32).
  * ``f.n_rows(consumed, T)`` -> the rows a call on ``T`` samples reads after ``consumed``.
  * ``f.new_state(S)`` -> :class:`LpcFilterState`, to continue streams block by block; blocks of any lengths give the
    bits of one call.
  * ``f.chunks(S, T)`` -> the chunks per stream a call of that shape is cut into (1: sequential).

  ``time_parallel`` lets the synthesis of few long streams, which one thread per stream walks slowly, run in chunks
  (``include/alz_b200_lpcscan.h``): each chunk's response to its start state is summarized, the chunk start states are
  scanned, and every chunk is rerun from its own.  ``False`` (the default) always walks sequentially; ``True`` lets a
  cost model pick the chunk count, which is 1 unless the chunks pay; a positive int forces that count, lowered so that
  every chunk holds at least ``max(order, 1)`` samples.  A call cut into chunks differs from the sequential bits by the
  float64 rounding drift of the scan (``DESIGN.md`` gives the measured size); a stream whose chunk summaries or scanned
  states are not finite (NaN or infinite samples or rows, unstable rows that overflow) is walked sequentially in the
  same launches and keeps its bits.  Calls of either kind mix freely on one state.  The analysis is sample-parallel
  and exact already, and ignores the option."""

  def __init__(self, order, hop, kind="analysis", dtype=None, time_parallel=False):
    self.order = _int_arg("order", order, 0, MAX_ORDER)
    self.hop = _int_arg("hop", hop, 1, 2 ** 62)
    if not isinstance(kind, str) or kind not in LPCFILT_KINDS:
      raise ValueError("kind must be 'analysis' or 'synthesis' (got %r)" % (kind,))
    self.kind = kind
    if dtype is None:
      import torch
      dtype = torch.float32
    if str(dtype) not in ("torch.float32", "torch.float64"):
      raise ValueError("dtype must be torch.float32 or torch.float64")
    self.dtype = dtype
    if isinstance(time_parallel, bool):
      self.time_parallel = time_parallel
    elif isinstance(time_parallel, Integral):
      if time_parallel < 1:
        raise ValueError("time_parallel must be True, False or a positive chunk count (got %d)" % time_parallel)
      self.time_parallel = int(time_parallel)
    else:
      raise TypeError("time_parallel must be a bool or a positive int, not %s" % type(time_parallel).__name__)

  def _key(self):
    return (self.order, self.hop, self.kind)

  def chunks(self, n_streams, n_samples):
    """Chunks per stream a call on ``n_streams`` x ``n_samples`` is cut into (1: sequential evaluation)."""
    S = _int_arg("n_streams", n_streams, 0, 2 ** 62)
    T = _int_arg("n_samples", n_samples, 0, 2 ** 62)
    if self.kind != "synthesis" or self.time_parallel is False or self.order == 0:
      return 1
    if self.time_parallel is True:
      return LPCSCAN_LIB.check(LPCSCAN_LIB.load().alz_lpcscan_chunks(S, T, self.order, self.hop))
    return max(1, min(self.time_parallel, T // self.order))

  def new_state(self, n_streams):
    return LpcFilterState(self, n_streams)

  def n_rows(self, consumed, T):
    """Rows a call on ``T`` samples reads after ``consumed`` samples (0 for an empty call)."""
    consumed = _int_arg("consumed", consumed, 0, 2 ** 62)
    T = _int_arg("T", T, 0, 2 ** 62)
    return (consumed + T - 1) // self.hop - consumed // self.hop + 1 if T else 0

  def apply(self, x, coef, state=None):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input64(x)
    if not isinstance(coef, torch.Tensor) or coef.dtype != torch.float64 or coef.dim() != 3 or not coef.is_cuda:
      raise ValueError("coef must be a CUDA float64 tensor [streams, rows, order + 1]")
    if coef.shape[0] != S or coef.shape[2] != self.order + 1:
      raise ValueError("coef is %s, x has %d streams and the order is %d: need [%d, rows, %d]"
                       % (tuple(coef.shape), S, self.order, S, self.order + 1))
    if coef.device != x.device:
      raise ValueError("coef lives on %s, x on %s" % (coef.device, x.device))
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      _engine.check_state(state, LpcFilterState, "LpcFilter", S, x.device)
      if state.key != self._key():
        raise ValueError("state belongs to an LpcFilter with another order, hop or kind")
      F = coef.shape[1]
      need = self.n_rows(state.consumed, T)
      if F < need:
        raise ValueError("coef has %d rows per stream; %d samples after %d need %d (hop %d)"
                         % (F, T, state.consumed, need, self.hop))
      if coef.stride(2) != 1 and self.order > 0:
        coef = coef.contiguous()
      out = torch.empty((S, T), dtype=self.dtype, device=x.device)
      P = self.chunks(S, T)
      stream = torch.cuda.current_stream(x.device).cuda_stream
      if P > 1:
        L = LPCSCAN_LIB.load()
        nbytes = LPCSCAN_LIB.check(L.alz_lpcscan_scratch_bytes(S, P, self.order))
        # on this stream: torch's allocator orders reuse
        scratch = torch.empty(max(8, nbytes), dtype=torch.uint8, device=x.device)
        LPCSCAN_LIB.check(L.alz_lpcscan_apply(
          x.data_ptr(), _sample_dtype(torch, x.dtype, "x"), xs, out.data_ptr(), _sample_dtype(torch, self.dtype, "dtype"),
          max(T, 1), coef.data_ptr(), coef.stride(1) if F > 1 else self.order + 1, coef.stride(0) if S > 1 else 0, F,
          state.tensor.data_ptr(), S, T, state.consumed, self.order, self.hop, P, scratch.data_ptr(), nbytes, stream))
      else:
        LPCFILT_LIB.check(LPCFILT_LIB.load().alz_lpcfilt_apply(
          x.data_ptr(), _sample_dtype(torch, x.dtype, "x"), xs, out.data_ptr(),
          _sample_dtype(torch, self.dtype, "dtype"), max(T, 1), coef.data_ptr(), coef.stride(1) if F > 1 else self.order + 1, coef.stride(0) if S > 1 else 0, F,
          state.tensor.data_ptr(), S, T, state.consumed, self.order, self.hop, LPCFILT_KINDS[self.kind], stream))
    state.consumed += T
    return out
