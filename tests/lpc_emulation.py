"""Python float64 emulation of AudioLazy's ``lpc.kautocor(block, order)`` over the blocks of ``Stream.blocks(size,
hop)``, operation for operation (include/alz_b200_lpc.h restates it; the kernel follows it).

On CPython >= 3.12 the builtin ``sum()`` over floats is a compensated (Neumaier) sum, and both hot sums of the
reference -- ``acorr`` and the ``inner`` product of ``levinson_durbin`` -- go through it, so a plain float64 loop does
not reproduce them: :func:`psum` does.  The reference's ``levinson_durbin`` works on ZFilter objects whose polynomials
drop coefficients equal to zero; :func:`kautocor` keeps the dense lists the ``inner`` products iterate over and applies
the same dropping to the coefficient updates.
"""
import hashlib
import math

import numpy as np


def psum(terms):
  """CPython 3.12's ``sum()`` of float items with start 0: the first item is added to 0 as is, the later ones with
  Neumaier's compensation, and the compensation is added at the end when it is finite and nonzero."""
  it = iter(terms)
  for first in it:
    f = 0.0 + first
    break
  else:
    return 0.0
  c = 0.0
  for x in it:
    t = f + x
    if abs(f) >= abs(x):
      c += (f - t) + x
    else:
      c += (x - t) + f
    f = t
  if c != 0.0 and math.isfinite(c):
    f += c
  return f


def acorr(b, order):
  """``[psum(b[n] * b[n + tau] for n) for tau in 0..order]`` of a float64 block; lags past the block give 0."""
  b = [float(v) for v in b]
  return [psum(b[n] * b[n + tau] for n in range(len(b) - tau)) for tau in range(order + 1)]


def _inner(r, a, b):
  return psum(r[abs(i - j)] * ai * bj for i, ai in enumerate(a) for j, bj in enumerate(b))


def _numlist(A):
  """The reference's ``A.numlist``: coefficients up to the highest one that is not zero (a_0 = 1 always is)."""
  hi = max(k for k, v in enumerate(A) if v != 0.0)
  return A[:hi + 1]


def levinson_durbin(r, order):
  """(coef [order + 1], error, failed) from the lags ``r[0..order]``: ``coef[0] = 1``, coefficients the reference
  drops as zero are 0.0.  ``failed`` when some step's denominator is zero (the reference's ``ParCorError``); coef and
  error are then NaN."""
  A = [1.0]
  for m in range(1, order + 1):
    B = [0.0] + A[::-1]                          # A(1 / z) * z^-m, dense, length m + 1
    Zm = [0.0] * m + [1.0]
    den = _inner(r, B, B)
    if den == 0.0:
      return [math.nan] * (order + 1), math.nan, True
    c = _inner(r, _numlist(A), Zm) / den
    A = A + [0.0]
    if c != 0.0:                                 # c == 0: c * B is the empty polynomial
      for k in range(m + 1):
        if B[k] != 0.0:
          p = c * B[k]
          if p != 0.0:
            v = A[k] - p
            A[k] = v if v != 0.0 else 0.0
  return A, _inner(r, _numlist(A), _numlist(A)), False


def kautocor(b, order):
  """``lpc.kautocor(b, order)`` of one float64 block: (acorr, coef, error, failed)."""
  r = acorr(b, order)
  coef, err, failed = levinson_durbin(r, order)
  return r, coef, err, failed


def frames(x, size, hop=None, window=None, final=True):
  """float64 frames of ``Stream(x).blocks(size, hop)`` of one float32 stream: frame k covers samples
  [k hop, k hop + size), each widened and multiplied by ``window[n]``; with ``final``, the padded last block when the
  reference emits one (samples past the end are 0.0)."""
  hop = size if hop is None else hop
  x = np.asarray(x, dtype=np.float32).astype(np.float64)
  N = len(x)
  n_full = max(0, (N - size) // hop + 1)
  ks = list(range(n_full))
  if final and N - n_full * hop > max(size - hop, 0):
    ks.append(n_full)
  w = None if window is None else np.asarray(window, dtype=np.float64)
  out = []
  for k in ks:
    blk = np.zeros(size)
    seg = x[k * hop:k * hop + size]
    blk[:len(seg)] = seg
    with np.errstate(invalid="ignore"):            # inf * 0.0 is NaN, as in the reference
      out.append(blk * w if w is not None else blk)
  return out


def lpc_frames(x, order, size, hop=None, window=None, final=True):
  """Stacked (acorr [F, order + 1], coef [F, order + 1], error [F], failed [F]) of every frame of one stream."""
  res = [kautocor(b, order) for b in frames(x, size, hop, window, final)]
  r = np.array([v[0] for v in res], dtype=np.float64).reshape(len(res), order + 1)
  c = np.array([v[1] for v in res], dtype=np.float64).reshape(len(res), order + 1)
  e = np.array([v[2] for v in res], dtype=np.float64)
  f = np.array([v[3] for v in res], dtype=np.uint8)
  return r, c, e, f


def canon(values):
  """float64 array with every NaN replaced by one quiet NaN, so that bit comparisons treat NaN as equal to NaN."""
  v = np.array(values, dtype=np.float64)
  v[np.isnan(v)] = np.nan
  return v


def digest(values):
  return hashlib.sha256(np.ascontiguousarray(canon(values), dtype="<f8").tobytes()).hexdigest()
