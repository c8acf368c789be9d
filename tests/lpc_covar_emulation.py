"""Python float64 emulation of AudioLazy's covariance-method LPC, ``lpc.kcovar(block, order)``, and of its
``lag_matrix(block, order)``, operation for operation (include/alz_b200_lpc.h restates it; the kernels follow it).

The reference's ``kcovar`` is a Gram-Schmidt lattice on ZFilter objects.  Their polynomials drop every coefficient
equal to zero, an addition keeps a term only one side has as it is, and ``inner`` runs over the *dense* ``numlist``s
(a missing power reads 0.0, a list stops at its highest power).  :func:`kcovar` keeps dense lists with +0.0 for a
missing power plus each list's ``numlist`` length, and applies the same dropping to every update.

``inner(A, z^-m)`` and ``inner(z^-(m+1), B[q])`` are mostly products with a factor 0.0.  Such a product is +-0 when
its other factors give a finite partial product, and adding +-0 leaves the compensated sum's state unchanged, so
``fast=True`` (what the kernel does) sums only the products of the unit coefficient, and returns NaN when one skipped
product is NaN (the dense sum is then NaN too).  ``fast=False`` sums every product, as the reference does.
"""
import math

import numpy as np

from lpc_emulation import canon, digest, frames, psum  # noqa: F401  (re-exported for the tests)

ZERO_DIVISION, UNSTABLE = 1, 2


def lag_matrix(b, order):
  """``[[psum(b[n - i] * b[n - j] for n in order .. size - 1) for i] for j]`` of a float64 block, as a float64
  ``[order + 1, order + 1]`` array.  The compensated sums run on all cells at once, one term per step."""
  b = np.asarray(b, dtype=np.float64)
  size, L = len(b), order + 1
  if order >= size:
    raise ValueError("Block length should be higher than order")
  J, I = np.meshgrid(np.arange(L), np.arange(L), indexing="ij")
  f = np.zeros((L, L))
  c = np.zeros((L, L))
  with np.errstate(invalid="ignore", over="ignore"):
    for n in range(order, size):
      x = b[n - I] * b[n - J]
      t = f + x
      c += np.where(np.abs(f) >= np.abs(x), (f - t) + x, (x - t) + f)
      f = t
    return np.where((c != 0.0) & np.isfinite(c), f + c, f)


def _dense_inner(phi, a, la, b, lb):
  return psum(phi[i][j] * a[i] * b[j] for i in range(la) for j in range(lb))


def _numlist_len(a):
  return max(k for k, v in enumerate(a) if v != 0.0) + 1


def kcovar(phi, fast=True):
  """(coef [order + 1], error, failed) of the lag matrix ``phi`` (a list of lists or an array, order >= 1).

  ``failed`` is 0, ZERO_DIVISION (the reference's ``ZeroDivisionError("Can't find next coefficient")``) or UNSTABLE
  (its ``ValueError("Unstable filter")``); coef and error of a failed frame are NaN.  Order 0 raises IndexError, as
  the reference does."""
  phi = [[float(v) for v in row] for row in phi]
  order = len(phi) - 1
  L = order + 1
  if order < 1:
    raise IndexError("list index out of range")
  maxphi = 0.0
  for row in phi:
    for v in row:
      maxphi = max(maxphi, abs(v)) if math.isfinite(v) else math.inf

  def maxabs(a, n):
    m = 0.0
    for v in a[:n]:
      m = max(m, abs(v)) if math.isfinite(v) else math.inf
    return m

  def quiet(bound):
    return math.isfinite(maxphi * bound)             # then every partial product is finite

  def inner_a_unit(A, la, m):
    # inner(A, z^-m): the products (phi[i][j] * A[i]) * 0.0 for j < m are skipped
    if not fast:
      return _dense_inner(phi, A, la, [0.0] * m + [1.0], m + 1)
    if not quiet(maxabs(A, la)):
      if any(not math.isfinite(phi[i][j] * A[i]) for i in range(la) for j in range(m)):
        return math.nan
    return psum(phi[i][m] * A[i] for i in range(la))

  def inner_unit_b(m1, Bq, lb):
    # inner(z^-m1, B[q]): the products (phi[i][j] * 0.0) * B[q][j] for i < m1 are skipped
    if not fast:
      return _dense_inner(phi, [0.0] * m1 + [1.0], m1 + 1, Bq, lb)
    if not quiet(maxabs(Bq, lb)):
      if any(not (math.isfinite(phi[i][j]) and math.isfinite(Bq[j])) for i in range(m1) for j in range(lb)):
        return math.nan
    return psum(phi[m1][j] * Bq[j] for j in range(lb))

  A = [1.0] + [0.0] * order
  la = 1
  B = [[0.0, 1.0]]                                   # B[q] has powers 1 .. q + 1; its numlist length is q + 2
  beta = [_dense_inner(phi, B[0], 2, B[0], 2)]
  m = 1
  while True:
    if beta[m - 1] == 0.0:
      return [math.nan] * L, math.nan, ZERO_DIVISION
    k = -inner_a_unit(A, la, m) / beta[m - 1]
    if k >= 1 or k <= -1:
      return [math.nan] * L, math.nan, UNSTABLE
    for p in range(1, m + 1):                      # A += k * B[m - 1]
      b = B[m - 1][p]
      if b != 0.0:
        t = k * b
        if t != 0.0:
          v = A[p] + t
          A[p] = v if v != 0.0 else 0.0
    la = _numlist_len(A)
    if m >= order:
      return A, _dense_inner(phi, A, la, A, la), 0
    gamma = [inner_unit_b(m + 1, B[q], q + 2) / beta[q] for q in range(m)]
    Bm = [0.0] * (m + 2)                           # z^-(m + 1) - sum(gamma[q] * B[q] for q < m)
    for p in range(1, m + 1):
      acc = 0.0
      for q in range(p - 1, m):
        b = B[q][p]
        if b != 0.0:
          t = gamma[q] * b
          if t != 0.0:
            v = acc + t
            acc = v if v != 0.0 else 0.0
      Bm[p] = -acc if acc != 0.0 else 0.0
    Bm[m + 1] = 1.0
    B.append(Bm)
    beta.append(_dense_inner(phi, Bm, m + 2, Bm, m + 2))
    m += 1


def lpc_frames(x, order, size, hop=None, window=None, final=True, fast=True):
  """Stacked (lagm [F, L, L], coef [F, L], error [F], failed [F]) of every frame of one stream, L = order + 1."""
  L = order + 1
  lagm, coef, err, failed = [], [], [], []
  for b in frames(x, size, hop, window, final):
    phi = lag_matrix(b, order)
    c, e, f = kcovar(phi, fast)
    lagm.append(phi)
    coef.append(c)
    err.append(e)
    failed.append(f)
  F = len(lagm)
  return (np.array(lagm, dtype=np.float64).reshape(F, L, L), np.array(coef, dtype=np.float64).reshape(F, L),
          np.array(err, dtype=np.float64), np.array(failed, dtype=np.uint8))
