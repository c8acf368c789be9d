"""Float64 emulation of the reference's amdf(lag, size)(x, zero=zero), operation for operation (test infrastructure).

For taps (delay k_j, coefficient c_j) of (1 - z ** -lag).linearize():
  d[n]    = c_0 x[n - k_0] + c_1 x[n - k_1] + ...  (each product rounded, summed left to right; no taps: zero)
  new[n]  = abs(d[n]) * (1. / size)
  mean[n] = (mean[n - 1] - old[n]) + new[n],  old[n] = new[n - size], or zero * (1. / size) for n < size
with x[j] = zero for j < 0 and mean[-1] = zero.  numpy float64 elementwise arithmetic rounds every operation, so this
reproduces the reference's Python-float sequence bit for bit."""
import hashlib

import numpy as np


def digest(y):
  """SHA-256 of a float64 array's little-endian bytes."""
  return hashlib.sha256(np.ascontiguousarray(y, dtype="<f8").tobytes()).hexdigest()


def differences(x, taps, zero=0.):
  """``d[..., n]`` for ``x[..., T]`` (float64)."""
  x = np.asarray(x, dtype=np.float64)
  T = x.shape[-1]
  if not taps:
    return np.full(x.shape, float(zero))
  K = max(k for k, _ in taps)
  xp = np.concatenate([np.full(x.shape[:-1] + (K,), float(zero)), x], axis=-1)
  d = None
  for k, c in taps:
    t = float(c) * xp[..., K - k:K - k + T]
    d = t if d is None else d + t
  return d


def amdf(x, taps, size, zero=0.):
  """The AMDF of ``x[..., T]`` at one lag (``taps``) -> float64 ``[..., T]``."""
  inv = 1. / size
  new = np.abs(differences(x, taps, zero)) * inv
  zinv = float(zero) * inv
  out = np.empty_like(new)
  mean = np.full(new.shape[:-1], float(zero))
  for n in range(new.shape[-1]):
    old = new[..., n - size] if n >= size else zinv
    mean = (mean - old) + new[..., n]
    out[..., n] = mean
  return out


def amdf_bank(x, taps_list, size, zero=0.):
  """``x[S, T]`` -> float64 ``[S, L, T]``: one :func:`amdf` per lag, the recursion vectorised over (stream, lag)."""
  x = np.asarray(x, dtype=np.float64)
  inv = 1. / size
  new = np.stack([np.abs(differences(x, taps, zero)) * inv for taps in taps_list], axis=1)
  zinv = float(zero) * inv
  out = np.empty_like(new)
  mean = np.full(new.shape[:-1], float(zero))
  for n in range(new.shape[-1]):
    old = new[..., n - size] if n >= size else zinv
    mean = (mean - old) + new[..., n]
    out[..., n] = mean
  return out
