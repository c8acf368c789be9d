"""Python float64 emulation of AudioLazy's ``resample(x, old, new, order, zero)`` as include/alz_b200_resample.h
restates it: a schedule walked from one pending position, Lagrange weights that depend on that position only, and
CPython 3.12's compensated ``sum()`` (:func:`lpc_emulation.psum`) of the rounded products, block by block."""
from functools import reduce
import operator

import numpy as np

from lpc_emulation import psum


def start_index(order):
  threshold = .5 * (order + 1)
  return float(int(threshold) + int(threshold + .5))


def schedule(order, step, idx, n_samples):
  """(pos, idx_out, idx_next) of a block of n_samples samples starting from the pending position idx."""
  threshold = .5 * (order + 1)
  pos, idxs, consumed = [], [], 0
  while True:
    while idx > threshold:
      if consumed == n_samples:
        return pos, idxs, idx
      consumed += 1
      idx -= 1
    pos.append(consumed)
    idxs.append(idx)
    idx += step


def weights(idx, order):
  L = order + 1
  return [reduce(operator.mul, [(idx - r) / (j - r) for r in range(L) if r != j]) for j in range(L)]


def resample_batch(x, old, new, order=3, zero=0.):
  """:func:`resample` of every row of the float32 array ``x[S, T]`` in one block, vectorised over streams and
  outputs: the same float64 operations in the same order, elementwise."""
  x = np.asarray(x, dtype=np.float32).astype(np.float64)
  S, T = x.shape
  L = order + 1
  pos, idxs, _ = schedule(order, old / new, start_index(order), T)
  pos, k = np.array(pos, dtype=np.int64), np.array(idxs, dtype=np.float64)
  data = np.concatenate([np.full((S, L), float(zero)), x], axis=1)
  f, c = np.zeros((S, len(pos))), np.zeros((S, len(pos)))
  with np.errstate(invalid="ignore", over="ignore"):
    for j in range(L):
      w = None
      for r in range(L):
        if r != j:
          q = (k - r) / (j - r)
          w = q if w is None else w * q
      term = data[:, pos + j] * w
      t = f + term
      big = np.abs(f) >= np.abs(term)
      c = c + np.where(big, (f - t) + term, (term - t) + f)
      f = t
    return np.where((c != 0) & np.isfinite(c), f + c, f)


def resample(x, old, new, order=3, zero=0., blocks=None):
  """float64 outputs of one stream of float32 samples ``x``, cut into ``blocks`` (lengths; default one block)."""
  x = [float(v) for v in np.asarray(x, dtype=np.float32)]
  L, step = order + 1, old / new
  hist = [float(zero)] * L
  idx, out, at = start_index(order), [], 0
  for n in (blocks if blocks is not None else [len(x)]):
    block = x[at:at + n]
    at += n
    pos, idxs, idx = schedule(order, step, idx, n)
    data = hist + block
    for p, k in zip(pos, idxs):
      ys = data[p:p + L]
      out.append(psum(y * w for y, w in zip(ys, weights(k, order))))
    hist = data[len(data) - L:]
  return out
