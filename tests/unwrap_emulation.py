"""The arithmetic of include/alz_b200_unwrap.h restated twice: in plain Python, operation by operation, and vectorised
with numpy (the float64 terms of every jump at once, then their sequential sum with ``np.add.accumulate``).  Both use
the header's convention for a jump with step 0: its term is NaN and its index is the failure the state records."""
import math

import numpy as np


def py_rem(v, w):
  """CPython 3.12's float_rem for w != 0 (C's fmod: NaN for an infinite v or a NaN operand, v for an infinite w)."""
  if math.isinf(v) or math.isnan(v) or math.isnan(w):
    mod = math.nan
  else:
    mod = v if math.isinf(w) else math.fmod(v, w)
  if mod != 0.0:                                   # NaN counts as nonzero
    if (w < 0) != (mod < 0):
      mod = mod + w
  else:
    mod = math.copysign(0.0, w)
  return mod


def unwrap(d, max_delta, step):
  """-> (out, fail): the header's recurrence over the float64 samples ``d``; ``fail`` is the index of the first jump
  taken with step 0, or -1."""
  M, P = float(max_delta), float(step)
  out, fail = [], -1
  delta, prev = 0.0, None
  for n, x in enumerate(float(v) for v in d):
    if n == 0:
      delta = x - x
      out.append(x)
    else:
      diff = x - prev
      if abs(diff) > M:
        if P == 0.0:
          fail = n if fail < 0 else fail
          term = math.nan
        else:
          a, b = py_rem(diff, P), py_rem(diff, -P)
          term = (-diff) + (b if abs(b) < abs(a) else a)
        delta = delta + term
      out.append(x + delta)
    prev = x
  return out, fail


def _rem(v, w):
  with np.errstate(invalid="ignore"):
    mod = np.fmod(v, w)
    adjust = (mod != 0) & ((w < 0) != (mod < 0))
    mod = np.where(adjust, mod + w, mod)
  return np.where(mod == 0, np.copysign(0.0, w), mod)


def unwrap_batch(x, max_delta, step):
  """Vectorised: ``x[S, T]`` (any float dtype, widened to float64) -> ``(out[S, T] float64, fail[S] int64)`` for
  streams that start with the call."""
  d = np.asarray(x, dtype=np.float64)
  if d.ndim == 1:
    d = d[None]
  S, T = d.shape
  M, P = float(max_delta), float(step)
  if T == 0:
    return d.copy(), np.full(S, -1, dtype=np.int64)
  with np.errstate(invalid="ignore", over="ignore"):
    diff = d[:, 1:] - d[:, :-1]
    jump = np.abs(diff) > M
    if P == 0.0:
      term = np.full_like(diff, np.nan)
    else:
      a, b = _rem(diff, P), _rem(diff, -P)
      term = -diff + np.where(np.abs(b) < np.abs(a), b, a)
    # delta is never -0.0 (it starts at +0.0 and a rounded sum is -0.0 only when both terms are), so adding +0.0 at the
    # samples without a jump leaves it unchanged, and accumulate adds in sample order
    e = np.concatenate([d[:, :1] - d[:, :1], np.where(jump, term, 0.0)], axis=1)
    delta = np.add.accumulate(e, axis=1)
    out = d + delta
  out[:, 0] = d[:, 0]
  first = jump.argmax(axis=1) + 1 if T > 1 else np.zeros(S, dtype=np.int64)
  fail = np.where(jump.any(axis=1) & (P == 0.0), first, -1).astype(np.int64)
  return out, fail


def clip(x, low, high):
  """The reference's clip in float64; ``None`` is no limit."""
  d = np.asarray(x, dtype=np.float64)
  with np.errstate(invalid="ignore"):
    if low is None and high is None:
      return d.copy()
    if low is None:
      return np.where(d < high, d, float(high))
    if high is None:
      return np.where(d > low, d, float(low))
    return np.where(d > high, float(high), np.where(d < low, float(low), d))
