"""numpy emulation of AudioLazy's zcross over float32 samples (include/alz_b200_zcross.h restates the semantics), and
of ``sum(block)`` over ``zcross(...).blocks(size, hop)``."""
import hashlib

import numpy as np


def start_sign(first_sign):
  return 0 if first_sign == 0 else (-1 if first_sign < 0 else 1)


def zcross(x, hysteresis=0., first_sign=0.):
  """uint8 crossing flags of the rows of ``x`` (float32, compared in float64 against the float64 ``hysteresis``)."""
  x = np.asarray(x, dtype=np.float32).astype(np.float64)
  h = float(hysteresis)
  s0 = start_sign(first_sign)
  with np.errstate(invalid="ignore"):
    decisive = (x > h) | (x < -h)
    sgn = np.where(x < 0, -1, 1)
    n = x.shape[-1]
    last = np.maximum.accumulate(np.where(decisive, np.arange(n), -1), axis=-1)   # last decisive sample at or before n
    s = np.where(last >= 0, np.take_along_axis(sgn, np.maximum(last, 0), axis=-1), s0)
    prev = np.concatenate([np.full(x.shape[:-1] + (1,), s0), s[..., :-1]], axis=-1)
    return ((prev != 0) & (x * prev < -h)).astype(np.uint8)


def block_sums(flags, size, hop=None, final=True):
  """[sum(b) for b in flags.blocks(size, hop)] along the last axis: blocks [k hop, k hop + size), then (if ``final``)
  the first incomplete block k, counting [k hop, N), when N - k hop > max(size - hop, 0)."""
  hop = size if hop is None else hop
  flags = np.asarray(flags, dtype=np.int64)
  N = flags.shape[-1]
  c = np.concatenate([np.zeros(flags.shape[:-1] + (1,), np.int64), np.cumsum(flags, axis=-1)], axis=-1)
  k = np.arange(max(0, (N - size) // hop + 1))
  sums = c[..., k * hop + size] - c[..., k * hop]
  kp = len(k)
  if final and N - kp * hop > max(size - hop, 0):
    sums = np.concatenate([sums, c[..., N:] - c[..., kp * hop:kp * hop + 1]], axis=-1)
  return sums.astype(np.int32)


def digest(values, dtype):
  return hashlib.sha256(np.ascontiguousarray(values, dtype=dtype).tobytes()).hexdigest()
