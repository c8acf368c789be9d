"""CPU restatement of the batched step-down of ``include/alz_b200_parcor.h``, row by row, with the host's own ``k ** 2``:
what ``parcor_batch`` computes for one row, as ``(k list, failed, stable)``."""
import math


def parcor_row(row):
  """(emitted k values, failure code 0 / 1 / 2 / 3, stable) of one row, as the header defines them."""
  a = [float(c) for c in row]
  if not a[0] == 1.0:
    return [], 3, False
  M = max((i for i, c in enumerate(a) if c != 0), default=0)
  ks = []
  for m in range(M, 0, -1):
    k = a[m] if a[m] != 0 else 0.0
    ks.append(k)
    try:
      q = k ** 2
    except OverflowError:
      return ks, 2, False
    d = 1 - q
    if d == 0:
      return ks, 1, False
    r = 1 / d
    new = [0.0] * (m + 1)
    for j in range(1, m):
      x, y = a[j], a[m - j]
      t = x if (k == 0 or y == 0) else x - k * y
      new[j] = 0.0 if (r == 0 or t == 0) else t * r
    new[0] = 1.0
    a = new
  return ks, 0, all(abs(k) < 1 for k in ks)


def same_float(x, y):
  """Equal bits, a NaN matching any NaN."""
  if math.isnan(x) or math.isnan(y):
    return math.isnan(x) and math.isnan(y)
  return x == y and math.copysign(1, x) == math.copysign(1, y)
