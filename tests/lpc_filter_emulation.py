"""Float64 restatement of the LPC filter kernels (include/alz_b200_lpcfilt.h) in their order of operations: per sample
``y = x[n]``, then ``y = y + c_k * x[n - k]`` (analysis) or ``y = y + (-c_k) * y[n - k]`` (synthesis) for k = 1 ..
order, each product and each sum rounded once.  numpy's float64 multiply and add are single IEEE operations, so this
is the reference's arithmetic, vectorized over streams (and, for the analysis, over samples)."""
import numpy as np


def row_index(consumed, T, hop):
  """The call's row of each of its samples."""
  n = consumed + np.arange(T)
  return n // hop - consumed // hop


def lpc_filter(kind, x, coef, hop, consumed=0, hist=None):
  """``kind`` "analysis" or "synthesis" of ``x[S, T]`` (float64) with ``coef[S, F, order + 1]`` (float64) after
  ``consumed`` samples whose last ``order`` inputs or outputs are ``hist[S, order]`` (zeros when None).  Returns
  ``(y[S, T], hist)``."""
  x = np.asarray(x, np.float64)
  coef = np.asarray(coef, np.float64)
  S, T = x.shape
  order = coef.shape[2] - 1
  hist = np.zeros((S, order)) if hist is None else np.asarray(hist, np.float64)
  rows = row_index(consumed, T, hop)
  with np.errstate(all="ignore"):
    if kind == "analysis":
      full = np.concatenate([hist, x], axis=1)                   # sample n at column n + order
      y = x.copy()
      for k in range(1, order + 1):
        c = coef[:, rows, k] if T else np.zeros((S, 0))
        y = y + c * full[:, order - k:order - k + T]
      return y, full[:, full.shape[1] - order:]
    y = np.concatenate([hist, np.zeros((S, T))], axis=1)
    for n in range(T):
      acc = x[:, n].copy()
      c = coef[:, rows[n]]
      for k in range(1, order + 1):
        acc = acc + (-c[:, k]) * y[:, order + n - k]
      y[:, order + n] = acc
    return y[:, order:], y[:, y.shape[1] - order:]


def same_bits(got, want):
  """Equal float64 values bit for bit, every NaN equal to every NaN."""
  got = np.asarray(got, np.float64)
  want = np.asarray(want, np.float64)
  nan = np.isnan(want)
  return got.shape == want.shape and np.array_equal(np.isnan(got), nan) and \
      np.array_equal(got[~nan].view(np.uint64), want[~nan].view(np.uint64))
