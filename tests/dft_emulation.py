"""Float64 emulation of the arithmetic of include/alz_b200_dft.h: the reference's dft under CPython 3.12, one multiply
and one add per part and term in n order from +0.0, then CPython's _Py_c_quot by complex(size, 0.0)."""
import cmath

import numpy as np


def dft(blk, freqs, normalize=True):
  """The reference's ``dft(blk, freqs, normalize)``, restated term by term (``blk`` of floats)."""
  blk = [float(v) for v in blk]
  if not blk:
    if freqs and normalize:
      raise ZeroDivisionError("division by zero")
    return [0] * len(freqs)
  L = float(len(blk))
  out = []
  for f in freqs:
    re = im = 0.0
    for n, x in enumerate(blk):
      w = cmath.exp(-1j * n * f)
      re = re + x * w.real
      im = im + x * w.imag
    if normalize:
      re, im = (re + im * 0.0) / L, (im - re * 0.0) / L
    out.append(complex(re, im))
  return out


def dft_batch(b, table, normalize=True):
  """``b[R, size]`` float64 frame values, ``table[size, n_freqs]`` complex128 twiddles -> ``[R, n_freqs]`` complex128:
  the same arithmetic, vectorised over frames and frequencies (numpy rounds every product and sum on its own)."""
  b = np.asarray(b, dtype=np.float64)
  R, size = b.shape
  re = np.zeros((R, table.shape[1]))
  im = np.zeros((R, table.shape[1]))
  wr, wi = table.real, table.imag
  with np.errstate(all="ignore"):
    for n in range(size):
      re = re + b[:, n:n + 1] * wr[n]
      im = im + b[:, n:n + 1] * wi[n]
    if normalize:
      re, im = (re + im * 0.0) / size, (im - re * 0.0) / size
  out = np.empty(re.shape, dtype=np.complex128)
  out.real, out.imag = re, im
  return out


def frames(x, size, hop, window=None, final=True):
  """The float64 values of the blocks of ``Stream(x).blocks(size, hop)`` (the padded last block included when the
  reference emits it), times ``window``: ``[F, size]``."""
  x = np.asarray(x, dtype=np.float64)
  N = len(x)
  F = max(0, (N - size) // hop + 1)
  kp = F
  if final and N - kp * hop > max(size - hop, 0):
    F += 1
  out = np.zeros((F, size))
  for k in range(F):
    seg = x[k * hop:k * hop + size]
    out[k, :len(seg)] = seg
  if window is not None:
    with np.errstate(all="ignore"):
      out = out * np.asarray(window, dtype=np.float64)
  return out
