"""A numpy restatement of the reference's stft / overlap_add arithmetic, the yardstick of the STFT kernels: the frame
rule of ``Stream.blocks``, the window products, numpy's rfft / irfft and shifts, and the overlap-add sums in the
reference's order (each frame's sum starting from the older frames' open sums, the first ``size - hop`` samples of
the stream from +0.0)."""
import numpy as np


def frames(x, size, hop):
  """The float64 blocks of ``Stream(x).blocks(size, hop)`` (the padded last block included)."""
  x = np.asarray(x, dtype=np.float64)
  out, k = [], 0
  while True:
    blk = x[k * hop:k * hop + size]
    # Stream.blocks emits a block when it is full, and at the end one padded block if samples are left over
    if len(blk) == size:
      out.append(blk)
    else:
      if len(x) - k * hop > max(size - hop, 0):
        out.append(np.concatenate([blk, np.zeros(size - len(blk))]))
      break
    k += 1
  return np.array(out).reshape(-1, size)


def analysis(x, size, hop, wnd=None, before=True):
  b = frames(x, size, hop)
  if wnd is not None:
    b = b * np.asarray(wnd, dtype=np.float64)
  if before:
    b = np.fft.ifftshift(b, axes=-1)
  return np.fft.rfft(b, size, axis=-1) if len(b) else np.zeros((0, size // 2 + 1), complex)


def synthesis_frames(spec, size, after=True):
  v = np.fft.irfft(spec, size, axis=-1) if len(spec) else np.zeros((0, size))
  return np.fft.fftshift(v, axes=-1) if after else v


def ola(v, size, hop, w=None):
  """float64 overlap-add of the frames v[F, size] times w (None: no multiply), all pending samples included."""
  v = np.asarray(v, dtype=np.float64).reshape(-1, size)
  old = np.zeros(size)
  out = []
  for blk in v:
    blk = blk * w if w is not None else blk.copy()
    blk[:size - hop] += old[hop:]
    out.append(blk[:hop])
    old = blk
  out.append(old[hop:])
  return np.concatenate(out)


def stft(x, size, hop, func, wnd=None, before=True, after=True, ola_w=None, overlap=True):
  """The reference's stft(func, size, hop, ...) of the samples x with numpy's transforms: the float64 samples, or the
  frames [F, size] when not ``overlap``.  ``func`` acts on the spectra [F, size // 2 + 1], one frame a row; ``ola_w`` is
  the normalized overlap-add window (None: no multiply)."""
  spec = analysis(x, size, hop, wnd, before)
  v = synthesis_frames(func(spec) if len(spec) else spec, size, after)
  return ola(v, size, hop, ola_w) if overlap else v
