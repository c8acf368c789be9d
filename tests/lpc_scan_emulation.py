"""Float64 restatement of the time-parallel LPC synthesis (include/alz_b200_lpcscan.h): the chunk summaries, the scan
of the chunk start states and the rerun, with the kernels' walks in their order of operations (the walks of
tests/lpc_filter_emulation.py) and the fallback of streams whose summaries or scanned states are not finite.  The
scan is a plain float64 matrix product here, as it has no bit contract on the device either."""
import numpy as np

from lpc_filter_emulation import lpc_filter, row_index


def chunk_bounds(T, P):
  """First sample of each of the P chunks of T samples, then T."""
  q, r = divmod(T, P)
  return np.array([p * q + min(p, r) for p in range(P + 1)], dtype=np.int64)


def max_chunks(T, order):
  return max(1, T // max(order, 1))


def _walk(x, coef, rows, lo, h, use_input, store=None):
  """Walks chunk p of every stream over samples [lo[p], lo[p + 1]) from h[S, P, R, order] (newest first), the runs R
  with ``use_input`` reading x and the others zero input; stores outputs into ``store[S, T]`` when given.  Returns the
  final states."""
  S, P, R, order = h.shape
  lens = lo[1:] - lo[:-1]
  for i in range(int(lens.max()) if P else 0):
    active = i < lens                                          # [P]
    n = np.minimum(lo[:-1] + i, max(x.shape[1] - 1, 0))
    acc = np.where(use_input[None, None, :], x[:, n][:, :, None], 0.0)
    c = coef[:, rows[n]]                                       # [S, P, order + 1]
    for k in range(1, order + 1):
      acc = acc + (-c[:, :, None, k]) * h[..., k - 1]
    if order:
      h = np.where(active[None, :, None, None], np.concatenate([acc[..., None], h[..., :-1]], axis=3), h)
    if store is not None:
      store[:, n[active]] = acc[:, active, 0]
  return h


def lpc_scan(x, coef, hop, P, consumed=0, hist=None):
  """The synthesis of ``x[S, T]`` (float64) with ``coef[S, F, order + 1]`` in P chunks per stream after ``consumed``
  samples whose last ``order`` outputs are ``hist[S, order]`` (oldest first; zeros when None).  Returns ``(y[S, T],
  hist, flagged[S])``: flagged streams are the sequential walk's, bit for bit."""
  x = np.asarray(x, np.float64)
  coef = np.asarray(coef, np.float64)
  S, T = x.shape
  order = coef.shape[2] - 1
  hist = np.zeros((S, order)) if hist is None else np.asarray(hist, np.float64)
  assert 1 <= P <= max_chunks(T, order)
  rows = row_index(consumed, T, hop)
  lo = chunk_bounds(T, P)
  R = order + 1
  with np.errstate(all="ignore"):
    h0 = np.zeros((S, P, R, order))
    for u in range(1, R):
      h0[:, :, u, u - 1] = 1.0
    use = np.arange(R) == 0
    h = _walk(x, coef, rows, lo, h0, use)
    F = h[:, :, 0, :]                                          # [S, P, order]
    M = np.swapaxes(h[:, :, 1:, :], 2, 3)                      # [S, P, i, j]: column j is the response to e_j
    states = np.zeros((S, P + 1, order))
    states[:, 0] = hist[:, ::-1]
    for p in range(P):
      states[:, p + 1] = F[:, p] + np.einsum("sij,sj->si", M[:, p], states[:, p])
    flagged = ~(np.isfinite(F).all(axis=(1, 2)) & np.isfinite(M).all(axis=(1, 2, 3)) &
                np.isfinite(states).all(axis=(1, 2)))
    y = np.zeros((S, T))
    h = _walk(x, coef, rows, lo, states[:, :P, None, :].copy(), np.array([True]), store=y)
    out_hist = h[:, P - 1, 0, ::-1].copy()
  for s in np.nonzero(flagged)[0]:
    ys, hs = lpc_filter("synthesis", x[s:s + 1], coef[s:s + 1], hop, consumed, hist[s:s + 1])
    y[s], out_hist[s] = ys[0], hs[0]
  return y, out_hist, flagged


def within_bar(got, want, bar=1e-9):
  """Per stream, max |got - want| <= bar * max |want| (equal values where want is not finite)."""
  got = np.asarray(got, np.float64)
  want = np.asarray(want, np.float64)
  if got.shape != want.shape:
    return False
  for g, w in zip(got.reshape(len(got), -1), want.reshape(len(want), -1)):
    if not np.array_equal(np.isnan(g), np.isnan(w)) or not np.array_equal(g[np.isinf(w)], w[np.isinf(w)]):
      return False
    fin = np.isfinite(w)
    if not fin.any():
      continue
    with np.errstate(all="ignore"):
      if not np.max(np.abs(g[fin] - w[fin])) <= bar * np.max(np.abs(w[fin])):
        return False
  return True


def kautocor_rows(x, order, size, hop):
  """The autocorrelation-method rows of every frame [k hop, k hop + size) of x (1-D), through Levinson-Durbin in
  float64: stable rows, as LpcFrames(order, size, hop) gives them up to rounding."""
  x = np.asarray(x, np.float64)
  out = []
  for k0 in range(0, len(x) - size + 1, hop):
    b = x[k0:k0 + size]
    r = np.array([b[:size - m] @ b[m:] for m in range(order + 1)])
    r[0] *= 1 + 1e-9                                             # a white-noise floor keeps the tone rows regular
    a = np.array([1.0])
    err = r[0]
    for m in range(1, order + 1):
      k = -(a @ r[m:0:-1]) / err
      a = np.concatenate([a, [0.0]])
      a = a + k * a[::-1]
      err *= 1 - k * k
    out.append(a)
  return np.array(out)
