"""Device engine: compiled plans, device buffers and the lazy block pump.

Everything numeric happens in the native library (``_capi``); PyTorch is used only as
the container of device memory, CUDA streams and (in :mod:`audiolazy_b200.parallel`)
``torch.distributed``. No filtering arithmetic is done in Python or numpy here.
"""
from __future__ import annotations

import itertools as it
import threading
from array import array
from collections import deque

import numpy as np

from . import _capi
from .stream import Stream

#: block sizes of the lazy pump: start small (low latency for ``take(few)``), grow
#: geometrically, cap at MAX_BLOCK samples per launch.
FIRST_BLOCK = 256
MAX_BLOCK = 1 << 20

_lock = threading.Lock()
_cache = {}


def torch_mod():
  import torch
  if not torch.cuda.is_available():
    raise _capi.NativeError("audiolazy_b200 needs a CUDA device (there is no CPU evaluator)")
  return torch


def stream_input(x):
  """The input of a batched call: a CUDA float32 tensor ``x[streams, samples]`` (1-D: one stream) ->
  ``(x, S, T, row_stride)``, its rows made contiguous."""
  torch = torch_mod()
  if x.dim() == 1:
    x = x.unsqueeze(0)
  if x.dtype != torch.float32 or x.dim() != 2 or x.device.type != "cuda":
    raise ValueError("x must be a CUDA float32 tensor [streams, samples]")
  if x.stride(1) != 1:
    x = x.contiguous()
  S, T = x.shape
  return x, S, T, x.stride(0) if S > 1 else max(T, 1)     # a length-1 axis may carry any stride


def stream_input64(x):
  """As :func:`stream_input`, for calls that also take float64 samples: a CUDA float32 or float64 tensor
  ``x[streams, samples]`` (1-D: one stream) -> ``(x, S, T, row_stride)``, its rows made contiguous."""
  torch = torch_mod()
  if x.dim() == 1:
    x = x.unsqueeze(0)
  if x.dtype not in (torch.float32, torch.float64) or x.dim() != 2 or x.device.type != "cuda":
    raise ValueError("x must be a CUDA float32 or float64 tensor [streams, samples]")
  if x.stride(1) != 1:
    x = x.contiguous()
  S, T = x.shape
  return x, S, T, x.stride(0) if S > 1 else max(T, 1)


def check_state(state, cls, owner, S, device):
  """The checks every streaming state takes before its own: ``state`` is a ``cls`` (from ``<owner>.new_state``) made
  for ``S`` streams on ``device``."""
  if not isinstance(state, cls):
    raise ValueError("state must come from %s.new_state" % owner)
  if state.n_streams != S:
    raise ValueError("state was created for %d streams, x has %d" % (state.n_streams, S))
  if state.device != device:
    raise ValueError("state lives on %s, x on %s" % (state.device, device))


def n_blocks(consumed, T, size, hop, final):
  """Blocks of ``Stream(x).blocks(size, hop)`` a call on ``T`` samples emits after ``consumed`` samples: the blocks it
  completes, plus, with ``final``, the padded last block when the reference emits one (``alz_lpc_frames``)."""
  ka = max(0, (consumed - size) // hop + 1)
  kc = (consumed + T - size) // hop
  n = max(0, kc - ka + 1)
  if final and consumed + T - max(kc + 1, 0) * hop > max(size - hop, 0):
    n += 1
  return n


def _key(bank_sections):
  return tuple(tuple((tuple(b), tuple(a)) for b, a in channel) for channel in bank_sections)


class DeviceBank(object):
  """A plan (bank of cascades) bound to the current CUDA device plus the torch-side
  helpers to allocate state / output and launch on torch's current stream."""

  def __init__(self, bank_sections, parallel=False):
    torch = torch_mod()
    self.device = torch.device("cuda", torch.cuda.current_device())
    _capi.set_device(self.device.index)
    self.plan = _capi.Plan(bank_sections, parallel=parallel)
    self.parallel = parallel
    self.n_channels = self.plan.n_channels
    self._sections = bank_sections

  # ---- state -------------------------------------------------------------------------
  def _pad_init(self, init, depth):
    if init is None:
      return None
    C, K = self.plan.n_channels, self.plan.n_sections
    arr = np.zeros((C, K, max(depth, 1)), dtype=np.float64)
    for c, channel in enumerate(init):
      for k, hist in enumerate(channel):
        if len(hist) > depth:
          raise ValueError("initial history longer than the section's delay line")
        arr[c, k, :len(hist)] = hist
    return arr[:, :, :depth] if depth else None

  def new_state(self, n_streams, xinit=None, yinit=None):
    """Device state (torch float64) for ``n_streams`` streams; ``xinit`` / ``yinit`` are
    per channel, per section lists of initial delays (``zero`` / ``memory``)."""
    torch = torch_mod()
    n = max(1, self.plan.state_doubles(n_streams))
    state = torch.empty(n, dtype=torch.float64, device=self.device)
    xi = self._pad_init(xinit, self.plan.xd)
    yi = self._pad_init(yinit, self.plan.yd)
    if xi is not None and not xi.any():
      xi = None
    if yi is not None and not yi.any():
      yi = None
    self.plan.state_init(state.data_ptr(), n_streams, xi, yi, torch.cuda.current_stream(self.device).cuda_stream)
    return state

  # ---- launches ----------------------------------------------------------------------
  def apply(self, x, state, out=None, channel_major=False):
    """``x``: CUDA float32 tensor ``[S, T]`` (rows may be strided); returns ``[S, C, T]``, or ``[C, S, T]`` with
    ``channel_major=True`` (``alz_apply_f32_ex``: the 32 rows a warp stores are then 64 KB apart instead of C x 64 KB,
    which the HBM write path likes better: +7 % on the store-bound bank)."""
    torch = torch_mod()
    if x.dim() == 1:
      x = x.unsqueeze(0)
    if x.dtype != torch.float32 or x.device != self.device or x.dim() != 2:
      raise ValueError("x must be a float32 tensor [streams, samples] on the bank's CUDA device (%s)" % self.device)
    if x.stride(1) != 1:
      x = x.contiguous()
    S, T = x.shape
    shape = (self.n_channels, S, T) if channel_major else (S, self.n_channels, T)
    if out is None:
      out = torch.empty(shape, dtype=torch.float32, device=x.device)
    elif out.shape != shape or out.dtype != torch.float32 or not out.is_contiguous():
      raise ValueError("out must be a contiguous float32 tensor %s" % ("[C, S, T]" if channel_major else "[S, C, T]"))
    xs = x.stride(0) if S > 1 else max(T, 1)
    cur = torch.cuda.current_stream(x.device).cuda_stream
    if channel_major and S > 0 and T > 0:
      self.plan.apply_ex(x.data_ptr(), out.data_ptr(), state.data_ptr(), S, T, xs, S * T, T, cur)
    else:
      self.plan.apply(x.data_ptr(), out.data_ptr(), state.data_ptr(), S, T, xs, T, cur)
    return out

  def freq_response(self, freqs):
    """Complex response of every channel on ``freqs`` (rad/sample; array-like or CUDA float64
    tensor): CUDA complex128 tensor ``[C, n]`` (reference ``lazy_filters.py:267-301`` per filter)."""
    torch = torch_mod()
    w = torch.as_tensor(freqs, dtype=torch.float64).to(self.device).contiguous().reshape(-1)
    out = torch.empty((self.n_channels, w.numel(), 2), dtype=torch.float64, device=self.device)
    self.plan.freq_response(w.data_ptr(), out.data_ptr(), w.numel(), torch.cuda.current_stream(self.device).cuda_stream)
    return torch.view_as_complex(out)

  def apply_sum(self, x, state):
    """ParallelFilter: ``x[S, T]`` -> ``out[S, T]`` = the left-associated sum of every channel's output. One kernel
    (float64 accumulation, channel outputs never reach memory) when the plan allows it, else bank launch + channel sum."""
    torch = torch_mod()
    if x.dim() == 1:
      x = x.unsqueeze(0)
    S, T = x.shape
    if self.parallel and self.plan.kind == _capi.KIND_BIQUAD and self.plan.num_taps <= 3:
      # rows padded to 16 bytes: the fused kernel moves its tiles with TMA
      Tp = (T + 3) & ~3
      xp = x if (T == Tp and x.is_contiguous() and x.data_ptr() % 16 == 0) else None
      if xp is None:
        xp = torch.zeros((S, Tp), dtype=torch.float32, device=x.device)
        xp[:, :T] = x
      out = torch.empty((S, Tp), dtype=torch.float32, device=x.device)
      try:
        self.plan.apply_sum(xp.data_ptr(), out.data_ptr(), state.data_ptr(), S, T, Tp, Tp,
                            torch.cuda.current_stream(x.device).cuda_stream)
        return out[:, :T]
      except _capi.NativeError:
        pass                              # more channels than one parameter block, ...: the two-kernel path below
    return self.sum_channels(self.apply(x, state))

  def sum_channels(self, y):
    torch = torch_mod()
    S, C, T = y.shape
    out = torch.empty((S, T), dtype=torch.float32, device=y.device)
    _capi.sum_channels(y.data_ptr(), out.data_ptr(), S, C, T, T, T, torch.cuda.current_stream(y.device).cuda_stream)
    return out


def device_bank(bank_sections, parallel=False):
  """Cached :class:`DeviceBank` for a bank given as channels -> sections -> (b, a). ``parallel``: the bank is the
  member list of a ParallelFilter (plain float64 sections, summed inside one kernel)."""
  torch = torch_mod()
  key = (torch.cuda.current_device(), bool(parallel), _key(bank_sections))
  with _lock:
    db = _cache.get(key)
    if db is None:
      if len(_cache) > 256:
        _cache.clear()
      db = _cache[key] = DeviceBank(bank_sections, parallel=parallel)
  return db


def _to_f32(chunk):
  """list / tuple of Python numbers -> float32 ndarray. ``array('d', ...)`` walks the objects in C about twice as
  fast as ``np.asarray`` does; anything it refuses (complex, nested, None) goes the numpy way and raises there."""
  try:
    return np.frombuffer(array("d", chunk), dtype=np.float64).astype(np.float32)
  except (TypeError, OverflowError):
    return np.asarray(chunk, dtype=np.float32)


def _blocks(seq):
  """Yield float32 numpy blocks of the input iterable (whole thing at once when it is a
  sized container, geometrically growing read-ahead otherwise)."""
  if isinstance(seq, np.ndarray) and seq.ndim == 1:
    for i in range(0, len(seq), MAX_BLOCK):
      yield np.ascontiguousarray(seq[i:i + MAX_BLOCK], dtype=np.float32)
    return
  if isinstance(seq, (list, tuple)):
    for i in range(0, len(seq), MAX_BLOCK):
      yield _to_f32(seq if len(seq) <= MAX_BLOCK else seq[i:i + MAX_BLOCK])
    return
  src = iter(seq)
  n = FIRST_BLOCK
  while True:
    chunk = list(it.islice(src, n))
    if not chunk:
      return
    yield _to_f32(chunk)
    if len(chunk) < n:
      return
    n = min(n * 4, MAX_BLOCK)


class _Blocks(object):
  """Marker: an iterable of ready float32 blocks (see :func:`_pre_blocks`)."""

  def __init__(self, gen):
    self.gen = gen


def _pre_blocks(seq, pre):
  def gen():
    for xb in _blocks64(seq):
      yield pre(xb).astype(np.float32)
  return _Blocks(gen())


def _blocks64(seq):
  """As :func:`_blocks` but float64 blocks (the pre-op runs on the values the reference's Stream arithmetic sees)."""
  if isinstance(seq, np.ndarray) and seq.ndim == 1:
    for i in range(0, len(seq), MAX_BLOCK):
      yield np.asarray(seq[i:i + MAX_BLOCK], dtype=np.float64)
    return
  src = iter(seq)
  n = FIRST_BLOCK if not isinstance(seq, (list, tuple)) else MAX_BLOCK
  while True:
    chunk = list(it.islice(src, n))
    if not chunk:
      return
    try:
      yield np.frombuffer(array("d", chunk), dtype=np.float64)
    except (TypeError, OverflowError):
      yield np.asarray(chunk, dtype=np.float64)
    if len(chunk) < n:
      return
    n = min(n * 4, MAX_BLOCK)


def _pump(db, seq, xinit, yinit, sum_channels):
  """Generator of per-block results: numpy float32 ``[C, n]`` (or ``[n]`` when summed)."""
  torch = torch_mod()
  state = None
  for xb in (seq.gen if isinstance(seq, _Blocks) else _blocks(seq)):
    if state is None:
      state = db.new_state(1, xinit, yinit)
    x_dev = torch.from_numpy(xb).to(db.device, non_blocking=False)
    if sum_channels:
      yield db.apply_sum(x_dev, state)[0].cpu().numpy()
    else:
      yield db.apply(x_dev, state)[0].cpu().numpy()


def filter_stream(bank_sections, seq, xinit, yinit, sum_channels=False, pre=None, post=None):
  """Lazy Stream of a single-output filter call (one channel, or the channel sum). ``pre`` / ``post``: numpy
  ufunc-like callables applied to each input block (float64, before the float32 conversion) / output block
  (float64) -- the x**2, abs, sqrt around the lowpass of ``envelope.*`` without a Python frame per sample."""
  db = device_bank(bank_sections, parallel=sum_channels)   # errors (zero gain, no device) raise at call time, like the reference
  if pre is not None:
    seq = _pre_blocks(seq, pre)

  def rows():
    for block in _pump(db, seq, xinit, yinit, sum_channels):
      row = block if sum_channels else block[0]
      yield (row if post is None else post(row.astype(np.float64))).tolist()

  # chain.from_iterable walks the per-block lists in C: no Python frame per sample
  return Stream(it.chain.from_iterable(rows()))


def bank_streams(bank_sections, seq, xinit, yinit):
  """One lazy Stream per channel, fed by a shared pump (like a tee: a channel consumed
  far ahead of the others buffers their samples)."""
  db = device_bank(bank_sections)
  return tee_streams(_pump(db, seq, xinit, yinit, False), db.n_channels)


def tee_streams(pump, C):
  """``pump``: generator of per-block ``[C, n]`` arrays -> ``C`` lazy Streams, one per row, that share it (a row
  consumed far ahead of the others buffers their blocks)."""
  queues = [deque() for _ in range(C)]

  def channel(c):      # generator of per-block lists of channel c
    while True:
      while not queues[c]:
        try:
          block = next(pump)
        except StopIteration:
          return
        for q, row in zip(queues, block):
          q.append(row.tolist())
      yield queues[c].popleft()

  return [Stream(it.chain.from_iterable(channel(c))) for c in range(C)]


# --------------------------------------------------------------------------------------
# time-varying coefficients (reference lazy_filters.py:169-176, 200-216, 262-263)
# --------------------------------------------------------------------------------------
def filter_stream_tv(num_terms, den_terms, seq, memory_init, zero):
  """Lazy Stream of a single filter whose coefficients may be Streams.

  ``num_terms`` / ``den_terms``: ``[(delay, coeff)]`` sorted by delay (``den_terms`` includes
  delay 0); ``coeff`` is a number or an iterator advanced once per input sample. A Stream a0
  becomes a variable gain exactly as the reference rewrites it: ``inv = 1 / a0`` and every
  other coefficient is multiplied by ``inv``. The per-sample coefficient values of a block
  are evaluated on the host (they are the USER's streams) and uploaded with the block.
  When a coefficient Stream ends before the input, the Stream yields the samples before that
  point and then raises ``RuntimeError``, as the reference does."""
  torch = torch_mod()
  device = torch.device("cuda", torch.cuda.current_device())
  _capi.set_device(device.index)
  a0 = dict(den_terms)[0]
  num = [(d, c) for d, c in num_terms]
  den = [(d, c) for d, c in den_terms if d != 0]
  sections = [([1.0 if any(d == k for d, _ in num) else 0.0 for k in range(max([d for d, _ in num] + [0]) + 1)] or [1.0],
               [1.0] + [1.0 if any(d == k for d, _ in den) else 0.0 for k in range(1, max([d for d, _ in den] + [0]) + 1)])]
  if not num:
    sections[0] = ([0.0], sections[0][1])
  plan = _capi.Plan([sections], force_generic=True)
  taps = plan.taps()
  sources = []
  for delay, is_den in taps:
    table = dict(den) if is_den else dict(num)
    sources.append((is_den, table.get(delay, 0.0)))
  state = torch.empty(max(1, plan.state_doubles(1)), dtype=torch.float64, device=device)
  xi = np.zeros((1, 1, max(plan.xd, 1)))[:, :, :plan.xd]
  yi = np.zeros((1, 1, max(plan.yd, 1)))[:, :, :plan.yd]
  xi[...] = float(zero)
  yi[0, 0, :len(memory_init)] = memory_init[:plan.yd]
  cur = lambda: torch.cuda.current_stream(device).cuda_stream
  plan.state_init(state.data_ptr(), 1, xi if plan.xd else None, yi if plan.yd else None, cur())

  def pull(src, n):
    if hasattr(src, "__next__"):
      return list(it.islice(src, n))
    return None    # constant

  def gen():
    for xb in _blocks(seq):
      n = len(xb)
      cols = [pull(src, n) for _, src in sources]
      a0_vals = pull(a0, n)
      lens = [len(c) for c in cols if c is not None] + ([len(a0_vals)] if a0_vals is not None else [])
      m = min([n] + lens)           # samples before the shortest coefficient stream ends
      if m == 0:
        raise _coefficients_ended()
      inv = None if a0_vals is None else 1.0 / np.asarray(a0_vals[:m], dtype=np.float64)
      coef = np.empty((len(sources), m), dtype=np.float64)
      for row, (col, (is_den, src)) in enumerate(zip(cols, sources)):
        vals = np.full(m, float(src)) if col is None else np.asarray(col[:m], dtype=np.float64)
        vals = vals * inv if inv is not None else vals / float(a0)
        coef[row] = -vals if is_den else vals
      x_dev = torch.from_numpy(np.ascontiguousarray(xb[:m])).to(device)
      c_dev = torch.from_numpy(coef).to(device)
      y_dev = torch.empty(m, dtype=torch.float32, device=device)
      plan.apply_tv(x_dev.data_ptr(), y_dev.data_ptr(), state.data_ptr(), 1, m, m, m, c_dev.data_ptr(), m, cur())
      yield y_dev.cpu().numpy().tolist()
      if m < n:
        raise _coefficients_ended()

  return Stream(it.chain.from_iterable(gen()))


def _coefficients_ended():
  """What the reference raises at the first input sample after a coefficient Stream ends: its generated filter loop
  calls ``next()`` on the Stream, and Python turns a StopIteration leaving a generator into RuntimeError (PEP 479)."""
  return RuntimeError("generator raised StopIteration")
