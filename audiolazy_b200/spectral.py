"""Short-time Fourier analysis and resynthesis: ``window`` / ``wsymm``, ``overlap_add`` and ``stft`` with the
reference's names and signatures (``audiolazy/lazy_analysis.py``), and their batched forms :class:`Stft` and
:class:`OverlapAdd`, evaluated by the sm_90a kernels behind ``include/alz_b200_stft.h``.

The windows are host lists, the reference's values bit for bit.  Framing, windowing, the float64 FFTs and the
overlap-add run on the GPU: the overlap-add is the reference's float64 arithmetic exactly (its float32 output is the
float32 of the reference's values), the FFTs are float64 transforms accurate to a few ulps of each frame's peak.
"""
from __future__ import annotations

import ctypes
import itertools as it
from collections.abc import Iterable
from math import ceil, cos, pi, sin
from numbers import Integral

import numpy as np

from . import _build, _capi, _engine
from .core import StrategyDict
from .stream import Stream

# ---------------------------------------------------------------------------------------------------------------------
# Windows (host, float64 lists)
# ---------------------------------------------------------------------------------------------------------------------

window = StrategyDict("window")
wsymm = StrategyDict("wsymm")
for _sd in (window, wsymm):                 # attributes, not strategies (StrategyDict.__setattr__ would register them)
  object.__setattr__(_sd, "symm", wsymm)
  object.__setattr__(_sd, "periodic", window)


def _hann(n, size):
  return .5 * (1 - cos(2 * pi * n / size))


def _hamming(n, size):
  return .54 - .46 * cos(2 * pi * n / size)


def _bartlett(n, size):
  return 1 - 2.0 / size * abs(n - size / 2.0)


def _triangular(n, size):
  return 1 - 2.0 / (size + 2) * abs(n - size / 2.0)


def _blackman(n, size, alpha):
  return (1 - alpha) / 2 + alpha / 2 * cos(4 * pi * n / size) - .5 * cos(2 * pi * n / size)


def _cos(n, size, alpha):
  return sin(pi * n / size) ** alpha


#: (names, value of sample n for a window length `size`, default parameters): the periodic window of length L uses
#: size = L, the symmetric one size = L - 1 (and is [1.0] for L == 1)
_WINDOWS = [
  (("hann", "hanning"), _hann, {}),
  (("hamming",), _hamming, {}),
  (("rect", "dirichlet", "rectangular"), None, {}),
  (("bartlett",), _bartlett, {}),
  (("triangular", "triangle"), _triangular, {}),
  (("blackman",), _blackman, {"alpha": .16}),
  (("cos",), _cos, {"alpha": 1}),
]


def _make_window(value, defaults, symm):
  if "alpha" in defaults:
    def wnd(size, alpha=defaults["alpha"]):
      if symm and size == 1:
        return [1.0]
      m = size - 1 if symm else size
      return [value(n, m, alpha) for n in range(size)]
  else:
    def wnd(size):
      if symm and size == 1:
        return [1.0]
      m = size - 1 if symm else size
      return [value(n, m) for n in range(size)]
  return wnd


def _rect(size):
  return [1.0 for n in range(size)]


def _register_windows():
  for names, value, defaults in _WINDOWS:
    if value is None:                        # the rectangular window: one strategy shared by both dicts, which wsymm
      window.strategy(*names)(_rect)         # knows by its first name only (as the reference's does)
      wsymm.strategy(names[0])(_rect)
      _rect.periodic = _rect.symm = _rect
      continue
    periodic = _make_window(value, defaults, False)
    symmetric = _make_window(value, defaults, True)
    window.strategy(*names)(periodic)
    wsymm.strategy(*names)(symmetric)
    for f in (periodic, symmetric):
      f.periodic, f.symm = periodic, symmetric


_register_windows()


# ---------------------------------------------------------------------------------------------------------------------
# Overlap-add gains (host)
# ---------------------------------------------------------------------------------------------------------------------

def _hop_blocks(values, hop):
  """The ``hop``-long blocks of ``values``, the last one padded with 0.0 (``Stream(values).blocks(hop)``)."""
  return [list(values[i:i + hop]) + [0.0] * max(0, i + hop - len(values)) for i in range(0, len(values), hop)]


def _window_values(wnd, size):
  """``wnd`` (None, a callable ``wnd(size)`` or an iterable of reals) as a list of floats, or None."""
  if wnd is None:
    return None
  if callable(wnd) and not isinstance(wnd, Stream):
    wnd = wnd(size)
  if not isinstance(wnd, Iterable):
    raise TypeError("Window should be an iterable or a callable")
  values = list(wnd)
  if len(values) != size:
    raise ValueError("Incompatible window size")
  return values


def ola_window(size, hop, wnd=None, normalize=True, strategy="numpy"):
  """The float64 window w' the overlap-add multiplies each frame by, normalized as the reference's ``overlap_add``
  strategy does: ``numpy`` divides by ``np.sum(np.abs(np.vstack(hop blocks)), 0).max()``, ``list`` by the ``max`` of
  the builtin ``sum`` of each column of ``|w|`` blocks (``[1 / ceil(size / hop)] * size`` without a window); a zero gain
  leaves the window as it is.  ``None`` (``list`` with no window and no normalization) means no multiply at all."""
  values = _window_values(wnd, size)
  if strategy == "numpy":
    w = np.ones(size) if values is None else np.array(values, dtype=np.float64)
    if normalize and size:
      gain = np.sum(np.abs(np.vstack([np.array(b) for b in _hop_blocks(list(w), hop)])), 0).max()
      if gain:
        w = w / gain
    return w
  if strategy != "list":
    raise ValueError("unknown overlap-add strategy %r" % (strategy,))
  if normalize:
    if values:
      gain = max(map(sum, zip(*_hop_blocks([abs(v) for v in values], hop))))
      if gain:
        values = [v / gain for v in values]
    else:
      values = [1 / ceil(size / hop)] * size
  return None if not values else np.array(values, dtype=np.float64)


# ---------------------------------------------------------------------------------------------------------------------
# The native library (include/alz_b200_stft.h)
# ---------------------------------------------------------------------------------------------------------------------

MAX_SIZE = 8192

_i32, _i64, _vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
LIB = _capi.NativeLib(_build.LIBRARIES["stft"].path, "STFT", {
  "alz_stft_last_error": (ctypes.c_char_p, []),
  "alz_stft_frames": (_i64, [_i64, _i64, _i32, _i32, _i32]),
  "alz_stft_analysis_state_bytes": (_i64, [_i64, _i32]),
  "alz_stft_analysis_state_init": (_i32, [_vp, _i64, _i32, _vp]),
  "alz_stft_ola_state_bytes": (_i64, [_i64, _i32, _i32]),
  "alz_stft_ola_state_init": (_i32, [_vp, _i64, _i32, _i32, _vp]),
  "alz_stft_analysis": (_i32, [_vp, _i64, _vp, _vp, _vp, _i32, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _i32, _vp]),
  "alz_stft_synthesis": (_i32, [_vp, _i32, _i64, _i64, _vp, _i32, _vp, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32,
                                _i32, _vp]),
  "alz_stft_ola_f64": (_i32, [_vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _vp]),
  "alz_stft_ola_f32": (_i32, [_vp, _i64, _i64, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _i32, _i32, _vp]),
}, {_capi.ALZ_ERR_INVALID: ValueError})
#: every function include/alz_b200_stft.h declares
SYMBOLS = LIB.symbols
lib = LIB.load
_check = LIB.check


def _size_hop(size, hop):
  if not isinstance(size, Integral) or isinstance(size, bool):
    raise TypeError("size must be an integer, not %s" % type(size).__name__)
  if not 1 <= size <= MAX_SIZE:
    raise ValueError("size must be in 1 .. %d (got %d)" % (MAX_SIZE, size))
  hop = size if hop is None else hop
  if not isinstance(hop, Integral) or isinstance(hop, bool):
    raise TypeError("hop must be an integer, not %s" % type(hop).__name__)
  if hop > size:
    raise ValueError("Hop value can't be higher than size")
  if hop < 1:
    raise ValueError("hop must be >= 1 (got %d)" % hop)
  return int(size), int(hop)


class _Plan(object):
  """Device tensors of one transform size: the twiddle table and windows, built once per device."""

  def __init__(self, size):
    self.size = size
    self._dev = {}

  def tensors(self, device, *host):
    got = self._dev.get(device)
    if got is None:
      torch = _engine.torch_mod()
      m = np.arange(self.size)
      ang = 2 * np.pi * m / self.size
      tw = np.empty((self.size, 2))
      tw[:, 0], tw[:, 1] = np.cos(ang), -np.sin(ang)
      got = self._dev[device] = [torch.from_numpy(tw).to(device)] + [
        None if h is None else torch.from_numpy(np.ascontiguousarray(h, dtype=np.float64)).to(device) for h in host]
    return got


class OlaState(object):
  """Device state of an :class:`OverlapAdd` (or :class:`Stft` synthesis) over ``n_streams`` streams: the frames
  consumed and the ``size - hop`` sums still open.  A call with ``final=True`` ends it."""

  def __init__(self, owner, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.key = owner._key()
    self.frames = 0
    self.ended = False
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_stft_ola_state_bytes(self.n_streams, owner.size, owner.hop))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_stft_ola_state_init(self.tensor.data_ptr(), self.n_streams, owner.size, owner.hop,
                                           torch.cuda.current_stream(device).cuda_stream))

  @property
  def device(self):
    return self.tensor.device


class StftState(object):
  """Device state of :class:`Stft` calls over ``n_streams`` streams: for the analysis the samples consumed and the
  last ``size`` samples; for the synthesis an :class:`OlaState` (``.ola``).  ``analyze(..., final=True)`` ends the
  analysis, ``synthesize(..., final=True)`` the synthesis."""

  def __init__(self, owner, n_streams):
    torch = _engine.torch_mod()
    self.n_streams = int(n_streams)
    if self.n_streams < 0:
      raise ValueError("n_streams must be >= 0")
    self.key = owner._key()
    self.consumed = 0
    self.ended = False
    device = torch.device("cuda", torch.cuda.current_device())
    with torch.cuda.device(device):
      nbytes = _check(lib().alz_stft_analysis_state_bytes(self.n_streams, owner.size))
      self.tensor = torch.empty(max(8, nbytes), dtype=torch.uint8, device=device)
      _check(lib().alz_stft_analysis_state_init(self.tensor.data_ptr(), self.n_streams, owner.size,
                                                torch.cuda.current_stream(device).cuda_stream))
    self.ola = OlaState(owner, n_streams)

  @property
  def device(self):
    return self.tensor.device


def _check_state(state, cls, owner, S, device, key, part=None):
  """``part``: the attribute of the state whose ``ended`` counts (the synthesis' ``ola``), or None for the state."""
  _engine.check_state(state, cls, type(owner).__name__, S, device)
  if state.key != key:
    raise ValueError("state belongs to a %s with another size, hop, window or option" % type(owner).__name__)
  if (getattr(state, part) if part else state).ended:
    raise ValueError("state was ended by a call with final=True")


def _out_samples(F, size, hop, final):
  return F * hop + (size - hop if final else 0)


class OverlapAdd(object):
  """The reference's ``overlap_add`` (strategy ``"numpy"`` or ``"list"``) of many streams of frames.

  * ``ola.apply(frames, state=None, final=False)`` for a CUDA float32 or float64 ``frames[S, F, size]`` (any strides
    between frames and streams) -> float32 ``[S, F * hop]``, plus the ``size - hop`` pending samples when ``final``:
    the float32 of the reference's float64 values, bit for bit.
  * ``ola.new_state(S)`` -> :class:`OlaState`, to continue streams block by block."""

  def __init__(self, size, hop=None, wnd=None, normalize=True, strategy="numpy"):
    self.size, self.hop = _size_hop(size, hop)
    self.strategy = strategy
    self.normalize = bool(normalize)
    self.window = ola_window(self.size, self.hop, wnd, normalize, strategy)
    self._plan = _Plan(self.size)

  def _key(self):
    return (self.size, self.hop, None if self.window is None else self.window.tobytes())

  def new_state(self, n_streams):
    return OlaState(self, n_streams)

  def apply(self, frames, state=None, final=False):
    torch = _engine.torch_mod()
    if not (torch.is_tensor(frames) and frames.is_cuda and frames.dim() == 3 and
            frames.dtype in (torch.float32, torch.float64)):
      raise ValueError("frames must be a CUDA float32 or float64 tensor [streams, frames, size]")
    S, F, n = frames.shape
    if n != self.size:
      raise ValueError("Wrong block size or declared")
    if frames.stride(2) != 1:
      frames = frames.contiguous()
    with torch.cuda.device(frames.device):
      if state is None:
        state = self.new_state(S)
      _check_state(state, OlaState, self, S, frames.device, self._key())
      dev = frames.device
      _, w = self._plan.tensors(dev, self.window)
      y = torch.empty((S, _out_samples(F, self.size, self.hop, final)), dtype=torch.float32, device=dev)
      fn = lib().alz_stft_ola_f64 if frames.dtype == torch.float64 else lib().alz_stft_ola_f32
      _check(fn(frames.data_ptr(), frames.stride(1), frames.stride(0), None if w is None else w.data_ptr(),
                y.data_ptr(), y.shape[1], state.tensor.data_ptr(), S, F, self.size, self.hop, int(bool(final)),
                torch.cuda.current_stream(dev).cuda_stream))
    state.frames += F
    state.ended = bool(final)
    return y


class Stft(object):
  """Short-time Fourier analysis and resynthesis of many streams: the reference's ``stft`` with its default
  ``numpy.fft.rfft`` / ``irfft`` transforms.

  Frame ``k`` is the block ``[k hop, k hop + size)`` of ``Stream(x).blocks(size, hop)`` (``hop`` defaults to ``size``,
  at most ``size``), times ``wnd`` when given (``None``, a callable ``wnd(size)`` or ``size`` reals), rotated by
  ``ifftshift`` when ``before``; its spectrum is ``rfft`` of that, ``size // 2 + 1`` bins of ``dtype`` (complex64 or
  complex128).  The synthesis takes ``irfft(X, size)``, rotates it back with ``fftshift`` when ``after``, and
  overlap-adds with the ``ola`` strategy (``"numpy"``, ``"list"``, or ``None`` for the float64 frames), window
  ``ola_wnd`` and ``ola_normalize``.

  * ``st.analyze(x, state=None, final=False)`` -> spectra ``[S, F, size // 2 + 1]`` of a CUDA float32 ``x[S, T]``;
  * ``st.synthesize(spec, state=None, final=False)`` -> float32 ``[S, F * hop]`` (plus ``size - hop`` samples when
    ``final``), or float64 frames ``[S, F, size]`` when ``ola`` is None;
  * ``st.apply(x, func, state=None, final=False)``: analysis, ``func(spec)`` once on the whole batch (it must act on
    the last axis), synthesis;
  * ``st.new_state(S)`` -> :class:`StftState`; ``st.n_frames(consumed, T, final)``."""

  def __init__(self, size, hop=None, wnd=None, before=True, after=True, ola_wnd=None, ola_normalize=True, ola="numpy",
               dtype=None):
    torch = _engine.torch_mod()
    self.size, self.hop = _size_hop(size, hop)
    values = _window_values(wnd, self.size)
    self.window = None if values is None else np.array(values, dtype=np.float64)
    self.before, self.after = bool(before), bool(after)
    if ola not in ("numpy", "list", None):
      raise ValueError("ola must be 'numpy', 'list' or None")
    self.ola = ola
    self.ola_window = None if ola is None else ola_window(self.size, self.hop, ola_wnd, ola_normalize, ola)
    dtype = torch.complex64 if dtype is None else dtype
    if dtype not in (torch.complex64, torch.complex128):
      raise ValueError("dtype must be torch.complex64 or torch.complex128")
    self.dtype = dtype
    self.bins = self.size // 2 + 1
    self._plan = _Plan(self.size)

  def _key(self):
    return (self.size, self.hop, None if self.window is None else self.window.tobytes(), self.before, self.after,
            self.ola, None if self.ola_window is None else self.ola_window.tobytes())

  def new_state(self, n_streams):
    return StftState(self, n_streams)

  def n_frames(self, consumed, T, final):
    """Frames an analysis call on ``T`` samples emits after ``consumed`` samples."""
    return _engine.n_blocks(consumed, T, self.size, self.hop, final)

  def analyze(self, x, state=None, final=False):
    torch = _engine.torch_mod()
    x, S, T, xs = _engine.stream_input(x)
    with torch.cuda.device(x.device):
      if state is None:
        state = self.new_state(S)
      _check_state(state, StftState, self, S, x.device, self._key())
      F = self.n_frames(state.consumed, T, final)
      dev = x.device
      tw, w = self._plan.tensors(dev, self.window, self.ola_window)[:2]
      spec = torch.empty((S, F, self.bins), dtype=self.dtype, device=dev)
      _check(lib().alz_stft_analysis(x.data_ptr(), xs, None if w is None else w.data_ptr(), tw.data_ptr(),
                                     spec.data_ptr(), int(self.dtype == torch.complex128), F, state.tensor.data_ptr(),
                                     S, T, self.size, self.hop, int(self.before), int(bool(final)),
                                     torch.cuda.current_stream(dev).cuda_stream))
    state.consumed += T
    state.ended = bool(final)
    return spec

  def _spectra(self, spec):
    """``spec`` as a complex CUDA tensor [S, F, size // 2 + 1] with unit stride along the bins (irfft's length rule:
    truncated or zero-padded)."""
    torch = _engine.torch_mod()
    if not (torch.is_tensor(spec) and spec.is_cuda and spec.dim() == 3):
      raise ValueError("spec must be a CUDA tensor [streams, frames, bins]")
    if not spec.is_complex():
      spec = spec.to(torch.complex128 if spec.dtype == torch.float64 else torch.complex64)
    if spec.dtype not in (torch.complex64, torch.complex128):
      raise ValueError("spec must be complex64 or complex128")
    n = spec.shape[2]
    if n > self.bins:
      spec = spec[:, :, :self.bins]
    elif n < self.bins:
      spec = torch.nn.functional.pad(torch.view_as_real(spec), (0, 0, 0, self.bins - n))
      spec = torch.view_as_complex(spec.contiguous())
    if spec.stride(2) != 1:
      spec = spec.contiguous()
    return spec

  def synthesize(self, spec, state=None, final=False):
    torch = _engine.torch_mod()
    spec = self._spectra(spec)
    S, F, _ = spec.shape
    with torch.cuda.device(spec.device):
      if state is None:
        state = self.new_state(S)
      _check_state(state, StftState, self, S, spec.device, self._key(), "ola")
      dev = spec.device
      tw, _, ow = self._plan.tensors(dev, self.window, self.ola_window)
      frames = torch.empty((S, F, self.size), dtype=torch.float64, device=dev)
      y = None
      if self.ola is not None:
        y = torch.empty((S, _out_samples(F, self.size, self.hop, final)), dtype=torch.float32, device=dev)
      _check(lib().alz_stft_synthesis(spec.data_ptr(), int(spec.dtype == torch.complex128), spec.stride(1),
                                      spec.stride(0), tw.data_ptr(), int(self.after), frames.data_ptr(),
                                      None if ow is None else ow.data_ptr(), None if y is None else y.data_ptr(),
                                      0 if y is None else y.shape[1], state.ola.tensor.data_ptr(), S, F, self.size,
                                      self.hop, int(bool(final)), torch.cuda.current_stream(dev).cuda_stream))
    if y is not None:
      state.ola.frames += F
      state.ola.ended = bool(final)
      return y
    return frames

  def apply(self, x, func, state=None, final=False):
    """Analysis, ``func`` on the spectra of the whole batch, synthesis."""
    x, S, _, _ = _engine.stream_input(x)
    if state is None:
      state = self.new_state(S)
    spec = self.analyze(x, state, final)
    return self.synthesize(func(spec), state, final)


# ---------------------------------------------------------------------------------------------------------------------
# The reference's lazy API
# ---------------------------------------------------------------------------------------------------------------------

_OLA_CHUNK = 1024          # frames an overlap_add call hands the kernel at once


def _frame_chunks(blk_sig, size):
  chunk = []
  for blk in blk_sig:
    values = np.asarray(list(blk) if not isinstance(blk, np.ndarray) else blk, dtype=np.float64)
    if values.shape != (size,):
      raise ValueError("Wrong block size or declared")
    chunk.append(values)
    if len(chunk) == _OLA_CHUNK:
      yield np.stack(chunk)
      chunk = []
  if chunk:
    yield np.stack(chunk)


def _f32_values(y):
  return y[0].cpu().numpy().astype(np.float64).tolist()


def _make_overlap_add(strategy):
  def ola(blk_sig, size=None, hop=None, wnd=None, normalize=True):
    if size is None:
      blk_sig = Stream(blk_sig)
      size = len(blk_sig.peek())
    op = OverlapAdd(size, hop, wnd, normalize, strategy)
    torch = _engine.torch_mod()
    state = op.new_state(1)
    device = state.device

    def gen():
      for chunk in _frame_chunks(blk_sig, op.size):
        yield _f32_values(op.apply(torch.from_numpy(chunk).to(device).unsqueeze(0), state))
      yield _f32_values(op.apply(torch.empty((1, 0, op.size), dtype=torch.float64, device=device), state, final=True))

    return Stream(it.chain.from_iterable(gen()))
  ola.__doc__ = ("Overlap-add of an iterable of blocks (the reference's ``overlap_add.%s``): the float32 of the "
                 "reference's float64 samples, from the sm_90a overlap-add kernel." % strategy)
  return ola


overlap_add = StrategyDict("overlap_add")
overlap_add.strategy("numpy")(_make_overlap_add("numpy"))
overlap_add.strategy("list")(_make_overlap_add("list"))


class _NotSpecified(object):
  pass


def _shift_flag(name, value, shifts):
  """True for the default (numpy's or torch's ifftshift / fftshift), False for None."""
  if value is _NotSpecified:
    return True
  if value is None:
    return False
  torch = _engine.torch_mod()
  if value in shifts(torch):
    return True
  raise NotImplementedError("'%s' other than the default shift or None is not supported on the GPU" % name)


def _ola_strategy(ola):
  if ola is None:
    return None
  if ola is overlap_add or ola is overlap_add.numpy:
    return "numpy"
  if ola is overlap_add.list:
    return "list"
  raise NotImplementedError("'ola' must be overlap_add, one of its strategies, or None")


def _bins_of(result, bins, device):
  torch = _engine.torch_mod()
  r = result if torch.is_tensor(result) else torch.as_tensor(np.asarray(result))
  r = r.to(device).reshape(-1).to(torch.complex128)
  if r.numel() >= bins:
    return r[:bins]
  return torch.cat([r, torch.zeros(bins - r.numel(), dtype=torch.complex128, device=device)])


def _stft_rfft(func=None, **kwparams):
  """Short-time Fourier block processor (the reference's ``stft``, strategy ``rfft``): ``stft(func, size=..., hop=...,
  wnd=..., before=..., after=..., ola=..., ola_wnd=..., ola_normalize=...)(sig)`` -> Stream.  ``func`` is called once
  per frame on a 1-D complex128 CUDA tensor of ``size // 2 + 1`` bins (Python operators and torch functions work on it,
  numpy-only functions do not); its result, real or complex, is truncated or zero-padded to that length.  Called
  without ``func`` it returns the same function with other defaults (partial evaluation, decorator).

  The samples of ``sig`` are taken as float32, as every entry point of this package takes them; the reference windows
  and transforms the float64 values themselves.  For float32-representable input (audio decoded from 8 to 24 bits
  included) the two agree to 1e-7 of the output's peak; other float64 input adds its own float32 rounding on top."""
  if func is None:
    return lambda f=None, **new_kws: _stft_rfft(f, **dict(kwparams, **new_kws))

  def wrapper(sig, **kwargs):
    kws = dict(kwparams, **kwargs)
    if "size" not in kws:
      raise TypeError("Missing 'size' argument")
    if "hop" in kws and kws["hop"] is not None and kws["hop"] > kws["size"]:
      raise ValueError("Hop value can't be higher than size")
    size, hop = kws.pop("size"), kws.pop("hop", None)
    wnd = kws.pop("wnd", None)
    ola = _ola_strategy(kws.pop("ola", overlap_add))
    for name, default in (("transform", np.fft.rfft), ("inverse_transform", np.fft.irfft)):
      if name in kws and kws.pop(name) is not default:
        raise NotImplementedError("'%s' other than numpy's rfft / irfft is not supported on the GPU" % name)
    before = _shift_flag("before", kws.pop("before", _NotSpecified),
                         lambda torch: (np.fft.ifftshift, torch.fft.ifftshift))
    after = _shift_flag("after", kws.pop("after", _NotSpecified), lambda torch: (np.fft.fftshift, torch.fft.fftshift))
    ola_params = {}
    for k, v in kws.items():
      if k.startswith("ola_"):
        if ola is None:
          raise TypeError("Extra '{}' argument with no overlap-add strategy".format(k))
        if k not in ("ola_wnd", "ola_normalize"):
          raise TypeError("overlap_add got an unexpected keyword argument '%s'" % k[len("ola_"):])
        ola_params[k] = v
      else:
        raise TypeError("Unknown '{}' extra argument".format(k))
    torch = _engine.torch_mod()
    st = Stft(size, hop, wnd, before, after, ola_params.get("ola_wnd"), ola_params.get("ola_normalize", True), ola,
              dtype=torch.complex128)
    state = st.new_state(1)
    device = state.device

    def process(spec, final):
      if spec.shape[1]:
        spec = torch.stack([_bins_of(func(spec[0, f]), st.bins, device) for f in range(spec.shape[1])]).unsqueeze(0)
      out = st.synthesize(spec, state, final)
      if ola is None:
        return list(out[0].cpu().numpy())
      return _f32_values(out)

    def gen():
      for xb in _engine._blocks(sig):
        yield process(st.analyze(torch.from_numpy(xb).to(device).unsqueeze(0), state), False)
      empty = torch.empty((1, 0), dtype=torch.float32, device=device)
      yield process(st.analyze(empty, state, final=True), True)

    return Stream(it.chain.from_iterable(gen()))

  try:
    wrapper.__name__ = func.__name__
  except (AttributeError, TypeError):
    pass
  return wrapper


def _stft_unsupported(name):
  def strategy(func=None, **kwparams):
    raise NotImplementedError("stft.%s (complex transforms) is not supported on the GPU: 'transform' and "
                              "'inverse_transform' other than numpy's rfft / irfft" % name)
  return strategy


stft = StrategyDict("stft")
stft.strategy("rfft", "base", "real")(_stft_rfft)
stft.strategy("cfft", "complex")(_stft_unsupported("cfft"))
stft.strategy("cfftr", "complex_real")(_stft_unsupported("cfftr"))
