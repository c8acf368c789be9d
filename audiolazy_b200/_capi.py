"""ctypes binding of the C ABI declared in ``include/alz_b200.h``.

This is the only place Python meets native code.  There is no CPU fallback: if the
library cannot be loaded, or a compute entry point is called without a usable CUDA
device, a :class:`NativeError` is raised.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _build

ALZ_OK = 0
ALZ_ERR_INVALID = -1
ALZ_ERR_NONCAUSAL = -2
ALZ_ERR_ZERO_GAIN = -3
ALZ_ERR_CUDA = -4
ALZ_ERR_NOMEM = -5
ALZ_ERR_UNSUPPORTED = -6
KIND_BIQUAD = 1
KIND_GENERIC = 2
PLAN_FORCE_GENERIC = 1
PLAN_EXACT = 2
PLAN_DESIGN_ONLY = 4
PLAN_SEQUENTIAL = 8
PLAN_PARALLEL = 16


class NativeError(RuntimeError):
  """The native CUDA library is missing or a native call failed."""


class NativeLib(object):
  """The ctypes binding of one of the package's native libraries.

  ``prototypes`` maps every function the library's header declares to its ``(restype, argtypes)``; :attr:`symbols`
  is that list.  :meth:`load` opens the library once (``path``, or the file the environment variable ``env`` names)
  and binds the prototypes.  :meth:`check` turns a negative status code into the exception ``errors`` maps it to
  (called with the message of the library's ``*_last_error`` function), or into a :class:`NativeError`."""

  def __init__(self, path, name, prototypes, errors, env=None):
    self.path = path
    self.name = name
    self.prototypes = prototypes
    self.symbols = tuple(prototypes)
    self.errors = errors
    self.env = env
    self.last_error = next(s for s in prototypes if s.endswith("_last_error"))
    self.cdll = None

  def load(self, reload=False):
    """Load the library once (again with ``reload``); raise :class:`NativeError` if it is absent or cannot be loaded."""
    if self.cdll is not None and not reload:
      return self.cdll
    path = os.environ.get(self.env, self.path) if self.env else self.path
    if not os.path.exists(path):
      raise NativeError(
        "audiolazy_b200 %s library not found at %s -- build it with "
        "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)" % (self.name, path))
    try:
      L = ctypes.CDLL(path)
    except OSError as exc:
      raise NativeError("cannot load %s: %s" % (path, exc))
    for symbol, (restype, argtypes) in self.prototypes.items():
      fn = getattr(L, symbol)
      fn.restype, fn.argtypes = restype, argtypes
    self.cdll = L
    return L

  def check(self, rc):
    if rc < 0:
      msg = getattr(self.load(), self.last_error)().decode("utf-8", "replace")
      if rc in self.errors:
        raise self.errors[rc](msg)
      raise NativeError("%s error %d: %s" % (self.last_error[:-len("_last_error")], rc, msg))
    return rc


class PlanInfo(ctypes.Structure):
  _fields_ = [(n, ctypes.c_int32) for n in
              ("abi_version", "kind", "n_channels", "n_sections", "num_taps", "monic", "state_doubles", "fp64_ops",
               "device", "n_fp32_channels", "tier_tol_e9", "time_parallel")] + [("reserved", ctypes.c_int32 * 4)]


_i32, _i64, _f64, _vp, _p = ctypes.c_int32, ctypes.c_int64, ctypes.c_double, ctypes.c_void_p, ctypes.POINTER
LIB = NativeLib(_build.LIB_PATH, "native", {
  "alz_last_error": (ctypes.c_char_p, []),
  "alz_abi_version": (_i32, []),
  "alz_device_count": (_i32, []),
  "alz_set_device": (_i32, [_i32]),
  "alz_plan_create": (_i32, [_vp, _vp, _i32, _i32, _p(_vp)]),
  "alz_plan_create_ex": (_i32, [_vp, _vp, _i32, _i32, _i32, _p(_vp)]),
  "alz_plan_destroy": (None, [_vp]),
  "alz_plan_taps": (_i32, [_vp, _vp, _vp, _i32]),
  "alz_plan_tiers": (_i32, [_vp, _vp, _vp, _i32]),
  "alz_plan_info_get": (_i32, [_vp, _p(PlanInfo)]),
  "alz_plan_state_doubles": (_i64, [_vp, _i64]),
  "alz_state_init": (_i32, [_vp, _vp, _i64, _vp, _vp, _vp]),
  "alz_plan_history": (_i32, [_vp, _p(_i32), _p(_i32)]),
  "alz_apply_f32": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp]),
  "alz_apply_f32_ex": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i64, _vp]),
  "alz_apply_tv_f32": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp, _i64, _vp]),
  "alz_apply_sum_f32": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _vp]),
  "alz_apply_envelope_f32": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _f64, _f64, _vp]),
  "alz_apply_envelope_f32_host": (_i32, [_vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _f64, _f64]),
  "alz_apply_envelope_f32_ex": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _f64, _f64,
                                       _vp]),
  "alz_apply_envelope_f32_host_ex": (_i32, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _i32, _i32, _i32, _f64,
                                            _f64]),
  "alz_stream_create_partition": (_i32, [_i32, _i32, _p(_vp), _p(_i32)]),
  "alz_stream_destroy_partition": (_i32, [_vp]),
  "alz_host_alloc": (_i32, [_p(_vp), _i64, _i32, _p(_i32)]),
  "alz_host_free": (_i32, [_vp]),
  "alz_apply_f32_host": (_i32, [_vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64]),
  "alz_sum_channels_f32": (_i32, [_vp, _vp, _i64, _i32, _i64, _i64, _i64, _vp]),
  "alz_freq_response_f64": (_i32, [_vp, _vp, _vp, _i64, _vp]),
  "alz_launch_count": (_i64, []),
}, {
  ALZ_ERR_ZERO_GAIN: lambda msg: ZeroDivisionError("Invalid filter gain"),   # same exception as lazy_filters.py:177-178
  ALZ_ERR_INVALID: ValueError,
}, env="ALZ_B200_LIB")
#: every function include/alz_b200.h declares
SYMBOLS = LIB.symbols
_check = LIB.check
#: the loaded filter library; None until :func:`lib` loads it, and setting it back to None makes the next call load it
#: again (from the file ``ALZ_B200_LIB`` names then)
_lib = None


def lib():
  """Load (once) ``_native/libalz_b200.so``, or the file ``ALZ_B200_LIB`` names; raise :class:`NativeError` if it
  cannot be loaded."""
  global _lib
  if _lib is None:
    _lib = LIB.load(reload=True)
  return _lib


def pack_sections(bank):
  """``bank``: list (channels) of lists (sections) of ``(b, a)`` float lists ->
  ``(coef float64[], desc int32[], C, KM)`` in the alz_plan_create layout."""
  C = len(bank)
  KM = max([len(ch) for ch in bank] + [1])
  desc = np.zeros((C, KM, 3), dtype=np.int32)
  coef = []
  for c, ch in enumerate(bank):
    for k, (b, a) in enumerate(ch):
      b = [float(v) for v in b] or [0.0]
      a = [float(v) for v in a]
      desc[c, k] = (len(b), len(a), len(coef))
      coef.extend(b)
      coef.extend(a)
  return np.asarray(coef or [0.0], dtype=np.float64), np.ascontiguousarray(desc.reshape(-1)), C, KM


class Plan(object):
  """A compiled bank of cascades living on the current CUDA device."""

  def __init__(self, bank, force_generic=False, exact=False, design_only=False, sequential=False, parallel=False):
    L = lib()
    coef, desc, C, KM = pack_sections(bank)
    handle = ctypes.c_void_p()
    flags = (PLAN_FORCE_GENERIC if force_generic else 0) | (PLAN_EXACT if exact else 0) | \
            (PLAN_DESIGN_ONLY if design_only else 0) | (PLAN_SEQUENTIAL if sequential else 0) | (PLAN_PARALLEL if parallel else 0)
    _check(L.alz_plan_create_ex(coef.ctypes.data, desc.ctypes.data, C, KM, flags, ctypes.byref(handle)))
    self._h = handle
    info = PlanInfo()
    _check(L.alz_plan_info_get(self._h, ctypes.byref(info)))
    self.kind = info.kind
    self.n_channels = info.n_channels
    self.n_sections = info.n_sections
    self.num_taps = info.num_taps
    self.monic = bool(info.monic)
    self.monic_mode = info.monic          # 0 plain sections, 1 gain on the float64 output, 2 gain on the float32 input
    self.state_doubles_per_recurrence = info.state_doubles
    self.fp64_ops = info.fp64_ops
    self.device = info.device
    self.n_fp32_channels = info.n_fp32_channels
    self.tier_tol = info.tier_tol_e9 * 1e-9
    self.time_parallel = bool(info.time_parallel)   # few long streams may be evaluated time-parallel
    xd, yd = ctypes.c_int32(), ctypes.c_int32()
    _check(L.alz_plan_history(self._h, ctypes.byref(xd), ctypes.byref(yd)))
    self.xd, self.yd = xd.value, yd.value

  def __del__(self):
    h, self._h = getattr(self, "_h", None), None
    if h and _lib is not None:
      _lib.alz_plan_destroy(h)

  def state_doubles(self, n_streams):
    return _check(lib().alz_plan_state_doubles(self._h, int(n_streams)))

  def state_init(self, state_ptr, n_streams, xinit=None, yinit=None, stream=0):
    xi = None if xinit is None else np.ascontiguousarray(xinit, dtype=np.float64)
    yi = None if yinit is None else np.ascontiguousarray(yinit, dtype=np.float64)
    for arr, depth in ((xi, self.xd), (yi, self.yd)):
      if arr is not None and arr.size != self.n_channels * self.n_sections * depth:
        raise ValueError("initial history must have shape [%d][%d][%d]" % (self.n_channels, self.n_sections, depth))
    _check(lib().alz_state_init(self._h, state_ptr, int(n_streams),
                                None if xi is None else xi.ctypes.data,
                                None if yi is None else yi.ctypes.data, stream))

  def apply(self, x_ptr, y_ptr, state_ptr, n_streams, n_samples, x_stride, y_stride, stream=0):
    _check(lib().alz_apply_f32(self._h, x_ptr, y_ptr, state_ptr, int(n_streams), int(n_samples), int(x_stride),
                               int(y_stride), stream))

  def apply_sum(self, x_ptr, out_ptr, state_ptr, n_streams, n_samples, x_stride, out_stride, stream=0):
    """ParallelFilter in one kernel (plans created with ``parallel=True``); raises :class:`NativeError`
    (ALZ_ERR_UNSUPPORTED) for unaligned rows or non-biquad members."""
    _check(lib().alz_apply_sum_f32(self._h, x_ptr, out_ptr, state_ptr, int(n_streams), int(n_samples), int(x_stride),
                                   int(out_stride), stream))

  ENVELOPE_MODES = {"abs": 0, "squared": 1, "rms": 2}

  def apply_envelope(self, x_ptr, env_ptr, state_ptr, env_state_ptr, n_streams, n_samples, x_stride, env_stride, decim,
                     mode, g, R, stream=0):
    """Bank + fused envelope consumer on device buffers (``alz_apply_envelope_f32``)."""
    _check(lib().alz_apply_envelope_f32(self._h, x_ptr, env_ptr, state_ptr, env_state_ptr, int(n_streams), int(n_samples),
                                        int(x_stride), int(env_stride), int(decim), self.ENVELOPE_MODES[mode], float(g),
                                        float(R), stream))

  def apply_envelope_host(self, x, env=None, decim=48, mode="abs", g=None, R=None):
    """``x``: float32 ndarray [S][T] on the host -> ``env`` [S][C][T // decim]: the bank's channel envelopes
    (``mode``: abs / squared / rms; one-pole lowpass ``e = g r + R e1``), decimated on the device."""
    x = np.asarray(x, dtype=np.float32)
    if x.ndim == 1:
      x = x[None, :]
    S, T = x.shape
    if g is None or R is None:
      R = 0.99 if R is None else R
      g = 1.0 - R if g is None else g
    if env is None:
      env = np.empty((S, self.n_channels, T // decim), dtype=np.float32)
    assert env.dtype == np.float32 and env.shape == (S, self.n_channels, T // decim) and env.flags.c_contiguous
    _check(lib().alz_apply_envelope_f32_host(self._h, x.ctypes.data, env.ctypes.data, S, T, x.strides[0] // 4 if S > 1 else T,
                                             T // decim, int(decim), self.ENVELOPE_MODES[mode], float(g), float(R)))
    return env

  def apply_envelope_ex(self, x_ptr, env_ptr, state_ptr, env_state_ptr, n_streams, n_samples, x_stride, env_stride, decim,
                        phase, mode, g, R, stream=0):
    """:meth:`apply_envelope` for a block of an endless stream (``alz_apply_envelope_f32_ex``): any ``n_samples``;
    ``phase`` samples of the current decimation window were consumed before the block, which yields
    ``(phase + n_samples) // decim`` values per row."""
    _check(lib().alz_apply_envelope_f32_ex(self._h, x_ptr, env_ptr, state_ptr, env_state_ptr, int(n_streams),
                                           int(n_samples), int(x_stride), int(env_stride), int(decim), int(phase),
                                           self.ENVELOPE_MODES[mode], float(g), float(R), stream))

  def apply_envelope_host_ex(self, x, env=None, state_ptr=None, env_state_ptr=None, decim=48, phase=0, mode="abs", g=None,
                             R=None):
    """:meth:`apply_envelope_host` for a block of an endless stream (``alz_apply_envelope_f32_host_ex``): device states
    (``None``: zero, discarded) and ``phase``; returns ``env`` [S][C][(phase + T) // decim]."""
    x = np.asarray(x, dtype=np.float32)
    if x.ndim == 1:
      x = x[None, :]
    if x.strides[1] != 4:
      x = np.ascontiguousarray(x)
    S, T = x.shape
    if g is None or R is None:
      R = 0.99 if R is None else R
      g = 1.0 - R if g is None else g
    n_out = (int(phase) + T) // decim
    if env is None:
      env = np.empty((S, self.n_channels, n_out), dtype=np.float32)
    assert env.dtype == np.float32 and env.shape == (S, self.n_channels, n_out) and env.flags.c_contiguous
    _check(lib().alz_apply_envelope_f32_host_ex(self._h, x.ctypes.data, env.ctypes.data, state_ptr, env_state_ptr, S, T,
                                                x.strides[0] // 4 if S > 1 else max(T, 1), max(n_out, 1), int(decim),
                                                int(phase), self.ENVELOPE_MODES[mode], float(g), float(R)))
    return env

  def tiers(self):
    """``(tier int32[C], probe_err float64[C])``: precision tier of every channel (0 float64, 1 float32) and the
    float32 error the plan-time probe measured for it (< 0: not probed)."""
    tier = np.zeros(self.n_channels, dtype=np.int32)
    err = np.zeros(self.n_channels, dtype=np.float64)
    _check(lib().alz_plan_tiers(self._h, tier.ctypes.data, err.ctypes.data, self.n_channels))
    return tier, err

  def apply_ex(self, x_ptr, y_ptr, state_ptr, n_streams, n_samples, x_stride, y_stride, y_stream_stride, stream=0):
    """:meth:`apply` with an explicit distance between the output rows of consecutive streams (channel slices
    written into a wider ``y[S][C_total][T]``, possibly on a peer GPU)."""
    _check(lib().alz_apply_f32_ex(self._h, x_ptr, y_ptr, state_ptr, int(n_streams), int(n_samples), int(x_stride),
                                  int(y_stride), int(y_stream_stride), stream))

  def taps(self):
    """``[(delay, is_den), ...]`` in coefficient-table order (generic plans only)."""
    n = _check(lib().alz_plan_taps(self._h, None, None, 0))
    delay = np.zeros(n, dtype=np.int32)
    is_den = np.zeros(n, dtype=np.int32)
    _check(lib().alz_plan_taps(self._h, delay.ctypes.data, is_den.ctypes.data, n))
    return list(zip(delay.tolist(), [bool(v) for v in is_den.tolist()]))

  def freq_response(self, w_ptr, out_ptr, n, stream=0):
    """Bank response on a grid: ``out[C][n][2]`` float64 (re, im) for ``w[n]`` rad/sample (device pointers)."""
    _check(lib().alz_freq_response_f64(self._h, w_ptr, out_ptr, int(n), stream))

  def apply_tv(self, x_ptr, y_ptr, state_ptr, n_streams, n_samples, x_stride, y_stride, coef_ptr, coef_stride, stream=0):
    _check(lib().alz_apply_tv_f32(self._h, x_ptr, y_ptr, state_ptr, int(n_streams), int(n_samples), int(x_stride),
                                  int(y_stride), coef_ptr, int(coef_stride), stream))

  def apply_host(self, x, y=None, state_ptr=None):
    """``x``: float32 ndarray [S][T] (C-contiguous rows). Returns ``y`` [S][C][T]."""
    x = np.asarray(x, dtype=np.float32)
    if x.ndim == 1:
      x = x[None, :]
    if x.strides[1] != 4:
      x = np.ascontiguousarray(x)
    S, T = x.shape
    if y is None:
      y = np.empty((S, self.n_channels, T), dtype=np.float32)
    assert y.dtype == np.float32 and y.shape == (S, self.n_channels, T) and y.flags.c_contiguous
    x_stride = x.strides[0] // 4 if S > 1 else max(T, 1)   # a length-1 axis may carry any stride
    _check(lib().alz_apply_f32_host(self._h, x.ctypes.data, y.ctypes.data, state_ptr, S, T, x_stride, T))
    return y


class PartitionStream(object):
  """A CUDA stream confined to ``sm_count`` SMs of ``device`` (green context, ``alz_stream_create_partition``).
  ``.handle`` is the ``cudaStream_t``; ``.sm_count`` what was granted. Wrap it with ``torch.cuda.ExternalStream``."""

  def __init__(self, sm_count, device=-1):
    h, granted = ctypes.c_void_p(), ctypes.c_int32(0)
    _check(lib().alz_stream_create_partition(int(device), int(sm_count), ctypes.byref(h), ctypes.byref(granted)))
    self.handle = h.value
    self.sm_count = granted.value

  def close(self):
    h, self.handle = self.handle, None
    if h:
      _check(lib().alz_stream_destroy_partition(h))


class HostBuffer(object):
  """Pinned float32 host array on the NUMA node of a CUDA device (``alz_host_alloc``): ``.array`` is a numpy view.
  Call :meth:`free` when done (the memory is not garbage collected while views may exist)."""

  def __init__(self, shape, device=-1):
    shape = tuple(int(v) for v in (shape if isinstance(shape, (tuple, list)) else (shape,)))
    n = int(np.prod(shape)) if shape else 1
    ptr, node = ctypes.c_void_p(), ctypes.c_int32(-1)
    _check(lib().alz_host_alloc(ctypes.byref(ptr), max(4, n * 4), int(device), ctypes.byref(node)))
    self._ptr = ptr
    self.numa_node = node.value
    self.array = np.ctypeslib.as_array(ctypes.cast(ptr, ctypes.POINTER(ctypes.c_float)), shape=(max(n, 1),))[:n].reshape(shape)

  def free(self):
    ptr, self._ptr = self._ptr, None
    if ptr:
      self.array = None
      _check(lib().alz_host_free(ptr))


def sum_channels(y_ptr, out_ptr, n_streams, n_channels, n_samples, y_stride, out_stride, stream=0):
  _check(lib().alz_sum_channels_f32(y_ptr, out_ptr, int(n_streams), int(n_channels), int(n_samples), int(y_stride),
                                    int(out_stride), stream))


def device_count():
  return lib().alz_device_count()


def set_device(index):
  _check(lib().alz_set_device(int(index)))


def launch_count():
  return lib().alz_launch_count()
