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

#: every symbol include/alz_b200.h declares (tests check the library exports them all)
SYMBOLS = (
  "alz_last_error", "alz_abi_version", "alz_device_count", "alz_set_device", "alz_plan_create", "alz_plan_create_ex",
  "alz_plan_destroy", "alz_plan_taps", "alz_apply_tv_f32", "alz_plan_tiers", "alz_apply_f32_ex", "alz_host_alloc",
  "alz_host_free", "alz_stream_create_partition", "alz_stream_destroy_partition", "alz_apply_sum_f32", "alz_apply_envelope_f32", "alz_apply_envelope_f32_host",
  "alz_apply_envelope_f32_ex", "alz_apply_envelope_f32_host_ex",
  "alz_plan_info_get", "alz_plan_state_doubles", "alz_state_init", "alz_plan_history", "alz_apply_f32",
  "alz_apply_f32_host", "alz_sum_channels_f32", "alz_freq_response_f64", "alz_launch_count",
)


class NativeError(RuntimeError):
  """The native CUDA library is missing or a native call failed."""


class PlanInfo(ctypes.Structure):
  _fields_ = [(n, ctypes.c_int32) for n in
              ("abi_version", "kind", "n_channels", "n_sections", "num_taps", "monic", "state_doubles", "fp64_ops",
               "device", "n_fp32_channels", "tier_tol_e9")] + [("reserved", ctypes.c_int32 * 5)]


_lib = None


def lib():
  """Load (once) ``_native/libalz_b200.so``; raise :class:`NativeError` if absent."""
  global _lib
  if _lib is not None:
    return _lib
  path = os.environ.get("ALZ_B200_LIB", _build.LIB_PATH)
  if not os.path.exists(path):
    raise NativeError(
      "audiolazy_b200 native library not found at %s -- build it with "
      "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)" % path)
  try:
    L = ctypes.CDLL(path)
  except OSError as exc:  # pragma: no cover
    raise NativeError("cannot load %s: %s" % (path, exc))
  i32, i64, vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
  L.alz_last_error.restype = ctypes.c_char_p
  L.alz_last_error.argtypes = []
  L.alz_abi_version.restype = i32
  L.alz_device_count.restype = i32
  L.alz_set_device.restype = i32
  L.alz_set_device.argtypes = [i32]
  L.alz_plan_create.restype = i32
  L.alz_plan_create.argtypes = [vp, vp, i32, i32, ctypes.POINTER(vp)]
  L.alz_plan_create_ex.restype = i32
  L.alz_plan_create_ex.argtypes = [vp, vp, i32, i32, i32, ctypes.POINTER(vp)]
  L.alz_plan_taps.restype = i32
  L.alz_plan_taps.argtypes = [vp, vp, vp, i32]
  L.alz_plan_tiers.restype = i32
  L.alz_plan_tiers.argtypes = [vp, vp, vp, i32]
  L.alz_apply_tv_f32.restype = i32
  L.alz_apply_tv_f32.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, vp, i64, vp]
  L.alz_plan_destroy.restype = None
  L.alz_plan_destroy.argtypes = [vp]
  L.alz_plan_info_get.restype = i32
  L.alz_plan_info_get.argtypes = [vp, ctypes.POINTER(PlanInfo)]
  L.alz_plan_state_doubles.restype = i64
  L.alz_plan_state_doubles.argtypes = [vp, i64]
  L.alz_state_init.restype = i32
  L.alz_state_init.argtypes = [vp, vp, i64, vp, vp, vp]
  L.alz_plan_history.restype = i32
  L.alz_plan_history.argtypes = [vp, ctypes.POINTER(i32), ctypes.POINTER(i32)]
  L.alz_apply_f32.restype = i32
  L.alz_apply_f32.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, vp]
  L.alz_apply_f32_ex.restype = i32
  L.alz_apply_f32_ex.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, i64, vp]
  L.alz_apply_sum_f32.restype = i32
  L.alz_apply_sum_f32.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64, vp]
  f64 = ctypes.c_double
  L.alz_apply_envelope_f32.restype = i32
  L.alz_apply_envelope_f32.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i32, i32, f64, f64, vp]
  L.alz_apply_envelope_f32_host.restype = i32
  L.alz_apply_envelope_f32_host.argtypes = [vp, vp, vp, i64, i64, i64, i64, i32, i32, f64, f64]
  L.alz_apply_envelope_f32_ex.restype = i32
  L.alz_apply_envelope_f32_ex.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i32, i32, i32, f64, f64, vp]
  L.alz_apply_envelope_f32_host_ex.restype = i32
  L.alz_apply_envelope_f32_host_ex.argtypes = [vp, vp, vp, vp, vp, i64, i64, i64, i64, i32, i32, i32, f64, f64]
  L.alz_stream_create_partition.restype = i32
  L.alz_stream_create_partition.argtypes = [i32, i32, ctypes.POINTER(vp), ctypes.POINTER(i32)]
  L.alz_stream_destroy_partition.restype = i32
  L.alz_stream_destroy_partition.argtypes = [vp]
  L.alz_host_alloc.restype = i32
  L.alz_host_alloc.argtypes = [ctypes.POINTER(vp), i64, i32, ctypes.POINTER(i32)]
  L.alz_host_free.restype = i32
  L.alz_host_free.argtypes = [vp]
  L.alz_apply_f32_host.restype = i32
  L.alz_apply_f32_host.argtypes = [vp, vp, vp, vp, i64, i64, i64, i64]
  L.alz_sum_channels_f32.restype = i32
  L.alz_sum_channels_f32.argtypes = [vp, vp, i64, i32, i64, i64, i64, vp]
  L.alz_freq_response_f64.restype = i32
  L.alz_freq_response_f64.argtypes = [vp, vp, vp, i64, vp]
  L.alz_launch_count.restype = i64
  _lib = L
  return L


def _check(rc):
  if rc < 0:
    msg = lib().alz_last_error().decode("utf-8", "replace")
    if rc == ALZ_ERR_ZERO_GAIN:
      raise ZeroDivisionError("Invalid filter gain")   # same exception as lazy_filters.py:177-178
    if rc == ALZ_ERR_INVALID:
      raise ValueError(msg)
    raise NativeError("alz error %d: %s" % (rc, msg))
  return rc


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
