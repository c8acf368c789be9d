"""CPU oracle for the AudioLazy filter hot path -- TEST INFRASTRUCTURE ONLY.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package; nothing under ``audiolazy_b200/``
does (``tests/test_no_oracle_in_product.py`` enforces it).

Two restatements of the reference's evaluator (``LinearFilter.__call__``, reference
``audiolazy/lazy_filters.py:141-264``; ``CascadeFilter.__call__``, ``:988-990``):

* :func:`bank_apply` -- plain C (``alz_oracle.c``), float64, same term order and
  separately rounded operations as the generated Python source; fast enough for the
  parity tests (a 64-channel bank over 20 000 samples in ~50 ms).
* :func:`py_section` / :func:`py_cascade` -- pure-Python loops mirroring the generated
  generator body statement by statement; used on small cases to pin the C file.

Both are pinned against golden vectors produced by the reference itself
(``tests/golden/make_golden.py``) in ``tests/test_oracle.py``.

:func:`tv_apply` states the time-varying contract of ``alz_apply_tv_f32`` (per-sample coefficient tables) in numpy;
``tests/test_time_varying.py`` pins it to the reference's outputs (``tests/golden/make_tv.py``).
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


def build(force: bool = False) -> str:
  """Compile ``alz_oracle.c`` with gcc (idempotent). Returns the library path."""
  so = os.path.join(_HERE, "libalz_oracle.so")
  src = os.path.join(_HERE, "alz_oracle.c")
  if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
    subprocess.check_call(["make", "-C", _HERE, "-s", "-B"])
  return so


def _lib():
  global _LIB
  if _LIB is None:
    lib = ctypes.CDLL(build())
    i32, i64, vp = ctypes.c_int32, ctypes.c_int64, ctypes.c_void_p
    lib.orc_bank_apply.restype = ctypes.c_int
    lib.orc_bank_apply.argtypes = [vp, vp, vp, vp, i32, i32, i64, i64, i64, i64, vp, i32, vp, i32, i64, i64]
    lib.orc_bank_apply_f32.restype = ctypes.c_int
    lib.orc_bank_apply_f32.argtypes = [vp, vp, vp, vp, i32, i32, i64, i64, i64, i64, i64, i64]
    _LIB = lib
  return _LIB


def pack_bank(bank):
  """``bank``: list (channels) of lists (sections) of ``(b, a)`` coefficient lists
  -> ``(coef float64[], desc int32[C*KM*3], C, KM)`` in the include/alz_b200.h layout."""
  C = len(bank)
  KM = max((len(ch) for ch in bank), default=0)
  coef, desc = [], np.zeros((C, max(KM, 1), 3), dtype=np.int32)
  for c, ch in enumerate(bank):
    for k, (b, a) in enumerate(ch):
      b = [float(v) for v in b]
      a = [float(v) for v in a]
      if len(b) == 0:
        b = [0.0]
      desc[c, k] = (len(b), len(a), len(coef))
      coef.extend(b)
      coef.extend(a)
  if KM == 0:
    KM = 1
  return np.asarray(coef if coef else [0.0], dtype=np.float64), np.ascontiguousarray(desc.reshape(-1)), C, KM


def bank_apply(x, bank, xinit=None, yinit=None, threads: int = 1):
  """Filter float32 rows ``x[S][T]`` through every channel of ``bank``.

  Returns the reference's float64 result ``y[S][C][T]``. ``xinit``/``yinit``:
  ``[C][KM][h]`` initial input/output histories (``zero`` / ``memory``)."""
  x = np.ascontiguousarray(np.atleast_2d(x), dtype=np.float32)
  S, T = x.shape
  coef, desc, C, KM = pack_bank(bank)
  y = np.empty((S, C, T), dtype=np.float64)
  hx = hy = 0
  xi = yi = None
  if xinit is not None:
    xi = np.ascontiguousarray(xinit, dtype=np.float64).reshape(C, KM, -1)
    hx = xi.shape[2]
  if yinit is not None:
    yi = np.ascontiguousarray(yinit, dtype=np.float64).reshape(C, KM, -1)
    hy = yi.shape[2]
  lib = _lib()

  def run(lo, hi):
    rc = lib.orc_bank_apply(x.ctypes.data, y.ctypes.data, coef.ctypes.data, desc.ctypes.data, C, KM, S, T, T, T,
                            xi.ctypes.data if xi is not None else None, hx,
                            yi.ctypes.data if yi is not None else None, hy, lo, hi)
    if rc != 0:
      raise RuntimeError("oracle failed")

  _threaded(run, S, threads)
  return y


def bank_apply_f32(x, bank, threads: int = 1, out=None):
  """Same as :func:`bank_apply` with zero initial state and float32-rounded output
  (what the device stores); this is the leg ``bench.py`` times as the CPU baseline."""
  x = np.ascontiguousarray(np.atleast_2d(x), dtype=np.float32)
  S, T = x.shape
  coef, desc, C, KM = pack_bank(bank)
  y = out if out is not None else np.empty((S, C, T), dtype=np.float32)
  lib = _lib()

  def run(lo, hi):
    if lib.orc_bank_apply_f32(x.ctypes.data, y.ctypes.data, coef.ctypes.data, desc.ctypes.data, C, KM, S, T, T, T,
                              lo, hi) != 0:
      raise RuntimeError("oracle failed")

  _threaded(run, S, threads)
  return y


def tv_apply(x, sections, table, xinit=None, yinit=None):
  """The time-varying contract of ``alz_apply_tv_f32`` in float64, vectorised over streams.

  ``x``: float32 rows ``[S][T]``.  ``sections``: the cascade, one list of ``(delay, is_den)`` taps per section, in
  the order ``alz_plan_taps`` lists them (section by section, numerator then feedback taps, ascending delay).
  ``table[i][n]``: the coefficient of tap ``i`` (counted over all sections) at sample ``n`` (``b_k / a_0`` for a
  numerator tap, ``-a_k / a_0`` for a feedback tap); every stream uses the same table.  ``xinit`` / ``yinit``:
  ``[K][h]`` initial input / output histories of each section as ``alz_state_init`` takes them (entry ``j`` is delay
  ``j + 1``), or None for zeros.  Each product is rounded, then added to the sum in table order, starting from 0.0.
  Returns ``y[S][T]`` float64, the last section's output."""
  x = np.atleast_2d(np.asarray(x, dtype=np.float32)).astype(np.float64)
  S, T = x.shape
  table = np.asarray(table, dtype=np.float64)

  def seeds(init, k, depth):
    row = [] if init is None else [float(v) for v in np.asarray(init, dtype=np.float64)[k]]
    row = (row + [0.0] * depth)[:depth]
    return [np.full(S, v) for v in row]          # hist[d - 1] = the value at delay d

  rows, xh, yh, first = [], [], [], 0      # rows[k]: (table row, delay, is_den) of section k's taps
  for k, taps in enumerate(sections):
    rows.append([(first + i, int(d), bool(den)) for i, (d, den) in enumerate(taps)])
    first += len(taps)
    xh.append(seeds(xinit, k, max([d for d, den in taps if not den] + [0])))
    yh.append(seeds(yinit, k, max([d for d, den in taps if den] + [0])))
  y = np.empty((S, T), dtype=np.float64)
  for n in range(T):
    inp = x[:, n]
    for k, taps in enumerate(rows):
      acc = np.zeros(S)
      for i, d, den in taps:
        past = yh[k][d - 1] if den else (inp if d == 0 else xh[k][d - 1])
        acc = acc + table[i, n] * past
      if xh[k]:
        xh[k].insert(0, inp)
        xh[k].pop()
      if yh[k]:
        yh[k].insert(0, acc)
        yh[k].pop()
      inp = acc
    y[:, n] = inp
  return y


def _threaded(run, S, threads):
  threads = max(1, min(int(threads), S))
  if threads == 1:
    run(0, S)
    return
  bounds = np.linspace(0, S, threads + 1).astype(np.int64)
  with ThreadPoolExecutor(threads) as ex:   # ctypes releases the GIL during the C call
    list(ex.map(lambda i: run(int(bounds[i]), int(bounds[i + 1])), range(threads)))


# --------------------------------------------------------------------------------------
# pure-Python restatement (small cases only)
# --------------------------------------------------------------------------------------
def py_section(b, a, seq, memory=None, zero=0.0):
  """One section, statement by statement as the reference's generated ``gen``
  (lazy_filters.py:239-257). Returns a list."""
  b = list(b)
  a = list(a)
  while len(b) > 1 and b[-1] == 0:
    b.pop()   # Poly drops zero terms; a trailing zero shortens numlist (lazy_poly.py:132-139)
  while len(a) > 1 and a[-1] == 0:
    a.pop()
  if a[0] == 0:
    raise ZeroDivisionError("Invalid filter gain")
  la, lb = len(a), len(b)
  lm = la - 1
  if memory is None:
    m = [zero] * lm
  else:
    m = list(memory)[:lm]
    m = [zero] * (lm - len(m)) + m   # zero_pad(memory, lm - len) pads on the LEFT (lazy_misc.py:132-160)
  d = [zero] * (lb - 1)
  out = []
  gain = a[0]
  for d0 in seq:
    terms = []
    hist = [d0] + d
    for k, c in enumerate(b):
      if c == 1:
        terms.append(hist[k])
      elif c == -1:
        terms.append(-hist[k])
      elif c != 0:
        terms.append(c * hist[k])
    for k in range(1, la):
      c = a[k]
      if c == -1:
        terms.append(m[k - 1])
      elif c == 1:
        terms.append(-m[k - 1])
      elif c != 0:
        terms.append(-c * m[k - 1])
    if not terms:
      m0 = zero
    else:
      acc = terms[0]
      for t in terms[1:]:
        acc = acc + t
      if gain == -1:
        m0 = -acc
      elif gain != 1:
        m0 = acc / gain
      else:
        m0 = acc
    out.append(m0)
    if lm:
      m = [m0] + m[:-1]
    if lb > 1:
      d = [d0] + d[:-1]
  return out


def py_cascade(sections, seq, memory=None, zero=0.0):
  """CascadeFilter.__call__ (lazy_filters.py:988-990): ``memory``/``zero`` are
  forwarded identically to every section."""
  data = list(seq)
  for b, a in sections:
    data = py_section(b, a, data, memory=memory, zero=zero)
  return data


# --------------------------------------------------------------------------------------
# compiled-source Python restatement: what CPython costs the reference per sample
# --------------------------------------------------------------------------------------
def py_compiled_section(b, a, zero=0.0):
  """A generator FUNCTION ``gen(seq)`` for one section, built the way the reference builds its
  evaluator (``lazy_filters.py:197-260``): the difference equation is written out as ONE Python
  expression over local delay variables, compiled with ``exec``, and the histories are shifted
  by plain assignments -- so that its per-sample cost in CPython is the reference's. Same term
  order, +-1 elision, zero dropping and ``/ a0`` on the sum as :func:`py_section`."""
  b = [float(v) for v in b]
  a = [float(v) for v in a]
  while len(b) > 1 and b[-1] == 0:
    b.pop()
  while len(a) > 1 and a[-1] == 0:
    a.pop()
  if a[0] == 0:
    raise ZeroDivisionError("Invalid filter gain")
  terms = []
  for k, c in enumerate(b):
    if c == 1:
      terms.append("x%d" % k)
    elif c == -1:
      terms.append("-x%d" % k)
    elif c != 0:
      terms.append("%r * x%d" % (c, k))
  for k, c in enumerate(a):
    if k == 0 or c == 0:
      continue
    terms.append("y%d" % k if c == -1 else ("-y%d" % k if c == 1 else "-%r * y%d" % (c, k)))
  body = ["def gen(seq):"]
  if not terms:
    body += ["  for x0 in seq:", "    yield %r" % zero]
  else:
    expr = " + ".join(terms)
    if a[0] == -1:
      expr = "-(%s)" % expr
    elif a[0] != 1:
      expr = "(%s) / %r" % (expr, a[0])
    for k in range(1, len(a)):
      body.append("  y%d = %r" % (k, zero))
    for k in range(1, len(b)):
      body.append("  x%d = %r" % (k, zero))
    body += ["  for x0 in seq:", "    y0 = " + expr, "    yield y0"]
    body += ["    y%d = y%d" % (k, k - 1) for k in range(len(a) - 1, 0, -1)]
    body += ["    x%d = x%d" % (k, k - 1) for k in range(len(b) - 1, 0, -1)]
  scope = {}
  exec("\n".join(body), scope)
  return scope["gen"]


def py_compiled_cascade(sections, seq, zero=0.0):
  """Nested generators, one per section, consumed lazily (``CascadeFilter.__call__``,
  ``lazy_filters.py:988-990``). Returns the outermost generator."""
  data = iter(seq)
  for b, a in sections:
    data = py_compiled_section(b, a, zero)(data)
  return data
