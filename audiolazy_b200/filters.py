"""Linear filters behind AudioLazy's API, evaluated on the GPU.

Host-side mirror of the hot path of reference ``audiolazy/lazy_filters.py``:

* :class:`LinearFilter` / :class:`ZFilter` / ``z`` -- rational transfer functions in
  ``z**-1`` with the reference's operator algebra (``lazy_filters.py:692-892``);
  calling one with an iterable returns a lazy :class:`~audiolazy_b200.stream.Stream`
  of the filtered samples (``lazy_filters.py:141-264``).
* :class:`CascadeFilter` / :class:`ParallelFilter` -- series / parallel composites
  (``lazy_filters.py:970-1084``).
* ``comb``, ``resonator``, ``lowpass``, ``highpass`` -- the coefficient builders
  (``lazy_filters.py:1087-1495``), same formulas in the same floating-point order.

What differs from the reference, by design:

* the per-sample difference equation is not interpreted in Python: a filter call
  flattens the filter into a table of direct-form-I sections and streams blocks of
  samples through hand-written sm_90a CUDA kernels (:mod:`audiolazy_b200._engine`,
  C ABI in ``include/alz_b200.h``). There is no CPU evaluator here: without the
  native library / a CUDA device the call raises.
* samples cross the device boundary as float32 (the north-star contract); the
  recurrence itself runs in float64. Outputs therefore agree with the reference's
  float64 iterator to float32 rounding (<= 1e-5 relative is the tested bar; ~6e-8 is
  typical), and are Python floats whatever the input type was.
* input is pulled in blocks (read-ahead), not sample by sample.
* time-varying coefficients (Stream-valued ``b_k`` / ``a_k``, reference
  ``lazy_filters.py:169-176, 200-216``): the coefficient Streams are the user's Python
  iterables, so their per-sample values are pulled on the host block by block and uploaded
  with the samples; the difference equation itself still runs in the CUDA kernel
  (``alz_apply_tv_f32``).
"""
from __future__ import annotations

import cmath
import itertools as it
import operator
from collections import OrderedDict
from collections.abc import Iterable
from functools import reduce
import math
from math import pi, inf, e, nan
from numbers import Real

from .core import StrategyDict
from .misc import elementwise
from .poly import Poly
from .stream import Stream, avoid_stream, thub

__all__ = ["LinearFilterProperties", "LinearFilter", "ZFilter", "z", "FilterList", "CascadeFilter",
           "ParallelFilter", "comb", "resonator", "lowpass", "highpass"]


class LinearFilterProperties(object):
  """Coefficient read-out shared by filters and filter lists; needs ``numpoly`` and
  ``denpoly`` (reference ``lazy_filters.py:47-95``)."""

  def _dense(self, poly):
    """Coefficients of ``poly`` by ascending delay, zeros included; non-causal filters raise."""
    if any(power < 0 for power, _ in poly.terms()):
      raise ValueError("Non-causal filter")
    return list(poly.values())

  numlist = numerator = property(lambda self: self._dense(self.numpoly))
  denlist = denominator = property(lambda self: self._dense(self.denpoly))
  #: delay -> coefficient, non-zero terms only, in ascending delay order
  numdict = property(lambda self: OrderedDict(self.numpoly.terms()))
  dendict = property(lambda self: OrderedDict(self.denpoly.terms()))
  #: the same polynomials written in ``z`` instead of ``z**-1`` (for root finding)
  numpolyz = property(lambda self: Poly(self.numerator[::-1]))
  denpolyz = property(lambda self: Poly(self.denominator[::-1]))


def _is_real_number(value):
  return isinstance(value, Real) or type(value).__module__ == "numpy" and hasattr(value, "dtype") and \
    value.dtype.kind in "fiub" and getattr(value, "ndim", 1) == 0


def _seed_histories(sections, memory, zero):
  """memory= / zero= of the reference call signature -> per-section initial histories
  ``(xinit, yinit)`` as lists (per section) of lists (delay 1, 2, ...).

  Reference ``lazy_filters.py:181-195``: every section receives the same arguments;
  ``memory`` gives ``m1, m2, ...`` from its FIRST ``la-1`` items and, when shorter, is
  padded with ``zero`` on the LEFT (``zero_pad(memory, lm - len)`` pads before);
  a callable is called with the size; input pre-history ``d1, d2, ...`` is ``zero``."""
  zero = float(zero)
  xinit, yinit = [], []
  for b, a in sections:
    lm = len(a) - 1
    if memory is None:
      mem = [zero] * lm
    else:
      src = memory(lm) if not isinstance(memory, Iterable) else memory
      mem = [float(v) for v in it.islice(iter(src), lm)]
      mem = [zero] * (lm - len(mem)) + mem
    xinit.append([zero] * max(len(b) - 1, 0))
    yinit.append(mem)
  return xinit, yinit


@avoid_stream
class LinearFilter(LinearFilterProperties):
  """Rational transfer function ``numpoly / denpoly`` in ``x = z**-1``."""

  def __init__(self, numerator=None, denominator=None):
    if isinstance(numerator, LinearFilter):      # copy constructor, optionally divided by `denominator`
      source = numerator if denominator is None else operator.truediv(numerator, denominator)
      num, den = source.numpoly, source.denpoly
    else:
      num, den = Poly(numerator), Poly({0: 1} if denominator is None else denominator)
    # normalise so that the denominator's lowest power is z**0 (reference lazy_filters.py:126-132)
    lowest = min(power for power, _ in den.terms())
    if lowest != 0:
      advance = Poly([0, 1]) ** -lowest
      num, den = num * advance, den * advance
    self.numpoly, self.denpoly = num, den

  def _polys(self):
    return self.numpoly, self.denpoly

  def __iter__(self):
    return iter((self.numdict, self.dendict))

  def __hash__(self):
    return hash(tuple(power for poly in self._polys() for power, _ in poly.terms()))

  def __eq__(self, other):
    return isinstance(other, LinearFilter) and all(mine == theirs for mine, theirs in zip(self._polys(), other._polys()))

  def __ne__(self, other):   # as in the reference: true only when BOTH polynomials differ
    return isinstance(other, LinearFilter) and all(mine != theirs for mine, theirs in zip(self._polys(), other._polys()))

  # -- the hot path ------------------------------------------------------------------
  def _check_callable(self):
    """Call-time validation, same errors as reference ``lazy_filters.py:164-178``."""
    terms = list(self.numpoly.terms()) + list(self.denpoly.terms())
    if any(power < 0 for power, _ in terms):
      raise ValueError("Non-causal filter")
    a0 = self.denpoly[0]
    if not isinstance(a0, Stream) and a0 == 0:
      raise ZeroDivisionError("Invalid filter gain")
    if not all(isinstance(c, Stream) or _is_real_number(c) for _, c in terms):
      raise NotImplementedError("only real-number (or Stream-of-number) coefficients run on the accelerated path")

  def sections(self):
    """``[(b, a)]``: this filter as one direct-form-I section (float lists)."""
    self._check_callable()
    if not self.is_lti():
      raise NotImplementedError("a time-varying filter has no constant section table")
    b = [float(v) for v in self.numlist] or [0.0]
    a = [float(v) for v in self.denlist]
    return [(b, a)]

  def __call__(self, seq, memory=None, zero=0.):
    """Filter any iterable; returns a Stream (reference ``lazy_filters.py:141-264``).

    ``memory`` seeds the output history (iterable: its first items; callable: called
    with the size), ``zero`` the input pre-history and missing memory entries."""
    from . import _engine
    if not self.is_lti():
      self._check_callable()
      lm = max(p for p, _ in self.denpoly.terms())
      _, yinit = _seed_histories([([0.0], [1.0] * (lm + 1))], memory, zero)
      as_source = lambda c: iter(c) if isinstance(c, Stream) else c
      num = [(p, as_source(c)) for p, c in self.numpoly.terms()]
      den = [(p, as_source(c)) for p, c in self.denpoly.terms()]
      return _engine.filter_stream_tv(num, den, seq, yinit[0], float(zero))
    sections = self.sections()
    (b, a), = sections
    if not any(b) and not any(a[1:]):
      # nothing to sum: the reference's generated loop yields `zero` for every input sample (lazy_filters.py:224-228)
      return Stream(zero for _ in seq)
    xinit, yinit = _seed_histories(sections, memory, zero)
    return _engine.filter_stream([sections], seq, [xinit], [yinit])

  # -- batch API (no reference counterpart: arrays in, arrays out, no per-sample Python) ---
  def as_bank(self):
    """This filter as a one-channel :class:`~audiolazy_b200.bank.FilterBank`."""
    from .bank import FilterBank
    return FilterBank([self])

  def apply(self, x, state=None):
    """CUDA float32 tensor ``x[S, T]`` (or ``[T]``) -> tensor ``[S, T]``: S independent streams."""
    y = self.as_bank().apply(x, state=state)
    return y[:, 0] if x.dim() == 2 else y[0, 0]

  def apply_host(self, x):
    """float32 ndarray ``x[S, T]`` (or ``[T]``) on the host -> ndarray of the same shape."""
    import numpy as np
    x = np.asarray(x, dtype=np.float32)
    y = self.as_bank().apply_host(x)
    return y[:, 0] if x.ndim == 2 else y[0, 0]

  # -- analysis ----------------------------------------------------------------------
  @elementwise("freq", 1)
  def freq_response(self, freq):
    """Complex response at ``freq`` rad/sample (iterables map elementwise)."""
    z_ = cmath.exp(-1j * freq)
    num = self.numpoly(z_)
    den = self.denpoly(z_)
    if den == 0:
      return nan
    return num / den

  def is_lti(self):
    return not any(isinstance(c, Iterable) for _, c in it.chain(self.numpoly.terms(), self.denpoly.terms()))

  def is_causal(self):
    return all(power >= 0 for power, _ in self.numpoly.terms())

  def copy(self):
    return type(self)(self.numpoly.copy(), self.denpoly.copy())

  def linearize(self):
    """Fractional delays become their two integer neighbours, weighted linearly: a term ``v * z**-(m + f)`` with
    ``0 < f < 1`` is replaced by ``v (1 - f) z**-m + v f z**-(m+1)``; terms that land on the same delay add up
    (reference ``lazy_filters.py:339-373``; e.g. ``(z ** -4.3).linearize()`` is ``0.7 z^-4 + 0.3 z^-5``)."""
    def spread(poly):
      out = {}
      for power, coeff in poly.terms():
        whole = int(power)
        frac = power - whole
        shares = [(whole, coeff)] if frac == 0 else [(whole, coeff * (1. - frac)), (whole + 1, coeff * frac)]
        for delay, share in shares:
          out[delay] = out[delay] + share if delay in out else share
      return out
    return self.__class__(spread(self.numpoly), spread(self.denpoly))

  @property
  def poles(self):
    return self.denpolyz.roots

  @property
  def zeros(self):
    return self.numpolyz.roots


@avoid_stream
class ZFilter(LinearFilter):
  """Linear filter with the Z-transform operator algebra: build filters from ``z``
  (``(1 + z**-1) / (1 - 0.5 * z**-1)``) or from coefficient lists ``ZFilter(b, a)``.

  >>> filt = ZFilter([1, 1], [1, -1])          # doctest: +SKIP
  >>> list(filt([1, 5, -4, -7, 9]))            # doctest: +SKIP
  [1.0, 7.0, 8.0, -3.0, -1.0]
  """

  @staticmethod
  def _wrap(other):
    if isinstance(other, ZFilter):
      return other
    if isinstance(other, LinearFilter):
      raise ValueError("Filter equations have different domains")
    return ZFilter([other])   # probably a number

  def __add__(self, other):
    other = self._wrap(other)
    if self.denpoly == other.denpoly:
      return ZFilter(self.numpoly + other.numpoly, self.denpoly)
    return ZFilter(self.numpoly * other.denpoly.copy() + other.numpoly * self.denpoly.copy(),
                   self.denpoly * other.denpoly)

  def __radd__(self, other):
    return self._wrap(other) + self

  def __sub__(self, other):
    return self + (-other)

  def __rsub__(self, other):
    return self._wrap(other) - self

  def __mul__(self, other):
    if isinstance(other, ZFilter):
      return ZFilter(self.numpoly * other.numpoly, self.denpoly * other.denpoly)
    if isinstance(other, LinearFilter):
      raise ValueError("Filter equations have different domains")
    return ZFilter(self.numpoly * other, self.denpoly)

  def __rmul__(self, other):
    return self._wrap(other) * self

  def __truediv__(self, other):
    if isinstance(other, ZFilter):
      return ZFilter(self.numpoly * other.denpoly, self.denpoly * other.numpoly)
    if isinstance(other, LinearFilter):
      raise ValueError("Filter equations have different domains")
    return self * operator.truediv(1, other)

  def __rtruediv__(self, other):
    return self._wrap(other) / self

  def __pow__(self, exponent):
    single_terms = len(self.numpoly) < 2 and len(self.denpoly) < 2
    if exponent < 0 and not single_terms:      # invert first: Poly powers of sums need exponent >= 0
      return ZFilter(self.denpoly, self.numpoly) ** -exponent
    if not isinstance(exponent, (int, float)):
      raise ValueError("Z-transform powers only valid with integers")
    return ZFilter(self.numpoly ** exponent, self.denpoly ** exponent)

  def __neg__(self):
    return ZFilter(-self.numpoly, self.denpoly)

  def __pos__(self):
    return ZFilter(+self.numpoly, self.denpoly)

  def diff(self, n=1, mul_after=1):
    """``n``-th derivative with respect to ``z``; after each differentiation the result is multiplied by
    ``mul_after`` (a number or a ZFilter), as ``gammatone.sampled`` needs with ``mul_after=-z`` (reference
    ``lazy_filters.py:819-838``).

    Quotient rule, kept in the form ``N_m / D**(m+1)``: with ``H_m = N_m / D**m``,
    ``H_m' = (N_m' D - m N_m D') / D**(m+1)``, so ``N_{m+1} = mul_after (N_m' D - m N_m D')`` and only the numerator is
    carried through the loop; the denominator is ``D**(n+1)`` at the end."""
    if isinstance(mul_after, ZFilter):
      carried, base = ZFilter(self.numpoly), ZFilter(self.denpoly)
      for m in range(1, n + 1):
        carried = mul_after * (carried.diff() * base - m * carried * base.diff())
      return carried / base ** (n + 1)
    to_z = Poly({-1: 1})                       # the polynomials are in z**-1: substitute to differentiate in z
    carried, base = self.numpoly(to_z), self.denpoly(to_z)
    for m in range(1, n + 1):
      carried = mul_after * (carried.diff() * base - m * carried * base.diff())
    return ZFilter(carried(to_z), self.denpoly ** (n + 1))

  def __call__(self, seq, memory=None, zero=0.):
    """Filter an iterable; given another ZFilter ``g`` instead, return the composition ``H(g)``: every ``z**-k``
    of both polynomials becomes ``g**-k`` (reference ``lazy_filters.py:885-887``)."""
    if isinstance(seq, ZFilter):
      def at(poly):
        total = 0
        for power, coeff in poly.terms():
          total = total + coeff * seq ** -power
        return total
      return at(self.numpoly) / at(self.denpoly)
    return super(ZFilter, self).__call__(seq, memory=memory, zero=zero)

  def __repr__(self):
    def side(poly):
      parts = []
      for power, value in poly.terms():
        if value == 0:
          continue
        mono = "" if power == 0 else ("z^%s" % -power if -power != 1 else "z")
        if mono and value == 1:
          parts.append(mono)
        elif mono and value == -1:
          parts.append("-" + mono)
        else:
          parts.append(("%g" % value) + (" * " + mono if mono else ""))
      return " + ".join(parts).replace("+ -", "- ") or "0"
    num, den = side(self.numpoly), side(self.denpoly)
    return num if den == "1" else "(%s) / (%s)" % (num, den)

  __str__ = __repr__


z = ZFilter({-1: 1})


# --------------------------------------------------------------------------------------
# composites
# --------------------------------------------------------------------------------------
class FilterList(list, LinearFilterProperties):
  """Common part of CascadeFilter / ParallelFilter: a list of filters."""

  def __init__(self, *filters):
    if len(filters) == 1 and not callable(filters[0]) and isinstance(filters[0], Iterable):
      filters = filters[0]
    list.__init__(self)
    self.extend(filters)

  def _rewrap(self, result):
    return type(self)(result)

  def __add__(self, other):
    return self._rewrap(list.__add__(self, list(other)))

  def __radd__(self, other):
    return self._rewrap(list(other) + list(self))

  def __mul__(self, other):
    return self._rewrap(list.__mul__(self, other))

  __rmul__ = __mul__

  def __getitem__(self, item):
    result = list.__getitem__(self, item)
    return self._rewrap(result) if isinstance(item, slice) else result

  def is_linear(self):
    return all(isinstance(f, LinearFilter) or (hasattr(f, "is_linear") and f.is_linear()) for f in self.callables)

  def is_lti(self):
    return self.is_linear() and all(f.is_lti() for f in self.callables)

  def is_causal(self):
    return all(f.is_causal() for f in self.callables if hasattr(f, "is_causal"))

  def __eq__(self, other):
    return type(other) is type(self) and list(self) == list(other)

  def __ne__(self, other):
    return not self == other

  __hash__ = None

  @property
  def callables(self):
    """Members, with bare numbers cast to constant-gain filters."""
    return [(f if callable(f) else LinearFilter(f)) for f in self]

  def _fold(self, combine, attribute):
    """``combine`` over one attribute of every member; members without it are non-linear."""
    try:
      return reduce(combine, (getattr(f, attribute) for f in self.callables))
    except AttributeError:
      raise AttributeError("Non-linear filter")

  def _roots(self, attribute):
    """All members' ``poles`` / ``zeros`` concatenated (LTI lists only)."""
    if not self.is_lti():
      raise AttributeError("Not a LTI filter")
    return [root for f in self.callables for root in getattr(f, attribute)]

  def _flat_sections(self):
    """Sections of an all-LTI list whose members are filters or cascades, else None."""
    out = []
    for f in self.callables:
      if isinstance(f, CascadeFilter):
        sub = f._flat_sections()
        if sub is None:
          return None
        out.append(sub)
      elif isinstance(f, LinearFilter) and f.is_lti():
        try:
          out.append(f.sections())
        except NotImplementedError:
          return None
      else:
        return None
    return out


@avoid_stream
class CascadeFilter(FilterList):
  """Filters applied in series. A filter is any callable that receives an iterable and
  returns a Stream (reference ``lazy_filters.py:970-1021``). When every member is an
  LTI filter the whole cascade is ONE device plan: intermediate signals never leave
  the registers of the kernel."""

  def _flat_sections(self):
    nested = FilterList._flat_sections(self)
    return None if nested is None else [sec for member in nested for sec in member]

  def __call__(self, *args, **kwargs):
    sections = self._flat_sections()
    if sections is not None and len(args) == 1 and set(kwargs) <= {"memory", "zero"}:
      from . import _engine
      xinit, yinit = _seed_histories(sections, kwargs.get("memory"), kwargs.get("zero", 0.))
      return _engine.filter_stream([sections], args[0], [xinit], [yinit])
    return reduce(lambda data, filt: filt(data, *args[1:], **kwargs), self.callables, args[0])

  # batch API, as LinearFilter.apply / apply_host
  def as_bank(self):
    from .bank import FilterBank
    return FilterBank([self])

  apply = LinearFilter.apply
  apply_host = LinearFilter.apply_host

  # the cascade as one transfer function: products of the members' polynomials / responses
  numpoly = property(lambda self: self._fold(operator.mul, "numpoly"))
  denpoly = property(lambda self: self._fold(operator.mul, "denpoly"))
  poles = property(lambda self: self._roots("poles"))
  zeros = property(lambda self: self._roots("zeros"))

  @elementwise("freq", 1)
  def freq_response(self, freq):
    return reduce(operator.mul, (f.freq_response(freq) for f in self.callables))


@avoid_stream
class ParallelFilter(FilterList):
  """Filters fed by the same input whose outputs are summed (reference
  ``lazy_filters.py:1024-1084``). All-LTI lists run as one bank launch followed by the
  left-associated channel sum on the device."""

  def __call__(self, *args, **kwargs):
    if len(self) == 0:
      zero = kwargs["zero"] if "zero" in kwargs else 0.
      return Stream(zero for _ in args[0])
    nested = self._flat_sections()
    if nested is not None and len(args) == 1 and set(kwargs) <= {"memory", "zero"}:
      from . import _engine
      seeds = [_seed_histories(ch, kwargs.get("memory"), kwargs.get("zero", 0.)) for ch in nested]
      return _engine.filter_stream(nested, args[0], [s[0] for s in seeds], [s[1] for s in seeds], sum_channels=True)
    arg0 = thub(args[0], len(self))
    return reduce(operator.add, (f(arg0, *args[1:], **kwargs) for f in self.callables))

  def _as_one_filter(self):
    if not self.is_linear():
      raise AttributeError("Non-linear filter")
    return reduce(operator.add, (ZFilter(f) for f in self.callables))

  # the sum as one transfer function: summed over a common denominator
  numpoly = property(lambda self: self._as_one_filter().numpoly)
  denpoly = property(lambda self: self._fold(operator.mul, "denpoly"))
  poles = property(lambda self: self._roots("poles"))

  @property
  def zeros(self):
    if not self.is_lti():
      raise AttributeError("Not a LTI filter")
    return reduce(operator.add, (ZFilter(f) for f in self)).zeros

  @elementwise("freq", 1)
  def freq_response(self, freq):
    return reduce(operator.add, (f.freq_response(freq) for f in self.callables))


# --------------------------------------------------------------------------------------
# coefficient builders (float64 host arithmetic, same operation order as the reference)
#
# A design parameter may be a Stream (one value per sample): the math functions below map
# over iterables, every intermediate that the formula reads more than once goes through
# ``thub`` with its read count (a no-op for plain numbers), and the result is a ZFilter with
# Stream coefficients, i.e. a time-varying filter (reference ``lazy_filters.py:1202-1206``,
# ``examples/lptv.py:28-38``).
# --------------------------------------------------------------------------------------
cos, sin, exp, sqrt = (elementwise("x", 0)(f) for f in (math.cos, math.sin, math.exp, math.sqrt))


def _unit_if_zero(values):
  """``values`` with zeros replaced by one (number or Stream)."""
  if isinstance(values, Iterable):
    return Stream(v if v else 1 for v in values)
  return values if values else 1


comb = StrategyDict("comb")


@comb.strategy("fb", "alpha", "fb_alpha", "feedback_alpha")
def comb(delay, alpha=1):
  """Feedback comb ``y[n] = x[n] + alpha * y[n - delay]`` (ref ``lazy_filters.py:1090-1116``)."""
  return 1 / (1 - alpha * z ** -delay)


@comb.strategy("tau", "fb_tau", "feedback_tau")
def comb(delay, tau=inf):
  """Feedback comb from a time constant: ``alpha = e ** (-delay / tau)`` (ref ``:1119-1146``)."""
  alpha = e ** (-delay / tau)
  return 1 / (1 - alpha * z ** -delay)


@comb.strategy("ff", "ff_alpha", "feedforward_alpha")
def comb(delay, alpha=1):
  """Feedforward comb ``y[n] = x[n] + alpha * x[n - delay]`` (ref ``:1149-1173``)."""
  return 1 + alpha * z ** -delay


resonator = StrategyDict("resonator")


@resonator.strategy("poles_exp")
def resonator(freq, bandwidth):
  """Two-pole resonator, 0 dB at ``freq``; ``R = exp(-bandwidth / 2)`` (ref ``:1179-1209``)."""
  R = thub(exp(-bandwidth * .5), 5)
  cost = thub(cos(freq) * (2 * R) / (1 + R ** 2), 2)
  gain = (1 - R ** 2) * sqrt(1 - cost ** 2)
  denominator = 1 - 2 * R * cost * z ** -1 + R ** 2 * z ** -2
  return gain / denominator


@resonator.strategy("freq_poles_exp")
def resonator(freq, bandwidth):
  """Two-pole resonator whose ``freq`` is the pole angle (ref ``:1212-1242``)."""
  R = thub(exp(-bandwidth * .5), 3)
  freq = thub(freq, 2)
  gain = (1 - R ** 2) * sin(freq)
  denominator = 1 - 2 * R * cos(freq) * z ** -1 + R ** 2 * z ** -2
  return gain / denominator


@resonator.strategy("z_exp")
def resonator(freq, bandwidth):
  """Two-pole resonator with zeros at DC and Nyquist, 0 dB at ``freq`` (ref ``:1245-1276``)."""
  R = thub(exp(-bandwidth * .5), 5)
  cost = cos(freq) * (1 + R ** 2) / (2 * R)
  gain = (1 - R ** 2) * .5
  numerator = 1 - z ** -2
  denominator = 1 - 2 * R * cost * z ** -1 + R ** 2 * z ** -2
  return gain * numerator / denominator


@resonator.strategy("freq_z_exp")
def resonator(freq, bandwidth):
  """Like ``z_exp`` with ``freq`` as the pole angle (ref ``:1279-1310``)."""
  R = thub(exp(-bandwidth * .5), 3)
  gain = (1 - R ** 2) * .5
  numerator = 1 - z ** -2
  denominator = 1 - 2 * R * cos(freq) * z ** -1 + R ** 2 * z ** -2
  return gain * numerator / denominator


lowpass = StrategyDict("lowpass")
highpass = StrategyDict("highpass")


@lowpass.strategy("pole")
def lowpass(cutoff):
  """One-pole lowpass, -3.0103 dB at ``cutoff`` rad/sample, 0 dB at DC (ref ``:1370-1378``)."""
  x = thub(2 - cos(cutoff), 2)
  R = thub(x - sqrt(x ** 2 - 1), 2)
  return (1 - R) / (1 - R * z ** -1)


@highpass.strategy("pole")
def highpass(cutoff):
  """One-pole highpass, 0 dB at Nyquist (ref ``:1381-1389``)."""
  x = thub(2 + cos(cutoff), 2)
  R = thub(x - sqrt(x ** 2 - 1), 2)
  return (1 - R) / (1 + R * z ** -1)


@lowpass.strategy("z")
def lowpass(cutoff):
  """One-pole one-zero lowpass (ref ``:1392-1405``)."""
  cutoff = thub(cutoff, 2)
  numR = sin(cutoff) - 1
  denR = _unit_if_zero(cos(cutoff))   # where cos is zero the numerator is zero too
  R = thub(numR / denR, 2)
  gain = (1 + R) / 2
  return gain * (1 + z ** -1) / (1 + R * z ** -1)


@highpass.strategy("z")
def highpass(cutoff):
  """One-pole one-zero highpass (ref ``:1408-1421``)."""
  cutoff = thub(cutoff, 2)
  numR = 1 - sin(cutoff)
  denR = _unit_if_zero(cos(cutoff))
  R = thub(numR / denR, 2)
  gain = (1 + R) / 2
  return gain * (1 - z ** -1) / (1 - R * z ** -1)


@lowpass.strategy("pole_exp")
def lowpass(cutoff):
  """Matched-Z one-pole lowpass, ``R = exp(-cutoff)`` (ref ``:1424-1437``)."""
  R = thub(exp(-cutoff), 2)
  return (1 - R) / (1 - R * z ** -1)


@highpass.strategy("pole_exp")
def highpass(cutoff):
  """Matched-Z one-pole highpass, ``R = exp(cutoff - pi)`` (ref ``:1440-1454``)."""
  R = thub(exp(cutoff - pi), 2)
  return (1 - R) / (1 + R * z ** -1)


@lowpass.strategy("z_exp")
def lowpass(cutoff):
  """Matched-Z one-pole one-zero lowpass, ``R = exp(cutoff - pi)`` (ref ``:1457-1472``)."""
  R = thub(exp(cutoff - pi), 2)
  G = (R + 1) / 2
  return G * (1 + z ** -1) / (1 + R * z ** -1)


@highpass.strategy("z_exp")
def highpass(cutoff):
  """Matched-Z one-pole one-zero highpass, ``R = exp(-cutoff)`` (ref ``:1475-1490``)."""
  R = thub(exp(-cutoff), 2)
  G = (R + 1) / 2
  return G * (1 - z ** -1) / (1 - R * z ** -1)


lowpass.default = lowpass.pole
highpass.default = highpass.z
