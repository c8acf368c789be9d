"""Laurent-polynomial coefficient container used by the filter algebra.

A :class:`Poly` is a sum of powers ``sum(c_p * x**p)`` with integer (possibly negative)
powers; the linear filters store their numerator and denominator as polynomials in
``x = z**-1`` (reference ``audiolazy/lazy_poly.py:66-487`` and
``lazy_filters.py:114-132``). The evaluator and the builders read it through
``terms()`` / ``values()`` (reference ``lazy_poly.py:159-198``).

Semantics kept from the reference because results depend on them:

* coefficients equal to ``zero`` are dropped at construction (``lazy_poly.py:132-139``),
  so a filter ``[1, 0, 2]`` has two numerator terms;
* terms remember their insertion order (a plain ``dict``): products accumulate in the
  order ``for a in self: for b in other`` and sums list ``self``'s powers first, which
  fixes the floating-point summation order of every design formula;
* ``terms()`` sorts by power, ``values()`` is the dense ascending list.

Coefficients may be :class:`~audiolazy_b200.stream.Stream` instances (time-varying
filters): as in the reference they are kept whatever their values, compared by identity,
tee-copied by :meth:`Poly.copy`, and fanned out with ``thub`` when a product or a division
uses them more than once (``lazy_poly.py:388-402, 449-462``). ``lagrange`` and ``resample``
(``lazy_poly.py:493-603``) live in :mod:`audiolazy_b200.resampling`.
"""
from __future__ import annotations

import operator
from collections.abc import Iterable
from functools import reduce

from .stream import Stream, thub

__all__ = ["Poly", "x"]


def _is_int_like(p):
  return isinstance(p, int) or (isinstance(p, float) and p.is_integer())


class Poly(object):
  """Sum of powers with number coefficients. Build from a list (index = power), a
  dict ``{power: coeff}``, another Poly or a single number (constant term)."""
  __slots__ = ("_terms", "_zero", "_hash")

  def __init__(self, data=None, zero=None):
    self._zero = 0.0 if zero is None else zero
    if isinstance(data, Poly):
      items = list(data._terms.items())
      if zero is None:
        self._zero = data._zero
    elif isinstance(data, dict):
      items = list(data.items())
    elif isinstance(data, (list, tuple)):
      items = list(enumerate(data))
    elif data is None:
      items = []
    elif isinstance(data, Stream):            # a (possibly endless) coefficient stream: constant term
      items = [(0, data)]
    elif isinstance(data, Iterable) and not isinstance(data, (str, bytes)):
      items = list(enumerate(data))
    else:
      items = [(0, data)]
    terms = {}
    for power, coeff in items:
      if isinstance(power, float) and power.is_integer():
        power = int(power)
      if not isinstance(coeff, Stream) and coeff == self._zero:   # Stream coefficients are kept
        terms.pop(power, None)
        continue
      terms[power] = coeff
    self._terms = terms

  # -- read-out ----------------------------------------------------------------------
  @property
  def zero(self):
    return self._zero

  def terms(self, sort="auto", reverse=False):
    """``(power, coeff)`` pairs; sorted by power when all powers are integers."""
    if sort == "auto":
      sort = self.is_laurent()
    keys = sorted(self._terms, reverse=reverse) if sort else (
      list(reversed(self._terms)) if reverse else list(self._terms))
    return ((k, self._terms[k]) for k in keys)

  def values(self):
    """Dense coefficient list for powers ``0..order`` (needs natural powers)."""
    if not self._terms:
      return iter(())
    return (self[k] for k in range(self.order + 1))

  def __getitem__(self, power):
    return self._terms.get(power, self._zero)

  def __len__(self):
    return len(self._terms)

  def __iter__(self):
    raise TypeError("Poly is not iterable; use terms() or values()")

  def is_polynomial(self):
    return all(isinstance(k, int) and k >= 0 for k in self._terms)

  def is_laurent(self):
    return all(isinstance(k, int) for k in self._terms)

  @property
  def order(self):
    if not self.is_polynomial():
      raise AttributeError("Power needs to be positive integers")
    return max(self._terms) if self._terms else 0

  def copy(self, zero=None):
    """Same terms; Stream coefficients are tee-copied so both polynomials stay usable."""
    return Poly({k: (v.copy() if isinstance(v, Stream) else v) for k, v in self._terms.items()},
                zero=self._zero if zero is None else zero)

  # -- arithmetic --------------------------------------------------------------------
  def _coerce(self, other):
    return other if isinstance(other, Poly) else Poly(other, zero=self._zero)

  def __neg__(self):
    return Poly({k: -v for k, v in self._terms.items()}, zero=self._zero)

  def __pos__(self):
    return Poly({k: +v for k, v in self._terms.items()}, zero=self._zero)

  def __add__(self, other):
    other = self._coerce(other)
    out = dict(self._terms)            # self's powers first, then other's new ones;
    for k, v in other._terms.items():  # a shared power keeps its place, values add
      out[k] = out[k] + v if k in self._terms else v
    return Poly(out, zero=self._zero)

  def __radd__(self, other):
    return Poly(other, zero=self._zero) + self

  def __sub__(self, other):
    return self + (-self._coerce(other))

  def __rsub__(self, other):
    return Poly(other, zero=self._zero) + (-self)

  def __mul__(self, other):
    other = self._coerce(other)
    out = {}
    mine = [(k, thub(v, len(other._terms))) for k, v in self._terms.items()]      # Streams are used
    theirs = [(k, thub(v, len(self._terms))) for k, v in other._terms.items()]    # once per partner term
    for p1, c1 in mine:
      for p2, c2 in theirs:
        p = p1 + p2
        if p in out:
          out[p] += c1 * c2
        else:
          out[p] = c1 * c2
    return Poly(out, zero=self._zero)

  def __rmul__(self, other):
    return Poly(other, zero=self._zero) * self

  def __pow__(self, exponent):
    if isinstance(exponent, Poly):
      if any(k != 0 for k in exponent._terms):
        raise NotImplementedError("Can't power general Poly instances")
      exponent = exponent[0]
    if exponent == 0:
      return Poly(1, zero=self._zero)
    if not self._terms:
      return Poly(zero=self._zero)
    if len(self._terms) == 1:
      (p, c), = self._terms.items()
      return Poly({p * exponent: 1 if c == 1 else c ** exponent}, zero=self._zero)
    if not _is_int_like(exponent) or exponent < 0:
      raise NotImplementedError("Can't power a multi-term Poly to %r" % (exponent,))
    return reduce(operator.mul, [self] * int(exponent))

  def __truediv__(self, other):
    if isinstance(other, Poly):
      if len(other) == 1:
        (delta, value), = other._terms.items()
        return Poly({k - delta: operator.truediv(v, value) for k, v in self._terms.items()}, zero=self._zero)
      if len(other) == 0:
        raise ZeroDivisionError("Dividing Poly instance by zero")
      raise NotImplementedError("Can't divide general Poly instances")
    other = thub(other, len(self._terms))
    return Poly({k: operator.truediv(v, other) for k, v in self._terms.items()}, zero=self._zero)

  def diff(self, n=1):
    """n-th derivative with respect to ``x``."""
    terms = self._terms
    for _ in range(n):
      terms = {k - 1: k * v for k, v in terms.items() if k != 0}
    return Poly(terms, zero=self._zero)

  def integrate(self):
    if -1 in self._terms:
      raise ValueError("Unable to integrate term that powers to -1")
    return Poly({k + 1: v / (k + 1) for k, v in self._terms.items()}, zero=self._zero)

  # -- evaluation --------------------------------------------------------------------
  def __call__(self, value, horner="auto"):
    """Evaluate at ``value``; a Poly argument composes. Simple polynomials use the
    Horner scheme from the highest power down, merging gaps into one power
    (same operation order as reference ``lazy_poly.py:284-349``)."""
    if isinstance(value, Poly):
      return Poly(sum((c * value ** p for p, c in self._terms.items()), Poly(zero=self._zero)), zero=self._zero)
    if not self._terms:
      return self._zero
    if value == 0:
      return self[0]
    if horner == "auto":
      horner = self.is_polynomial()
    if horner:
      pairs = list(self.terms(sort=True, reverse=True))
      power, result = pairs[0]
      for npower, ncoeff in pairs[1:]:
        scale = value if power == npower + 1 else value ** (power - npower)
        result = ncoeff + result * scale
        power = npower
      return result * value ** power
    return sum(c * value ** p for p, c in self.terms())

  # -- comparison / hashing ----------------------------------------------------------
  def __eq__(self, other):
    if not isinstance(other, Poly):
      other = Poly(other, zero=self._zero)

    def same(a, b):
      return a is b if isinstance(a, Stream) or isinstance(b, Stream) else a == b

    return same(self._zero, other._zero) and len(self._terms) == len(other._terms) and \
      all(k in other._terms and same(v, other._terms[k]) for k, v in self._terms.items())

  def __ne__(self, other):
    return not (self == other)

  def __hash__(self):
    return hash((frozenset((k, id(v) if isinstance(v, Stream) else v) for k, v in self._terms.items()), self._zero))

  @property
  def roots(self):
    import numpy as np
    return np.roots(list(self.values())[::-1]).tolist()

  def __repr__(self):
    if not self._terms:
      return "0"
    parts = []
    for p, c in self.terms():
      parts.append("%r" % (c,) if p == 0 else ("%r * x" % (c,) if p == 1 else "%r * x^%s" % (c, p)))
    return " + ".join(parts)


x = Poly({1: 1})
