"""Small helpers the filter path and its tests use: ``sHz``, ``almost_eq``,
``zero_pad``, ``elementwise``, ``freq2lag`` / ``lag2freq`` (reference ``audiolazy/lazy_misc.py``)."""
from __future__ import annotations

import functools
import itertools as it
from collections.abc import Iterable
from math import pi

from .core import StrategyDict

__all__ = ["sHz", "almost_eq", "zero_pad", "elementwise", "rint", "freq2lag", "lag2freq", "DEFAULT_SAMPLE_RATE"]

DEFAULT_SAMPLE_RATE = 44100   # reference lazy_misc.py:41


def rint(x, step=1):
  """Round to the nearest multiple of ``step``, as an int."""
  return int(round(x / step) * step) if step != 1 else int(round(x))


def sHz(rate):
  """``(s, Hz)`` unit constants: samples per second and radians per sample per hertz,
  so that ``440 * Hz`` is a frequency in rad/sample (reference ``lazy_misc.py:300-320``)."""
  return float(rate), 2 * pi / rate


def freq2lag(v):
  """Frequency (rad/sample) to lag (samples): ``2 * pi / v`` (reference ``lazy_misc.py:323-325``)."""
  return 2 * pi / v


def lag2freq(v):
  """Lag (samples) to frequency (rad/sample): ``2 * pi / v`` (reference ``lazy_misc.py:329-331``)."""
  return 2 * pi / v


def zero_pad(seq, left=0, right=0, zero=0.0):
  """Generator padding ``seq`` with ``left`` leading and ``right`` trailing ``zero`` items
  (reference ``lazy_misc.py:132-160``)."""
  return it.chain(it.repeat(zero, left), seq, it.repeat(zero, right))


def elementwise(name="", pos=None):
  """Decorator: when the argument called ``name`` (or at position ``pos``) is an
  iterable, map the function over it and return a Stream/list-like of results
  (reference ``lazy_misc.py:163-228``). Lists/tuples/sets keep their type."""
  from .stream import Stream
  if (name == "") and (pos is None):
    pos = 0

  def decorator(func):
    @functools.wraps(func)
    def wrapper(*args, **kwargs):
      positional = (pos is not None) and (pos < len(args))
      arg = args[pos] if positional else kwargs.get(name)
      if isinstance(arg, Iterable) and not isinstance(arg, (str, bytes)):
        def call(value):
          if positional:
            new_args = args[:pos] + (value,) + args[pos + 1:]
            return func(*new_args, **kwargs)
          new_kwargs = dict(kwargs)
          new_kwargs[name] = value
          return func(*args, **new_kwargs)
        if isinstance(arg, (list, tuple, set)):
          return type(arg)(call(v) for v in arg)
        return Stream(call(v) for v in arg)
      return func(*args, **kwargs)
    return wrapper
  return decorator


almost_eq = StrategyDict("almost_eq")


def _pairwise(check, a, b, pad):
  ia, ib = isinstance(a, Iterable), isinstance(b, Iterable)
  if ia != ib:
    return False
  if ia:
    return all(_pairwise(check, x, y, pad) for x, y in it.zip_longest(a, b, fillvalue=pad))
  return check(a, b)


@almost_eq.strategy("bits")
def almost_eq(a, b, bits=32, tol=1, ignore_type=True, pad=0.0):
  """``|a-b| <= 2**(tol - significand - 1) * |a+b|`` elementwise over (nested) iterables;
  ``bits`` picks the IEEE significand (32 -> 23 bits), reference ``lazy_misc.py:234-267``."""
  if not (ignore_type or type(a) == type(b)):
    return False
  scale = 2.0 ** (tol - {32: 23, 64: 52, 80: 63, 128: 112}[bits] - 1)
  return _pairwise(lambda x, y: abs(x - y) <= scale * abs(x + y), a, b, pad)


@almost_eq.strategy("diff")
def almost_eq(a, b, max_diff=1e-7, ignore_type=True, pad=0.0):
  """``|a-b| <= max_diff`` elementwise (reference ``lazy_misc.py:270-297``)."""
  if not (ignore_type or type(a) == type(b)):
    return False
  return _pairwise(lambda x, y: abs(x - y) <= max_diff, a, b, pad)
