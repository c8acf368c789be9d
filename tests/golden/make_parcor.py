#!/usr/bin/env python
"""Generate tests/golden/parcor_cases.json by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_parcor.py

For every row (the coefficients of a FIR ZFilter, row[0] the constant term), the reference's parcor(ZFilter(row)): the
values the generator yields before it ends or raises, and the exception's type name when it raises (ParCorError, or
OverflowError from `k ** 2`); and parcor_stable(1 / ZFilter(row)) (or the exception it raises).  Floats are stored as
JSON numbers written by repr(), NaN and the infinities as Python's json writes them, so -0.0 keeps its sign; one
case per line.
The rows are regenerated from seeds by rows() below.
"""
import json
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
#: the LPC orders of the analysis-filter rows
ORDERS = [1, 2, 3, 4, 5, 6, 8, 12, 16, 24, 32, 40, 48, 64]


def step_up(ks):
  """The FIR analysis filter whose reflection coefficients, highest order first, are `ks` (Levinson step-up).  With
  dyadic ks every operation is exact, so the step-down meets them again exactly."""
  a = [1.0]
  for k in reversed(ks):
    padded = a + [0.0]
    a = [x + k * y for x, y in zip(padded, reversed(padded))]
  return a


def near_midpoint_squares(rng, n, misrounded=0):
  """n doubles k in (-1, 1) whose exact square lies within 2**-8 ulp of a rounding midpoint: there a pow that is not
  correctly rounded most often differs from k * k.  The first `misrounded` of them are ones where this host's `k ** 2`
  does differ from k * k."""
  out = []
  while len(out) < n:
    k = float(rng.uniform(-1, 1))
    m, e = math.frexp(abs(k))
    mi = int(m * 2 ** 53)                     # k = mi * 2**(e - 53), mi has 53 bits
    sq = mi * mi                              # 105 or 106 bits
    drop = sq.bit_length() - 53               # bits below the rounded square's last place
    rem = sq & ((1 << drop) - 1)
    half = 1 << (drop - 1)
    if abs(rem - half) * 256 < (1 << drop) and (len(out) >= misrounded or k ** 2 != k * k):
      out.append(k)
  return out


def rows(al):
  """name -> list of rows."""
  rng = np.random.default_rng(2026)
  out = {}
  n = np.arange(1024)
  blocks = {
    "noise": rng.standard_normal(1024),
    "tone": np.sin(2 * np.pi * 0.0371 * n + .4) + .25 * np.sin(2 * np.pi * 0.213 * n),
    "dc": np.full(1024, .75),
    "impulse": np.r_[1.0, np.zeros(1023)],
  }
  for name, blk in blocks.items():
    lpc_rows = []
    for order in ORDERS:
      try:
        filt = al.lpc.kautocor(blk.tolist(), order)
      except al.ParCorError:
        continue
      num = [float(c) for c in filt.numerator]
      lpc_rows.append(num + [0.0] * (order + 1 - len(num)))
    out["lpc_" + name] = lpc_rows
  out["stable"] = [step_up(rng.uniform(-.99, .99, int(rng.integers(1, 65))).tolist()) for _ in range(16)]
  out["unstable"] = [[1.0] + (rng.standard_normal(int(rng.integers(1, 65))) * rng.choice([.3, 1., 4.])).tolist()
                     for _ in range(16)]
  out["doctest"] = [[float(c) for c in al.levinson_durbin([1, 2, 3, 4, 5, 3, 2, 1]).numerator]]
  out["unit_k"] = [step_up([1.0, .5, -.25]), step_up([-1.0, .5]), step_up([.5, -1.0, .25]), step_up([.25, .5, 1.0]),
                   step_up([.5, .25, .125, -1.0]), step_up([-.5, 1.0, .5, .25, -.125]), [1.0, 0.0, 1.0],
                   [1.0, -1.0], [1.0, 1.0]]
  out["overflow"] = [[1.0, 3.0, 1e200], [1.0, 1e160, .5], [1.0, .5, -2e154], [1.0, .5, 1.3e154], [1.0, 0.0, 1.5e154],
                     [1.0, 2.0, 3.0, 1e155], [1.0, 1e300, 1e-300]]
  nan, inf = math.nan, math.inf
  tiny = 5e-324
  out["specials"] = [[1.0, nan], [1.0, .5, nan], [1.0, nan, .5], [1.0, inf], [1.0, .5, -inf], [1.0, inf, .25],
                     [1.0, -inf, 0.0, .5], [1.0, 0.0, inf, 0.0, .5], [1.0, nan, 0.0, 0.0, .25],
                     [1.0, -0.0, .5], [1.0, .5, -0.0], [1.0, -0.0, -0.0, .3], [1.0, tiny], [1.0, .5, tiny],
                     [1.0, tiny, .5], [1.0, 2.2250738585072014e-308, -.4], [1.0, -1e-310, 1e-200, .3],
                     [1.0, 1e-160, 1e-170], [1.0, 0.3, inf, 0.7], [1.0, .5, .25, inf, -.125]]
  out["zeros"] = [[1.0, 0.0, 0.0, .5], [1.0, .5, 0.0, 0.0], [1.0, .3, 0.0, -.2, 0.0, .1], [1.0, 0.0, .9, 0.0],
                  [1.0, 0.0], [1.0, 0.0, 0.0, 0.0], step_up([.5, 0.0, .25]), step_up([0.0, 0.0, .5, 0.0]),
                  [1.0, .5, .25, 0.0, 0.0, 0.0, 0.0]]
  out["one"] = [[1.0]]
  out["not_monic"] = [[2.0, 1.0, .5], [nan, .5], [-1.0, .25], [0.5]]
  out["midpoint"] = [[1.0, float(rng.integers(-64, 65)) / 64 or .5, k] for k in near_midpoint_squares(rng, 300, 200)]
  return out


def run_one(al, row):
  """(ks, error name or None, stable or error name) of the reference on one row."""
  ks, err = [], None
  try:
    for k in al.parcor(al.ZFilter(row)):
      ks.append(k)
  except Exception as exc:
    err = type(exc).__name__
  try:
    stable = bool(al.parcor_stable(1 / al.ZFilter(row)))
  except Exception as exc:
    stable = type(exc).__name__
  return [float(k) for k in ks], err, stable


def main():
  warnings.simplefilter("ignore")
  sys.path.insert(0, os.environ["ALZ_REFERENCE"])
  import audiolazy as al  # the reference
  from audiolazy import lazy_lpc
  al.ParCorError = lazy_lpc.ParCorError
  cases = []
  for name, group in rows(al).items():
    for i, row in enumerate(group):
      row = [float(c) for c in row]
      ks, err, stable = run_one(al, row)
      cases.append({"name": "%s_%d" % (name, i), "row": row, "k": ks, "error": err, "stable": stable})
  with open(os.path.join(HERE, "parcor_cases.json"), "w") as f:
    f.write('{"python": "%d.%d", "cases": [\n' % sys.version_info[:2])
    f.write(",\n".join(json.dumps(c, separators=(",", ":")) for c in cases))
    f.write("\n]}\n")
  print(len(cases), "cases")


if __name__ == "__main__":
  main()
