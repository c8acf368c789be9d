#!/usr/bin/env python
"""Generate tests/golden/lpc_filter_cases.npz by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_lpc_filter.py

Every case is one stream of samples x and a table of LPC rows coef[F][order + 1] (column 0 is 1.0) switched every
`hop` samples.  With held(k) the reference's Stream of each row's coef[r][k] repeated `hop` times, the reference
computes

    analysis:   (1 + sum(held(k) * z ** -k for k in 1 .. order))(x)
    synthesis:  (1 / (1 + sum(held(k) * z ** -k for k in 1 .. order)))(x)

with its defaults (memory of zeros, zero = 0.0); at order 0 both filters are ZFilter(1).  The script records the
generator source the reference writes for one filter of each kind and asserts its form: a plain left-to-right float64
sum, in ascending delay, of `d0` and one product per tap (`next(bk) * dk`, or `-next(ak) * mk`).

The file holds `meta`, a JSON list of {"name", "kind", "order", "hop", "x_f32"} (x_f32: every sample is a float32
value, so the case also runs from float32 input), and per case i the float64 arrays `x_i`, `coef_i` and `y_i`.  Every
input and row is regenerated from seeds by cases() below.
"""
import itertools as it
import json
import math
import os
import re
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORDERS = [0, 1, 2, 3, 8, 16, 32, 64]
#: hop -> samples of the case; the last hop is longer than its input
HOPS = {1: 70, 7: 300, 160: 700, 512: 1300, 1000: 230}
F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.float32(1e-45))                       # the smallest float32 subnormal


def step_up(ks):
  """The monic FIR filter whose reflection coefficients, highest order first, are `ks` (Levinson step-up)."""
  a = [1.0]
  for k in reversed(ks):
    padded = a + [0.0]
    a = [x + k * y for x, y in zip(padded, reversed(padded))]
  return a


def f32(v):
  return np.asarray(v, np.float32).astype(np.float64)


def inputs(rng, T, kind):
  """A float64 input of T samples: float32 values widened (kind "noise", "tone", "specials") or float64 values that
  are not float32 ("f64")."""
  n = np.arange(T)
  if kind == "noise":
    return f32(rng.standard_normal(T) * .3)
  if kind == "tone":
    return f32(np.sin(2 * np.pi * .0137 * n) + .3 * np.sin(2 * np.pi * .21 * n + .5))
  if kind == "f64":
    x = rng.standard_normal(T) * .3
    x[rng.random(T) < .05] = 0.1
    x[:3] = [1e300, 5e-324, -2.5e-310][:min(3, T)]
    return x
  x = f32(rng.standard_normal(T) * .3)
  specials = [math.nan, math.inf, -math.inf, -0.0, 0.0, F32_TINY, -F32_TINY, F32_MAX, -F32_MAX,
              float(np.float32(1.1754942e-38))]
  where = rng.choice(T, min(T, 2 * len(specials)), replace=False)
  for i, w in enumerate(where):
    x[w] = specials[i % len(specials)]
  return x


def lpc_rows(al, rng, order, F, source):
  """F rows of order + 1 coefficients.  "noise", "tone", "impulse": the reference's own lpc.kautocor of frames of
  those signals (zero-padded to order + 1, as LpcFrames gives them); "stable": step-up of random |k| < 1; "unstable":
  random rows that make the synthesis overflow to inf and then NaN; "specials": rows with 0.0, -0.0, +-inf and NaN."""
  rows = []
  for r in range(F):
    if order == 0:
      rows.append([1.0])
      continue
    if source in ("noise", "tone", "impulse"):
      m = np.arange(256)
      blk = {"noise": rng.standard_normal(256),
             "tone": np.sin(2 * np.pi * (.01 + .02 * r) * m) + .1 * rng.standard_normal(256),
             "impulse": np.r_[np.zeros(r % 5), 1.0, np.zeros(255 - r % 5)]}[source]
      filt = al.lpc.kautocor([float(v) for v in blk], order)
      num = [float(c) for c in filt.numerator]
      rows.append(num + [0.0] * (order + 1 - len(num)))
    elif source == "stable":
      rows.append(step_up(rng.uniform(-.95, .95, order).tolist()))
    elif source == "unstable":
      rows.append([1.0] + (rng.standard_normal(order) * 2.5).tolist())
    else:
      row = [1.0] + (rng.standard_normal(order) * .2).tolist()
      specials = [0.0, -0.0, math.inf, -math.inf, math.nan]
      for j in range(1, order + 1):
        if rng.random() < .3:
          row[j] = specials[int(rng.integers(len(specials)))]
      rows.append(row)
  return rows


def cases(al):
  """(name, kind, order, hop, x, rows) of every case."""
  rng = np.random.default_rng(2027)
  sources = ["noise", "tone", "impulse", "stable", "unstable", "specials"]
  xkinds = ["noise", "tone", "specials", "f64"]
  out = []
  i = 0
  for kind in ("analysis", "synthesis"):
    for order in ORDERS:
      for hop, T in HOPS.items():
        source = sources[i % len(sources)]
        xkind = xkinds[(i // len(sources) + i) % len(xkinds)]
        i += 1
        F = -(-T // hop)
        x = inputs(rng, T, xkind)
        out.append(("%s_o%d_h%d_%s_%s" % (kind, order, hop, source, xkind), kind, order, hop, x,
                    lpc_rows(al, rng, order, F, source)))
  # every source and input kind at order 16 and hop 160, both kinds
  for kind in ("analysis", "synthesis"):
    for source in sources:
      for xkind in xkinds:
        x = inputs(rng, 500, xkind)
        out.append(("%s_all_%s_%s" % (kind, source, xkind), kind, 16, 160, x, lpc_rows(al, rng, 16, 4, source)))
  # hand-made: 0 * inf in a silent row, a NaN tap, -0.0 through the sums, the README row
  nan, inf = math.nan, math.inf
  readme = [1.0, 0.0, .5, 0.0, -.5]
  for kind in ("analysis", "synthesis"):
    out.append(("%s_zero_tap_times_inf" % kind, kind, 3, 4, [1.0, inf, 0.5, -0.25, 1.0, 2.0, 0.0, -0.0, 3.0, 1.0],
                [[1.0, 0.0, 0.0, 0.0], [1.0, .5, -0.0, 0.0], [1.0, 0.0, 0.0, 0.0]]))
    out.append(("%s_nan_tap" % kind, kind, 2, 3, [0.5, -1.0, 0.25, 0.0, 1.0, 2.0, -1.0, 0.5, 0.0],
                [[1.0, .5, .25], [1.0, nan, 0.0], [1.0, -.5, .25]]))
    out.append(("%s_signed_zeros" % kind, kind, 2, 2, [-0.0, -0.0, 0.0, -0.0, -0.0, -0.0],
                [[1.0, -0.0, 0.0], [1.0, 0.0, -0.0], [1.0, -1.0, -0.0]]))
    out.append(("%s_readme" % kind, kind, 4, 200, [-1., 0., 1., 0.] * 50, [readme]))
    out.append(("%s_inf_rows" % kind, kind, 2, 5, inputs(rng, 20, "noise"),
                [[1.0, inf, 0.0], [1.0, -inf, .5], [1.0, .5, inf], [1.0, 0.0, 0.0]]))
  return out


GENERATED = []


def run(al, kind, order, hop, x, rows):
  """The reference's output of one case (a list of floats)."""
  z = al.z

  def held(k):
    return al.Stream(it.chain.from_iterable(it.repeat(row[k], hop) for row in rows))

  if order == 0:
    filt = al.ZFilter(1)
  else:
    filt = 1 + sum(held(k) * z ** -k for k in range(1, order + 1))
  if kind == "synthesis":
    filt = 1 / filt
  return [float(v) for v in filt(list(x))]


def check_generated(al, lazy_filters):
  """Record the generator source of an order-3 filter of each kind, print it and assert its form."""
  orig = lazy_filters._exec_eval

  def spy(data, expr):
    GENERATED.append(data)
    return orig(data, expr)

  lazy_filters._exec_eval = spy
  try:
    for kind in ("analysis", "synthesis"):
      run(al, kind, 3, 2, [1.0, 2.0, 3.0], [[1.0, .1, .2, .3]] * 2)
  finally:
    lazy_filters._exec_eval = orig
  ana, syn = GENERATED
  print(ana, syn, sep="\n\n")
  assert re.search(r"^    m0 = d0 \+ next\(b1\) \* d1 \+ next\(b2\) \* d2 \+ next\(b3\) \* d3$", ana, re.M), ana
  assert re.search(r"^  d1 = d2 = d3 = zero$", ana, re.M), ana
  assert re.search(r"^    m0 = d0 \+ -next\(a1\) \* m1 \+ -next\(a2\) \* m2 \+ -next\(a3\) \* m3$", syn, re.M), syn
  assert re.search(r"^  m1 , m2 , m3 , = memory$", syn, re.M), syn


def main():
  warnings.simplefilter("ignore")
  sys.path.insert(0, os.environ["ALZ_REFERENCE"])
  import audiolazy as al  # the reference
  from audiolazy import lazy_filters
  check_generated(al, lazy_filters)
  meta, arrays = [], {}
  for i, (name, kind, order, hop, x, rows) in enumerate(cases(al)):
    x = [float(v) for v in x]
    y = run(al, kind, order, hop, x, rows)
    assert len(y) == len(x)
    xa = np.asarray(x, np.float64)
    with np.errstate(all="ignore"):
      is_f32 = bool(np.array_equal(xa.astype(np.float32).astype(np.float64), xa, equal_nan=True))
    meta.append({"name": name, "kind": kind, "order": order, "hop": hop, "x_f32": is_f32})
    arrays["x_%d" % i] = xa
    arrays["coef_%d" % i] = np.asarray(rows, np.float64).reshape(len(rows), order + 1)
    arrays["y_%d" % i] = np.asarray(y, np.float64)
  np.savez_compressed(os.path.join(HERE, "lpc_filter_cases.npz"), meta=np.array(json.dumps(meta)), **arrays)
  print(len(meta), "cases;", sum(len(arrays["x_%d" % i]) for i in range(len(meta))), "samples")


if __name__ == "__main__":
  main()
