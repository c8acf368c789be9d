#!/usr/bin/env python
"""Generate tests/golden/tv_cases.json by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_tv.py

Every case is a filter whose coefficients include Streams (advanced once per input sample, reference
``LinearFilter.__call__``), called on a float32 test signal given as a list or as an iterator.  The case stores how
many values the reference yields, the float64 values at the samples :func:`kept` lists, and, when a coefficient Stream
ends before the input, the type of the exception it raises there (under CPython >= 3.7 a StopIteration inside the
generator becomes ``RuntimeError``, PEP 479).  The designs are built by :func:`design` from either library's ``z`` /
``Stream`` / ``CascadeFilter``, so the tests build the same filters from the package; the inputs are regenerated with
:func:`signal`.  Every design is stable.
"""
import json
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
#: the lazy pump's block ends for an iterator input (blocks of 256, 1024, 4096, ... samples)
PUMP_EDGES = (256, 1280, 5376)


def kept(n):
  """Samples of an n-sample output whose values a case stores: the first 40 (the seeded histories and the rings' first
  wraps), 6 either side of every pump block edge, the last 8, and every 97th.  A wrong coefficient or history at any
  sample of a recursive filter shows in the samples after it."""
  edges = {i for e in PUMP_EDGES for i in range(e - 6, e + 6)}
  return [i for i in range(n) if i < 40 or i >= n - 8 or i % 97 == 0 or i in edges]


def signal(seed, n):
  """The float32 test signal of tests/conftest.py, as Python floats."""
  return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32).astype(np.float64).tolist()


def memory3(size):
  """A callable ``memory=``: called with the memory size."""
  return [.25, -.5, .125, .75][:size]


def _feedback(M, d, values):
  """One Stream feedback tap at delay ``d`` plus a constant one at delay 1 when ``d > 1``: |poles| < 1."""
  z, St = M.z, M.Stream
  den = 1 - St(*values) * z ** -d
  if d > 1:
    den = den - .2 * z ** -1
  return (.5 + .25 * z ** -1) / den


def design(M, name):
  """The filter of case ``name`` built from module ``M`` (the reference or the package)."""
  z, St = M.z, M.Stream
  if name == "num_streams_stream_a0":
    return (St(1., 2., 3.) + St(.5, -.5) * z ** -1 + St(.1, .2, .3, .4) * z ** -3) / (St(2., 4., 8.) - .5 * z ** -1)
  if name == "const_a0":
    return (1 + St(.5, -.25, .75) * z ** -1 + St(-.3, .2) * z ** -2) / (2 - .6 * z ** -1 + .2 * z ** -2)
  if name == "delay0":
    return St(1., -1., .5) + .25 * z ** -1
  if name == "fb_two_streams":
    return 1 / (1 - St(.5, -.3) * z ** -2 - St(.1, .2, -.25) * z ** -17)
  if name.startswith("fb"):
    return _feedback(M, int(name[2:]), (.6, -.45, .3, 0., -.7))
  if name == "finite_list":
    coef = np.random.default_rng(77).uniform(-.6, .6, 700).tolist()
    return (1 - St([.5 * v for v in coef]) * z ** -4) / (1 - St(coef) * z ** -1)
  if name == "int_streams":
    return (St(1, 2, 3) + St(2, 1) * z ** -1) / (St(4, 2) - St(1, -1, 0) * z ** -1)
  if name == "int_feedback":
    return 1 / (2 - St(1, -1) * z ** -1)
  if name == "cascade_lti":
    return M.CascadeFilter(1 / (1 - .3 * z ** -1), St(1., .5, -.5) * z ** -1 + 1, .5 + .25 * z ** -2)
  if name == "cascade_two_tv":
    return M.CascadeFilter(1 / (1 - St(.2, -.4) * z ** -3), 1 - .5 * z ** -1, (1 + St(.5, 0.) * z ** -1) / 2)
  if name.startswith("short"):
    n = {"short300": 300, "short700": 700, "short256": 256, "short0": 0, "short_a0": 40}[name]
    if name == "short_a0":
      return (1 + .5 * z ** -1) / (St([2.] * n) - .5 * z ** -1)
    return (1 + St([1., -.5] * (n // 2) + [1.] * (n % 2)) * z ** -1) / (1 - St([.5, -.25, .125] * (n // 3) + [.5] * (n % 3)) * z ** -2)
  raise KeyError(name)


#: (name, design, seed, length, "list" / "iter", call keyword arguments)
CASES = [
  ("num_streams_stream_a0", "num_streams_stream_a0", 1, 600, "list", {}),
  ("num_streams_stream_a0_iter", "num_streams_stream_a0", 2, 6000, "iter", {}),
  ("const_a0", "const_a0", 3, 500, "list", {}),
  ("delay0", "delay0", 4, 300, "list", {}),
] + [("fb%d" % d, "fb%d" % d, 10 + d, 700 if d < 256 else 1400, "list", {}) for d in (1, 2, 15, 16, 17, 63, 64, 65, 300)] + [
  ("fb_two_streams", "fb_two_streams", 5, 800, "list", {}),
  ("fb65_iter", "fb65", 6, 6000, "iter", {}),
  ("finite_list", "finite_list", 7, 650, "list", {}),
  ("int_streams", "int_streams", 8, 400, "list", {}),
  ("int_feedback", "int_feedback", 9, 400, "list", {}),
  ("cascade_lti", "cascade_lti", 10, 500, "list", {}),
  ("cascade_two_tv_iter", "cascade_two_tv", 11, 6000, "iter", {}),
  ("memory_list", "fb2", 12, 300, "list", {"memory": [.5, -.25], "zero": .125}),
  ("memory_short", "fb17", 13, 300, "list", {"memory": [.5, -.25, .75], "zero": -.25}),
  ("memory_callable", "const_a0", 14, 300, "list", {"memory": "memory3", "zero": .5}),
  ("memory_cascade", "cascade_lti", 15, 300, "list", {"memory": [.3, -.6], "zero": .25}),
  ("short_list", "short300", 16, 500, "list", {}),
  ("short_iter", "short700", 17, 6000, "iter", {}),
  ("short_block_edge", "short256", 18, 600, "iter", {}),
  ("short_empty", "short0", 19, 50, "list", {}),
  ("short_stream_a0", "short_a0", 20, 100, "iter", {}),
  ("short_exact", "short300", 21, 300, "list", {}),
]


def call_kwargs(kwargs):
  return {k: (memory3 if v == "memory3" else v) for k, v in kwargs.items()}


def run(filt, x, mode, kwargs):
  """-> (the values the filter yields, the exception type name or None)."""
  out = []
  try:
    for v in filt(iter(x) if mode == "iter" else x, **call_kwargs(kwargs)):
      out.append(float(v))
  except Exception as exc:         # the case records it
    return out, type(exc).__name__
  return out, None


def main():
  sys.path.insert(0, os.environ["ALZ_REFERENCE"])
  sys.dont_write_bytecode = True
  warnings.simplefilter("ignore")
  import audiolazy as al  # the reference
  cases = []
  for name, dname, seed, n, mode, kwargs in CASES:
    y, exc = run(design(al, dname), signal(seed, n), mode, kwargs)
    cases.append({"name": name, "design": dname, "seed": seed, "length": n, "input": mode, "kwargs": kwargs,
                  "raises": exc, "n": len(y), "y": [y[i] for i in kept(len(y))]})
  path = os.path.join(HERE, "tv_cases.json")
  with open(path, "w") as fh:      # one case per line; json writes floats with repr(): they read back exactly
    fh.write('{"python": "%d.%d", "cases": [\n' % sys.version_info[:2])
    fh.write(",\n".join(json.dumps(case) for case in cases))
    fh.write("\n]}\n")
  print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
