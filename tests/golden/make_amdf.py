#!/usr/bin/env python
"""Generate tests/golden/amdf_cases.json by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_amdf.py

For every case, the reference's amdf(lag, size)(x, zero=zero) over a seeded float32 signal widened to Python floats:
the SHA-256 digest of its float64 output, every STEP-th value, and the taps of the reference's
(1 - z ** -lag).linearize().  The error cases record which exception the reference raises, with its message, and
whether it comes from the call or from the first value.
"""
import hashlib
import json
import os
import sys
import warnings

import numpy as np

REF = os.environ["ALZ_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
warnings.simplefilter("ignore")
import audiolazy as al  # noqa: E402  (the reference)

HERE = os.path.dirname(os.path.abspath(__file__))
LENGTH, STEP = 6000, 50

#: (lag, size, zero): integer and fractional lags (below 1 too), lag 0, a lag longer than the input, size 1, a size
#: longer than the input, size 1024, zero 0 / 0.25 / -0.3, a negative lag the reference's linearize makes causal, and a
#: lag so small that its z^0 coefficient cancels (one tap)
CASES = [
  (1, 1, 0.), (3, 4, 0.), (2.5, 4, 0.), (37.25, 100, 0.), (0, 12, 0.), (150, 64, .25), (0.4, 3, 0.), (7, 1000, -.3),
  (48, 1024, 0.), (800, 1024, .25), (113.7, 1024, -.3), (6500, 16, 0.), (5, 7000, -.3), (0, 5, -.3), (0.4, 1, .25),
  (1.5, 2, .25), (-0.5, 4, 0.), (260.125, 333, .25), (1e-20, 8, .25),
]
ERRORS = [(3, 0), (-2, 4), (-7.5, 16), (3, 2.5), (3, -2)]


def signal(seed, n):
  return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32)


def digest(y):
  return hashlib.sha256(np.ascontiguousarray(y, dtype="<f8").tobytes()).hexdigest()


def main():
  cases = []
  for i, (lag, size, zero) in enumerate(CASES):
    seed = 500 + i
    x = signal(seed, LENGTH).astype(np.float64).tolist()
    y = np.array(list(al.amdf(lag, size)(x, zero=zero)), dtype=np.float64)
    taps = [[int(k), float(v)] for k, v in (1 - al.z ** -lag).linearize().numdict.items()]
    cases.append({"lag": lag, "size": size, "zero": zero, "seed": seed, "length": LENGTH, "taps": taps,
                  "digest": digest(y), "step": STEP, "values": y[::STEP].tolist()})
  errors = []
  for lag, size in ERRORS:
    where = "call"
    try:
      s = al.amdf(lag, size)([1., 2., 3.])
      where = "first value"
      next(iter(s))
      raise AssertionError("no error for lag=%r size=%r" % (lag, size))
    except (ValueError, TypeError, ZeroDivisionError) as exc:
      errors.append({"lag": lag, "size": size, "error": type(exc).__name__, "message": str(exc), "raised_at": where})
  path = os.path.join(HERE, "amdf_cases.json")
  with open(path, "w") as fh:
    json.dump({"cases": cases, "errors": errors}, fh, indent=0)
  print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
