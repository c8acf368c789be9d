#!/usr/bin/env python
"""Generate tests/golden/unwrap_cases.json by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_unwrap.py

For every (input, max_delta, step) case, the reference's unwrap(x, max_delta, step) over float64 values: the number of
values it yields, the SHA-256 digest of them as float64 (every NaN written as the one quiet NaN numpy makes, so NaN
matches by NaN-ness and -0.0 by sign), every STEP-th value, and the exception that ends the Stream when one does (step
0, the empty input).  For every (input, low, high) clip case the same, or the exception the call raises.
The inputs are regenerated from seeds by inputs() below.
"""
import hashlib
import json
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
PI = math.pi
#: (max_delta, step) as Python expressions: the default, the reference tests' ints, negative / zero / NaN / inf
#: max_delta, negative / inf / NaN / tiny / huge step, and the zero steps that raise at the first jump
PARAMS = ["(pi, 2 * pi)", "(8, 10)", "(4., 10.)", "(-1., 2 * pi)", "(0., 2 * pi)", "(nan, 2 * pi)", "(inf, 2 * pi)",
          "(pi, -2 * pi)", "(pi, inf)", "(pi, nan)", "(pi, 1e-300)", "(pi, 1e300)", "(.5, 1e-3)", "(pi, 0)",
          "(pi, 0.)", "(pi, -0.)"]
#: (low, high) of clip: both, one-sided, signed zeros, NaN limits, limits that are not float32, ints, high < low
CLIPS = ["(-1., 1.)", "(None, 0.)", "(0., None)", "(-0., None)", "(None, -0.)", "(-0., 0.)", "(nan, 1.)", "(-1., nan)",
         "(nan, nan)", "(.1, .3)", "(-3, 5)", "(None, None)", "(2., 1.)", "(4, 3.9)"]
CLIP_INPUTS = ["specials", "uniform", "reference_ints", "starts_neg_zero"]
STEP = 97


def env():
  return {"pi": math.pi, "nan": math.nan, "inf": math.inf}


def inputs():
  """name -> float64 array: wrapped phases of a tone and a chirp, uniform random phases, the reference's own test data,
  IEEE specials, short inputs whose first samples are special, ties |d % P| == |d % -P|, values that are not float32,
  and long inputs (several 2048-sample tiles) whose samples jump never, sometimes, always or first after 5000."""
  rng = np.random.default_rng(1234)
  out = {}
  n = np.arange(10007)
  out["tone"] = np.angle(np.exp(1j * (2 * np.pi * 441 / 48000 * n + .3)))
  out["chirp"] = np.angle(np.exp(1j * (2 * np.pi * (50 + 3000 * n / len(n)) / 48000 * n)))[:7001]
  out["uniform"] = rng.uniform(-np.pi, np.pi, 5003)
  out["reference_ints"] = np.array([0, 27, 11, 19, -1, -19, 48, 12, 0, 10, -10, 20, -20, 30, -30, 40, -40, 50, -55, -49,
                                    -40, -38, -29, -17, -25], dtype=np.float64)
  f32max = float(np.finfo(np.float32).max)
  pool = np.array([0., -0., np.nan, np.inf, -np.inf, 5e-324, -5e-324, 2.2250738585072014e-308, f32max, -f32max, 1e300,
                   -1e300, .1, np.pi, -np.pi, 2 * np.pi, 1 / 3, -7.5, 40.], dtype=np.float64)
  out["specials"] = pool[rng.integers(0, len(pool), 3001)]
  out["starts_neg_zero"] = np.array([-0., -0., 1., -0., 0., -0.])
  out["starts_nan"] = np.array([np.nan, 1., 2., 9., 1.])
  out["starts_inf"] = np.array([np.inf, 1., 2., 9.])
  out["starts_minus_inf"] = np.array([-np.inf, -0., 5.])
  out["nan_mid"] = np.array([0., np.nan, 1., 10., 20., np.nan, np.nan, 3., -4.])
  out["inf_mid"] = np.array([0., np.inf, 1., 2.])
  out["half_pi"] = np.array([0., np.pi, 0., -np.pi, 2 * np.pi])
  out["ties"] = np.cumsum(rng.choice([5., -5., 15., -25., 1.], 2003))
  out["not_float32"] = rng.uniform(-100, 100, 3001) + 1e-9
  out["huge"] = rng.choice([1e300, -1e300, 3e299, 1., -2.], 1001) * rng.uniform(.5, 1, 1001)
  out["single"] = np.array([-0.])
  out["empty"] = np.array([], dtype=np.float64)
  out["long_never"] = 1e-3 * np.arange(9001)
  out["long_sometimes"] = np.angle(np.exp(1j * 2 * np.pi * 960 / 48000 * np.arange(9001)))
  out["long_always"] = rng.uniform(-50, 50, 9001)
  late = 1e-3 * np.arange(6001)
  late[5000:] += 10.                               # the first jump (and the step-0 failure) lies in the third tile
  out["late_jump"] = late
  return out


def canon(values):
  a = np.array(values, dtype=np.float64).reshape(-1)
  a[np.isnan(a)] = np.nan
  return a


def digest(values):
  return hashlib.sha256(canon(values).tobytes()).hexdigest()


def run(make):
  """The values a reference Stream yields, and the exception that ends it ([type, message]) if one does."""
  got = []
  try:
    s = make()
  except Exception as exc:
    return None, [type(exc).__name__, str(exc)], "call"
  try:
    for v in s:
      got.append(v)
  except Exception as exc:
    return got, [type(exc).__name__, str(exc)], "iteration"
  return got, None, None


def record(name, params, got, exc, where):
  rec = {"input": name, "params": params}
  if got is not None:
    rec.update({"n": len(got), "digest": digest(got) if got else "", "values": [float(v) for v in got[::STEP]]})
  if exc is not None:
    rec.update({"exception": exc, "raised_at": where})
  return rec


def main():
  sys.path.insert(0, os.environ["ALZ_REFERENCE"])
  sys.dont_write_bytecode = True
  warnings.simplefilter("ignore")
  import audiolazy as al  # the reference
  xs = inputs()
  cases = []
  for name, x in xs.items():
    xl = x.tolist()
    for params in PARAMS:
      m, p = eval(params, env())
      got, exc, where = run(lambda: al.unwrap(xl, max_delta=m, step=p))
      cases.append(record(name, params, got, exc, where))
  clips = []
  for name in CLIP_INPUTS:
    xl = xs[name].tolist()
    for params in CLIPS:
      lo, hi = eval(params, env())
      got, exc, where = run(lambda: al.clip(xl, low=lo, high=hi))
      clips.append(record(name, params, got, exc, where))
  errors = []
  for params in ("('a', 2 * pi)", "(pi, 1j)", "(None, 2 * pi)"):
    m, p = eval(params, env())
    got, exc, where = run(lambda: al.unwrap([0., 10.], max_delta=m, step=p))
    errors.append({"params": params, "exception": exc, "raised_at": where, "n": len(got or [])})
  path = os.path.join(HERE, "unwrap_cases.json")
  with open(path, "w") as fh:
    json.dump({"step": STEP, "cases": cases, "clips": clips, "errors": errors}, fh, indent=0)
  print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
