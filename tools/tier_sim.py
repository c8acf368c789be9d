#!/usr/bin/env python
"""Numerical experiment behind the per-channel precision tier (DESIGN.md section 3).

Emulates the monic cascade of csrc/alz_biquad.cuh in float32 arithmetic on the CPU (numpy,
vectorised over channels and streams, serial in time) for several candidate schemes and
prints each channel's error against the float64 oracle:

  f32      float32 coefficients, float32 state, FFMA
  ds       double-single coefficients (hi + lo float32), float32 state, 2 FFMA per tap
  delta    float32 state, feedback written as y1 + (y1 - y2) + e1*y1 + e2*y2 (e = small parts)
  dform    DIFFERENCE form: state (y1, d1 = y1 - y2), d = d1 + (t - h y1 - e2 d1), y = y1 + d with h = |1 - p|^2,
           e2 = 1 - A^2 (small coefficients keep their relative precision, rounding noise shaped by 1 - A^2 z^-1)
  dform2   dform with the numerator taken from the previous section's difference

Round-2 outcome (DESIGN.md section 3): on white noise the difference form holds 1.6e-6 from ERB channel 6 upward
(direct float32: 1e-3 ... 1e-5 there), but (i) it needs a 4-deep dependency chain per section and sample for the
arithmetic alone, (ii) it misses the bar on short rows (64
samples: 6e-5 relative to the early transient's peak) and on inputs without in-band content (pure Nyquist: 4e-3).
It is NOT in the product; this script keeps the experiment reproducible.

Test infrastructure: imports oracle/.
"""
import argparse
import sys
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

f32 = np.float32


def fma32(a, b, c):
  return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def monic_tables(sections):
  """-> c1[C][K], c2[C][K], na1[C][K], na2[C][K], G[C] (float64)."""
  C, K = len(sections), max(len(ch) for ch in sections)
  c1 = np.zeros((C, K)); c2 = np.zeros((C, K)); na1 = np.zeros((C, K)); na2 = np.zeros((C, K)); G = np.ones(C)
  for c, ch in enumerate(sections):
    for k, (b, a) in enumerate(ch):
      b = [v / a[0] for v in b] + [0.0] * 3
      a = [v / a[0] for v in a] + [0.0] * 3
      G[c] *= b[0]
      c1[c, k], c2[c, k] = b[1] / b[0], b[2] / b[0]
      na1[c, k], na2[c, k] = -a[1], -a[2]
  return c1, c2, na1, na2, G


def run(sections, x, scheme):
  """x[S][T] float32 -> y[S][C][T] float32 with the emulated arithmetic."""
  c1, c2, na1, na2, G = monic_tables(sections)
  C, K = c1.shape
  S, T = x.shape
  Gf = G.astype(f32)
  hi = lambda v: v.astype(f32)
  lo = lambda v: (v - v.astype(f32).astype(np.float64)).astype(f32)
  u = np.zeros((K + 1, 2, S, C), dtype=f32)
  dstate = np.zeros((K, S, C), dtype=f32)
  dprev = None
  y = np.empty((S, C, T), dtype=f32)
  bc = lambda v: np.broadcast_to(v[None, :], (S, C))
  for n in range(T):
    inp = (x[:, n:n + 1] * Gf[None, :]).astype(f32)
    in1, in2 = u[0, 0].copy(), u[0, 1].copy()
    u[0, 1] = in1
    u[0, 0] = inp
    for k in range(K):
      y1, y2 = u[k + 1, 0].copy(), u[k + 1, 1].copy()
      t = inp
      if scheme == "f32":
        if np.any(c1[:, k]): t = fma32(bc(hi(c1[:, k])), in1, t)
        if np.any(c2[:, k]): t = fma32(bc(hi(c2[:, k])), in2, t)
        t = fma32(bc(hi(na2[:, k])), y2, t)
        o = fma32(bc(hi(na1[:, k])), y1, t)
      elif scheme == "ds":
        for cf, v in ((c1[:, k], in1), (c2[:, k], in2), (na2[:, k], y2)):
          if np.any(cf):
            t = fma32(bc(lo(cf)), v, t)
            t = fma32(bc(hi(cf)), v, t)
        t = fma32(bc(lo(na1[:, k])), y1, t)
        o = fma32(bc(hi(na1[:, k])), y1, t)
      elif scheme == "delta":
        # na1 = 2 - e1, na2 = -1 + e2 : y = t + e2*y2 - e1*y1 + (y1 - y2) + y1   (differences of neighbours are exact-ish)
        e1 = (2.0 - na1[:, k]); e2 = (na2[:, k] + 1.0)
        if np.any(c1[:, k]): t = fma32(bc(hi(c1[:, k])), in1, t)
        if np.any(c2[:, k]): t = fma32(bc(hi(c2[:, k])), in2, t)
        t = fma32(bc(hi(e2)), y2, t)
        t = fma32(bc(hi(-e1)), y1, t)
        d = (y1 - y2).astype(f32)
        o = ((t + d).astype(f32) + y1).astype(f32)
      elif scheme in ("dform", "dform2"):
        # state (y1, d1 = y1 - y2):  d = d1 + (t - h*y1 - e2*d1),  y = y1 + d   (h = 1 - na1 - na2, e2 = 1 + na2)
        h = 1.0 - na1[:, k] - na2[:, k]; e2 = 1.0 + na2[:, k]
        d1 = dstate[k]
        if scheme == "dform2" and k > 0:
          # numerator from the previous section's difference: in + c1*in1 = (in - in1) + (1 + c1)*in1
          t = fma32(bc(hi(1.0 + c1[:, k])), in1, dprev)
        else:
          if np.any(c1[:, k]): t = fma32(bc(hi(c1[:, k])), in1, t)
        if np.any(c2[:, k]): t = fma32(bc(hi(c2[:, k])), in2, t)
        wv = fma32(bc(hi(-h)), y1, t)
        wv = fma32(bc(hi(-e2)), d1, wv)
        dn = (d1 + wv).astype(f32)
        o = (y1 + dn).astype(f32)
        dstate[k] = dn
        dprev = dn
      else:
        raise ValueError(scheme)
      u[k + 1, 1] = y1
      u[k + 1, 0] = o
      inp, in1, in2 = o, y1, y2
    y[:, :, n] = inp
  return y


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--strategy", default="slaney")
  ap.add_argument("--samples", type=int, default=20000)
  ap.add_argument("--streams", type=int, default=2)
  ap.add_argument("--schemes", default="f32,ds")
  args = ap.parse_args()
  import audiolazy_b200 as ab
  import oracle
  bank = ab.gammatone_bank(strategy=args.strategy)
  secs = bank.sections()
  if any(len(b) > 3 for ch in secs for b, a in ch):
    print("head-FIR bank: emulation covers biquad sections only"); return
  x = np.random.default_rng(0).uniform(-1, 1, (args.streams, args.samples)).astype(f32)
  want = oracle.bank_apply(x, secs)
  peak = np.max(np.abs(want), axis=-1)
  res = {}
  for sch in args.schemes.split(","):
    got = run(secs, x, sch).astype(np.float64)
    res[sch] = np.max(np.max(np.abs(got - want), axis=-1) / peak, axis=0)
  c1, c2, na1, na2, G = monic_tables(secs)
  print("ch   fc[Hz]     R        " + "  ".join("%-9s" % s for s in res))
  for c in range(len(secs)):
    R = np.sqrt(abs(na2[c, 0]))
    print("%2d  %8.1f  %.5f  " % (c, bank.freqs[c] if bank.freqs is not None else -1, R) +
          "  ".join("%.3e" % res[s][c] for s in res))


if __name__ == "__main__":
  main()
