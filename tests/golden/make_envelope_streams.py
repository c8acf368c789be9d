#!/usr/bin/env python
"""Generate tests/golden/envelope_streams.npz by RUNNING THE REFERENCE ITSELF:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_envelope_streams.py

The reference's envelope.abs / .rms / .squared (default cutoff pi / 512) of six channels of the 64-channel slaney bank
(designed as make_golden.py designs it), over signal(77, 12000) widened to Python floats.  Every STEP-th value of each
row is stored (the envelope is smooth at that spacing: its lowpass has a time constant of ~160 samples), which keeps
the fixture small; tests/test_envelope_stream_gpu.py compares FilterBank.envelope_streams with decim 1 against them.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden import Hz, al, erb_space, signal  # noqa: E402  (imports the reference from ALZ_REFERENCE)

CHANNELS = [0, 9, 21, 33, 47, 63]
SEED, LENGTH, STEP = 77, 12000, 40


def main():
  x = signal(SEED, LENGTH).astype(np.float64).tolist()
  fcs = erb_space()
  out = {"channels": np.array(CHANNELS), "index": np.arange(0, LENGTH, STEP)}
  for mode in ("abs", "rms", "squared"):
    rows = []
    for c in CHANNELS:
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fcs[c] * Hz, Hz)
      filt = al.gammatone.slaney(fcs[c] * Hz, bw)
      rows.append(np.array(list(al.envelope[mode](filt(x))), dtype=np.float64)[::STEP])
    out[mode] = np.stack(rows)
  path = os.path.join(HERE, "envelope_streams.npz")
  np.savez_compressed(path, **out)
  print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
