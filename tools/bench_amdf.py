"""Time the batched AMDF (AmdfBank.apply, libalz_b200_amdf.so) on the device and print one JSON line.

* A: 4096 streams x 16384 samples, 256 lags over 48...800 samples (integer and fractional), size 1024, decim 256;
  reports lag-samples per second.  Its output is compared with float32 of the float64 emulation on four streams (and
  with a plan created with ALZ_AMDF_PLAN_SEQUENTIAL, which at this shape runs the same sequential path).
* B: one stream of 2 880 000 samples (a minute at 48 kHz), the same bank, time-parallel (the default plan) against
  the sequential plan; their outputs are compared (max error relative to each row's peak).

The card's name and power limit are read in the same run and are part of the record (profiles/h100_amdf.json).

    python tools/bench_amdf.py [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZE, DECIM = 1024, 256


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


def lags():
  """256 lags over 48...800 samples: 128 integer and 128 fractional, as a 60 Hz - 1 kHz pitch range at 48 kHz."""
  rng = np.random.default_rng(0)
  whole = np.linspace(48, 800, 128).round().astype(int).tolist()
  frac = rng.uniform(48, 800, 128).tolist()
  return whole + frac


def fp64_ops(bank):
  """FP64 operations per sample of all lags: per lag 2 x (products + sums of the taps) + 2 scalings + 2 adds."""
  return sum(2 * (2 * len(t) - 1) + 4 if t else 4 for t in bank.taps)


def timed(torch, bank, x, steps, warm):
  """Median ms per apply over a resident batch (each call continues the streams of one state)."""
  S = x.shape[0]
  state = bank.new_state(S, decim=DECIM)
  for _ in range(warm):
    bank.apply(x, decim=DECIM, state=state)
  times = []
  for _ in range(steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    bank.apply(x, decim=DECIM, state=state)
    e1.record()
    torch.cuda.synchronize()
    times.append(e0.elapsed_time(e1))
  return {"ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times), "steps": steps}


def emulation_check(torch, bank, x, streams):
  """Whether the timed shape's output equals float32 of the float64 emulation of AudioLazy's amdf
  (tests/amdf_emulation.py) on the sampled ``streams``, at every stored (decim-th) sample."""
  sys.path.insert(0, os.path.join(ROOT, "tests"))
  from amdf_emulation import amdf_bank
  got = fresh(torch, bank, x)[streams].cpu().numpy()
  want = amdf_bank(x[streams].cpu().numpy(), bank.taps, SIZE)[:, :, DECIM - 1::DECIM].astype(np.float32)
  return {"streams": streams, "equal": bool(np.array_equal(got, want))}


def fresh(torch, bank, x):
  y = bank.apply(x, decim=DECIM, state=bank.new_state(x.shape[0], decim=DECIM))
  torch.cuda.synchronize()
  return y


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_amdf needs a CUDA device")
  torch.cuda.set_device(0)
  L = lags()
  par, seq = ab.AmdfBank(L, SIZE), ab.AmdfBank(L, SIZE, sequential=True)
  ops = fp64_ops(par)
  rec = {"workload": "AmdfBank.apply: 256 lags over 48...800 (128 integer, 128 fractional), size 1024, decim 256, "
                     "float32 device buffers", "card": card()}

  S, T = 4096, 16384
  x = torch.rand((S, T), device="cuda", generator=torch.Generator("cuda").manual_seed(1)) * 2 - 1
  a = timed(torch, par, x, steps=10, warm=2)
  a.update({"streams": S, "samples": T, "lags": len(L), "chunks": par.chunks(S, T),
            "lag_samples_per_s": S * T * len(L) / (a["ms"] * 1e-3),
            "fp64_ops_per_s": S * T * ops / (a["ms"] * 1e-3),
            "equal_to_sequential_plan": bool(torch.equal(fresh(torch, par, x), fresh(torch, seq, x))),
            "equal_to_sequential_plan_note": "trivial at this shape: the default plan evaluates it sequentially (chunks "
                                             "= 1), so both calls run the same path",
            "equal_to_float64_emulation": emulation_check(torch, par, x, [0, 1365, 2730, 4095])})
  rec["A_4096x16384"] = a
  del x

  S, T = 1, 2880000
  x = torch.rand((S, T), device="cuda", generator=torch.Generator("cuda").manual_seed(2)) * 2 - 1
  fast = timed(torch, par, x, steps=10, warm=2)
  slow = timed(torch, seq, x, steps=3, warm=1)
  yp, ys = fresh(torch, par, x).double(), fresh(torch, seq, x).double()
  err = ((yp - ys).abs().amax(dim=-1) / ys.abs().amax(dim=-1).clamp_min(1e-30)).max().item()
  rec["B_1x2880000"] = {"time_parallel": dict(fast, chunks=par.chunks(S, T)), "sequential": slow,
                        "speedup": slow["ms"] / fast["ms"], "max_rel_err_vs_sequential": err,
                        "lag_samples_per_s_time_parallel": S * T * len(L) / (fast["ms"] * 1e-3)}
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
