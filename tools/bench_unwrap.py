"""Time the batched unwrap and clip kernels (Unwrap, Clip; libalz_b200_unwrap.so) on the device and print one JSON line.

* A: 4096 streams x 16384 float32 wrapped phases of tones (a jump every 8 to 200 samples) -> float64.
* B: A with float64 input.
* C: one stream of 2,880,000 float32 phases of a tone with a jump every ~50 samples -> float64 (the tile chain), and
  C0: the same stream without a jump (every carry-in comes from the look-back).
* D: A with a jump on every sample (every tile walks 2048 dependent adds: the serial-chain worst case).
* E: 2,101,248 rows (513 bins x 4096 streams) of 32 float32 frames -> float64 (the phase-vocoder layout).
* F: Clip(-1, 1) on A's shape, float32 -> float32.

Each case reports the time per call from CUDA events around many back-to-back calls (a call is the new state and its
clearing, the scratch clear and the kernel), the bytes it must move (samples in and out, and the per-stream state), their share of the H100 SXM
data-sheet HBM3 bandwidth (3.35 TB/s), and the floor that binds among the HBM floor and the chain floor: the longest
stream's jumps, one dependent float64 add each, at CHAIN_NS per add.  The baseline is a torch float64 composition of
the same recurrence in the same run (diff, remainder, where, cumsum; torch.clamp for F), timed too; its cumsum does not
add in the reference's order, so its maximum deviation from the exact result is reported.  The card's name, power limit
and SM clock are read with nvidia-smi in the same run (profiles/h100_unwrap.json).

    python tools/bench_unwrap.py [--out FILE]
"""
import argparse
import json
import math
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12
#: an estimate, not a measurement: one dependent DADD of about 8 cycles at the 1.98 GHz boost clock, the chain floor's
#: unit
CHAIN_NS = 4.0


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


def torch_unwrap(torch, x, M=math.pi, P=2 * math.pi):
  """The recurrence composed from torch float64 operations (its cumsum is not the reference's sequential sum)."""
  d = x.double()
  diff = d[:, 1:] - d[:, :-1]
  a, b = torch.remainder(diff, P), torch.remainder(diff, -P)
  term = torch.where(diff.abs() > M, -diff + torch.where(b.abs() < a.abs(), b, a), torch.zeros_like(diff))
  return torch.cat([d[:, :1], d[:, 1:] + term.cumsum(dim=1)], dim=1)


def timed(torch, fn, reps, warm=3):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    fn()
  e1.record()
  torch.cuda.synchronize()
  return e0.elapsed_time(e1) / reps


def workload(torch, fn, base, nbytes, max_jumps, reps, base_reps):
  ms = timed(torch, fn, reps)
  got, want = fn(), base()
  torch.cuda.synchronize()
  hbm_ms = nbytes / PEAK_BYTES_PER_S * 1e3
  chain_ms = max_jumps * CHAIN_NS * 1e-6
  dev = (got.double() - want.double()).abs()
  rec = {"ms": ms, "calls_timed": reps, "bytes": nbytes, "GB_per_s": nbytes / (ms * 1e-3) / 1e9,
         "share_of_3.35TB_per_s": hbm_ms / ms, "hbm_floor_ms": hbm_ms, "longest_chain_jumps": max_jumps,
         "chain_floor_ms": chain_ms, "binding_floor": "hbm" if hbm_ms >= chain_ms else "chain",
         "share_of_binding_floor": max(hbm_ms, chain_ms) / ms,
         "baseline_max_abs_deviation": float(torch.nan_to_num(dev, nan=0.).max()),
         "baseline_bit_equal": bool(torch.equal(got.double(), want.double()))}
  bms = timed(torch, base, base_reps, warm=1)
  rec.update({"torch_baseline_ms": bms, "speedup_vs_torch_baseline": bms / ms})
  return rec


def jumps(torch, x, M=math.pi):
  d = x.double()
  return int(((d[:, 1:] - d[:, :-1]).abs() > M).sum(dim=1).max()) if x.shape[1] > 1 else 0


def tones(torch, S, T, gen):
  """Wrapped phases of one tone per stream, 8 to 200 samples per period."""
  f = 1. / (8 + 192 * torch.rand((S, 1), device="cuda", generator=gen, dtype=torch.float64))
  ph = 2 * math.pi * f * torch.arange(T, device="cuda", dtype=torch.float64)
  return torch.remainder(ph + math.pi, 2 * math.pi) - math.pi


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_unwrap needs a CUDA device")
  torch.cuda.set_device(0)
  uw = ab.Unwrap()
  rec = {"workload": "Unwrap(max_delta=pi, step=2 pi) and Clip(-1, 1) on CUDA tensors", "card": card()}
  gen = torch.Generator("cuda").manual_seed(1)

  S, T = 4096, 16384
  x64 = tones(torch, S, T, gen)
  x = x64.float()
  st = 32 * 2 * S                                  # the state, read and written
  rec["A_4096x16384_f32_to_f64"] = workload(torch, lambda: uw.apply(x), lambda: torch_unwrap(torch, x),
                                            S * T * 12 + st, jumps(torch, x), reps=50, base_reps=5)
  rec["B_4096x16384_f64_to_f64"] = workload(torch, lambda: uw.apply(x64), lambda: torch_unwrap(torch, x64),
                                            S * T * 16 + st, jumps(torch, x64), reps=50, base_reps=5)
  xd = torch.where(torch.arange(T, device="cuda") % 2 == 0, 0., 5.).expand(S, T).contiguous()
  rec["D_4096x16384_jump_every_sample"] = workload(torch, lambda: uw.apply(xd), lambda: torch_unwrap(torch, xd),
                                                   S * T * 12 + st, jumps(torch, xd), reps=20, base_reps=5)
  del xd
  c = ab.Clip(-1., 1.)
  xs = x * 1.25
  rec["F_clip_4096x16384_f32"] = workload(torch, lambda: c.apply(xs), lambda: torch.clamp(xs, -1., 1.), S * T * 8, 0,
                                          reps=100, base_reps=20)
  del x, x64, xs

  T = 2880000
  xc = (torch.remainder(2 * math.pi / 50.3 * torch.arange(T, device="cuda", dtype=torch.float64) + math.pi,
                        2 * math.pi) - math.pi).float()[None]
  rec["C_1x2880000_jump_every_50"] = workload(torch, lambda: uw.apply(xc), lambda: torch_unwrap(torch, xc), T * 12 + 64,
                                              jumps(torch, xc), reps=20, base_reps=5)
  xc0 = (1e-6 * torch.arange(T, device="cuda", dtype=torch.float64)).float()[None]
  rec["C0_1x2880000_no_jump"] = workload(torch, lambda: uw.apply(xc0), lambda: torch_unwrap(torch, xc0), T * 12 + 64,
                                         0, reps=50, base_reps=5)
  del xc, xc0

  S, T = 513 * 4096, 32
  xe = tones(torch, S, T, gen).float()
  rec["E_2101248x32_f32_to_f64"] = workload(torch, lambda: uw.apply(xe), lambda: torch_unwrap(torch, xe),
                                            S * T * 12 + 32 * 2 * S, jumps(torch, xe), reps=50, base_reps=5)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
