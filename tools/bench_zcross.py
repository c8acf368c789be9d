"""Time the batched zero-crossing kernel (Zcross, libalz_b200_zcross.so) on the device and print one JSON line.

* A: 4096 streams x 16384 samples of uniform noise, flags (5 bytes per sample: 4 in, 1 out).
* B: the same input, block counts only, size 2048, hop 1024 (4 bytes per sample).
* C: one stream of 2^27 samples of noise, flags.
* D: one stream of 2^27 samples of silence after one decisive sample, flags: every tile after the first has no
  decisive sample, so every carry-in comes from the look-back (its worst case).

Each workload reports the time per call from CUDA events around many back-to-back calls (a call is the scratch clear,
the scan kernel and the finish kernel), the bytes it must move over that time, their share of the H100 SXM data-sheet
HBM3 bandwidth (3.35 TB/s), and an exact comparison with a torch-composed evaluation of the same semantics in the same
run (decisive mask, cummax of indices, gather), which is timed too.  That baseline exists for this comparison only.
The card's name, power limit and SM clock are read with nvidia-smi in the same run (profiles/h100_zcross.json).

    python tools/bench_zcross.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12
H = .01


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


def torch_zcross(torch, x, h, s0=0):
  """The semantics of include/alz_b200_zcross.h composed from torch operations."""
  xd = x.double()
  decisive = (xd > h) | (xd < -h)
  n = torch.arange(x.shape[-1], device=x.device).expand_as(x)
  last = torch.where(decisive, n, torch.full_like(n, -1)).cummax(dim=-1).values
  sgn = torch.where(x < 0, -1, 1).to(torch.int8)
  s = torch.where(last >= 0, sgn.gather(-1, last.clamp_min(0)), torch.full_like(sgn, s0))
  prev = torch.cat([torch.full_like(s[:, :1], s0), s[:, :-1]], dim=-1)
  return ((prev != 0) & (xd * prev < -h)).to(torch.uint8)


def torch_counts(torch, flags, size, hop):
  """Block sums of complete blocks [k hop, k hop + size) from a cumulative sum."""
  c = torch.nn.functional.pad(flags.to(torch.int64).cumsum(dim=-1), (1, 0))
  k = torch.arange((flags.shape[-1] - size) // hop + 1, device=flags.device)
  return (c[:, k * hop + size] - c[:, k * hop]).to(torch.int32)


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


def workload(torch, fn, base, nbytes, reps, base_reps):
  ms = timed(torch, fn, reps)
  got, want = fn(), base()
  torch.cuda.synchronize()
  rec = {"ms": ms, "calls_timed": reps, "bytes": nbytes, "GB_per_s": nbytes / (ms * 1e-3) / 1e9,
         "share_of_3.35TB_per_s": nbytes / (ms * 1e-3) / PEAK_BYTES_PER_S,
         "equal_to_torch_baseline": bool(torch.equal(got, want))}
  bms = timed(torch, base, base_reps, warm=1)
  rec.update({"torch_baseline_ms": bms, "speedup_vs_torch_baseline": bms / ms})
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_zcross needs a CUDA device")
  torch.cuda.set_device(0)
  zc = ab.Zcross(H, 0)
  rec = {"workload": "Zcross(hysteresis=%g, first_sign=0), float32 device buffers" % H, "card": card()}
  gen = torch.Generator("cuda").manual_seed(1)

  S, T = 4096, 16384
  x = torch.rand((S, T), device="cuda", generator=gen) * 2 - 1
  rec["A_4096x16384_flags"] = workload(torch, lambda: zc.apply(x), lambda: torch_zcross(torch, x, H),
                                       S * T * 5, reps=200, base_reps=5)
  rec["B_4096x16384_counts_2048_1024"] = workload(
      torch, lambda: zc.counts(x, 2048, 1024), lambda: torch_counts(torch, torch_zcross(torch, x, H), 2048, 1024),
      S * T * 4, reps=200, base_reps=5)
  del x

  T = 1 << 27
  x = torch.rand((1, T), device="cuda", generator=gen) * 2 - 1
  rec["C_1x2^27_flags"] = workload(torch, lambda: zc.apply(x), lambda: torch_zcross(torch, x, H), T * 5, reps=50,
                                   base_reps=2)
  x.zero_()
  x[0, 0] = .5
  rec["D_1x2^27_silence_flags"] = workload(torch, lambda: zc.apply(x), lambda: torch_zcross(torch, x, H), T * 5,
                                           reps=50, base_reps=2)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
