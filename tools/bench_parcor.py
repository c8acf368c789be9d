"""Time the batched PARCOR kernel (parcor_batch; libalz_b200_parcor.so) on the device and print one JSON line.

* A: the flagship LpcFrames coefficients: LpcFrames(16, 1024, 512) of 4096 x 16384 float32 samples, 4096 x 31 rows of
  17 (127k rows); also the time of LpcFrames.apply itself on that input, and of apply followed by parcor_batch.
* B: 10**6 random rows of order 64 (L = 65), a quarter of them unstable.
* Baseline: the same step-down composed from torch float64 operations on A's and B's rows (one vectorized step per
  order, `k * k` for the square and no failure bookkeeping), timed in the same run; it is not the reference's
  arithmetic, so its largest deviation from parcor_batch over the rows both finish is reported.

Each time is per call, from CUDA events around back-to-back calls after a warm-up.  The HBM floor is the bytes a call
must move (the rows in; k, count, failed and stable out) over the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s).  The
card's name, power limit and SM clock are read with nvidia-smi in the same run (profiles/h100_parcor.json).

    python tools/bench_parcor.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


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


def torch_step_down(torch, rows):
  """k of every row, highest order first, from torch float64 operations: k * k for the square, no dropped terms."""
  a = rows[:, 1:].clone()
  L1 = a.shape[1]
  ks = []
  for m in range(L1, 0, -1):
    k = a[:, m - 1]
    ks.append(k)
    r = 1 / (1 - k * k)
    if m > 1:
      a[:, :m - 1] = (a[:, :m - 1] - k[:, None] * a[:, :m - 1].flip(1)) * r[:, None]
  return torch.stack(ks, dim=1)


def case(torch, ab, rows, reps):
  n, L = rows.shape
  t = timed(torch, lambda: ab.parcor_batch(rows), reps)
  tb = timed(torch, lambda: torch_step_down(torch, rows), max(3, reps // 10))
  res = ab.parcor_batch(rows)
  base = torch_step_down(torch, rows)
  full = (res.failed == 0) & (res.count == L - 1) & torch.isfinite(res.k).all(dim=1) & torch.isfinite(base).all(dim=1)
  dev = (res.k[full] - base[full]).abs().max().item() if bool(full.any()) else None
  nbytes = n * L * 8 + n * (L - 1) * 8 + n * (4 + 1 + 1)
  floor_ms = nbytes / PEAK_BYTES_PER_S * 1e3
  return {"rows": n, "L": L, "ms": round(t, 4), "bytes": nbytes, "hbm_floor_ms": round(floor_ms, 4),
          "share_of_hbm_floor": round(floor_ms / t, 3), "torch_k_times_k_ms": round(tb, 4),
          "torch_max_abs_deviation": dev, "torch_rows_compared": int(full.sum().item()),
          "failed_rows": int((res.failed != 0).sum().item()), "stable_rows": int(res.stable.sum().item())}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  torch.cuda.set_device(0)
  g = torch.Generator(device="cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=g) * 2 - 1
  lp = ab.LpcFrames(16, 1024, 512)
  coef = lp.apply(x).coef
  out = {"card": card(), "torch": torch.__version__}
  a = case(torch, ab, coef.reshape(-1, 17), 200)
  a["lpc_apply_ms"] = round(timed(torch, lambda: lp.apply(x), 20), 4)
  a["lpc_apply_then_parcor_ms"] = round(timed(torch, lambda: ab.parcor_batch(lp.apply(x).coef), 20), 4)
  out["A_lpc_frames_order16"] = a
  rng = torch.Generator(device="cuda").manual_seed(2)
  b = torch.randn((1_000_000, 65), dtype=torch.float64, device="cuda", generator=rng)
  b *= torch.where(torch.rand((1_000_000, 1), device="cuda", generator=rng) < .25, .5, .02).double()
  b[:, 0] = 1.0
  out["B_random_order64"] = case(torch, ab, b, 50)
  line = json.dumps(out)
  print(line)
  if args.out:
    with open(args.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
