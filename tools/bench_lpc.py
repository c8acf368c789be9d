"""Time frame-wise LPC (LpcFrames, libalz_b200_lpc.so) on the device and print one JSON line.

* A: 4096 streams x 16384 samples of noise, order 16, size 1024, hop 512, Hann window, coefficients and errors.
* B: the same, autocorrelation only (no Levinson-Durbin stage).
* C: one stream of 2 880 000 samples (one minute at 48 kHz), order 16, size 1024, hop 512, Hann window.
* D: A at order 32.

Each workload reports the time per call from CUDA events around back-to-back calls after a warm-up, frames/s, and
the FP64 instructions per second COUNTED FROM THE ALGORITHM (not profiled): 6 per acorr term (one product, the
compensated add: add, compare, two adds, add into the compensation), 7 per Levinson-Durbin term (two products),
with the share of the H100 SXM data-sheet FP64 peak they imply (34 TFLOPS = 1.7e13 FP64 instructions/s).  A
torch-composed float64 baseline (unfold, window, FFT autocorrelation, batched Levinson-Durbin loop) is timed in the
same run, with its largest deviation from the exact result.  The card's name, power limit and SM clock are read with
nvidia-smi in the same run (profiles/h100_lpc.json).

    python tools/bench_lpc.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_FP64_INSTR_PER_S = 1.7e13


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


def counted_fp64(order, size, levinson):
  """FP64 instructions per frame, counted from the algorithm (dense sums, as the kernels run them)."""
  acorr = 6 * sum(max(size - tau, 0) for tau in range(order + 1))
  if not levinson:
    return acorr
  terms = sum((m + 1) ** 2 + m * (m + 1) for m in range(1, order + 1)) + (order + 1) ** 2   # at most
  return acorr + 7 * terms


def torch_lpc(torch, x, order, size, hop, w, levinson=True):
  """float64 frames, FFT autocorrelation and a batched Levinson-Durbin recursion, all in torch operations."""
  fr = x.double().unfold(-1, size, hop) * w
  n = 1 << (2 * size - 1).bit_length()
  X = torch.fft.rfft(fr, n=n)
  r = torch.fft.irfft(X.real ** 2 + X.imag ** 2, n=n)[..., :order + 1]
  if not levinson:
    return r
  a = torch.zeros(r.shape[:-1] + (order + 1,), dtype=torch.float64, device=x.device)
  a[..., 0] = 1
  e = r[..., 0].clone()
  for m in range(1, order + 1):
    k = -(a[..., :m] * r[..., 1:m + 1].flip(-1)).sum(-1) / e
    a[..., 1:m + 1] = a[..., 1:m + 1] + k[..., None] * a[..., :m].flip(-1)
    e = e * (1 - k * k)
  return a, e


def workload(torch, ab, x, order, size, hop, levinson, reps, base_reps):
  w = np.hanning(size)
  lp = ab.LpcFrames(order, size, hop, w)
  wd = torch.tensor(w, device="cuda")
  fn = (lambda: lp.apply(x)) if levinson else (lambda: lp.acorr(x))
  ms = timed(torch, fn, reps)
  S, T = x.shape
  F = lp.n_frames(0, T, False)
  instr = counted_fp64(order, size, levinson) * S * F
  rec = {"ms": ms, "calls_timed": reps, "frames": S * F, "frames_per_s": S * F / (ms * 1e-3),
         "fp64_instr_per_call_counted": instr, "fp64_instr_per_s_counted": instr / (ms * 1e-3),
         "share_of_fp64_peak_counted": instr / (ms * 1e-3) / PEAK_FP64_INSTR_PER_S}
  base = lambda: torch_lpc(torch, x, order, size, hop, wd, levinson)
  bms = timed(torch, base, base_reps, warm=1)
  exact, approx = fn(), base()
  if levinson:
    ok = exact.failed == 0
    dev = (approx[0] - exact.coef).abs()[ok].max().item()
    rel_err = ((approx[1] - exact.error).abs() / exact.error.abs())[ok].max().item()
    rec.update({"torch_baseline_max_abs_coef_deviation": dev, "torch_baseline_max_rel_error_deviation": rel_err,
                "failed_frames": int((~ok).sum())})
  else:
    dev = ((approx - exact).abs().amax(-1) / exact[..., 0].abs()).max().item()
    rec["torch_baseline_max_acorr_deviation_rel_to_lag0"] = dev
  rec.update({"torch_baseline_ms": bms, "kernel_time_over_baseline_time": ms / bms})
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_lpc needs a CUDA device")
  torch.cuda.set_device(0)
  rec = {"workload": "LpcFrames(order, size=1024, hop=512, Hann window), float32 device input", "card": card(),
         "fp64_peak_instr_per_s": PEAK_FP64_INSTR_PER_S}
  gen = torch.Generator("cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  rec["A_4096x16384_order16"] = workload(torch, ab, x, 16, 1024, 512, True, reps=20, base_reps=3)
  rec["B_4096x16384_order16_acorr"] = workload(torch, ab, x, 16, 1024, 512, False, reps=20, base_reps=3)
  rec["D_4096x16384_order32"] = workload(torch, ab, x, 32, 1024, 512, True, reps=10, base_reps=2)
  del x
  x = torch.rand((1, 2880000), device="cuda", generator=gen) * 2 - 1
  rec["C_1x2880000_order16"] = workload(torch, ab, x, 16, 1024, 512, True, reps=50, base_reps=5)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
