"""Time the short-time Fourier kernels (Stft, libalz_b200_stft.so) on the device and print one JSON line.

Size 1024, hop 512 and a Hann window unless stated, float32 noise on the device:

* A: analysis of 4096 x 16384 samples, complex64 spectra;
* B: the same with complex128 spectra;
* C: the round trip of examples/robotize.py (analysis, ``abs`` on the spectra, synthesis with a Hann overlap-add),
  4096 x 16384, complex64;
* D: the same round trip on 1 x 2 880 000 samples (one minute at 48 kHz) at hop 441;
* E: analysis (complex64) of 1024 x 16384 at sizes 256, 4096, 8192, 1000 (2^3 5^3) and the prime 1021, hop size / 2.

Each time is the median of 5 repetitions of CUDA events around back-to-back calls after a warm-up (min and max
reported as the spread).  Bytes are computed from the shapes: the samples read, the spectra written (and, for the round
trip, read back) and the samples written; the HBM floor is those bytes at 3.35 TB/s (the H100 SXM data sheet).  FP64
instructions are COUNTED FROM THE ALGORITHM as the kernels run it (window product, twiddle products as 4 instructions,
butterfly additions, the direct DFT of a prime stage), over 1.7e13 FP64 instructions/s (34 TFLOPS).  ``bound`` names the
larger of the two floors.  Baselines timed in the same run: a torch composition (unfold, window product, roll, torch.fft
rfft / irfft, fold for the overlap-add) in float64 / complex128 and in float32 / complex64 (cuFFT).  The card's name,
power limit and SM clock are read with nvidia-smi in the same run (profiles/h100_stft.json).

    python tools/bench_stft.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
PEAK_FP64_INSTR_PER_S = 1.7e13


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


def timed(torch, fn, reps, repeats=5, warm=3):
  for _ in range(warm):
    fn()
  torch.cuda.synchronize()
  out = []
  for _ in range(repeats):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
      fn()
    e1.record()
    torch.cuda.synchronize()
    out.append(e0.elapsed_time(e1) / reps)
  return {"ms": float(np.median(out)), "ms_min": min(out), "ms_max": max(out), "calls_per_repeat": reps}


def factor(n):
  out, m = [], n
  while m % 4 == 0:
    out.append(4)
    m //= 4
  while m % 2 == 0:
    out.append(2)
    m //= 2
  p = 3
  while m > 1:
    while m % p == 0:
      out.append(p)
      m //= p
    p += 2
  return out


def fft_instr(n):
  """FP64 instructions of one transform of length n as the kernels run it."""
  total = 0
  for r in factor(n):
    if r == 2:
      total += n // 2 * (4 + 4)                   # one twiddle product, 4 additions
    elif r == 4:
      total += n // 4 * (3 * 4 + 16)              # three twiddle products, 16 additions
    elif r <= 7:
      total += n // r * ((r - 1) * 4 + r * (r - 1) * 6)   # twiddles, then the direct R-point DFT
    else:
      total += n * (r - 1) * 6                    # each output a direct R-term sum
  return total


def torch_analysis(torch, x, size, hop, w, dtype):
  fr = x.to(dtype).unfold(-1, size, hop) * w
  return torch.fft.rfft(torch.roll(fr, -(size // 2), -1), dim=-1)


def torch_round_trip(torch, x, size, hop, w, ow, dtype):
  spec = torch_analysis(torch, x, size, hop, w, dtype)
  v = torch.roll(torch.fft.irfft(spec.abs(), n=size, dim=-1), size // 2, -1) * ow
  F = v.shape[-2]
  out = torch.nn.functional.fold(v.transpose(-1, -2), (1, (F - 1) * hop + size), (1, size), stride=(1, hop))
  return out.reshape(x.shape[0], -1)


def case(torch, ab, x, size, hop, dtype, round_trip, reps, base_reps):
  S, T = x.shape
  w = ab.window.hann(size)
  st = ab.Stft(size, hop, wnd=w, ola_wnd=ab.window.hann, dtype=dtype)
  F = st.n_frames(0, T, False)
  B = size // 2 + 1
  esize = 8 if dtype == torch.complex64 else 16
  if round_trip:
    fn = lambda: st.apply(x, abs)
    nbytes = S * T * 4 + 2 * S * F * B * esize + S * F * hop * 4
  else:
    fn = lambda: st.analyze(x)
    nbytes = S * T * 4 + S * F * B * esize
  instr = S * F * (size + fft_instr(size)) * (2 if round_trip else 1)   # window or overlap-add products, transform
  rec = timed(torch, fn, reps)
  ms = rec["ms"]
  hbm_ms, fp64_ms = nbytes / HBM_BYTES_PER_S * 1e3, instr / PEAK_FP64_INSTR_PER_S * 1e3
  rec.update({"streams": S, "samples": T, "size": size, "hop": hop, "frames": S * F, "bytes_from_shapes": nbytes,
              "hbm_floor_ms": hbm_ms, "fp64_instr_counted": instr, "fp64_floor_ms": fp64_ms,
              "bound": "bytes" if hbm_ms >= fp64_ms else "fp64 issue", "share_of_floor": max(hbm_ms, fp64_ms) / ms,
              "achieved_gb_per_s": nbytes / (ms * 1e-3) / 1e9})
  for name, real in (("torch_f64_c128", torch.float64), ("torch_f32_c64", torch.float32)):
    wd = torch.tensor(w, dtype=real, device="cuda")
    owd = torch.tensor(st.ola_window, dtype=real, device="cuda")
    if round_trip:
      base = lambda: torch_round_trip(torch, x, size, hop, wd, owd, real)
    else:
      base = lambda: torch_analysis(torch, x, size, hop, wd, real)
    b = timed(torch, base, base_reps, repeats=3, warm=1)
    rec[name] = {"ms": b["ms"], "ms_min": b["ms_min"], "ms_max": b["ms_max"], "kernel_over_baseline": ms / b["ms"]}
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_stft needs a CUDA device")
  torch.cuda.set_device(0)
  rec = {"workload": "Stft(size, hop, Hann), float32 device noise", "card": card(),
         "hbm_bytes_per_s": HBM_BYTES_PER_S, "fp64_peak_instr_per_s": PEAK_FP64_INSTR_PER_S}
  gen = torch.Generator("cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  rec["A_analysis_c64"] = case(torch, ab, x, 1024, 512, torch.complex64, False, 20, 5)
  rec["B_analysis_c128"] = case(torch, ab, x, 1024, 512, torch.complex128, False, 20, 5)
  rec["C_robotize_round_trip"] = case(torch, ab, x, 1024, 512, torch.complex64, True, 10, 3)
  del x
  x = torch.rand((1, 2880000), device="cuda", generator=gen) * 2 - 1
  rec["D_1x2880000_hop441_round_trip"] = case(torch, ab, x, 1024, 441, torch.complex64, True, 20, 5)
  del x
  x = torch.rand((1024, 16384), device="cuda", generator=gen) * 2 - 1
  for size in (256, 4096, 8192, 1000, 1021):
    rec["E_analysis_size%d" % size] = case(torch, ab, x, size, size // 2, torch.complex64, False, 10, 3)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
