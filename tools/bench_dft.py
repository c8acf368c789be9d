"""Time the DFT kernel (Dft, libalz_b200_dft.so) on the device and print one JSON line.

Hann windows, float32 noise on the device, complex128 output unless stated; frequencies of MIDI notes at 48 kHz:

* A: 4096 x 16384 samples, size 1024, hop 512, 64 frequencies (MIDI notes 36 - 99);
* B: A with 256 frequencies (MIDI 36 - 99 in quarter tones, then above);
* C: 1 x 2 880 000 samples (one minute at 48 kHz), size 2048, hop 480, the 88 piano keys (MIDI 21 - 108);
* D: 4096 x 16384, size 256, hop 128, 32 frequencies (MIDI 60 - 91);
* E: A with complex64 output.

``kernel`` is the library's apply (the DFT kernel and the state commit) on a table already on the device, ``call``
Dft.apply end to end.  Each time is the median of 5 repetitions of CUDA events around back-to-back calls after a
warm-up (min and max reported as the spread).  FP64 instructions are COUNTED FROM THE ALGORITHM: per frame, frequency
and sample one product and one addition per part (4), plus one window product per frame and sample; their floor is
1.7e13 FP64 instructions/s.  Bytes are computed from the shapes (samples read, spectra written); the HBM floor is those
bytes at 3.35 TB/s (the H100 SXM data sheet).  ``share_of_floor`` is the larger floor over the kernel time.  Baseline
timed in the same run: torch in float64, ``unfold``, the window product and a complex128 matmul against the same
table (cuBLAS, free to use FP64 tensor cores and fused multiply-adds, so it is not bit-exact); its largest deviation
from the kernel's output is reported.  The card's name, power limit and SM clock are read with nvidia-smi in the same
run (profiles/h100_dft.json).

    python tools/bench_dft.py [--out FILE]
"""
import argparse
import json
import math
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_stft import HBM_BYTES_PER_S, PEAK_FP64_INSTR_PER_S, card, timed  # noqa: E402  (same floors and timer)


def midi(notes, rate=48000.):
  return [2 * math.pi * 440 * 2 ** ((m - 69) / 12) / rate for m in notes]


def case(torch, ab, x, size, hop, freqs, dtype, reps, base_reps):
  from audiolazy_b200 import fourier
  S, T = x.shape
  nf = len(freqs)
  w = ab.window.hann(size)
  d = ab.Dft(freqs, size, hop, w, dtype=dtype)
  F = d.n_frames(0, T, False)
  esize = 16 if dtype == torch.complex128 else 8
  tw, wd = d._tensors(x.device)
  out = torch.empty((S, F, nf), dtype=dtype, device="cuda")
  state = d.new_state(S)
  cur = torch.cuda.current_stream().cuda_stream

  def kernel():
    fourier._check(fourier.lib().alz_dft_apply_f32(
      x.data_ptr(), x.stride(0), wd.data_ptr(), tw.data_ptr(), nf, 1, out.data_ptr(), int(esize == 16), F,
      state.tensor.data_ptr(), S, T, size, hop, 0, cur))

  rec = {"streams": S, "samples": T, "size": size, "hop": hop, "n_freqs": nf, "frames": S * F,
         "dtype": str(dtype).replace("torch.", "")}
  k = timed(torch, kernel, reps)
  ms = k["ms"]
  nbytes = S * T * 4 + S * F * nf * esize
  instr = S * F * size * (4 * nf + 1)
  hbm_ms, fp64_ms = nbytes / HBM_BYTES_PER_S * 1e3, instr / PEAK_FP64_INSTR_PER_S * 1e3
  rec.update({"kernel": k, "call": timed(torch, lambda: d.apply(x), max(1, reps // 2)),
              "bytes_from_shapes": nbytes, "table_bytes": size * nf * 16, "hbm_floor_ms": hbm_ms,
              "fp64_instr_counted": instr, "fp64_floor_ms": fp64_ms,
              "bound": "bytes" if hbm_ms >= fp64_ms else "fp64 issue",
              "share_of_floor": max(hbm_ms, fp64_ms) / ms,
              "achieved_fp64_instr_per_s": instr / (ms * 1e-3)})
  w64 = torch.tensor(w, dtype=torch.float64, device="cuda")

  def base():
    fr = x.double().unfold(-1, size, hop) * w64
    return (fr.to(torch.complex128) @ tw) / size

  b = timed(torch, base, base_reps, repeats=3, warm=1)
  y = d.apply(x).to(torch.complex128)
  dev = float((base()[:, :F] - y).abs().max().item())
  rec["torch_f64_unfold_matmul"] = {"ms": b["ms"], "ms_min": b["ms_min"], "ms_max": b["ms_max"],
                                    "kernel_over_baseline": ms / b["ms"], "max_abs_deviation": dev}
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_dft needs a CUDA device")
  torch.cuda.set_device(0)
  rec = {"workload": "Dft(freqs, size, hop, Hann), float32 device noise", "card": card(),
         "hbm_bytes_per_s": HBM_BYTES_PER_S, "fp64_peak_instr_per_s": PEAK_FP64_INSTR_PER_S}
  gen = torch.Generator("cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  a_freqs = midi(range(36, 100))
  b_freqs = midi([36 + k / 2 for k in range(128)]) + midi([100 + k / 4 for k in range(128)])
  rec["A_4096x16384_size1024_hop512_f64"] = case(torch, ab, x, 1024, 512, a_freqs, torch.complex128, 10, 3)
  rec["B_4096x16384_size1024_hop512_f256"] = case(torch, ab, x, 1024, 512, b_freqs, torch.complex128, 3, 2)
  rec["D_4096x16384_size256_hop128_f32"] = case(torch, ab, x, 256, 128, midi(range(60, 92)), torch.complex128, 10, 3)
  rec["E_4096x16384_size1024_hop512_f64_c64"] = case(torch, ab, x, 1024, 512, a_freqs, torch.complex64, 10, 3)
  del x
  x = torch.rand((1, 2880000), device="cuda", generator=gen) * 2 - 1
  rec["C_1x2880000_size2048_hop480_f88"] = case(torch, ab, x, 2048, 480, midi(range(21, 109)), torch.complex128, 10,
                                                 3)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
