"""Time the Lagrange resampler (Resampler, libalz_b200_resample.so) on the device and print one JSON line.

Float32 noise on the device, order 3 unless stated:

* A: 4096 x 16384 samples, 44100 -> 48000;
* B: the same, 48000 -> 16000;
* C: 1 x 2 880 000 samples (one minute at 48 kHz), 48000 -> 44100;
* D: A at order 15;
* E: A streamed in blocks of 1024 samples (16 calls continuing one state).

Three times per case: ``kernel`` (the library's apply, its three kernels, on schedule tables already on the device),
``schedule`` (the host walk of the schedule, a perf_counter median) and ``call`` (Resampler.apply end to end: schedule,
table upload, kernels, float32 output).  Each device time is the median of 5 repetitions of CUDA events around
back-to-back calls after a warm-up (min and max reported as the spread).  Bytes are computed from the shapes: the
samples read and the float32 outputs written (the tables, shared by every stream, are listed apart); the HBM floor is
those bytes at 3.35 TB/s (the H100 SXM data sheet).  FP64 instructions are COUNTED FROM THE ALGORITHM: per output and
stream one product and four additions per tap of the compensated sum plus the final one; per output, once, the
(order + 1) order quotients and products of the weights, a division counted as 8 instructions.  Their floor is
1.7e13 FP64 instructions/s.  Baseline timed in the same run: torch in float64, a gather of the same schedule's windows,
a product with the same weights and ``sum``; its largest deviation from the kernel's float64 output is reported (it is
not bit-exact: torch's sum is not compensated).  The card's name, power limit and SM clock are read with nvidia-smi in
the same run (profiles/h100_resample.json).

    python tools/bench_resample.py [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bench_stft import HBM_BYTES_PER_S, PEAK_FP64_INSTR_PER_S, card, timed  # noqa: E402  (same floors and timer)

DIV_INSTR = 8


def host_timed(fn, repeats=5):
  fn()
  out = []
  for _ in range(repeats):
    t0 = time.perf_counter()
    fn()
    out.append((time.perf_counter() - t0) * 1e3)
  return {"ms": float(np.median(out)), "ms_min": min(out), "ms_max": max(out)}


def case(torch, ab, x, old, new, order, reps, block=None):
  from audiolazy_b200 import resampling
  S, T = x.shape
  L = order + 1
  r = ab.Resampler(old, new, order)
  idx0 = resampling.start_index(order)
  pos, idxs, _ = r.schedule(idx0, T)
  n = len(pos)
  rec = {"streams": S, "samples": T, "old": old, "new": new, "order": order, "outputs_per_stream": n}
  nbytes = S * T * 4 + S * n * 4
  instr = S * n * (5 * L + 1) + n * L * (L - 1) * (2 + DIV_INSTR)
  if block is None:
    out = torch.empty((S, n), dtype=torch.float32, device="cuda")
    state = r.new_state(S)
    w = torch.empty((n, L), dtype=torch.float64, device="cuda")
    pos_d, idx_d = torch.from_numpy(pos).cuda(), torch.from_numpy(idxs).cuda()
    cur = torch.cuda.current_stream().cuda_stream

    def kernel():
      resampling._check(resampling.lib().alz_resample_apply(
        x.data_ptr(), out.data_ptr(), 0, state.tensor.data_ptr(), pos_d.data_ptr(), idx_d.data_ptr(), w.data_ptr(), n,
        S, T, x.stride(0), n, order, cur))

    k = timed(torch, kernel, reps)
    rec["kernel"] = k
    rec["schedule_host"] = host_timed(lambda: r.schedule(idx0, T))
    rec["call"] = timed(torch, lambda: r.apply(x), reps)
    ms = k["ms"]
    hbm_ms, fp64_ms = nbytes / HBM_BYTES_PER_S * 1e3, instr / PEAK_FP64_INSTR_PER_S * 1e3
    rec.update({"bytes_from_shapes": nbytes, "table_bytes": n * (8 + 8 + 2 * 8 * L), "hbm_floor_ms": hbm_ms,
                "fp64_instr_counted": instr, "fp64_floor_ms": fp64_ms,
                "bound": "bytes" if hbm_ms >= fp64_ms else "fp64 issue",
                "kernel_share_of_hbm_floor": hbm_ms / ms, "kernel_share_of_fp64_floor": fp64_ms / ms,
                "achieved_gb_per_s": nbytes / (ms * 1e-3) / 1e9})
    # torch float64 baseline: same schedule and weights
    wt = torch.empty((n, L), dtype=torch.float64, device="cuda")
    resampling._check(resampling.lib().alz_resample_apply(
      x.data_ptr(), out.data_ptr(), 0, r.new_state(S).tensor.data_ptr(), pos_d.data_ptr(), idx_d.data_ptr(),
      wt.data_ptr(), n, S, T, x.stride(0), n, order, cur))
    gather = pos_d[:, None] + torch.arange(L, device="cuda")[None, :]

    def base():
      data = torch.cat([torch.zeros((S, L), dtype=torch.float64, device="cuda"), x.double()], dim=1)
      return (data[:, gather] * wt).sum(-1)

    b = timed(torch, base, max(1, reps // 4), repeats=3, warm=1)
    ref64 = r.apply(x, dtype=torch.float64)
    dev = float((base() - ref64).abs().max().item())
    del ref64
    rec["torch_f64_gather"] = {"ms": b["ms"], "ms_min": b["ms_min"], "ms_max": b["ms_max"],
                               "kernel_over_baseline": ms / b["ms"], "max_abs_deviation": dev}
  else:
    def streamed():
      state = r.new_state(S)
      for i in range(0, T, block):
        r.apply(x[:, i:i + block], state=state)

    c = timed(torch, streamed, max(1, reps // 2))
    sched = host_timed(lambda: [r.schedule(idx0 + 0., block) for _ in range(0, T, block)])
    rec.update({"block": block, "calls": -(-T // block), "call_total": c, "schedule_host_total": sched,
                "bytes_from_shapes": nbytes, "hbm_floor_ms": nbytes / HBM_BYTES_PER_S * 1e3,
                "share_of_hbm_floor": nbytes / HBM_BYTES_PER_S * 1e3 / c["ms"]})
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_resample needs a CUDA device")
  torch.cuda.set_device(0)
  rec = {"workload": "Resampler(old, new, order), float32 device noise", "card": card(),
         "hbm_bytes_per_s": HBM_BYTES_PER_S, "fp64_peak_instr_per_s": PEAK_FP64_INSTR_PER_S}
  gen = torch.Generator("cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  rec["A_4096x16384_44100_48000_o3"] = case(torch, ab, x, 44100, 48000, 3, 20)
  rec["B_4096x16384_48000_16000_o3"] = case(torch, ab, x, 48000, 16000, 3, 20)
  rec["D_4096x16384_44100_48000_o15"] = case(torch, ab, x, 44100, 48000, 15, 10)
  rec["E_4096x16384_44100_48000_o3_blocks1024"] = case(torch, ab, x, 44100, 48000, 3, 10, block=1024)
  del x
  x = torch.rand((1, 2880000), device="cuda", generator=gen) * 2 - 1
  rec["C_1x2880000_48000_44100_o3"] = case(torch, ab, x, 48000, 44100, 3, 20)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
