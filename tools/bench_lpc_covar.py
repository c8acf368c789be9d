"""Time covariance-method LPC (LpcFrames(method="kcovar"), libalz_b200_lpc.so) on the device and print one JSON line.

* A: 4096 streams x 16384 samples of noise, order 16, size 1024, hop 512, Hann window, coefficients and errors.
* B: the same, lag matrices only (LpcFrames.lag_matrix, no recursion).
* C: one stream of 2 880 000 samples (one minute at 48 kHz), order 16, size 1024, hop 512, Hann window.
* D: A at order 32.
* E: 256 streams x 16384 samples at order 64.

Each workload reports the time per call from CUDA events around back-to-back calls after a warm-up, frames/s, and
the FP64 instructions per second COUNTED FROM THE ALGORITHM (not profiled), with the share of the H100 SXM data-sheet
FP64 peak they imply (see tools/bench_lpc.py): 6 per term of a sum of single products (a lag-matrix cell, the sums of
k and gamma, whose products of zero coefficients the kernel skips), 7 per term of a sum of double products (beta,
the error), 2 per coefficient update; the divisions are not counted.  A torch-composed float64 baseline (unfold,
window, the lag matrices by one batched matmul, torch.linalg.solve_ex of the normal equations) is timed in the same
run, in chunks of streams that fit the device, with its largest deviation from the kernel's result on the frames
both solve.  The card's name, power limit and SM clock are read with nvidia-smi in the same run
(profiles/h100_lpc_covar.json).

    python tools/bench_lpc_covar.py [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)
from bench_lpc import PEAK_FP64_INSTR_PER_S, card, timed  # noqa: E402


def counted_fp64(order, size, solve):
  """FP64 instructions per frame, counted from the algorithm as the kernels run it."""
  p = order
  lagm = 6 * (p + 1) * (p + 2) // 2 * (size - p)
  if not solve:
    return lagm
  single = sum(m + sum(q + 2 for q in range(m)) for m in range(1, p + 1))        # k and gamma sums
  double = 4 + sum((m + 2) ** 2 for m in range(1, p)) + (p + 1) ** 2             # beta and the error
  updates = sum(m + m * (m + 1) // 2 for m in range(1, p + 1))
  return lagm + 6 * single + 7 * double + 2 * updates


def torch_covar(torch, x, order, size, hop, w, solve=True, chunk=256):
  """float64 frames, the lag matrices as one batched matmul and the normal equations solved, chunk streams at a
  time; returns (phi, coef, error) or phi."""
  outs = []
  p = order
  for x0 in x.split(chunk):
    fr = x0.double().unfold(-1, size, hop) * w                   # [S, F, size]
    X = fr.unfold(-1, size - p, 1).flip(-2)                      # [S, F, p + 1, size - p]: X[i][n'] = b[p + n' - i]
    phi = X @ X.transpose(-1, -2)
    if not solve:
      outs.append(phi)
      continue
    sol, _ = torch.linalg.solve_ex(phi[..., 1:, 1:], -phi[..., 1:, :1])
    c = sol[..., 0]
    e = phi[..., 0, 0] + (phi[..., 0, 1:] * c).sum(-1)
    coef = torch.cat([torch.ones_like(c[..., :1]), c], -1)
    outs.append((phi, coef, e))
  if not solve:
    return torch.cat(outs)
  return tuple(torch.cat([o[j] for o in outs]) for j in range(3))


def workload(torch, ab, x, order, size, hop, solve, reps, base_reps, chunk):
  w = np.hanning(size)
  lp = ab.LpcFrames(order, size, hop, w, method="kcovar")
  wd = torch.tensor(w, device="cuda")
  fn = (lambda: lp.apply(x)) if solve else (lambda: lp.lag_matrix(x))
  ms = timed(torch, fn, reps)
  S, T = x.shape
  F = lp.n_frames(0, T, False)
  instr = counted_fp64(order, size, solve) * S * F
  rec = {"ms": ms, "calls_timed": reps, "frames": S * F, "frames_per_s": S * F / (ms * 1e-3),
         "fp64_instr_per_call_counted": instr, "fp64_instr_per_s_counted": instr / (ms * 1e-3),
         "share_of_fp64_peak_counted": instr / (ms * 1e-3) / PEAK_FP64_INSTR_PER_S}
  base = lambda: torch_covar(torch, x, order, size, hop, wd, solve, chunk)
  bms = timed(torch, base, base_reps, warm=1)
  exact, approx = fn(), base()
  if solve:
    ok = (exact.failed == 0) & torch.isfinite(approx[1]).all(-1) & torch.isfinite(approx[2])
    dev = (approx[1] - exact.coef).abs()[ok].max().item()
    rel_err = ((approx[2] - exact.error).abs() / exact.error.abs())[ok].max().item()
    rec.update({"torch_baseline_max_abs_coef_deviation": dev, "torch_baseline_max_rel_error_deviation": rel_err,
                "frames_both_solve": int(ok.sum()), "failed_frames": int((exact.failed != 0).sum())})
  else:
    scale = exact[..., 0, 0].abs()[..., None, None]
    rec["torch_baseline_max_lagm_deviation_rel_to_phi00"] = ((approx - exact).abs() / scale).max().item()
  rec.update({"torch_baseline_ms": bms, "kernel_time_over_baseline_time": ms / bms})
  return rec


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None, help="also write the JSON record to this file")
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  if not torch.cuda.is_available():
    raise SystemExit("bench_lpc_covar needs a CUDA device")
  torch.cuda.set_device(0)
  rec = {"workload": "LpcFrames(order, size=1024, hop=512, Hann window, method='kcovar'), float32 device input",
         "card": card(), "fp64_peak_instr_per_s": PEAK_FP64_INSTR_PER_S}
  gen = torch.Generator("cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  rec["A_4096x16384_order16"] = workload(torch, ab, x, 16, 1024, 512, True, reps=10, base_reps=2, chunk=512)
  rec["B_4096x16384_order16_lag_matrix"] = workload(torch, ab, x, 16, 1024, 512, False, reps=10, base_reps=2,
                                                    chunk=512)
  rec["D_4096x16384_order32"] = workload(torch, ab, x, 32, 1024, 512, True, reps=5, base_reps=2, chunk=256)
  rec["E_256x16384_order64"] = workload(torch, ab, x[:256].contiguous(), 64, 1024, 512, True, reps=5, base_reps=2,
                                        chunk=64)
  del x
  x = torch.rand((1, 2880000), device="cuda", generator=gen) * 2 - 1
  rec["C_1x2880000_order16"] = workload(torch, ab, x, 16, 1024, 512, True, reps=20, base_reps=3, chunk=1)
  line = json.dumps(rec)
  print(line)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as fh:
      fh.write(line + "\n")


if __name__ == "__main__":
  main()
