"""Time the LPC filter kernels (LpcFilter; libalz_b200_lpcfilt.so) on the device and print one JSON line.

* A: 4096 x 16384 float32 samples, order 16, hop 512, the rows of LpcFrames(16, 1024, 512) of the same samples with the
  last row repeated to cover every sample (32 rows per stream); float32 output.  Analysis, and synthesis of A's
  residual.
* B: one stream of 2 880 000 samples, order 16, hop 480 (rows of LpcFrames(16, 960, 480)).
* C: A at order 64 (rows of LpcFrames(64, 1024, 512)).
* D: A with hop 1: 16384 rows per stream (A's rows, each repeated 512 times), so the coefficient traffic dominates.

For each: the call (a new state, the output and the launches, CUDA events around back-to-back calls) and the kernel
time (the device time of the alz_lpcfilt kernels in torch.profiler, per call).  Analysis floors, counted from the
shapes: the bytes a call must move (samples in and out, the rows once) at the H100 SXM data-sheet HBM3 bandwidth
(3.35 TB/s), and its 2 x order FP64 operations per sample at 1.7e13 FP64 operations/s.  Synthesis is set against the
chain estimate: T samples of order dependent additions at 4 ns each (an estimate, not a measurement).

Baselines, same run: the analysis as a torch float64 composition (unfold plus row-expanded coefficients, in stream
chunks), not bit-exact (its largest deviation is reported); the synthesis as scipy.signal.lfilter per frame with
carried zi on the host, on 8 streams of A (scaled to 4096) and on B.  The card's name, power limit and SM clock are
read with nvidia-smi in the same run (profiles/h100_lpc_filter.json).

    python tools/bench_lpc_filter.py [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PEAK_BYTES_PER_S = 3.35e12
PEAK_FP64_PER_S = 1.7e13
CHAIN_ADD_S = 4e-9


def card():
  try:
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True, timeout=30).stdout.splitlines()[0]
    name, power, clock = [v.strip() for v in out.split(",")]
    return {"name": name, "power_limit": power, "sm_clock_max": clock}
  except Exception as exc:
    return {"error": repr(exc)}


def timed(torch, fn, reps, warm=2):
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


def kernel_ms(torch, fn, reps):
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
  us = 0.0
  for e in prof.key_averages():
    if "alz_lpcfilt" in e.key:
      us += getattr(e, "device_time_total", None) or getattr(e, "cuda_time_total", 0.0)
  return us / reps / 1e3


def rows_for(torch, ab, x, order, size, hop):
  """LpcFrames(order, size, hop) rows of x, the last repeated so that they cover every sample at `hop`."""
  coef = ab.LpcFrames(order, size, hop).apply(x).coef
  F = ab.LpcFilter(order, hop).n_rows(0, x.shape[1])
  return torch.cat([coef, coef[:, -1:].expand(-1, F - coef.shape[1], -1)], dim=1).contiguous()


def torch_analysis(torch, x, coef, hop, chunk=256):
  """Residual from torch float64 ops: unfold the padded samples, multiply by each sample's row, sum the taps."""
  S, T = x.shape
  order = coef.shape[2] - 1
  rows = torch.arange(T, device=x.device) // hop
  out = torch.empty((S, T), dtype=torch.float64, device=x.device)
  for s0 in range(0, S, chunk):
    xs = torch.nn.functional.pad(x[s0:s0 + chunk].double(), (order, 0))
    frames = xs.unfold(1, order + 1, 1).flip(-1)               # [s, T, order + 1]: x[n], x[n - 1], ...
    out[s0:s0 + chunk] = (frames * coef[s0:s0 + chunk][:, rows]).sum(-1)
  return out


def scipy_synthesis_s(x, coef, hop):
  """Seconds of scipy.signal.lfilter([1], row, frame, zi=zi) per frame with carried zi, on the host."""
  import numpy as np
  from scipy.signal import lfilter
  x = np.asarray(x, np.float64)
  coef = np.asarray(coef, np.float64)
  t0 = time.perf_counter()
  for s in range(x.shape[0]):
    zi = np.zeros(coef.shape[2] - 1)
    for r in range(coef.shape[1]):
      seg = x[s, r * hop:(r + 1) * hop]
      if not len(seg):
        break
      _, zi = lfilter([1.0], coef[s, r], seg, zi=zi)
  return time.perf_counter() - t0


def analysis_case(torch, ab, x, coef, hop, reps, baseline=True):
  S, T = x.shape
  order = coef.shape[2] - 1
  f = ab.LpcFilter(order, hop, "analysis")
  call = timed(torch, lambda: f.apply(x, coef), reps)
  kern = kernel_ms(torch, lambda: f.apply(x, coef), reps)
  nbytes = S * T * (4 + 4) + coef.numel() * 8
  hbm = nbytes / PEAK_BYTES_PER_S * 1e3
  fp64 = S * T * 2 * order / PEAK_FP64_PER_S * 1e3
  floor = max(hbm, fp64)
  out = {"S": S, "T": T, "order": order, "hop": hop, "call_ms": round(call, 4), "kernel_ms": round(kern, 4),
         "bytes": nbytes, "hbm_floor_ms": round(hbm, 4), "fp64_floor_ms": round(fp64, 4),
         "share_of_floor_kernel": round(floor / kern, 3) if kern else None,
         "share_of_floor_call": round(floor / call, 3)}
  if baseline:
    fd = ab.LpcFilter(order, hop, "analysis", torch.float64)
    out["torch_float64_ms"] = round(timed(torch, lambda: torch_analysis(torch, x, coef, hop), 3, warm=1), 3)
    ours = fd.apply(x, coef)
    base = torch_analysis(torch, x, coef, hop)
    out["torch_max_abs_deviation"] = (ours - base).abs().max().item()
    del ours, base
  return out


def synthesis_case(torch, ab, e, coef, hop, reps, host_streams):
  S, T = e.shape
  order = coef.shape[2] - 1
  f = ab.LpcFilter(order, hop, "synthesis")
  call = timed(torch, lambda: f.apply(e, coef), reps, warm=1)
  kern = kernel_ms(torch, lambda: f.apply(e, coef), max(1, reps // 2))
  est = T * order * CHAIN_ADD_S * 1e3
  out = {"S": S, "T": T, "order": order, "hop": hop, "call_ms": round(call, 4), "kernel_ms": round(kern, 4),
         "chain_estimate_ms": round(est, 3), "chain_estimate_is_an_estimate": True,
         "ns_per_dependent_add": round(kern * 1e6 / (T * order), 3) if order else None}
  n = min(S, host_streams)
  host = scipy_synthesis_s(e[:n].double().cpu().numpy(), coef[:n].cpu().numpy(), hop)
  out["scipy_lfilter_per_frame_host_ms"] = round(host * 1e3 * S / n, 1)
  out["scipy_streams_timed"] = n
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--out", default=None)
  args = ap.parse_args()
  import torch
  import audiolazy_b200 as ab
  torch.cuda.set_device(0)
  out = {"card": card(), "torch": torch.__version__}
  g = torch.Generator(device="cuda").manual_seed(1)
  x = torch.rand((4096, 16384), device="cuda", generator=g) * 2 - 1

  coef = rows_for(torch, ab, x, 16, 1024, 512)
  out["A_analysis"] = analysis_case(torch, ab, x, coef, 512, 50)
  res = ab.LpcFilter(16, 512, "analysis").apply(x, coef)
  out["A_synthesis"] = synthesis_case(torch, ab, res, coef, 512, 10, 8)

  xb = torch.rand((1, 2_880_000), device="cuda", generator=g) * 2 - 1
  cb = rows_for(torch, ab, xb, 16, 960, 480)
  out["B_analysis"] = analysis_case(torch, ab, xb, cb, 480, 50)
  rb = ab.LpcFilter(16, 480, "analysis").apply(xb, cb)
  out["B_synthesis"] = synthesis_case(torch, ab, rb, cb, 480, 2, 1)

  cc = rows_for(torch, ab, x, 64, 1024, 512)
  out["C_analysis"] = analysis_case(torch, ab, x, cc, 512, 20)
  rc = ab.LpcFilter(64, 512, "analysis").apply(x, cc)
  out["C_synthesis"] = synthesis_case(torch, ab, rc, cc, 512, 3, 4)
  del cc, rc

  cd = coef.repeat_interleave(512, dim=1)[:, :16384].contiguous()   # hop 1: 16384 rows of 17 per stream, 9.1 GB
  out["D_analysis"] = analysis_case(torch, ab, x, cd, 1, 10, baseline=False)
  rd = ab.LpcFilter(16, 1, "analysis").apply(x, cd)
  out["D_synthesis"] = synthesis_case(torch, ab, rd, cd, 1, 3, 1)
  line = json.dumps(out)
  print(line)
  if args.out:
    with open(args.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
