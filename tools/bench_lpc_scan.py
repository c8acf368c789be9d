"""Time the time-parallel LPC synthesis (LpcFilter(..., time_parallel=True); libalz_b200_lpcscan.so) against the
sequential synthesis on the device and print one JSON line.

Shapes, each excited by its own LpcFrames residual (float32 samples, rows of LpcFrames(order, 2 hop, hop) with the last
row repeated to cover every sample), float32 output:

* B: one stream of 2 880 000 samples (one minute at 48 kHz), order 16, hop 480;
* B64: B at order 64;
* B8: 8 such streams, order 16;
* C: 64 x 262 144 samples, order 16, hop 480;
* B_tone: B with a tone plus a little noise, whose rows (two resonances) remember past a chunk, so the scan's drift
  shows;
* A: 4096 x 16384 samples, order 16, hop 512 (the flagship shape), with the chunk count the model picks, and a forced
  16 chunks for comparison.

For each: the chunk count P the cost model picks; the sequential and time-parallel call times (CUDA events around
back-to-back calls, the two alternated over rounds in one run, medians reported); the device time of each pass
(torch.profiler, in a separate run): the summaries, the scan and the rerun; and the largest per-stream deviation of
the float64 time-parallel output from the float64 sequential one, relative to the stream's peak.  For B, the host
baseline: scipy.signal.lfilter per frame with carried zi.  The card's name, power limit and SM clock are read with
nvidia-smi in the same run (profiles/h100_lpc_scan.json).

    python tools/bench_lpc_scan.py [--out FILE]
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_lpc_filter import card, rows_for, scipy_synthesis_s, timed  # noqa: E402


def pass_ms(torch, fn, reps):
  """Device milliseconds per call of each of the three lpcscan kernels a call launches, in launch order."""
  from torch.autograd import DeviceType
  from torch.profiler import ProfilerActivity, profile
  fn()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      fn()
    torch.cuda.synchronize()
  evs = sorted((e for e in prof.events() if "alz_lpcscan" in e.name and e.device_type == DeviceType.CUDA),
               key=lambda e: e.time_range.start)
  # each call is walk (summaries), scan, walk (rerun): take the triples around each scan the trace kept whole
  sums = {"summaries": [], "scan": [], "rerun": []}
  for i, e in enumerate(evs):
    if "scan_kernel" in e.name and 0 < i < len(evs) - 1 and "walk" in evs[i - 1].name and "walk" in evs[i + 1].name:
      for name, ev in zip(sums, evs[i - 1:i + 2]):
        sums[name].append(ev.time_range.elapsed_us())
  if not sums["scan"]:
    return {"error": "no whole call in the trace"}
  out = {name + "_ms": round(sum(v) / len(v) / 1e3, 4) for name, v in sums.items()}
  out["calls_traced"] = len(sums["scan"])
  return out


def case(torch, ab, x, order, hop, rounds, reps, forced=None, host=False):
  S, T = x.shape
  coef = rows_for(torch, ab, x, order, 2 * hop, hop)
  e = ab.LpcFilter(order, hop, "analysis").apply(x, coef)
  tp = True if forced is None else forced
  seq = ab.LpcFilter(order, hop, "synthesis")
  par = ab.LpcFilter(order, hop, "synthesis", time_parallel=tp)
  P = par.chunks(S, T)
  out = {"S": S, "T": T, "order": order, "hop": hop, "time_parallel": tp, "P": P}
  ts, tpar = [], []
  for _ in range(rounds):
    ts.append(timed(torch, lambda: seq.apply(e, coef), reps, warm=1))
    tpar.append(timed(torch, lambda: par.apply(e, coef), reps, warm=1))
  out["sequential_ms"] = round(statistics.median(ts), 4)
  out["time_parallel_ms"] = round(statistics.median(tpar), 4)
  out["sequential_ms_all"] = [round(t, 4) for t in ts]
  out["time_parallel_ms_all"] = [round(t, 4) for t in tpar]
  out["speedup"] = round(out["sequential_ms"] / out["time_parallel_ms"], 2)
  if P > 1:
    try:
      out["passes"] = pass_ms(torch, lambda: par.apply(e, coef), max(1, reps))
    except Exception as exc:
      out["passes"] = {"error": repr(exc)}
  y64 = ab.LpcFilter(order, hop, "synthesis", torch.float64).apply(e, coef)
  t64 = ab.LpcFilter(order, hop, "synthesis", torch.float64, time_parallel=tp).apply(e, coef)
  dev = ((t64 - y64).abs().amax(dim=1) / y64.abs().amax(dim=1)).max().item()
  out["max_rel_deviation"] = dev
  out["max_abs_deviation"] = (t64 - y64).abs().max().item()
  out["within_1e-9"] = dev <= 1e-9
  del y64, t64
  if host:
    out["scipy_lfilter_per_frame_host_ms"] = round(scipy_synthesis_s(e.double().cpu().numpy(),
                                                                    coef.cpu().numpy(), hop) * 1e3, 1)
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
  xb = torch.rand((8, 2_880_000), device="cuda", generator=g) * 2 - 1
  out["B"] = case(torch, ab, xb[:1], 16, 480, 3, 1, host=True)
  n = torch.arange(2_880_000, device="cuda", dtype=torch.float64)
  tone = (torch.sin(.05 * n) + .5 * torch.sin(.31 * n + 1)).float() + xb[1:2] * 1e-3
  out["B_tone"] = case(torch, ab, tone, 16, 480, 2, 1)
  out["B64"] = case(torch, ab, xb[:1], 64, 480, 2, 1)
  out["B8"] = case(torch, ab, xb, 16, 480, 3, 1)
  xc = torch.rand((64, 262_144), device="cuda", generator=g) * 2 - 1
  out["C"] = case(torch, ab, xc, 16, 480, 3, 3)
  xa = torch.rand((4096, 16384), device="cuda", generator=g) * 2 - 1
  out["A"] = case(torch, ab, xa, 16, 512, 3, 5)
  out["A_forced_16"] = case(torch, ab, xa, 16, 512, 3, 5, forced=16)
  out["acceptance"] = all(v["P"] == 1 or v["time_parallel_ms"] < v["sequential_ms"]
                          for k, v in out.items() if isinstance(v, dict) and "P" in v and v["time_parallel"] is True)
  line = json.dumps(out)
  print(line)
  if args.out:
    with open(args.out, "w") as f:
      f.write(line + "\n")


if __name__ == "__main__":
  main()
