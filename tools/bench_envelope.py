"""Time the bank with the fused envelope consumer (envelope.abs, default cutoff pi / 512, decim 48) on the device and
print one JSON line: the 4096 x 16384 shape of bench.py's headline, and 1 / 16 streams of 10^6 samples evaluated
time-parallel (the default plan) and sequentially (a plan created with ALZ_PLAN_SEQUENTIAL).  The card's name and power
limit are part of the record (profiles/h100_envelope.json is one such line).

    python tools/bench_envelope.py
"""
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
  try:
    import pynvml
    pynvml.nvmlInit()
    h = pynvml.nvmlDeviceGetHandleByIndex(0)
    name = pynvml.nvmlDeviceGetName(h)
    return {"name": name.decode() if isinstance(name, bytes) else name,
            "power_limit_w": pynvml.nvmlDeviceGetEnforcedPowerLimit(h) / 1000.0,
            "sm_clock_max_mhz": pynvml.nvmlDeviceGetMaxClockInfo(h, pynvml.NVML_CLOCK_SM)}
  except Exception as exc:
    return {"error": repr(exc)}


def record(torch, plan, S, T, steps, warm, decim=48):
  """Median ms per alz_apply_envelope_f32_ex call over a resident [S][T] batch (L2 flushed between timed calls)."""
  C, R = plan.n_channels, 0.99388
  n_out = T // decim
  x = torch.rand((S, T), device="cuda") * 2 - 1
  env = torch.empty((S, C, n_out), dtype=torch.float32, device="cuda")
  st = torch.zeros(max(1, plan.state_doubles(S)), dtype=torch.float64, device="cuda")
  es = torch.zeros(S * C, dtype=torch.float64, device="cuda")
  flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
  cur = torch.cuda.current_stream().cuda_stream
  call = lambda: plan.apply_envelope_ex(x.data_ptr(), env.data_ptr(), st.data_ptr(), es.data_ptr(), S, T, T, n_out, decim, 0,
                                        "abs", 1.0 - R, R, cur)
  for _ in range(warm):
    call()
  times = []
  for _ in range(steps):
    flush.zero_()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    call()
    e1.record()
    torch.cuda.synchronize()
    times.append(e0.elapsed_time(e1))
  ms = statistics.median(times)
  return {"ms": ms, "min_ms": min(times), "max_ms": max(times), "steps": steps, "input_samples_per_s": S * T / (ms * 1e-3),
          "streams": S, "samples": T, "channels": C, "decim": decim}


def main():
  import torch
  import audiolazy_b200 as ab
  from audiolazy_b200 import _capi
  torch.cuda.set_device(0)
  bank = ab.gammatone_bank(strategy="slaney")
  plan = bank.device_bank().plan
  seq = _capi.Plan(bank.sections(), sequential=True)
  out = {"workload": "64-ch slaney gammatone bank + envelope.abs (cutoff pi / 512), decim 48, device buffers "
                     "(alz_apply_envelope_f32_ex)",
         "card": card(),
         "cfg4_shape": record(torch, plan, 4096, 16384, steps=15, warm=3)}
  for S in (1, 16):
    fast = record(torch, plan, S, 1000000, steps=7, warm=2)
    slow = record(torch, seq, S, 1000000, steps=3, warm=1)
    out["%dx1e6" % S] = {"time_parallel": fast, "sequential": slow, "speedup": slow["ms"] / fast["ms"]}
  print(json.dumps(out))


if __name__ == "__main__":
  main()
