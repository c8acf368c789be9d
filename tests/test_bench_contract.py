"""bench.py's reference arm runs anywhere (it times the CPU port): its JSON line carries the
contract's keys.  The GPU arm prints the same keys plus roofline / clocks (profiles/h100_bench_n1.json
is a committed sample)."""
import json
import os
import subprocess
import sys

from conftest import ROOT

KEYS = {"metric", "value", "unit", "n_gpus", "steps", "warmup", "ms_per_step", "higher_is_better", "scaling",
        "vs_baseline", "dtype", "data", "config", "e2e", "cpu_baseline"}


def test_reference_arm_line():
  out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--impl", "reference", "--steps", "1",
                        "--warmup", "0"], capture_output=True, text=True, timeout=600, check=True).stdout
  line = json.loads(out.strip().splitlines()[-1])
  assert line["impl"] == "reference" and KEYS <= set(line)
  assert line["unit"] == "input-samples/s" and line["higher_is_better"] is True and line["value"] > 0
  assert line["cpu_baseline"]["kind"] == "port" and line["cpu_baseline"]["cores"] >= 1
  assert line["e2e"] == {"value": line["value"], "unit": line["unit"], "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0}
  assert "workload" in line["config"]


def test_round2_gpu_sample_has_the_contract_keys_and_the_new_records():
  line = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_n1.json")))
  assert KEYS | {"clocks", "gpu_launches", "roofline"} <= set(line)
  roof = line["roofline"]
  assert roof["bound"] == "hbm" and abs(roof["frac"] - roof["achieved"] / roof["peak"]) < 1e-9
  assert roof["sustained"]["seconds"] >= 2.0 and roof["sustained"]["frac"] <= roof["burst"]["frac"] * 1.02   # >= 2 s of back-to-back launches
  assert abs(roof["achieved"] - 260 * 4096 * 16384 / (line["ms_per_step"] * 1e-3) / 1e9) < 1e-6 * roof["achieved"]
  assert line["gpu_launches"] == line["steps"] and line["dtype"] == "f64"
  cpu = line["cpu_baseline"]
  assert cpu["kind"] == "port" and cpu["reps"] >= 5 and cpu["min"] <= cpu["value"] <= cpu["max"]
  assert cpu["cores"] <= cpu["host"]["affinity"]                      # never more threads than the process may use
  for key in ("strategies", "cfg2", "cfg3", "cfg5", "few_streams", "generic", "stream_api"):
    assert key in line and "error" not in line[key], key
  assert set(line["strategies"]) == {"klapuri", "sampled"}
  assert line["stream_api"]["cfg1"]["ours_samples_per_s"] > line["stream_api"]["cfg1"]["python_port_samples_per_s"]
  assert line["e2e"]["h2d_bytes_per_step"] == 4096 * 16384 * 4 and line["e2e"]["d2h_bytes_per_step"] == 4096 * 64 * 16384 * 4


def test_committed_gpu_sample_has_the_contract_keys():
  line = json.load(open(os.path.join(ROOT, "profiles", "h100_bench_n1.json")))
  assert KEYS | {"clocks", "gpu_launches", "roofline"} <= set(line)
  roof = line["roofline"]
  assert roof["bound"] == "hbm" and abs(roof["frac"] - roof["achieved"] / roof["peak"]) < 1e-9
  assert line["gpu_launches"] == line["steps"] and line["dtype"] == "f64"
  assert line["e2e"]["h2d_bytes_per_step"] == 4096 * 16384 * 4 and line["e2e"]["d2h_bytes_per_step"] == 4096 * 64 * 16384 * 4
