"""Where the flagship bank's time goes on the GPU this runs on, in one run.

  python tools/bank_decomposition.py [--repeats 5] [--iters 20]

Prints, in this order:
  * the card: name, power limit and maximum SM clock (nvidia-smi, read in the same run);
  * the HBM ceilings of tools/microbench_hbm_write.cu (compiled here with nvcc into a temporary directory): a
    sequential fill, fills of 32 rows at a time in 128 / 256 / 512 B pieces (the bank's store pattern), copy and read;
  * tools/prof_bank.py (best of --iters launches, CUDA events) for the slaney bank at 4096 x 16384 with
    ALZ_EXP = 0 (default), 1 (no tile loads after the first group), 2 (no tile stores), 3 (neither); the first1 ...
    first4 probes (only the first n sections of each cascade); klapuri; slaney at 8192 x 8192;
  * the default case again between the others (--repeats runs in all), so that the run-to-run spread is in the output;
  * a summary: per case the best and the spread of its runs, and each ALZ_EXP case against the default.

ALZ_EXP cases compute garbage; they exist to time the kernel with one side of its traffic switched off.
"""
import argparse
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
S, T = 4096, 16384


def sh(cmd, env=None):
  run = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, env=env)
  out = run.stdout + (run.stderr if run.returncode else "")
  if run.returncode:
    raise SystemExit("command failed (%d): %s\n%s" % (run.returncode, " ".join(cmd), out[-3000:]))
  return out


def card():
  return sh(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"]).strip()


def hbm_ceilings():
  nvcc = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
  with tempfile.TemporaryDirectory() as tmp:
    exe = os.path.join(tmp, "microbench_hbm_write")
    sh([nvcc, "-O3", "-gencode", "arch=compute_90a,code=sm_90a", "-o", exe,
        os.path.join(ROOT, "tools", "microbench_hbm_write.cu")])
    return sh([exe]).rstrip()


def prof(name, s, t, iters, exp=0):
  env = dict(os.environ, ALZ_EXP=str(exp))
  line = sh([sys.executable, os.path.join(ROOT, "tools", "prof_bank.py"), name, str(s), str(t), str(iters)], env=env)
  line = line.strip().splitlines()[-1]
  return float(re.search(r"best ([0-9.]+) ms", line).group(1)), line


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--repeats", type=int, default=5, help="runs of the default case, spread between the others")
  ap.add_argument("--iters", type=int, default=20, help="launches per prof_bank run (the best one counts)")
  args = ap.parse_args()
  print("== card\n" + card(), flush=True)
  print("== HBM ceilings (tools/microbench_hbm_write.cu)\n" + hbm_ceilings(), flush=True)

  cases = [("ALZ_EXP=%d" % e, ("slaney", S, T, e)) for e in (1, 2, 3)]
  cases += [(n, (n, S, T, 0)) for n in ("first1", "first2", "first3", "first4")]
  cases += [("klapuri", ("klapuri", S, T, 0)), ("8192x8192", ("slaney", 8192, 8192, 0))]
  # the default case first, last and evenly between the others
  order = []
  every = max(1, len(cases) // max(1, args.repeats - 1))
  for k, case in enumerate(cases):
    if k % every == 0 and sum(1 for c in order if c[0] == "default") < args.repeats - 1:
      order.append(("default", ("slaney", S, T, 0)))
    order.append(case)
  while sum(1 for c in order if c[0] == "default") < args.repeats:
    order.append(("default", ("slaney", S, T, 0)))

  print("== tools/prof_bank.py, best of %d launches per run" % args.iters, flush=True)
  times = {}
  for label, (name, s, t, exp) in order:
    ms, line = prof(name, s, t, args.iters, exp)
    times.setdefault(label, []).append(ms)
    print("%-10s %s" % (label, line), flush=True)

  print("== summary (ms: best run, [min .. max] over runs)")
  base = times["default"]
  lo, hi = min(base), max(base)
  print("%-10s %8.3f  [%.3f .. %.3f]  spread %.1f %% over %d runs" % ("default", lo, lo, hi, 100 * (hi - lo) / lo, len(base)))
  for label, _ in cases:
    v = times[label]
    rel = "  %+.1f %% vs default" % (100 * (min(v) / lo - 1)) if label.startswith("ALZ_EXP") else ""
    print("%-10s %8.3f%s" % (label, min(v), rel))
  gap = lo - min(times["ALZ_EXP=1"])
  print("default - ALZ_EXP=1 = %.3f ms (%s the default's spread of %.3f ms)"
        % (gap, "beyond" if gap > hi - lo else "within", hi - lo))


if __name__ == "__main__":
  main()
