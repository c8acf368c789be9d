"""Compare builds of the filter library on the bank kernel, alternating them within one run.

  python tools/bank_ab.py --lib parent=/path/a/libalz_b200.so --lib branch=/path/b/libalz_b200.so \
      [--case "slaney 4096 16384"] [--case "slaney 4096 16384 ALZ_EXP=1"] [--rounds 3] [--iters 20]

Every round runs every case on every library (ALZ_B200_LIB), through tools/prof_bank.py (best of --iters launches,
CUDA events), in a rotated library order, so that drift of the card's clock or of other work on the machine is shared
by all builds.  A case is "<bank> <streams> <samples> [VAR=VALUE ...]", the variables set for that run only.  The
summary gives per case and library the best run and the range over rounds.
"""
import argparse
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--lib", action="append", required=True, metavar="LABEL=PATH")
  ap.add_argument("--case", action="append", metavar='"BANK S T [VAR=VALUE ...]"')
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--iters", type=int, default=20)
  args = ap.parse_args()
  libs = [tuple(s.split("=", 1)) for s in args.lib]
  cases = args.case or ["slaney 4096 16384"]
  print(subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                       capture_output=True, text=True).stdout.strip(), flush=True)
  times = {}
  for r in range(args.rounds):
    for case in cases:
      words = case.split()
      env = dict(os.environ, **dict(w.split("=", 1) for w in words[3:]))
      for k in range(len(libs)):
        label, path = libs[(k + r) % len(libs)]
        env["ALZ_B200_LIB"] = os.path.abspath(path)
        run = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "prof_bank.py")] + words[:3] + [str(args.iters)],
                             capture_output=True, text=True, cwd=ROOT, env=env)
        if run.returncode:
          raise SystemExit("%s / %s failed:\n%s" % (label, case, (run.stdout + run.stderr)[-3000:]))
        line = run.stdout.strip().splitlines()[-1]
        ms = float(re.search(r"best ([0-9.]+) ms", line).group(1))
        times.setdefault((case, label), []).append(ms)
        print("round %d  %-10s %-36s %8.3f ms" % (r, label, case, ms), flush=True)
  print("== summary: best [min .. max] over %d rounds, ms" % args.rounds)
  for case in cases:
    first = min(times[(case, libs[0][0])])
    for label, _ in libs:
      v = times[(case, label)]
      print("%-36s %-10s %8.3f [%.3f .. %.3f]  %+.1f %% vs %s"
            % (case, label, min(v), min(v), max(v), 100 * (min(v) / first - 1), libs[0][0]))


if __name__ == "__main__":
  main()
