"""Writes design_routing.json: the plan shape of every case of tests/design_space.py (design-only plans, no GPU).

Run it after a deliberate change of the plan logic, and review the diff: every changed line is a real design that now
runs on another kernel, another gain mode or another precision tier.

  python tests/golden/make_design_routing.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))


def main():
  from audiolazy_b200 import _capi
  from design_space import CASES, routing
  table = {c.id: routing(_capi.Plan(c.bank, design_only=True, **c.plan_kw)) for c in CASES if not c.id.startswith("long-")}
  with open(os.path.join(HERE, "design_routing.json"), "w") as fh:
    json.dump(table, fh, indent=0, sort_keys=True)
    fh.write("\n")
  print("%d cases" % len(table))


if __name__ == "__main__":
  main()
