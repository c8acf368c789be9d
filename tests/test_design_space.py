"""The routing of the designs the public builders produce (``tests/design_space.py``), on any machine: a design-only plan
per case against ``tests/golden/design_routing.json``, so that a plan-logic change that moves a real design onto another
kernel, gain mode or precision tier fails without a GPU; and what the precision tier promises for every bank."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from design_space import CASES, RATES, STRATEGIES, pole_radius, routing

GOLDEN_ROUTING = os.path.join(GOLDEN, "design_routing.json")
ROUTED = [c for c in CASES if not c.id.startswith("long-")]     # a long case is its base case on another shape


@pytest.fixture(scope="module")
def plans():
  from audiolazy_b200 import _capi
  return {c.id: _capi.Plan(c.bank, design_only=True, **c.plan_kw) for c in ROUTED}


@pytest.fixture(scope="module")
def golden():
  with open(GOLDEN_ROUTING) as fh:
    return json.load(fh)


def test_golden_lists_every_case(golden):
  assert sorted(golden) == sorted(c.id for c in ROUTED)


@pytest.mark.parametrize("case", ROUTED, ids=lambda c: c.id)
def test_design_routing(plans, golden, case):
  assert routing(plans[case.id]) == golden[case.id], case.id


def test_designs_are_stable():
  """Every design has its poles inside the unit circle; maverage.recursive's pole at z = 1 is cancelled by its zero."""
  for c in CASES:
    for ch in c.bank:
      r = pole_radius(ch)
      assert r < 1.0 or (c.family == "maverage" and r == 1.0), (c.id, r)


def test_poles_near_the_unit_circle_stay_on_the_float64_tier(plans):
  """A channel with a pole within 0.01 of the unit circle never runs its recurrence in float32."""
  bad = []
  for c in ROUTED:
    plan = plans[c.id]
    if plan.kind != 1:
      continue
    tier, probe = plan.tiers()
    for ch, t, e in zip(c.bank, tier, probe):
      r = pole_radius(ch)
      if t == 1 and r > 0.99:
        bad.append("%s: radius %.6f, probe %.3g" % (c.id, r, e))
  assert not bad, "\n".join(bad)


@pytest.mark.parametrize("rate", RATES)
def test_tier_follows_the_probe_in_every_gammatone_bank(plans, rate):
  """The tier of every channel is its own measurement: float32 exactly when the probe error is within the tolerance
  and no pole lies farther out than 0.99; the lowest channel of every bank with more than one channel is on float64.

  The split is not monotone in centre frequency, and this does not assert it (DESIGN.md section 3): near the boundary
  the probe error of neighbouring channels differs by a factor of 2 to 9, so float64 channels sit above float32 ones."""
  for strategy in STRATEGIES:
    for c in ROUTED:
      if c.family == "gammatone" and c.meta["rate"] == rate and c.meta["strategy"] == strategy:
        plan = plans[c.id]
        tier, probe = plan.tiers()
        radius = np.array([pole_radius(ch) for ch in c.bank])
        assert np.array_equal(tier == 1, (probe >= 0) & (probe <= plan.tier_tol) & (radius <= 0.99)), c.id
        assert len(c.bank) == 1 or tier[0] == 0, c.id
