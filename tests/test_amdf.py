"""amdf without a GPU: the float64 emulation against the reference's answers (tests/golden/amdf_cases.json, made by
tests/golden/make_amdf.py from a reference checkout), the product's tap tables, input validation, freq2lag / lag2freq
and the AMDF library's exported symbols."""
import builtins
import json
import math
import os

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import analysis as amdf_mod
from amdf_emulation import amdf as emulate, digest
from conftest import GOLDEN


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "amdf_cases.json")) as fh:
    return json.load(fh)


def signal(seed, n):
  return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32)


def test_emulation_reproduces_every_reference_digest(golden):
  assert len(golden["cases"]) >= 15
  for case in golden["cases"]:
    x = signal(case["seed"], case["length"])
    y = emulate(x, [tuple(t) for t in case["taps"]], case["size"], case["zero"])
    assert digest(y) == case["digest"], case
    assert y[::case["step"]].tolist() == case["values"]


def test_tap_tables_match_the_reference(golden):
  for case in golden["cases"]:
    assert amdf_mod.lag_taps(case["lag"]) == [(k, v) for k, v in case["taps"]], case["lag"]


def test_golden_covers_the_edges(golden):
  cases = golden["cases"]
  assert any(c["lag"] == 0 for c in cases) and any(0 < c["lag"] < 1 for c in cases)
  assert any(c["lag"] != int(c["lag"]) and c["lag"] > 1 for c in cases)
  assert any(c["lag"] > c["length"] for c in cases) and any(c["size"] > c["length"] for c in cases)
  assert {1, 1024} <= {c["size"] for c in cases}
  assert {0., .25, -.3} <= {c["zero"] for c in cases}


def test_errors_are_the_references(golden):
  """The reference raises these from the call or from the first value; this package always raises from the call."""
  for err in golden["errors"]:
    filt = ab.amdf(err["lag"], err["size"])              # building the callable never raises, as in the reference
    with pytest.raises(getattr(builtins, err["error"])) as info:
      filt([1., 2., 3.])
    if err["raised_at"] == "call":
      assert str(info.value) == err["message"]


def test_bank_validation():
  with pytest.raises(ZeroDivisionError):
    ab.AmdfBank([3], 0)
  with pytest.raises(ValueError, match="Non-causal"):
    ab.AmdfBank([4, -2], 8)
  with pytest.raises(TypeError):
    ab.AmdfBank([3], 2.0)
  with pytest.raises(ValueError):
    ab.AmdfBank([3], -1)
  with pytest.raises(ValueError):
    ab.AmdfBank([], 4)
  bank = ab.AmdfBank(np.arange(48, 52), np.int64(16))
  assert len(bank) == 4 and bank.size == 16
  assert all(t == [(0, 1.0), (k, -1.0)] for t, k in zip(bank.taps, range(48, 52)))


def test_freq2lag_lag2freq():
  assert ab.freq2lag(math.pi / 4) == 8.0
  assert ab.lag2freq(8) == math.pi / 4
  s, Hz = ab.sHz(48000)
  assert abs(ab.freq2lag(1000 * Hz) - 48.0) < 1e-12
  assert ab.freq2lag(2 * math.pi / 37.25) == 2 * math.pi / (2 * math.pi / 37.25)
