"""unwrap and clip without a GPU: the emulation of include/alz_b200_unwrap.h against the reference's answers
(tests/golden/unwrap_cases.json, made by tests/golden/make_unwrap.py from a reference checkout), the vectorised
emulation against the plain one, and argument errors."""
import json
import math
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import unwrapping
from conftest import GOLDEN
import unwrap_emulation as em

sys.path.insert(0, GOLDEN)
import make_unwrap  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "unwrap_cases.json")) as fh:
    doc = json.load(fh)
  assert doc["step"] == make_unwrap.STEP
  return doc


def params(c):
  return eval(c["params"], make_unwrap.env())


def same_bits(got, want):
  got, want = make_unwrap.canon(got), make_unwrap.canon(want)
  return got.tobytes() == want.tobytes()


def check_case(c, values):
  """``values`` are the reference's for case ``c``: its length, sampled values and digest, bit for bit."""
  values = list(values)
  assert len(values) == c["n"], (c["input"], c["params"])
  assert same_bits(values[::make_unwrap.STEP], c["values"]), (c["input"], c["params"])
  if values:
    assert make_unwrap.digest(values) == c["digest"], (c["input"], c["params"])


def test_emulation_reproduces_every_golden(golden):
  xs = make_unwrap.inputs()
  assert len(golden["cases"]) == len(xs) * len(make_unwrap.PARAMS)
  for c in golden["cases"]:
    x = xs[c["input"]]
    out, fail = em.unwrap(x.tolist(), *params(c))
    exc = c.get("exception")
    if exc == ["RuntimeError", "generator raised StopIteration"]:
      assert len(x) == 0 and out == []
    elif exc == ["ZeroDivisionError", "float modulo"]:
      assert fail == c["n"], (c["input"], c["params"])
      check_case(c, out[:fail])
    else:
      assert exc is None and fail == -1
      check_case(c, out)


def test_emulation_reproduces_every_clip_golden(golden):
  xs = make_unwrap.inputs()
  for c in golden["clips"]:
    low, high = params(c)
    if "exception" in c:
      assert c["exception"][0] == "ValueError" and c["raised_at"] == "call" and high < low
      continue
    check_case(c, em.clip(xs[c["input"]], low, high))


def test_golden_covers_the_edges(golden):
  cases = golden["cases"]
  assert {c["exception"][0] for c in cases if "exception" in c} == {"ZeroDivisionError", "RuntimeError"}
  zero = [c for c in cases if c.get("exception", [None])[0] == "ZeroDivisionError"]
  assert {c["params"] for c in zero} == {"(pi, 0)", "(pi, 0.)", "(pi, -0.)"} and min(c["n"] for c in zero) >= 1
  assert any(c["n"] > 4096 for c in zero)                 # the failure lies beyond the first tiles
  xs = make_unwrap.inputs()
  M, P = math.pi, 2 * math.pi
  jumps = {name: int(np.sum(np.abs(np.diff(xs[name])) > M)) for name in ("long_never", "long_sometimes", "long_always")}
  assert jumps["long_never"] == 0 and 0 < jumps["long_sometimes"] < 9000 // 10 and jumps["long_always"] > 8000
  d = np.diff(xs["ties"])
  assert any(abs(em.py_rem(v, 10.)) == abs(em.py_rem(v, -10.)) for v in d)
  assert (xs["not_float32"] != xs["not_float32"].astype(np.float32)).all()
  assert {c["params"] for c in golden["clips"] if "exception" in c} == {"(2., 1.)", "(4, 3.9)"}


def test_the_issue_examples():
  assert em.unwrap([0., math.pi], .5, 2 * math.pi)[0] == [0.0, math.pi]
  got = em.unwrap([0., math.nan, 1., 10.], math.pi, 2 * math.pi)[0]
  assert math.isnan(got[1]) and got[::2] == [0.0, 1.0] and got[3] == 3.7168146928204138
  got = em.unwrap([0., math.inf, 1., 2.], math.pi, 2 * math.pi)[0]
  assert got[0] == 0.0 and all(math.isnan(v) for v in got[1:])
  got = em.unwrap([-0., -0.], math.pi, 2 * math.pi)[0]
  assert math.copysign(1, got[0]) == -1 and math.copysign(1, got[1]) == 1
  assert em.unwrap([0., 7.], math.pi, math.inf)[0] == [0., 7.]
  assert em.unwrap([0., 1., 5., 9.], 2., 0.)[1] == 2
  assert repr(em.clip([-2., math.nan, -0.], -0., 1.).tolist()) == "[-0.0, nan, -0.0]"


def test_vectorised_emulation_equals_the_emulation(golden):
  xs = make_unwrap.inputs()
  for c in golden["cases"]:
    x = xs[c["input"]]
    want, fail = em.unwrap(x.tolist(), *params(c))
    got, gfail = em.unwrap_batch(x, *params(c))
    assert same_bits(got[0], want) and gfail[0] == fail, (c["input"], c["params"])


def test_library_sizes_without_a_device():
  L = unwrapping.lib()
  assert L.alz_unwrap_state_bytes(3) == 96
  assert L.alz_unwrap_state_bytes(-1) < 0
  assert L.alz_unwrap_scratch_bytes(0, 0) == 16
  assert L.alz_unwrap_scratch_bytes(1, 2048 * 5) == 16 + 5 * 12 + 4      # five tiles of one row, rounded to 8 bytes
  assert L.alz_unwrap_scratch_bytes(64 * 3 + 1, 32) == 16 + 4 * 12 + 0   # 64 rows of 32 samples per tile
  assert L.alz_unwrap_scratch_bytes(1, -1) < 0


def test_c_abi_argument_errors():
  L = unwrapping.lib()
  F32, F64 = unwrapping.FLOAT32, unwrapping.FLOAT64

  def last():
    return L.alz_unwrap_last_error().decode()

  assert L.alz_unwrap_apply(None, F32, 1, None, F64, 1, None, -1, 1, 1., 1., None, 0, None) < 0 and "shape" in last()
  assert L.alz_unwrap_apply(None, 2, 1, None, F64, 1, None, 1, 1, 1., 1., None, 0, None) < 0 and "dtype" in last()
  assert L.alz_unwrap_apply(None, F32, 1, None, F64, 1, None, 1, 1, 1., 1., None, 0, None) < 0 and "NULL" in last()
  assert L.alz_unwrap_apply(8, F32, 1, 16, F64, 1, 32, 2, 4, 1., 1., 64, 1 << 20, None) < 0 and "stride" in last()
  assert L.alz_unwrap_apply(8, F32, 4, 12, F64, 4, 32, 2, 4, 1., 1., 64, 1 << 20, None) < 0 and "misaligned" in last()
  assert L.alz_unwrap_apply(8, F32, 4, 16, F64, 4, 32, 2, 4, 1., 1., 64, 8, None) < 0 and "scratch" in last()
  assert L.alz_unwrap_apply(None, F32, 1, None, F64, 1, None, 0, 5, 1., 1., None, 0, None) == 0   # nothing to do
  assert L.alz_unwrap_state_init(None, 2, None) < 0 and "NULL" in last()
  assert L.alz_unwrap_state_init(None, 0, None) == 0
  assert L.alz_clip_apply(8, F32, 4, 16, F64, 4, 2, 4, 2., 1, 1., 1, None) < 0 and "smaller" in last()
  assert L.alz_clip_apply(8, F32, 4, 16, 7, 4, 2, 4, 0., 1, 1., 1, None) < 0 and "dtype" in last()
  assert L.alz_clip_apply(None, F32, 4, None, F32, 4, 0, 4, 2., 1, 1., 1, None) < 0   # high < low is checked first
  assert L.alz_clip_apply(None, F32, 4, None, F32, 4, 0, 4, 0., 0, 0., 0, None) == 0


def test_python_argument_errors(golden):
  """The reference raises TypeError for a non-real parameter at the first jump; this package raises it at the call."""
  for err in golden["errors"]:
    assert err["exception"][0] == "TypeError" and err["raised_at"] == "iteration" and err["n"] == 1
    m, p = eval(err["params"], make_unwrap.env())
    with pytest.raises(TypeError):
      ab.unwrap([0., 10.], max_delta=m, step=p)
    with pytest.raises(TypeError):
      ab.Unwrap(m, p)
  with pytest.raises(ValueError, match="smaller than lower"):
    ab.clip([], low=4, high=3.9)
  with pytest.raises(ValueError, match="smaller than lower"):
    ab.Clip(1., -1.)
  with pytest.raises(TypeError):
    ab.clip([1.], low="a")
  with pytest.raises(TypeError):
    ab.Clip(None, 1j)
  assert list(ab.clip([1, "a", None], None, None)) == [1, "a", None]    # both limits None: the input Stream itself
  uw = ab.Unwrap(np.float32(.5), np.int64(3))
  assert (uw.max_delta, uw.step) == (.5, 3.)
  c = ab.Clip(-0., None)
  assert math.copysign(1, c.low) == -1 and c.high is None
