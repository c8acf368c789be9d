"""resample / lagrange against the reference's goldens on the CPU: the float64 emulation of the header's arithmetic
reproduces every digest (in one block and cut into blocks), lagrange's values and polynomial coefficients equal the
reference's, the library's host schedule equals the emulation's bit for bit, and the reference's errors."""
import builtins
import json
import math
import os
import re
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import resampling
from conftest import GOLDEN
import resample_emulation as em
from lpc_emulation import digest

sys.path.insert(0, GOLDEN)
import make_resample  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "resample_cases.json")) as fh:
    doc = json.load(fh)
  assert doc["step"] == make_resample.STEP
  return doc


@pytest.fixture(scope="module")
def inputs():
  return make_resample.inputs()


def case_id(c):
  return "%s-%s/%s-o%d-z%s" % (c["input"], c["old"], c["new"], c["order"], c["zero"])


def check_case(c, values):
  """``values`` (float64) are the reference's outputs of case ``c``: count, digest and sampled values."""
  values = np.asarray(values, dtype=np.float64)
  assert len(values) == c["n_out"]
  want = np.array([make_resample.dec(v) for v in c["sampled"]], dtype=np.float64)
  assert np.array_equal(values[::make_resample.STEP], want, equal_nan=True)
  assert digest(values) == c["digest"]


def test_emulation_reproduces_every_digest(golden, inputs):
  for c in golden["cases"]:
    x = inputs[c["input"]]
    check_case(c, em.resample(x, c["old"], c["new"], c["order"], make_resample.dec(c["zero"])))


def test_emulation_in_blocks_gives_the_bits_of_one_call(golden, inputs):
  rng = np.random.default_rng(7)
  for c in golden["cases"][::5]:
    x = inputs[c["input"]]
    cuts, left = [], len(x)
    while left:
      n = int(min(left, rng.choice([0, 1, 2, c["order"], 5, 17, 64])))
      cuts.append(n)
      left -= n
    check_case(c, em.resample(x, c["old"], c["new"], c["order"], make_resample.dec(c["zero"]), blocks=cuts + [0]))


def test_lagrange_equals_the_reference(golden):
  for g in golden["lagrange"]:
    pairs = [tuple(p) for p in g["pairs"]]
    f = ab.lagrange.func(pairs)
    assert [f(k) for k in g["k"]] == g["values"]
    assert ab.lagrange(pairs)(g["k"][0]) == g["values"][0]
    assert [[k, v] for k, v in ab.lagrange.poly(pairs).terms()] == g["poly"]


def test_lagrange_errors():
  with pytest.raises(ValueError, match="not enough values to unpack"):
    ab.lagrange.func([])
  with pytest.raises(TypeError, match="reduce"):
    ab.lagrange.func([(0, 1.)])(.5)


@pytest.mark.parametrize("order", [1, 2, 3, 4, 7, 15, 64])
@pytest.mark.parametrize("old,new", [(44100, 48000), (48000, 44100), (1, 3), (50, 1), (1., .75)])
def test_library_schedule_equals_the_emulation(order, old, new):
  step = old / new
  idx = em.start_index(order)
  assert resampling.start_index(order) == idx
  for n in (0, 1, 3, 100, 1001):
    pos, idxs, nxt = resampling.schedule(order, step, idx, n)
    wpos, widxs, wnxt = em.schedule(order, step, idx, n)
    assert pos.tolist() == wpos
    assert idxs.tobytes() == np.array(widxs, dtype=np.float64).tobytes()
    assert nxt == wnxt
    idx = nxt


def test_library_schedule_refuses_what_it_cannot_walk():
  with pytest.raises(NotImplementedError, match="order"):
    resampling.schedule(65, 1., 4., 10)
  for step in (0., -1., math.inf, math.nan):
    with pytest.raises(NotImplementedError, match="finite and positive"):
      resampling.schedule(3, step, 4., 10)
  with pytest.raises(NotImplementedError, match="never advances"):
    resampling.schedule(3, 1e-20, 4., 10)


def test_reference_errors_at_the_first_value(golden, inputs):
  for e in golden["errors"]:
    kw = dict(e["kwargs"])
    s = ab.resample(inputs["noise"][:e["length"]].tolist(), **kw)     # nothing raises at call time
    exc, msg = e["exception"]
    with pytest.raises(getattr(builtins, exc), match=re.escape(msg)):
      s.take()


def test_unsupported_steps_raise_not_implemented():
  for kw in ({"old": -1}, {"old": 0}, {"old": math.nan}, {"old": math.inf}, {"old": ab.Stream(1, 2)}):
    with pytest.raises(NotImplementedError):
      ab.resample([1., 2., 3.], **kw).take()
  with pytest.raises(NotImplementedError, match="time-varying"):
    ab.Resampler(ab.Stream(1.), 1)
  with pytest.raises(NotImplementedError, match="above 64"):
    ab.Resampler(1, 2, order=65)
  with pytest.raises(ValueError):
    ab.Resampler(1, 2, order=0)


def test_vectorised_emulation_reproduces_every_digest(golden, inputs):
  for c in golden["cases"]:
    x = inputs[c["input"]][None]
    check_case(c, em.resample_batch(x, c["old"], c["new"], c["order"], make_resample.dec(c["zero"]))[0])
