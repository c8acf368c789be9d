"""Time-varying coefficients (Stream-valued b_k / a_k, reference ``LinearFilter.__call__``) without a GPU.

* Every case of ``tests/golden/tv_cases.json`` (the reference's own outputs, ``tests/golden/make_tv.py``) through the
  lazy API with the native layer replaced by ``tests/fake_native.py``, at 1e-7 of the row peak.  The same check runs on
  the device in ``tests/test_time_varying_gpu.py``.
* ``oracle.tv_apply``, the float64 statement of the ``alz_apply_tv_f32`` contract, pinned to those goldens through the
  coefficient tables the host layer builds, and to ``FakePlan.apply_tv`` bit for bit.
* A coefficient Stream that ends before the input: the values before it, then ``RuntimeError``, as in the reference.
"""
import json
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
import fake_native
import oracle
from conftest import GOLDEN

sys.path.insert(0, GOLDEN)
import make_tv  # noqa: E402  (the case designs; only data comes from the reference)

#: float32 output against the float64 reference: 2^-24 of each value, and the kernel's own float64 rounding
TOL = 1e-7

with open(os.path.join(GOLDEN, "tv_cases.json")) as _fh:
  CASES = {c["name"]: c for c in json.load(_fh)["cases"]}


def peak_err(got, want):
  """max |got - want| / max |want| (0 for two empty rows)."""
  got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
  if want.size == 0:
    return 0.0
  return float(np.max(np.abs(got - want)) / max(np.max(np.abs(want)), 1e-300))


def run_case(lib, case):
  """The case through ``lib``'s lazy API: ``(values yielded, exception type name or None)``."""
  filt = make_tv.design(lib, case["design"])
  return make_tv.run(filt, make_tv.signal(case["seed"], case["length"]), case["input"], case["kwargs"])


def stored(case, values):
  """``values`` (a whole output) at the samples the case stores (``make_tv.kept``)."""
  return np.asarray(values, dtype=np.float64)[make_tv.kept(case["n"])]


def check_golden_case(lib, case):
  got, raised = run_case(lib, case)
  assert raised == case["raises"], (case["name"], raised)
  assert len(got) == case["n"], (case["name"], len(got), case["n"])
  err = peak_err(stored(case, got), case["y"])
  print("%-28s %6d samples  worst %.3g of the peak" % (case["name"], case["n"], err))
  assert err <= TOL, (case["name"], err)


@pytest.fixture
def fake(monkeypatch):
  fake_native.install(monkeypatch)
  return ab


@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_case_through_the_lazy_api(fake, name):
  check_golden_case(fake, CASES[name])


def test_cases_cover_delays_inputs_seeds_and_endings():
  """The goldens keep what they are for: feedback delays around the ring sizes, every input kind, every seeding
  kind, and Streams that end before, at and exactly with the input."""
  designs = {c["design"] for c in CASES.values()}
  assert {"fb%d" % d for d in (1, 2, 15, 16, 17, 63, 64, 65, 300)} <= designs
  assert {c["input"] for c in CASES.values()} == {"list", "iter"}
  assert max(c["length"] for c in CASES.values() if c["input"] == "iter") > 256 + 1024 + 4096
  assert {type(c["kwargs"].get("memory")).__name__ for c in CASES.values()} == {"NoneType", "list", "str"}
  ended = [c for c in CASES.values() if c["raises"]]
  assert ended and all(c["raises"] == "RuntimeError" for c in ended)
  assert any(not c["n"] for c in ended) and CASES["short_exact"]["raises"] is None
  assert all(len(c["y"]) == len(make_tv.kept(c["n"])) for c in CASES.values())


# ---- the oracle ------------------------------------------------------------------------------------------------------
def split_sections(taps):
  """``Plan.taps()`` -> one tap list per section: every section starts with its numerator tap at delay 0."""
  out = []
  for tap in taps:
    if tap == (0, False):
      out.append([])
    out[-1].append(tap)
  return out


def record_tables(monkeypatch):
  """Wrap ``FakePlan.apply_tv`` to keep what the host hands the native layer: per plan, the taps, the initial
  histories, and the x and coefficient columns of every block."""
  calls = []
  original = fake_native.FakePlan.apply_tv

  def apply_tv(plan, x_ptr, y_ptr, state_ptr, n_streams, n_samples, x_stride, y_stride, coef_ptr, coef_stride, stream=0):
    T, taps = int(n_samples), plan.taps()
    st = fake_native.FakePlan.states[int(state_ptr)]
    if st["tv"] is None:
      calls.append({"taps": taps, "xi": st["xi"], "yi": st["yi"], "x": [], "table": []})
    coef = fake_native._f64(coef_ptr, (len(taps) - 1) * coef_stride + T)
    calls[-1]["x"].append(fake_native._f32(x_ptr, T).copy())
    calls[-1]["table"].append(np.stack([coef[i * coef_stride:i * coef_stride + T] for i in range(len(taps))]))
    return original(plan, x_ptr, y_ptr, state_ptr, n_streams, n_samples, x_stride, y_stride, coef_ptr, coef_stride,
                    stream)

  monkeypatch.setattr(fake_native.FakePlan, "apply_tv", apply_tv)
  return calls


@pytest.mark.parametrize("name", sorted(n for n, c in CASES.items() if not c["design"].startswith("cascade")))
def test_oracle_reproduces_the_reference_from_the_host_tables(fake, monkeypatch, name):
  """The host's tables (a0 folded into every coefficient) through ``oracle.tv_apply`` give the reference's float64
  outputs up to reassociation: the reference divides the sum by a0 instead."""
  case = CASES[name]
  calls = record_tables(monkeypatch)
  run_case(fake, case)
  if not case["n"]:
    assert not calls
    return
  (call,) = calls
  x = np.concatenate(call["x"])
  table = np.concatenate(call["table"], axis=1)
  xi = None if call["xi"] is None else call["xi"][0]
  yi = None if call["yi"] is None else call["yi"][0]
  got = oracle.tv_apply(x[None, :], split_sections(call["taps"]), table, xi, yi)[0]
  assert got.shape == (case["n"],)
  err = peak_err(stored(case, got), case["y"])
  assert err <= 1e-12, err


@pytest.mark.parametrize("b, a", [([1.], [1.]), ([.5, 0., -.25], [1.]), ([1., .5], [1., -.3, 0., .2]),
                                  ([1., 0., 0., 1.], [1.] + [0.] * 15 + [.5]), ([.2, .1, .1, .1], [1., .4, -.3, .2])])
def test_oracle_equals_the_fake_plan_bit_for_bit(monkeypatch, b, a):
  """Single-stream, single-section tables with zeros at some samples and seeded histories: the oracle's float64
  result rounded to float32 is the stand-in native layer's, bit for bit."""
  fake_native.install(monkeypatch)
  rng = np.random.default_rng(len(b) * 7 + len(a))
  T = 97
  plan = fake_native.FakePlan([[(b, a)]], force_generic=True)
  taps = plan.taps()
  x = rng.uniform(-1, 1, T).astype(np.float32)
  xi = rng.uniform(-1, 1, plan.xd)
  yi = rng.uniform(-1, 1, plan.yd)
  table = rng.uniform(-.6, .6, (len(taps), T + 5)) / len(taps)     # coef_stride > T
  table[:, ::7] = 0.0
  state = np.zeros(1)
  plan.state_init(state.ctypes.data, 1, xi[None, None, :] if plan.xd else None, yi[None, None, :] if plan.yd else None)
  y = np.empty_like(x)
  plan.apply_tv(x.ctypes.data, y.ctypes.data, state.ctypes.data, 1, T, T, T, table.ctypes.data, table.shape[1])
  got = oracle.tv_apply(x[None, :], [taps], table, [xi], [yi])
  assert np.array_equal(got[0].astype(np.float32), y)


# ---- a coefficient Stream that ends before the input -----------------------------------------------------------------
def test_short_coefficients_raise_after_the_values_before_them(fake):
  z, St = fake.z, fake.Stream
  x = make_tv.signal(3, 40)
  filt = St([1., 2., 3.]) * z ** -1 + .5
  out = iter(filt(x))
  got = [next(out) for _ in range(3)]
  assert got == pytest.approx([.5 * x[0], .5 * x[1] + 2. * x[0], .5 * x[2] + 3. * x[1]], rel=1e-6)
  with pytest.raises(RuntimeError):
    next(out)
  # an empty coefficient Stream raises on the first sample, an input as long as the coefficients ends cleanly
  with pytest.raises(RuntimeError):
    list((St([]) * z ** -1 + 1)(x))
  assert len(list((St([1.] * 40) * z ** -1 + 1)(x))) == 40
  assert list((St([]) * z ** -1 + 1)([])) == []
  # a Stream a0 that ends, and an end on a block boundary of a lazy input
  with pytest.raises(RuntimeError):
    list((1 / (St([2.] * 5) - .5 * z ** -1))(iter(x)))
  n = 256
  out = (St([.5] * n) * z ** -1 + 1)(iter(make_tv.signal(4, n + 10)))
  assert len(out.take(n)) == n
  with pytest.raises(RuntimeError):
    out.take(1)
  assert len(list((St([.5] * n) * z ** -1 + 1)(iter(make_tv.signal(4, n))))) == n
