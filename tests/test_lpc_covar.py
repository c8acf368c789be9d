"""Covariance-method LPC without a GPU: the float64 emulation against the reference's answers
(tests/golden/lpc_covar_cases.json, made by tests/golden/make_lpc_covar.py from a reference checkout), with and without
skipping the products of zero coefficients, and the method names, limits and library entry points on the host."""
import json
import math
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import linear_prediction as lp
from conftest import GOLDEN
import lpc_covar_emulation as em

sys.path.insert(0, GOLDEN)
from make_lpc_covar import inputs  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "lpc_covar_cases.json")) as fh:
    return json.load(fh)


def failures(failed):
  return [[k, int(f)] for k, f in enumerate(failed) if f]


@pytest.mark.parametrize("fast", [True, False])
def test_emulation_reproduces_every_reference_digest_and_failure(golden, fast):
  """Both forms of the emulation -- every product summed, as the reference does, and the products of zero coefficients
  skipped, as the kernel does -- give the reference's bits.  The dense form takes O(order^4) per frame, so it skips
  the order-64 cases."""
  xs = inputs()
  step = golden["step"]
  for c in golden["cases"]:
    if not fast and c["order"] > 32:
      continue
    x = xs[c["input"]]
    assert len(x) == c["length"]
    key = (c["input"], c["order"], c["size"], c["hop"], c["window"])
    M, C, E, failed = em.lpc_frames(x, c["order"], c["size"], c["hop"], c["window_values"], fast=fast)
    assert len(failed) == c["frames"], key
    assert em.digest(M) == c["lagm"], key
    assert em.digest(C) == c["coef"] and em.digest(E) == c["error"], key
    assert failures(failed) == c["failed"], key
    want = em.canon([[float(v) for v in row] for row in c["sample_lagm_row0"]]).reshape(-1, c["order"] + 1)
    assert want.tobytes() == em.canon(M[::step, 0]).tobytes(), key
    want = em.canon([[float(v) for v in row] for row in c["sample_coef"]]).reshape(-1, c["order"] + 1)
    assert want.tobytes() == em.canon(C[::step]).tobytes(), key
    assert em.canon([float(v) for v in c["sample_error"]]).tobytes() == em.canon(E[::step]).tobytes(), key
    lengths = [max((k for k, v in enumerate(row) if v != 0), default=0) + 1 for row in C]
    assert [0 if f else n for n, f in zip(lengths, failed)] == c["lengths"], key


def test_golden_covers_the_edges(golden):
  cases = golden["cases"]
  assert golden["python"] >= "3.12"
  assert {1, 2, 12, 16, 32, 64} <= {c["order"] for c in cases}
  pairs = {(c["size"], c["hop"]) for c in cases}
  assert any(h < s for s, h in pairs) and any(h == s for s, h in pairs) and any(h > s for s, h in pairs)
  padded = {c["frames"] > max(0, (c["length"] - c["size"]) // c["hop"] + 1) for c in cases}
  assert padded == {True, False}
  kinds = {(c["input"], f[1]) for c in cases for f in c["failed"]}
  assert {("silence", 1), ("impulse", 1), ("dc", 2), ("alternating", 2), ("tone", 2)} <= kinds
  assert any(c["failed"] and c["failed"][0][0] > 0 for c in cases)      # a failure after frames that do not fail
  # NaN and inf inputs run through without failing, with NaN results
  assert any(c["input"] in ("nan", "inf") and not c["failed"] and c["order"] >= 12 for c in cases)
  assert golden["raises"] == [["IndexError", "list index out of range"],
                              ["ValueError", "Block length should be higher than order"]]


def test_order_zero_and_short_blocks_raise_as_the_reference():
  with pytest.raises(IndexError):
    em.kcovar(em.lag_matrix([1., 2., 3.], 0))
  with pytest.raises(ValueError, match="Block length should be higher than order"):
    em.lag_matrix([1., 2.], 2)


def test_lag_matrix_is_the_host_lag_matrix_and_symmetric():
  rng = np.random.default_rng(3)
  b = rng.uniform(-1, 1, 50)
  M = em.lag_matrix(b, 7)
  assert M.tobytes() == M.T.tobytes()
  assert M.tolist() == ab.lag_matrix(b.tolist(), 7)


def test_methods_and_aliases():
  for name in ("kautocor", "kacorr", "kautocorrelation", "kauto_correlation"):
    assert ab.LpcFrames(4, 32, method=name).method == "kautocor"
  for name in ("kcovar", "kcov", "kcovariance"):
    assert ab.LpcFrames(4, 32, method=name).method == "kcovar"
  assert ab.LpcFrames(4, 32).method == "kautocor"
  for name in ("covar", "cov", "covariance", "ncovar", "ncov", "ncovariance", "nautocor", "nacorr", "autocor",
               "acorr", "autocorrelation", "nope"):
    with pytest.raises(ValueError, match="kautocor.*kcovar|kcov"):
      ab.LpcFrames(4, 32, method=name)
  with pytest.raises(TypeError):
    ab.LpcFrames(4, 32, method=None)


def test_covariance_limits():
  assert ab.LpcFrames(1, 2, method="kcovar").order == 1
  assert ab.LpcFrames(64, 65, method="kcov").size == 65
  for order, size in ((0, 10), (10, 10), (11, 10), (64, 64)):
    with pytest.raises(ValueError):
      ab.LpcFrames(order, size, method="kcovar")
  with pytest.raises(ValueError, match="Block length"):
    ab.lpc_frames([1., 2., 3.], 3, 3, method="kcovar")
  # the key of a state holds the method
  assert ab.LpcFrames(4, 32)._key() != ab.LpcFrames(4, 32, method="kcovar")._key()


def test_covariance_library_without_a_device():
  L = lp.lib()
  assert L.alz_lpc_covar_scratch_bytes(2, 3, 16) == 2 * 3 * 17 * 18 // 2 * 8
  assert L.alz_lpc_covar_scratch_bytes(1, 1, 0) == 8
  assert L.alz_lpc_covar_scratch_bytes(2, 3, 65) < 0
  args = [None, 0, None, None, None, None, None, 0, None, 1, 0]
  assert L.alz_lpc_covar_apply_f32(*args, 4, 4, 1, 0, None, 0, None) < 0      # order >= size
  assert "order" in L.alz_lpc_last_error().decode()
  assert L.alz_lpc_covar_apply_f32(*args, 65, 100, 1, 0, None, 0, None) < 0
  # order 0 has a lag matrix but no recursion: refused when a failure flag (any non-NULL pointer: the call is refused
  # before it is used) is asked for
  assert L.alz_lpc_covar_apply_f32(None, 0, None, None, None, None, 8, 0, None, 1, 0, 0, 4, 1, 0, None, 0, None) < 0
  assert "order >= 1" in L.alz_lpc_last_error().decode()


def test_psum_terms_of_zero_leave_the_sum_alone():
  """The rule the skipping rests on: adding +-0 to a compensated sum changes no bit, unless the zero is a NaN."""
  rng = np.random.default_rng(8)
  pool = [1., -1., 1e308, -1e308, math.inf, -math.inf, math.nan, 5e-324, 1e16, -1e16, .1, 3.]
  for _ in range(5000):
    terms = [pool[i] for i in rng.integers(0, len(pool), rng.integers(1, 6))]
    mixed = list(terms)
    for _ in range(rng.integers(1, 4)):
      mixed.insert(int(rng.integers(0, len(mixed) + 1)), [0., -0.][int(rng.integers(0, 2))])
    a, b = em.psum(terms), em.psum(mixed)
    assert (math.isnan(a) and math.isnan(b)) or (a == b and math.copysign(1, a) == math.copysign(1, b))
