"""Frame-wise LPC without a GPU: the float64 emulation against the reference's answers (tests/golden/lpc_cases.json,
made by tests/golden/make_lpc.py from a reference checkout), the compensated sum, argument validation, the frame
count, and the LPC library's exports, target and arithmetic."""
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, crossing, linear_prediction as lp
from conftest import GOLDEN
from native_libs import cuobjdump
import lpc_emulation as em

sys.path.insert(0, GOLDEN)
from make_lpc import inputs  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "lpc_cases.json")) as fh:
    return json.load(fh)


def test_emulation_reproduces_every_reference_digest_and_failure(golden):
  xs = inputs()
  for c in golden["cases"]:
    x = xs[c["input"]]
    assert len(x) == c["length"]
    r, coef, err, failed = em.lpc_frames(x, c["order"], c["size"], c["hop"], c["window_values"])
    key = (c["input"], c["order"], c["size"], c["hop"], c["window"])
    assert len(failed) == c["frames"], key
    assert em.digest(r) == c["acorr"], key
    assert em.digest(coef) == c["coef"], key
    assert em.digest(err) == c["error"], key
    assert np.flatnonzero(failed).tolist() == c["failed"], key
    step = golden["step"]
    for name, got in (("sample_acorr", r), ("sample_coef", coef)):
      want = em.canon([[float(v) for v in row] for row in c[name]]).reshape(-1, c["order"] + 1)
      assert want.tobytes() == em.canon(got[::step]).tobytes(), (key, name)
    assert em.canon([float(v) for v in c["sample_error"]]).tobytes() == em.canon(err[::step]).tobytes(), key
    lengths = [max((k for k, v in enumerate(row) if v != 0), default=0) + 1 for row in coef]
    assert [0 if f else n for n, f in zip(lengths, failed)] == c["lengths"], key


def test_golden_covers_the_edges(golden):
  cases = golden["cases"]
  assert golden["python"] >= "3.12"
  assert {0, 1, 2, 12, 16, 32} <= {c["order"] for c in cases}
  assert any(c["order"] >= c["size"] for c in cases)
  pairs = {(c["size"], c["hop"]) for c in cases}
  assert any(h < s for s, h in pairs) and any(h == s for s, h in pairs) and any(h > s for s, h in pairs)
  padded = {c["frames"] > max(0, (c["length"] - c["size"]) // c["hop"] + 1) for c in cases}
  assert padded == {True, False}
  assert {c["input"] for c in cases if c["failed"]} >= {"silence", "impulse"}
  assert any(c["failed"] and c["failed"][0] > 0 for c in cases)         # a failure after frames that do not fail
  assert golden["doctest"] == {"numlist": [1, 0.0, 0.875], "error": 1.875}


def test_psum_is_cpython_sum():
  """On CPython >= 3.12 the builtin sum() of floats is compensated; psum restates it."""
  rng = np.random.default_rng(5)
  pool = [0., -0., 1., -1., 1e308, -1e308, math.inf, -math.inf, math.nan, 5e-324, -5e-324, 1e16, -1e16, .1, 3.]
  for _ in range(20000):
    terms = [pool[i] for i in rng.integers(0, len(pool), rng.integers(0, 7))]
    want, got = sum(terms), em.psum(terms)
    assert (math.isnan(want) and math.isnan(got)) or (want == got and math.copysign(1, want) == math.copysign(1, got))
  if sys.version_info >= (3, 12):
    assert sum([1e16, 1., -1e16]) == 1.0 and em.psum([1e16, 1., -1e16]) == 1.0


def test_the_doctest():
  r, coef, err, failed = em.kautocor([-1., 0., 1., 0.] * 4, 2)
  assert coef == [1.0, 0.0, 0.875] and err == 1.875 and not failed


def test_validation():
  f = ab.LpcFrames(np.int64(16), 1024, 512, np.hamming(1024))
  assert (f.order, f.size, f.hop) == (16, 1024, 512) and len(f.window) == 1024
  assert ab.LpcFrames(0, 1).hop == 1 and ab.LpcFrames(64, 8192, window=[1.] * 8192).window[0] == 1.
  for args, exc in [((-1, 10), ValueError), ((65, 100), ValueError), ((2, 0), ValueError), ((2, 8193), ValueError),
                    ((2, 10, 0), ValueError), ((2.0, 10), TypeError), ((2, "10"), TypeError), ((True, 10), TypeError),
                    ((2, 10, 1.5), TypeError), ((2, 4, None, [1., 1.]), ValueError),
                    ((2, 2, None, ["a", 1.]), TypeError), ((2, 2, None, 3.), TypeError)]:
    with pytest.raises(exc):
      ab.LpcFrames(*args)
  with pytest.raises(ValueError):
    ab.lpc_frames([1., 2.], 70, 4)


@pytest.mark.parametrize("consumed,T,size,hop,final", [
    (0, 10, 4, 3, True), (0, 10, 4, 3, False), (7, 0, 4, 3, True), (0, 3, 4, 1, True), (5, 20, 3, 7, True),
    (0, 1, 1, 1, False), (123, 4567, 64, 64, True), (0, 2, 4, 1, True), (0, 16384, 1024, 512, False)])
def test_frame_count(consumed, T, size, hop, final):
  """A call emits the frames of the whole stream minus those of what came before; the library agrees."""
  x = np.zeros(consumed + T, dtype=np.float32)
  before = len(em.frames(x[:consumed], size, hop, final=False))
  total = len(em.frames(x, size, hop, final=final))
  f = ab.LpcFrames(0, size, hop)
  assert f.n_frames(consumed, T, final) == total - before == crossing.n_blocks(consumed, T, size, hop, final)
  assert lp.lib().alz_lpc_frames(consumed, T, size, hop, int(final)) == total - before


def test_library_sizes_without_a_device():
  L = lp.lib()
  assert L.alz_lpc_state_bytes(3, 1024) == 3 * (16 + 4096)
  assert L.alz_lpc_state_bytes(1, 5) == 40
  assert L.alz_lpc_state_bytes(1, 0) < 0 and L.alz_lpc_state_bytes(1, 8193) < 0
  assert L.alz_lpc_scratch_bytes(2, 3, 16) == 2 * 3 * 17 * 8
  assert L.alz_lpc_scratch_bytes(2, 3, 65) < 0
  assert L.alz_lpc_apply_f32(None, 0, None, None, None, None, None, 0, None, 1, 0, 65, 4, 1, 0, None, 0, None) < 0
  assert "order" in L.alz_lpc_last_error().decode()


def test_lpc_library_has_no_fused_multiply_add():
  """Built with -fmad=false: no product is contracted into an add, as the reference's arithmetic requires.  The only
  DFMAs are the Newton steps of the one correctly rounded division in the Levinson-Durbin kernel (c = num / den)."""
  sass = subprocess.run([cuobjdump(), "-sass", _build.LIBRARIES["lpc"].path], capture_output=True, text=True).stdout
  functions = re.split(r"\n\s*Function : ", sass)[1:]
  assert len(functions) == 3
  by_name = {f.split(None, 1)[0]: f for f in functions}
  lev = [body for name, body in by_name.items() if "alz_lpc_levinson_kernel" in name]
  acorr = [body for name, body in by_name.items() if "alz_lpc_kernel" in name]
  assert len(lev) == 1 and len(acorr) == 1
  assert "DADD" in acorr[0] and "DMUL" in acorr[0]
  for name, body in by_name.items():
    if body is not lev[0]:
      assert "DFMA" not in body, name
  assert "MUFU.RCP64H" in lev[0] and len(re.findall(r"\bDFMA\b", lev[0])) <= 20
