"""zcross without a GPU: the numpy emulation against the reference's answers (tests/golden/zcross_cases.json, made by
tests/golden/make_zcross.py from a reference checkout), input validation, and the zero-crossing library's exports."""
import ast
import json
import math
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import crossing
from conftest import GOLDEN
from zcross_emulation import block_sums, digest, zcross as emulate

sys.path.insert(0, GOLDEN)
from make_zcross import inputs  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "zcross_cases.json")) as fh:
    return json.load(fh)


def test_emulation_reproduces_every_reference_digest_and_block_sum(golden):
  xs = inputs()
  assert len(golden["cases"]) == 5 * 6 * 5
  for case in golden["cases"]:
    x = xs[case["input"]]
    assert len(x) == case["length"]
    y = emulate(x, float(case["hysteresis"]), float(case["first_sign"]))
    assert digest(y, "u1") == case["digest"], case["input"]
    assert y[::case["step"]].tolist() == case["values"]
    for b in case["blocks"]:
      sums = block_sums(y, b["size"], b["hop"])
      assert len(sums) == b["n"] and digest(sums, "<i4") == b["digest"], (case["input"], b)
      assert sums[:len(b["head"])].tolist() == b["head"]


def test_golden_covers_the_edges(golden):
  cases = golden["cases"]
  assert {"0.0", "0.01", "0.15", "-0.5", "inf", "nan"} == {c["hysteresis"] for c in cases}
  assert {"0.0", "-0.0", "-3", "2", "nan"} == {c["first_sign"] for c in cases}
  sizes = {(b["size"], b["hop"]) for b in golden["cases"][0]["blocks"]}
  assert any(h < s for s, h in sizes) and any(h == s for s, h in sizes) and any(h > s for s, h in sizes)
  assert any(s == 1 for s, _ in sizes)
  padded = set()                                          # the reference's padded last block, emitted and not
  for c in cases:
    for b in c["blocks"]:
      full = max(0, (c["length"] - b["size"]) // b["hop"] + 1)
      padded.add(b["n"] > full)
  assert padded == {True, False}
  x = inputs()["zero_runs"]
  assert np.max(np.diff(np.flatnonzero(x))) > 3 * 4096


def test_the_issue_examples():
  assert emulate([.1, .2, np.nan, -.3, 0., -0., .4], -.5).tolist() == [0, 1, 0, 1, 1, 1, 1]
  assert block_sums(emulate([1., -1.] * 5), 4, 3).tolist() == [3, 4, 4]
  assert emulate([-.5, .5], 0, math.nan).tolist() == [1, 1]           # first_sign NaN starts at +1
  assert emulate([-.5, .5], 0, -0.).tolist() == [0, 1]                # -0. means "search"


def test_errors_are_the_references(golden):
  """The reference raises these while iterating; this package raises from the call."""
  assert len(golden["errors"]) >= 5
  for err in golden["errors"]:
    assert err["error"] == "TypeError"
    h, fs = ast.literal_eval(err["hysteresis"]), ast.literal_eval(err["first_sign"])
    with pytest.raises(TypeError):
      ab.zcross([1., -1.], hysteresis=h, first_sign=fs)
    with pytest.raises(TypeError):
      ab.Zcross(h, fs)


def test_validation():
  zc = ab.Zcross(np.float32(.25), np.int64(-2))            # numpy scalars are real numbers
  assert zc.hysteresis == .25 and zc.sign == -1
  assert ab.Zcross(0, -0.).sign == 0 and ab.Zcross(0, math.nan).sign == 1 and ab.Zcross(True, 3).sign == 1
  with pytest.raises(TypeError):
    ab.Zcross("0.1")


@pytest.mark.parametrize("consumed,T,size,hop,final", [
    (0, 10, 4, 3, True), (0, 10, 4, 3, False), (7, 0, 4, 3, True), (0, 3, 4, 1, True), (5, 20, 3, 7, True),
    (0, 1, 1, 1, False), (123, 4567, 64, 64, True), (0, 2, 4, 1, True)])
def test_n_blocks_matches_the_emulated_split(consumed, T, size, hop, final):
  """The count a call stores is the emulated block count of the whole stream minus that of what came before."""
  flags = np.zeros(consumed + T, dtype=np.uint8)
  before = len(block_sums(flags[:consumed], size, hop, final=False))
  total = len(block_sums(flags, size, hop, final=final))
  assert crossing.n_blocks(consumed, T, size, hop, final) == total - before


def test_library_sizes_without_a_device():
  """The state and scratch queries are host-only: per stream 16 bytes plus the open blocks' counts, 8-byte aligned."""
  L = crossing.lib()
  assert L.alz_zcross_state_bytes(3, 0, 1) == 48
  assert L.alz_zcross_state_bytes(3, 2048, 1024) == 3 * 24
  assert L.alz_zcross_state_bytes(1, 5, 2) == 32
  assert L.alz_zcross_state_bytes(1, 5, 0) < 0
  assert L.alz_zcross_scratch_bytes(1, 0, 0, 1) == 16
