"""dft against the reference's goldens on the CPU: the float64 emulation of the header's arithmetic reproduces every
golden, the library's host twiddles equal cmath.exp(-1j * n * f) bit for bit, the argument and frame-count checks,
and the DFT library's SASS."""
import builtins
import cmath
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, _engine, fourier
from conftest import GOLDEN
from native_libs import cuobjdump
import dft_emulation as em

sys.path.insert(0, GOLDEN)
import make_dft  # noqa: E402


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "dft_cases.json")) as fh:
    doc = json.load(fh)
  assert doc["step"] == make_dft.STEP
  return doc


def case_id(c):
  return "%s-%s-%d-%s" % (c["input"], c.get("length", c["size"]), c["size"], c.get("hop", ""))


def freqs_of(c):
  return [make_dft.dec_freq(f) for f in c["freqs"]]


def parts(v):
  return (v, v) if isinstance(v, int) else (v.real, v.imag)


def check_values(c, values):
  """``values`` (a flat list of complex, or of int 0 for an empty block) are the reference's result of case ``c``: the
  exact bits of both parts, NaN by NaN-ness."""
  values = list(values)
  assert len(values) == c["n"], case_id(c)
  if "values" in c:
    for got, want in zip(values, c["values"]):
      if isinstance(want, int):
        assert got == want and isinstance(got, int), case_id(c)
        continue
      for g, w in zip(parts(got), want):
        w = make_dft.dec(w)
        assert (np.isnan(g) and np.isnan(w)) or (g == w and np.signbit(g) == np.signbit(w)), (case_id(c), got, want)
  else:
    for got, want in zip(values[::make_dft.STEP], c["sampled"]):
      for g, w in zip(parts(got), want):
        w = make_dft.dec(w)
        assert (np.isnan(g) and np.isnan(w)) or (g == w and np.signbit(g) == np.signbit(w)), (case_id(c), got, want)
    assert make_dft.digest(values) == c["digest"], case_id(c)


def framed_blocks(c):
  x = make_dft.signal(c["input"], c["length"])
  return em.frames(x, c["size"], c["hop"], make_dft.window(c["window"], c["size"]))


def test_emulation_reproduces_every_golden(golden):
  for c in golden["cases"]:
    x = make_dft.signal(c["input"], c["size"]).astype(np.float64).tolist()
    if "exception" in c:
      exc, msg = c["exception"]
      with pytest.raises(getattr(builtins, exc), match=re.escape(msg)):
        em.dft(x, freqs_of(c), c["normalize"])
    else:
      check_values(c, em.dft(x, freqs_of(c), c["normalize"]))
  for c in golden["framed"]:
    b = framed_blocks(c)
    assert len(b) == c["frames"], case_id(c)
    check_values(c, [v for row in b for v in em.dft(row.tolist(), freqs_of(c), c["normalize"])])


def test_vectorised_emulation_equals_the_emulation(golden):
  for c in golden["framed"]:
    if not c["freqs"]:
      continue
    b = framed_blocks(c)
    got = em.dft_batch(b, fourier.twiddles(freqs_of(c), c["size"]), c["normalize"])
    check_values(c, got.reshape(-1).tolist())


def _bits(v):
  return np.array([v.real, v.imag], dtype=np.float64).tobytes()


def test_host_twiddles_equal_cmath(golden):
  freqs = sorted({f for c in golden["cases"] + golden["framed"] for f in freqs_of(c)}, key=repr)
  for f in freqs:
    for size in (1, 7, 1024):
      try:
        want = [cmath.exp(-1j * n * f) for n in range(size)]
      except ValueError:
        with pytest.raises(ValueError, match="math domain error"):
          fourier.twiddles([f], size)
        continue
      got = fourier.twiddles([f], size)[:, 0]
      assert all(_bits(g) == _bits(w) or (np.isnan(g.real) and np.isnan(w.real) and np.isnan(g.imag) and
                                          np.isnan(w.imag)) for g, w in zip(got, want)), f
  # 10^5 random (n, f) pairs, every one filled by the library itself
  rng = np.random.default_rng(5)
  fs = np.concatenate([rng.uniform(-7, 7, 40), rng.uniform(-1e4, 1e4, 5), 10.0 ** rng.uniform(-300, 5, 5)])
  table = np.zeros((2000, len(fs)), dtype=np.complex128)
  unfilled = np.zeros(len(fs), dtype=np.uint8)
  assert fourier.lib().alz_dft_twiddles(np.ascontiguousarray(fs).ctypes.data, len(fs), 2000, table.ctypes.data,
                                        unfilled.ctypes.data) == 0
  assert not unfilled.any()
  for j, f in enumerate(fs):
    want = np.array([cmath.exp(-1j * n * float(f)) for n in range(2000)], dtype=np.complex128)
    assert table[:, j].tobytes() == want.tobytes(), f


def test_twiddles_mark_the_columns_cmath_fills():
  fs = np.array([1., np.inf, np.nan, 1e308, -np.inf], dtype=np.float64)
  table = np.zeros((3, 5), dtype=np.complex128)
  unfilled = np.zeros(5, dtype=np.uint8)
  assert fourier.lib().alz_dft_twiddles(fs.ctypes.data, 5, 3, table.ctypes.data, unfilled.ctypes.data) == 4
  assert unfilled.tolist() == [0, 1, 1, 1, 1]
  assert fourier.lib().alz_dft_twiddles(fs.ctypes.data, 5, 2, table.ctypes.data, unfilled.ctypes.data) == 3
  assert unfilled.tolist() == [0, 1, 1, 0, 1]
  t = fourier.twiddles([np.inf, np.nan, 2], 4)
  assert np.isnan(t[:, :2].real).all() and np.isnan(t[:, :2].imag).all()
  with pytest.raises(ValueError, match="math domain error"):
    fourier.twiddles([1., 1e308], 3)


def test_frame_counts_and_argument_errors():
  L = fourier.lib()
  for consumed, T, size, hop, final in ((0, 100, 10, 3, 0), (5, 17, 7, 9, 1), (0, 3, 7, 2, 1), (40, 0, 8, 8, 1)):
    assert L.alz_dft_frames(consumed, T, size, hop, final) == _engine.n_blocks(consumed, T, size, hop, final)
    blocks = em.frames(np.zeros(consumed + T), size, hop, final=final)
    assert len(blocks) - em.frames(np.zeros(consumed), size, hop, final=False).shape[0] == \
      L.alz_dft_frames(consumed, T, size, hop, final)
  assert L.alz_dft_frames(-1, 0, 4, 1, 0) < 0 and L.alz_dft_frames(0, 0, 4, 0, 0) < 0
  assert L.alz_dft_state_bytes(3, 1024) == 3 * (16 + 4096)
  assert L.alz_dft_state_bytes(1, 0) < 0 and L.alz_dft_state_bytes(1, 8193) < 0
  assert L.alz_dft_apply_f32(None, 0, None, None, 1, 1, None, 1, 0, None, 1, 0, 8193, 1, 0, None) < 0
  assert "size" in L.alz_dft_last_error().decode()
  assert L.alz_dft_apply_f32(None, 0, None, None, 4097, 1, None, 1, 0, None, 1, 0, 8, 1, 0, None) < 0
  assert "n_freqs" in L.alz_dft_last_error().decode()
  assert L.alz_dft_apply_f32(None, 0, None, None, 1, 1, None, 1, 0, None, 1, 0, 8, 0, 0, None) < 0
  assert "hop" in L.alz_dft_last_error().decode()
  assert L.alz_dft_twiddles(None, -1, 4, None, None) < 0


def test_python_argument_errors():
  with pytest.raises(NotImplementedError, match="complex frequencies"):
    ab.dft([1., 2.], [1j])
  with pytest.raises(NotImplementedError, match="complex-valued"):
    ab.dft([1., 2j], [1.])
  assert ab.dft([1., 2.], []) == []
  assert ab.dft([], [1., 2.], normalize=False) == [0, 0]
  with pytest.raises(ZeroDivisionError, match="division by zero"):
    ab.dft([], [1.])


def test_dft_library_has_no_fused_multiply_add():
  """Built with -fmad=false: no product is contracted into an add.  The only DFMAs are the Newton steps of the
  library's one correctly rounded division (the normalization's quotient, an out-of-line function), whose IEEE result
  they do not change."""
  sass = subprocess.run([cuobjdump(), "-sass", _build.LIBRARIES["dft"].path], capture_output=True, text=True).stdout
  functions = re.split(r"\n\s*Function : ", sass)[1:]
  by_name = {f.split(None, 1)[0]: f for f in functions}
  assert sorted(n for n in by_name if "alz_dft" in n) == sorted(by_name)
  main = [body for name, body in by_name.items() if "alz_dft_kernel" in name]
  assert len(main) == 1 and len(by_name) == 2
  body = main[0]
  assert "DADD" in body and "DMUL" in body
  # the division is a subroutine of the kernel: every DFMA lies between its MUFU.RCP64H and the kernel's end
  assert "MUFU.RCP64H" in body and len(re.findall(r"\bDFMA\b", body)) <= 20
  first_dfma = body.index("DFMA")
  assert body.rfind("EXIT", 0, first_dfma) > 0, "a DFMA before the kernel's exit: a contracted product"
  for name, b in by_name.items():
    if b is not body:
      assert "DFMA" not in b, name
