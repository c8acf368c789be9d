"""window / wsymm and the overlap-add gains against the reference's goldens, the numpy emulation of overlap_add against
the reference's outputs, the frame-count rule and the reference's errors."""
import json
import math
import os

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _engine, spectral
from conftest import GOLDEN
import stft_emulation as em


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "stft_cases.json")) as fh:
    return json.load(fh)


def decode(values):
  return np.array([float(v) for v in values], dtype=np.float64)


def test_windows_equal_the_reference_bit_for_bit(golden):
  import hashlib
  for c in golden["windows"]:
    f = getattr(ab, c["dict"])[c["name"]]
    vals = f(c["size"]) if c["alpha"] is None else f(c["size"], c["alpha"])
    assert hashlib.sha256(np.asarray(vals, dtype=np.float64).tobytes()).hexdigest() == c["digest"], c


def test_window_names_and_cross_attributes():
  assert [k[0] for k in ab.window.keys()] == ["hann", "hamming", "rect", "bartlett", "triangular", "blackman", "cos"]
  assert ab.window.hanning is ab.window.hann and ab.window.triangle is ab.window.triangular
  assert ab.window.dirichlet is ab.window.rect is ab.wsymm.rect and "dirichlet" not in ab.wsymm
  assert ab.window.hann.symm is ab.wsymm.hann and ab.wsymm.hann.periodic is ab.window.hann
  assert ab.window.symm is ab.wsymm and ab.wsymm.periodic is ab.window
  assert ab.wsymm.hann(1) == [1.0] and ab.wsymm.blackman(1) == [1.0]


def _ola_case(c):
  import sys
  sys.path.insert(0, GOLDEN)
  from make_stft import ola_inputs
  blocks = np.array(ola_inputs(c["size"])[c["input"]], dtype=np.float64).reshape(-1, c["size"])
  wnd = getattr(ab.window, c["wnd"]) if isinstance(c["wnd"], str) else c["wnd"]
  return blocks, spectral.ola_window(c["size"], c["hop"], wnd, c["normalize"], c["strategy"])


def test_emulated_overlap_add_equals_the_reference(golden):
  for c in golden["ola"]:
    blocks, w = _ola_case(c)
    got = em.ola(blocks, c["size"], c["hop"], w)
    assert np.array_equal(got, decode(c["output"]), equal_nan=True), c


def golden_stft_case(c):
  """The inputs and keywords of an stft golden: samples, window values, shift flags, overlap-add window and strategy."""
  import sys
  sys.path.insert(0, GOLDEN)
  import make_stft
  kws = c["kwargs"]
  size = c["size"]
  hop = c["hop"] or size
  wnd = getattr(ab.window, kws["wnd"])(size) if kws.get("wnd") else None
  ola = kws.get("ola", "numpy")
  ola_wnd = getattr(ab.window, kws["ola_wnd"]) if kws.get("ola_wnd") else None
  ola_w = None if ola is None else spectral.ola_window(size, hop, ola_wnd, kws.get("ola_normalize", True), ola)
  return (make_stft.stft_input(c["input"], size), size, hop, wnd, kws.get("before", 0) is not None,
          kws.get("after", 0) is not None, ola, ola_w)


def emulated_func(name, size):
  import sys
  sys.path.insert(0, GOLDEN)
  import make_stft
  return {"identity": lambda b: b, "abs": np.abs, "ifftshift": lambda b: np.fft.ifftshift(b, axes=-1),
          "mask": lambda b: b * make_stft.mask(size)}[name]


def test_emulated_stft_equals_the_reference(golden):
  """Bit for bit on the numpy version the goldens were recorded with (the same pocketfft), to 1e-12 of the peak
  otherwise."""
  arrays = np.load(os.path.join(GOLDEN, "stft_cases.npz"))
  exact = np.__version__ == golden["numpy"]
  for i, c in enumerate(golden["stft"]):
    x, size, hop, wnd, before, after, ola, ola_w = golden_stft_case(c)
    got = em.stft(x.astype(np.float64), size, hop, emulated_func(c["func"], size), wnd, before, after, ola_w,
                  ola is not None)
    want = arrays["stft_%d" % i]
    assert got.shape == want.shape, c["name"]
    if exact:
      assert np.array_equal(got, want, equal_nan=True), c["name"]
    else:
      peak = np.max(np.abs(want[np.isfinite(want)]), initial=0.)
      assert np.array_equal(np.isnan(got), np.isnan(want)), c["name"]
      assert np.all(np.abs(np.nan_to_num(got - want)) <= 1e-12 * peak), c["name"]


def test_gain_rules():
  assert np.array_equal(spectral.ola_window(8, 3, None, True, "numpy"), np.ones(8) / 3)
  assert spectral.ola_window(8, 3, None, True, "list").tolist() == [1 / 3] * 8
  assert spectral.ola_window(8, 3, None, False, "list") is None
  assert np.array_equal(spectral.ola_window(8, 3, None, False, "numpy"), np.ones(8))
  assert spectral.ola_window(4, 2, [0., 0., 0., 0.], True, "numpy").tolist() == [0.] * 4     # zero gain: as it is
  w = [.1, .2, .3, .7, .11, .13, .17, .19, .23]
  gain = max(map(sum, zip(*[[.1, .2, .3], [.7, .11, .13], [.17, .19, .23]])))
  assert spectral.ola_window(9, 3, w, True, "list").tolist() == [v / gain for v in w]
  gain = np.sum(np.abs(np.vstack([np.array(w[i:i + 3]) for i in (0, 3, 6)])), 0).max()
  assert np.array_equal(spectral.ola_window(9, 3, w, True, "numpy"), np.array(w) / gain)


def test_frame_count_rule():
  """Frames a call emits: those it completes, plus the padded last block at the end of the stream."""
  for T, size, hop in [(0, 4, 2), (5, 4, 2), (13, 8, 3), (7, 64, 64), (64, 64, 64), (65, 64, 64), (10, 3, 3)]:
    assert _engine.n_blocks(0, T, size, hop, True) == len(em.frames(np.zeros(T), size, hop)), (T, size, hop)
    complete = len([k for k in range(T) if k * hop + size <= T])
    assert _engine.n_blocks(0, T, size, hop, False) == complete, (T, size, hop)
    for c in range(T + 1):        # any split gives the frames of one call
      assert (_engine.n_blocks(0, c, size, hop, False) + _engine.n_blocks(c, T - c, size, hop, True) ==
              len(em.frames(np.zeros(T), size, hop)))


def test_reference_errors_at_call_time():
  with pytest.raises(TypeError, match="Missing 'size' argument"):
    ab.stft(abs)([1.])
  with pytest.raises(ValueError, match="Hop value can't be higher than size"):
    ab.stft(abs, size=4, hop=5)([1.])
  with pytest.raises(ValueError, match="Hop value can't be higher than size"):
    ab.OverlapAdd(4, 5)
  for name in ("cfft", "complex", "cfftr", "complex_real"):
    with pytest.raises(NotImplementedError, match="cfft"):
      ab.stft[name](abs, size=4)
  assert ab.stft.base is ab.stft.real is ab.stft.rfft is ab.stft.default

