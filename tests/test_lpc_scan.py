"""Time-parallel LPC synthesis on the CPU: the three passes restated in float64 (tests/lpc_scan_emulation.py) against
the sequential restatement (tests/lpc_filter_emulation.py) within the bar, on the reference's golden rows and on long
streams of stable rows; the fallback of streams with non-finite summaries; the cost model; the LpcFilter option; the
time-parallel synthesis library's argument checks; and its SASS."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, _capi, linear_prediction as lp
from conftest import ROOT
from lpc_filter_emulation import lpc_filter, same_bits
from lpc_scan_emulation import chunk_bounds, kautocor_rows, lpc_scan, max_chunks, within_bar
from native_libs import cuobjdump

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "lpc_filter_cases.npz"))
META = json.loads(str(GOLDEN["meta"]))
SYNTHESIS = [i for i, m in enumerate(META) if m["kind"] == "synthesis"]


def check_against_sequential(x, coef, hop, P, consumed=0, hist=None):
  """The emulation in P chunks against the sequential restatement: within the bar, flagged streams bit for bit."""
  want, want_hist = lpc_filter("synthesis", x, coef, hop, consumed, hist)
  got, got_hist, flagged = lpc_scan(x, coef, hop, P, consumed, hist)
  for s in range(len(x)):
    if flagged[s]:
      assert same_bits(got[s], want[s]) and same_bits(got_hist[s], want_hist[s]), s
    else:
      assert within_bar(got[s:s + 1], want[s:s + 1]), s
      assert within_bar(got_hist[s:s + 1], want_hist[s:s + 1]), s
  return flagged


def test_chunk_bounds():
  assert chunk_bounds(10, 3).tolist() == [0, 4, 7, 10]
  assert chunk_bounds(9, 9).tolist() == list(range(10))
  assert max_chunks(100, 16) == 6 and max_chunks(10, 16) == 1 and max_chunks(5, 0) == 5


@pytest.mark.parametrize("i", SYNTHESIS, ids=[META[i]["name"] for i in SYNTHESIS])
def test_golden_rows_within_the_bar(i):
  m = META[i]
  x, coef, y = GOLDEN["x_%d" % i], GOLDEN["coef_%d" % i], GOLDEN["y_%d" % i]
  top = max_chunks(len(x), m["order"])
  for P in sorted({min(2, top), min(3, top), top}):
    got, _, flagged = lpc_scan(x[None], coef[None], m["hop"], P)
    if flagged[0]:
      assert same_bits(got[0], y), P
    else:
      assert within_bar(got, y[None]), P
    check_against_sequential(x[None], coef[None], m["hop"], P)


def long_rows(kind, T, order, hop, rng):
  """Rows for T samples at `hop`: the kautocor rows of frames of a signal of that kind (half-overlapping frames of
  max(2 order + 2, 64) samples), row r taking the frame that holds sample r hop."""
  size = max(2 * order + 2, 64)
  t = np.arange(T + size)
  if kind == "noise":
    sig = rng.standard_normal(len(t))
  elif kind == "tones":
    sig = np.sin(.05 * t) + .5 * np.sin(.31 * t + 1) + .01 * rng.standard_normal(len(t))
  else:
    sig = np.sin(1e-5 * t * t) + .01 * rng.standard_normal(len(t))
  frames = kautocor_rows(sig, order, size, size // 2)
  r = np.arange(-(-T // hop) + 1)
  return frames[np.minimum(r * hop // (size // 2), len(frames) - 1)]


@pytest.mark.parametrize("order", [1, 2, 16, 32, 64])
@pytest.mark.parametrize("hop", [1, 7, 480, 5000])
def test_long_stable_streams_within_the_bar(order, hop):
  """Noise, tones and a chirp through their own autocorrelation rows, at forced chunk counts up to the largest (hop
  5000 is longer than every chunk)."""
  rng = np.random.default_rng(order * 100 + hop)
  T = 6000 if order < 64 else 3000
  coef = np.stack([long_rows(kind, T, order, hop, rng) for kind in ("noise", "tones", "chirp")])
  x = rng.standard_normal((3, T))
  top = max_chunks(T, order)
  for P in sorted({2, 3, max(2, top // 7), top}):
    flagged = check_against_sequential(x, coef, hop, P)
    assert not flagged.any(), P


def test_state_carries_across_calls():
  rng = np.random.default_rng(3)
  coef = np.concatenate([np.ones((2, 40, 1)), rng.standard_normal((2, 40, 6)) * .05], axis=2)
  x = rng.standard_normal((2, 3900))
  want, want_hist = lpc_filter("synthesis", x, coef, 100)
  got, hist, n = [], None, 0
  for cut, P in ((1234, 7), (1000, 1), (1666, 50)):
    if P > 1:
      y, hist, _ = lpc_scan(x[:, n:n + cut], coef[:, n // 100:], 100, P, n, hist)
    else:
      y, hist = lpc_filter("synthesis", x[:, n:n + cut], coef[:, n // 100:], 100, n, hist)
    got.append(y)
    n += cut
  assert within_bar(np.concatenate(got, axis=1), want) and within_bar(hist, want_hist)


def test_fallback_flags_exactly_the_non_finite_streams():
  rng = np.random.default_rng(11)
  S, T, order, hop = 7, 2000, 8, 100
  coef = np.concatenate([np.ones((S, 20, 1)), rng.standard_normal((S, 20, order)) * .05], axis=2)
  x = rng.standard_normal((S, T))
  x[1, 1234] = np.inf                                           # inf sample mid-stream
  x[2, 77] = np.nan                                             # NaN sample
  coef[3, 9, 4] = np.nan                                        # NaN row (a failed LpcFrames frame)
  coef[4, 5:, 1] = -3.0                                         # unstable rows: the output overflows
  x[5, -1] = -np.inf                                            # inf in the last sample
  flagged = check_against_sequential(x, coef, hop, 16)
  assert flagged.tolist() == [False, True, True, True, True, True, False]
  want, _ = lpc_filter("synthesis", x[4:5], coef[4:5], hop)
  assert np.isinf(want).any() and np.isnan(want).any()


# --- the cost model and the option ----------------------------------------------------------------------------------

def test_cost_model():
  L = lp.LPCSCAN_LIB.load()
  assert L.alz_lpcscan_chunks(1, 2_880_000, 0, 480) == 1                 # order 0: nothing to carry
  assert L.alz_lpcscan_chunks(1, 300, 16, 480) == 1                      # short: the launches cost more
  assert L.alz_lpcscan_chunks(4096, 16384, 16, 512) == 1                 # many streams: sequential pays
  assert L.alz_lpcscan_chunks(0, 100, 16, 480) == 1 and L.alz_lpcscan_chunks(5, 0, 16, 480) == 1
  for S, T, order in ((1, 2_880_000, 16), (1, 2_880_000, 64), (8, 2_880_000, 16), (64, 262_144, 16)):
    P = L.alz_lpcscan_chunks(S, T, order, 480)
    assert 100 <= P <= T // order, (S, T, order, P)
  assert L.alz_lpcscan_chunks(1, 100, 65, 1) < 0 and "order" in L.alz_lpcscan_last_error().decode()
  assert L.alz_lpcscan_chunks(1, 100, 4, 0) < 0 and "hop" in L.alz_lpcscan_last_error().decode()


def test_chunks_of_the_option():
  syn = lambda tp, order=16: ab.LpcFilter(order, 480, "synthesis", time_parallel=tp)
  assert syn(False).chunks(1, 2_880_000) == 1
  assert syn(True).chunks(1, 2_880_000) == lp.LPCSCAN_LIB.load().alz_lpcscan_chunks(1, 2_880_000, 16, 480) > 1
  assert syn(True).chunks(4096, 16384) == 1
  assert syn(1000).chunks(1, 3200) == 200 and syn(1000).chunks(1, 32000) == 1000   # chunks of >= order samples
  assert syn(1000).chunks(1, 10) == 1 and syn(7, 0).chunks(1, 100) == 1 and syn(7, 1).chunks(1, 5) == 5
  assert syn(1).chunks(1, 10 ** 6) == 1
  assert ab.LpcFilter(16, 480, "analysis", time_parallel=64).chunks(1, 10 ** 6) == 1
  assert ab.LpcFilter(16, 480, "analysis", time_parallel=True).chunks(1, 10 ** 6) == 1


def test_constructor_errors():
  for bad in (0, -3):
    with pytest.raises(ValueError):
      ab.LpcFilter(4, 10, "synthesis", time_parallel=bad)
  for bad in (2.0, "yes", None, [4]):
    with pytest.raises(TypeError):
      ab.LpcFilter(4, 10, "synthesis", time_parallel=bad)
  assert ab.LpcFilter(4, 10, "synthesis").time_parallel is False
  assert ab.LpcFilter(4, 10, "synthesis", time_parallel=np.int64(9)).time_parallel == 9
  assert ab.LpcFilter(4, 10, time_parallel=True).time_parallel is True


# --- the library ----------------------------------------------------------------------------------------------------

def test_library_checks_without_a_device():
  L = lp.LPCSCAN_LIB.load()
  args = dict(x=None, xt=0, xs=8, out=None, ot=1, os=8, coef=None, crs=3, ccs=3, F=2, state=None, S=1, T=8, C=0,
              order=2, hop=4, P=2, scratch=None, nbytes=1 << 20, stream=None)

  def call(**kw):
    a = dict(args, **kw)
    return L.alz_lpcscan_apply(*a.values())

  def msg():
    return L.alz_lpcscan_last_error().decode()

  assert call(order=65) < 0 and "order" in msg()
  assert call(hop=0) < 0 and "hop" in msg()
  assert call(xt=3) < 0 and "dtype" in msg()
  assert call(P=0) < 0 and "n_chunks" in msg()
  assert call(P=5) < 0 and "n_chunks" in msg()                  # 8 samples at order 2: at most 4 chunks
  assert call(F=1) < 0 and "needs 2" in msg()
  assert call(nbytes=8) < 0 and "scratch" in msg()
  assert call() < 0 and "NULL" in msg()
  ok = dict(x=8, out=8, coef=8, state=8, scratch=8)
  assert call(crs=2, **ok) < 0 and "row stride" in msg()
  assert call(S=2, xs=4, **ok) < 0 and "stride" in msg()
  assert call(ccs=-1, **ok) < 0 and "stream stride" in msg()
  assert call(xt=1, **dict(ok, x=4)) < 0 and "misaligned" in msg()
  assert call(T=0, F=0, P=1) == 0 and call(S=0) == 0
  assert L.alz_lpcscan_scratch_bytes(1, 1, 0) == 8
  assert L.alz_lpcscan_scratch_bytes(3, 10, 16) == 8 * (3 * 10 * 16 * 17 + 3 * 11 * 16) + 16
  assert L.alz_lpcscan_scratch_bytes(1, 0, 4) < 0 and L.alz_lpcscan_scratch_bytes(1, 2, 65) < 0
  with pytest.raises(ValueError, match="n_chunks"):
    lp.LPCSCAN_LIB.check(call(P=0))


def test_apply_needs_a_device():
  torch = pytest.importorskip("torch")
  if torch.cuda.is_available():
    pytest.skip("a CUDA device is present")
  with pytest.raises(_capi.NativeError):
    ab.LpcFilter(2, 4, "synthesis", time_parallel=True).apply(torch.zeros((1, 8)),
                                                              torch.zeros((1, 2, 3), dtype=torch.float64))


def test_lpcscan_walks_contract_nothing():
  """Built with -fmad=false: the 33 walk kernels (the register walk for each order 1 .. 32 and the shared-memory
  walk), which give a flagged stream its sequential bits, hold no DFMA; only the scan contracts."""
  sass = subprocess.run([cuobjdump(), "-sass", _build.LIBRARIES["lpcscan"].path], capture_output=True, text=True).stdout
  functions = re.split(r"\n\s*Function : ", sass)[1:]
  assert len(functions) == 34
  names = [body.split(None, 1)[0] for body in functions]
  assert sum("alz_lpcscan_walk_reg_kernel" in n for n in names) == 32
  assert sum("alz_lpcscan_walk_kernel" in n for n in names) == 1
  assert sum("alz_lpcscan_scan_kernel" in n for n in names) == 1
  for name, body in zip(names, functions):
    if "scan_kernel" in name:
      assert "DFMA" in body, name
    else:
      assert not re.search(r"\bDFMA\b", body) and "DMUL" in body and "DADD" in body, name
