"""amdf / AmdfBank on the GPU: the lazy call against the reference's answers, the batched kernel against the float64
emulation, blocks carried through an AmdfState, the time-parallel evaluation of few long streams, and coverage of
every kernel in libalz_b200_amdf.so."""
import json
import os

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from amdf_emulation import amdf as emulate, amdf_bank as emulate_bank, digest
from conftest import GOLDEN, signal
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "amdf_cases.json")) as fh:
    return json.load(fh)


def mixed_lags(n, lo=0.4, hi=800.0, seed=3):
  """Integer and fractional lags over [lo, hi], lag 0 and a lag below 1."""
  rng = np.random.default_rng(seed)
  frac = rng.uniform(lo, hi, n // 2)
  whole = rng.integers(int(lo) + 1, int(hi), n - n // 2 - 2)
  return [0, 0.4] + [float(v) for v in frac] + [int(v) for v in whole]


def test_lazy_call_equals_the_reference(torch, golden):
  """list(amdf(lag, size)(x, zero=zero)) is float32(reference) exactly, for every golden case."""
  for case in golden["cases"]:
    x = signal(case["seed"], case["length"])
    got = np.array(list(ab.amdf(case["lag"], case["size"])(x.astype(np.float64).tolist(), zero=case["zero"])))
    want = emulate(x, [tuple(t) for t in case["taps"]], case["size"], case["zero"])
    assert digest(want) == case["digest"]                # the emulation is the reference, bit for bit
    assert len(got) == case["length"]
    assert np.array_equal(got, want.astype(np.float32).astype(np.float64)), case
    assert np.array_equal(got[::case["step"]], np.float32(case["values"]).astype(np.float64))


def test_lazy_call_on_an_endless_iterator(torch):
  import itertools as it
  x = signal(5, 3000)
  s = ab.amdf(12.5, 40)(iter(x.tolist()), zero=.25)
  got = np.array(list(it.islice(s, 3000)))
  want = emulate(x, ab.AmdfBank([12.5], 40).taps[0], 40, .25)
  assert np.array_equal(got, want.astype(np.float32).astype(np.float64))


def test_bank_streams(torch):
  x = signal(6, 2500)
  lags = [0.4, 7, 99.75]
  streams = ab.AmdfBank(lags, 64)(x.tolist(), zero=-.3)
  for lag, s in zip(reversed(lags), reversed(streams)):       # a lag consumed first buffers the others
    want = emulate(x, ab.AmdfBank([lag], 64).taps[0], 64, -.3)
    assert np.array_equal(np.array(list(s)), want.astype(np.float32).astype(np.float64))


def test_batched_apply_sequential_plan(torch):
  """64 streams x 20000 samples, 210 mixed lags: the sequential plan equals float32(emulation) exactly; the default
  plan (time-parallel at this shape) agrees to <= 1e-5 of each row's peak."""
  S, T, size, zero = 64, 20000, 333, .25
  lags = mixed_lags(210)
  x = np.random.default_rng(11).uniform(-1, 1, (S, T)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()
  seq = ab.AmdfBank(lags, size, sequential=True)
  assert seq.chunks(S, T) == 1
  y = seq.apply(xd, state=seq.new_state(S, zero=zero))
  par = ab.AmdfBank(lags, size)
  assert par.chunks(S, T) > 1
  yp = par.apply(xd, state=par.new_state(S, zero=zero))
  torch.cuda.synchronize()
  assert tuple(y.shape) == (S, len(lags), T)
  worst = 0.0
  for l0 in range(0, len(lags), 16):
    ls = list(range(l0, min(l0 + 16, len(lags))))
    want = emulate_bank(x, [seq.taps[l] for l in ls], size, zero).astype(np.float32)
    got = y[:, ls].cpu().numpy()
    assert np.array_equal(got, want), "lags %s" % [lags[l] for l in ls]
    gp = yp[:, ls].cpu().numpy().astype(np.float64)
    peak = np.maximum(np.max(np.abs(want), axis=-1), 1e-30)
    worst = max(worst, float(np.max(np.max(np.abs(gp - want), axis=-1) / peak)))
  print("time-parallel vs sequential at 64 x 20000: max rel err %.3g" % worst)
  assert worst <= 1e-5


def test_long_delay_plan_after_a_short_delay_plan(torch):
  """A plan whose tap window needs more than 48 KB of shared memory (delays over ~990 samples) keeps working after a
  plan with a short delay is created, batched and lazily."""
  x = signal(12, 5000)
  xd = torch.from_numpy(x).cuda()
  long_bank = ab.AmdfBank([1500, 1200.5, 48], 64)
  state = long_bank.new_state(1, zero=.25)
  short_bank = ab.AmdfBank([3], 4)
  short_bank.apply(xd, state=short_bank.new_state(1))
  got = long_bank.apply(xd, state=state)[0].cpu().numpy()
  for l, taps in enumerate(long_bank.taps):
    assert np.array_equal(got[l], emulate(x, taps, 64, .25).astype(np.float32)), long_bank.lags[l]
  a = ab.amdf(1500, 64)(x.tolist())
  b = ab.amdf(3, 4)(x.tolist())
  assert np.array_equal(np.array(list(a)), emulate(x, long_bank.taps[0], 64).astype(np.float32).astype(np.float64))
  assert np.array_equal(np.array(list(b)), emulate(x, short_bank.taps[0], 4).astype(np.float32).astype(np.float64))


def test_infinite_inputs_follow_the_reference(torch):
  """inf / -inf samples: a lag with one tap (its z^0 coefficient cancels), two, three or none gives what the float64
  emulation gives (inf, NaN from inf - inf), not a NaN from an unused tap."""
  x = signal(13, 400)
  x[[37, 200]] = [np.inf, -np.inf]
  for lags in ([1e-20, 3, 2.5, 0], [1e-20, 3]):                # a 3-tap and a 2-tap group with a 1-tap lag in it
    bank = ab.AmdfBank(lags, 8)
    assert [len(t) for t in bank.taps] == [1, 2, 3, 0][:len(lags)]
    got = bank.apply(torch.from_numpy(x).cuda(), state=bank.new_state(1, zero=.25))[0].cpu().numpy()
    for l, taps in enumerate(bank.taps):
      with np.errstate(invalid="ignore"):
        want = emulate(x, taps, 8, .25).astype(np.float32)
      assert np.array_equal(got[l], want, equal_nan=True), lags[l]
    assert np.isinf(got[0]).any()


def _split(T, decim, rng):
  lengths = [0, 1, decim - 1, 5, 0, 3, 301, 2]
  lengths += [int(v) for v in rng.integers(0, 700, 4)]
  return lengths + [T - sum(lengths)]


@pytest.mark.parametrize("decim", [1, 7, 256])
def test_block_splits_are_bit_identical(torch, decim):
  """Blocks of lengths 0, 1, decim - 1 and random ones, starting at unaligned addresses, carried through the state,
  give the same bits as one call; one call equals float32(emulation) at every decim-th sample."""
  S, T, size, zero = 3, 6000, 150, -.3
  lags = [0, 0.4, 3, 37.25, 150, 255.5, 799.9]
  bank = ab.AmdfBank(lags, size)
  x = np.random.default_rng(decim).uniform(-1, 1, (S, T + 1)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()[:, 1:]                     # rows start 4 bytes past an aligned address
  whole = bank.apply(xd, decim=decim, state=bank.new_state(S, decim=decim, zero=zero))
  want = emulate_bank(x[:, 1:], bank.taps, size, zero)[:, :, decim - 1::decim].astype(np.float32)
  assert np.array_equal(whole.cpu().numpy(), want)
  state = bank.new_state(S, decim=decim, zero=zero)
  parts, t = [], 0
  for n in _split(T, decim, np.random.default_rng(100 + decim)):
    parts.append(bank.apply(xd[:, t:t + n], decim=decim, state=state))
    t += n
  assert t == T and state.phase == T % decim
  assert torch.equal(torch.cat(parts, dim=-1), whole)


def test_state_checks(torch):
  bank = ab.AmdfBank([3, 4.5], 16)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    bank.apply(x, state=bank.new_state(3))
  with pytest.raises(ValueError, match="decim"):
    bank.apply(x, decim=2, state=bank.new_state(2, decim=3))
  with pytest.raises(ValueError, match="another bank"):
    bank.apply(x, state=ab.AmdfBank([3], 16).new_state(2))
  with pytest.raises(ValueError, match="AmdfBank.new_state"):
    bank.apply(x, state=object())
  if torch.cuda.device_count() > 1:
    with torch.cuda.device(1):
      other = bank.new_state(2)
    with pytest.raises(ValueError, match="lives on"):
      bank.apply(x, state=other)
  same = ab.AmdfBank([3, 4.5], 16)                           # an equal bank may use the state
  assert same.apply(x, state=bank.new_state(2)).shape == (2, 2, 100)


@pytest.mark.parametrize("S", [1, 3])
def test_time_parallel(torch, S):
  """Few long streams: T = 10^6 + 37 after a 5-sample block (nonzero phase), 256 lags over 48...800, against the
  sequential plan; then a short block continues both states."""
  T, size, decim, zero = 10 ** 6 + 37, 1024, 7, .25
  lags = mixed_lags(256, lo=48.0, hi=800.0, seed=S)
  x = torch.from_numpy(np.random.default_rng(S).uniform(-1, 1, (S, 5 + T + 999)).astype(np.float32)).cuda()
  outs = {}
  for name, bank in (("seq", ab.AmdfBank(lags, size, sequential=True)), ("par", ab.AmdfBank(lags, size))):
    state = bank.new_state(S, decim=decim, zero=zero)
    a = bank.apply(x[:, :5], decim=decim, state=state)
    assert state.phase == 5
    chunks = bank.chunks(S, T)
    b = bank.apply(x[:, 5:5 + T], decim=decim, state=state)
    c = bank.apply(x[:, 5 + T:], decim=decim, state=state)
    outs[name] = (torch.cat([a, b, c], dim=-1), chunks)
  (ys, cs), (yp, cp) = outs["seq"], outs["par"]
  assert cs == 1 and cp > 1, (cs, cp)
  assert ys.shape == (S, 256, (5 + T + 999) // decim)
  err = ((yp.double() - ys.double()).abs().amax(dim=-1) / ys.double().abs().amax(dim=-1).clamp_min(1e-30)).max().item()
  print("time-parallel, S=%d, %d chunks: max rel err %.3g" % (S, cp, err))
  assert err <= 1e-5


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.from_numpy(np.random.default_rng(8).uniform(-1, 1, 3000).astype(np.float32)).cuda()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for lags in ([3, 48], [2.5, 48.25]):          # the 2-tap and the 3-tap body
    bank = ab.AmdfBank(lags, 32)
    bank.apply(x, decim=4, state=bank.new_state(1, decim=4))
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_amdf" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_amdf_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["amdf"].path, _LAUNCH_PROBE)
