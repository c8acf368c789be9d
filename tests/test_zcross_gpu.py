"""zcross / Zcross on the GPU: the lazy call against the reference's answers, the batched flags and block counts
against the numpy emulation, blocks carried through a ZcrossState, long and silent streams, concurrent CUDA streams,
state misuse, and coverage of every kernel in libalz_b200_zcross.so.  Every comparison is exact."""
import itertools as it
import json
import math
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import GOLDEN
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
from zcross_emulation import block_sums, digest, zcross as emulate

sys.path.insert(0, GOLDEN)
from make_zcross import inputs  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "zcross_cases.json")) as fh:
    return json.load(fh)


def test_lazy_call_equals_the_reference(torch, golden):
  xs = inputs()
  for case in golden["cases"]:
    x = xs[case["input"]]
    got = list(ab.zcross(x.astype(np.float64).tolist(), float(case["hysteresis"]), float(case["first_sign"])))
    assert all(type(v) is int for v in got[:50])
    got = np.array(got, dtype=np.uint8)
    assert digest(got, "u1") == case["digest"], (case["input"], case["hysteresis"], case["first_sign"])
    zc = ab.Zcross(float(case["hysteresis"]), float(case["first_sign"]))
    xd = torch.from_numpy(x).cuda()
    for b in case["blocks"]:
      sums = zc.counts(xd, b["size"], b["hop"], final=True)[0].cpu().numpy()
      assert digest(sums, "<i4") == b["digest"], (case["input"], case["hysteresis"], case["first_sign"], b)


def test_lazy_call_on_an_endless_iterator(torch, golden):
  x = inputs()["tone"]
  case = next(c for c in golden["cases"] if c["input"] == "tone" and c["hysteresis"] == "0.01" and c["first_sign"] == "-3")
  src = it.chain(x.astype(np.float64).tolist(), it.repeat(0.))
  got = np.array(list(it.islice(ab.zcross(src, .01, -3), len(x))), dtype=np.uint8)
  assert digest(got, "u1") == case["digest"]


def noise(rng, S, T):
  x = rng.uniform(-1, 1, (S, T)).astype(np.float32)
  x[:, ::7] *= np.float32(1e-3)                  # samples inside the hysteresis band
  return x


@pytest.mark.parametrize("S", [1, 3, 33, 4096])
def test_apply_and_counts_against_the_emulation(torch, S):
  rng = np.random.default_rng(S)
  for T in ([0, 1, 5, 4095, 4096, 4097, 12289, 20000] if S < 4096 else [0, 1, 4099, 16384]):
    x = noise(rng, S, T)
    xd = torch.from_numpy(x).cuda()
    for h, fs in ((0., 0), (.01, -1), (-.5, 2)):
      zc = ab.Zcross(h, fs)
      want = emulate(x, h, fs)
      assert np.array_equal(zc.apply(xd).cpu().numpy(), want), (S, T, h, fs)
      for size, hop in ((2048, 1024), (5, 5), (3, 11)):
        got = zc.counts(xd, size, hop, final=True).cpu().numpy()
        assert np.array_equal(got, block_sums(want, size, hop)), (S, T, h, fs, size, hop)


def test_one_long_stream_strided_and_unaligned(torch):
  T = 10 ** 7 + 37
  rng = np.random.default_rng(7)
  x = noise(rng, 1, T + 3)
  xd = torch.from_numpy(x).cuda()
  zc = ab.Zcross(.01, 0)
  for o in (0, 1, 2, 3):                          # rows starting 0, 4, 8 and 12 bytes past a 16-byte boundary
    want = emulate(x[:, o:o + T], .01)
    assert np.array_equal(zc.apply(xd[:, o:o + T]).cpu().numpy(), want), o
  got = zc.counts(xd[:, 1:1 + T], 2048, 1024, final=True).cpu().numpy()
  assert np.array_equal(got, block_sums(emulate(x[:, 1:1 + T], .01), 2048, 1024))
  # several streams with a row stride that is not a multiple of 4 floats, and a column stride of 2
  y = noise(rng, 5, 2 * 9001)
  yd = torch.from_numpy(y).cuda()
  assert np.array_equal(zc.apply(yd[:, 3:9004]).cpu().numpy(), emulate(y[:, 3:9004], .01))
  assert np.array_equal(zc.apply(yd[:, ::2]).cpu().numpy(), emulate(y[:, ::2], .01))


def _split(T, rng):
  lengths = [0, 1, 3, 0, 4096, 1, 5000] + [int(v) for v in rng.integers(0, 9000, 6)]
  return lengths + [T - sum(lengths)]


@pytest.mark.parametrize("size,hop", [(None, None), (2048, 1024), (4, 3), (16, 40), (1, 1), (7, 7)])
def test_block_splits_equal_one_call(torch, size, hop):
  S, T = 3, 60000
  rng = np.random.default_rng(3 if size is None else size * 100 + hop)
  x = noise(rng, S, T + 1)
  xd = torch.from_numpy(x).cuda()[:, 1:]
  zc = ab.Zcross(.15, -0.)
  if size is None:
    whole = zc.apply(xd)
  else:
    whole = zc.counts(xd, size, hop, final=True)
  state = zc.new_state(S, size=size, hop=hop)
  parts, t = [], 0
  lengths = _split(T, rng)
  for i, n in enumerate(lengths):
    if size is None:
      parts.append(zc.apply(xd[:, t:t + n], state=state))
    else:
      parts.append(zc.counts(xd[:, t:t + n], size, hop, state=state, final=i == len(lengths) - 1))
    t += n
  assert t == T and state.consumed == T
  assert torch.equal(torch.cat(parts, dim=-1), whole)
  want = emulate(x[:, 1:], .15)
  assert np.array_equal(whole.cpu().numpy(), want if size is None else block_sums(want, size, hop))


def test_silent_streams(torch):
  """One decisive sample, then 10^6 zeros (the look-back crosses every tile), then a crossing; and a stream that is
  never decisive.  Both also carried over two calls."""
  T = 10 ** 6 + 2
  x = np.zeros((2, T), dtype=np.float32)
  x[0, 0], x[0, -1] = .5, -.5
  x[1] = 1e-3
  xd = torch.from_numpy(x).cuda()
  zc = ab.Zcross(.01)
  got = zc.apply(xd).cpu().numpy()
  assert np.array_equal(got, emulate(x, .01)) and got[0].sum() == 1 and got[0, -1] == 1 and got[1].sum() == 0
  state = zc.new_state(2, size=4096, hop=1000)
  a = zc.counts(xd[:, :T // 2], 4096, 1000, state=state)
  b = zc.counts(xd[:, T // 2:], 4096, 1000, state=state, final=True)
  assert np.array_equal(torch.cat([a, b], dim=-1).cpu().numpy(), block_sums(emulate(x, .01), 4096, 1000))
  one = ab.Zcross(0, 1).apply(torch.zeros((1, 3 * 4096 + 5), device="cuda"))
  assert int(one.sum()) == 0


def test_two_cuda_streams_at_once(torch):
  rng = np.random.default_rng(9)
  xa, xb = noise(rng, 64, 300000), noise(rng, 1, 5 * 10 ** 6)
  da, db = torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda()
  zc = ab.Zcross(.01, 0)
  sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
  torch.cuda.synchronize()
  outs = []
  for _ in range(3):
    with torch.cuda.stream(sa):
      ya = zc.apply(da)
      ca = zc.counts(da, 2048, 1024, final=True)
    with torch.cuda.stream(sb):
      yb = zc.apply(db)
      cb = zc.counts(db, 2048, 1024, final=True)
    outs.append((ya, ca, yb, cb))
  torch.cuda.synchronize()
  wa, wb = emulate(xa, .01), emulate(xb, .01)
  for ya, ca, yb, cb in outs:
    assert np.array_equal(ya.cpu().numpy(), wa) and np.array_equal(yb.cpu().numpy(), wb)
    assert np.array_equal(ca.cpu().numpy(), block_sums(wa, 2048, 1024))
    assert np.array_equal(cb.cpu().numpy(), block_sums(wb, 2048, 1024))


def test_state_checks(torch):
  zc = ab.Zcross(.1, 0)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    zc.apply(x, state=zc.new_state(3))
  with pytest.raises(ValueError, match="hysteresis"):
    zc.apply(x, state=ab.Zcross(.2, 0).new_state(2))
  with pytest.raises(ValueError, match="first_sign"):
    zc.apply(x, state=ab.Zcross(.1, -1).new_state(2))
  with pytest.raises(ValueError, match="size"):
    zc.apply(x, state=zc.new_state(2, size=8))
  with pytest.raises(ValueError, match="size"):
    zc.counts(x, 8, 4, state=zc.new_state(2, size=8))
  with pytest.raises(ValueError, match="size"):
    zc.counts(x, 8, state=zc.new_state(2))
  with pytest.raises(ValueError, match="Zcross.new_state"):
    zc.apply(x, state=object())
  with pytest.raises(ValueError):
    zc.counts(x, 0)
  with pytest.raises(ValueError):
    zc.counts(x, 8, 0)
  with pytest.raises(ValueError):
    zc.new_state(2, size=0)
  if torch.cuda.device_count() > 1:
    with torch.cuda.device(1):
      other = zc.new_state(2)
    with pytest.raises(ValueError, match="lives on"):
      zc.apply(x, state=other)
  state = zc.new_state(2, size=8)
  zc.counts(x, 8, state=state, final=True)
  with pytest.raises(ValueError, match="final"):
    zc.counts(x, 8, state=state)
  nan = ab.Zcross(math.nan, 2)                               # an equal Zcross may use the state, NaN hysteresis too
  assert ab.Zcross(math.nan, 5).apply(x, state=nan.new_state(2)).shape == (2, 100)


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  zc = ab.Zcross(.01)
  zc.apply(x)
  zc.counts(x, 64, 32, final=True)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_zcross" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_zcross_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["zcross"].path, _LAUNCH_PROBE)
