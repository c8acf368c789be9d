"""unwrap / Unwrap and clip / Clip on the GPU: every golden through the lazy and the batched calls, the batched kernel
against the emulation at tile edges, batch shapes, both dtypes, block cuts, long streams, strided rows and the
phase-vocoder shape, failures, concurrency, state misuse and coverage of every kernel in libalz_b200_unwrap.so.
Every comparison is bit for bit (NaN by NaN-ness)."""
import builtins
import itertools as it
import json
import math
import os
import re
import sys
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import GOLDEN
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
import unwrap_emulation as em

sys.path.insert(0, GOLDEN)
import make_unwrap  # noqa: E402

pytestmark = pytest.mark.gpu
TILE = 2048


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "unwrap_cases.json")) as fh:
    return json.load(fh)


def params(c):
  return eval(c["params"], make_unwrap.env())


def bits(a):
  a = np.array(a, dtype=np.float64)
  a[np.isnan(a)] = np.nan
  return a.tobytes()


def check_case(c, values):
  values = list(values)
  assert len(values) == c["n"], (c["input"], c["params"])
  if values:
    assert make_unwrap.digest(values) == c["digest"], (c["input"], c["params"])


def test_every_golden_lazily_and_batched(torch, golden):
  xs = make_unwrap.inputs()
  for c in golden["cases"]:
    x = xs[c["input"]]
    m, p = params(c)
    exc = c.get("exception")
    s = ab.unwrap(x.tolist(), m, p)
    if exc is None:
      got = list(s)
      assert all(type(v) is float for v in got[:20])
      check_case(c, got)
    else:
      got = []
      with pytest.raises(getattr(builtins, exc[0]), match=re.escape(exc[1])):
        for v in s:
          got.append(v)
      check_case(c, got)
    if len(x):
      uw = ab.Unwrap(m, p)
      state = uw.new_state(1)
      y = uw.apply(torch.from_numpy(x).cuda(), state=state)[0].cpu().numpy()
      fail = int(state.failures()[0])
      if exc is None:
        assert fail == -1
        check_case(c, y)
      else:
        assert fail == c["n"]
        check_case(c, y[:fail])
        assert np.isnan(y[fail:]).all()


def test_every_clip_golden(torch, golden):
  xs = make_unwrap.inputs()
  for c in golden["clips"]:
    low, high = params(c)
    if "exception" in c:
      with pytest.raises(ValueError, match="smaller than lower"):
        ab.clip(xs[c["input"]].tolist(), low, high)
      continue
    check_case(c, ab.clip(xs[c["input"]].tolist(), low, high))
    if low is None and high is None:
      continue
    x = torch.from_numpy(xs[c["input"]]).cuda()
    check_case(c, ab.Clip(low, high).apply(x)[0].cpu().numpy())


@pytest.mark.parametrize("S", [1, 3, 65, 1000, 100000])
def test_tile_edges_against_the_emulation(torch, S):
  rng = np.random.default_rng(S)
  Ts = [1, 2, 31, 32, 33, TILE // 2, TILE - 1, TILE, TILE + 1, 3 * TILE + 5, 9 * TILE]
  if S >= 1000:
    Ts = [1, 33, TILE - 1, TILE + 1] if S == 1000 else [1, 32, 33]
  for T in Ts:
    x = rng.uniform(-2 * np.pi, 2 * np.pi, (S, T))
    x[:, ::5] = np.angle(np.exp(1j * x[:, ::5]))
    want, _ = em.unwrap_batch(x, np.pi, 2 * np.pi)
    uw = ab.Unwrap()
    for xd in (torch.from_numpy(x).cuda(), torch.from_numpy(x.astype(np.float32)).cuda()):
      w = want if xd.dtype == torch.float64 else em.unwrap_batch(x.astype(np.float32), np.pi, 2 * np.pi)[0]
      y64 = uw.apply(xd).cpu().numpy()
      assert bits(y64) == bits(w), (S, T, xd.dtype)
      y32 = uw.apply(xd, out_dtype=torch.float32).cpu().numpy()
      assert y32.dtype == np.float32 and bits(y32) == bits(w.astype(np.float32)), (S, T, xd.dtype)


def _cuts(T, rng):
  lengths = [0, 1, 3, 0, TILE, 1, 5000] + [int(v) for v in rng.integers(0, 9000, 6)]
  return lengths + [T - sum(lengths)]


@pytest.mark.parametrize("S", [1, 5, 300])
def test_block_cuts_equal_one_call(torch, S):
  T = 60000 if S < 300 else 40000
  rng = np.random.default_rng(S + 11)
  x = np.angle(np.exp(1j * np.cumsum(rng.uniform(-.5, 3, (S, T + 1)), axis=1)))
  xd = torch.from_numpy(x).cuda()[:, 1:]
  uw = ab.Unwrap(2., 2 * np.pi)
  whole = uw.apply(xd)
  state = uw.new_state(S)
  parts, t = [], 0
  for n in _cuts(T, rng):
    parts.append(uw.apply(xd[:, t:t + n], state=state))
    t += n
  assert t == T and state.consumed == T
  assert bits(torch.cat(parts, dim=-1).cpu().numpy()) == bits(whole.cpu().numpy())
  assert bits(whole.cpu().numpy()) == bits(em.unwrap_batch(x[:, 1:], 2., 2 * np.pi)[0])


@pytest.mark.parametrize("kind", ["never", "every_50", "every_sample"])
def test_one_long_stream(torch, kind):
  T = 2880000
  n = np.arange(T)
  if kind == "never":
    x = 1e-6 * n
  elif kind == "every_50":
    x = np.angle(np.exp(1j * 2 * np.pi * n / 50.3))
  else:
    x = np.where(n % 2 == 0, 0., 5.) + 1e-7 * n
  want, _ = em.unwrap_batch(x, np.pi, 2 * np.pi)
  got = ab.Unwrap().apply(torch.from_numpy(x).cuda())[0].cpu().numpy()
  assert bits(got) == bits(want[0])


def test_strided_and_misaligned_rows(torch):
  rng = np.random.default_rng(4)
  x = rng.uniform(-6, 6, (7, 2 * 5001 + 3))
  xd = torch.from_numpy(x).cuda()
  uw = ab.Unwrap()
  for sl in (np.s_[:, 1:5002], np.s_[:, 3:5004], np.s_[:, ::2], np.s_[::2, 5:4100]):
    want = em.unwrap_batch(x[sl], np.pi, 2 * np.pi)[0]
    assert bits(uw.apply(xd[sl]).cpu().numpy()) == bits(want), sl
    x32 = x.astype(np.float32)
    want32 = em.unwrap_batch(x32[sl], np.pi, 2 * np.pi)[0]
    assert bits(uw.apply(torch.from_numpy(x32).cuda()[sl]).cpu().numpy()) == bits(want32), sl
  c = ab.Clip(-.5, .25)
  assert bits(c.apply(xd[:, 3:5004]).cpu().numpy()) == bits(em.clip(x[:, 3:5004], -.5, .25))
  assert bits(c.apply(xd[:, ::2], out_dtype=torch.float32).cpu().numpy()) == \
    bits(em.clip(x[:, ::2], -.5, .25).astype(np.float32))


def test_phase_vocoder_shape(torch):
  """513 bins x 4096 streams of 32 frames each (2.1M rows), phases of a float32 STFT table."""
  S, T = 513 * 4096, 32
  g = torch.Generator("cuda").manual_seed(3)
  xd = (torch.rand((S, T), device="cuda", generator=g) * 2 - 1) * math.pi
  xd += torch.arange(T, device="cuda") * 1.3
  xd = torch.remainder(xd + math.pi, 2 * math.pi) - math.pi
  y = ab.Unwrap().apply(xd)
  rows = np.r_[0:2000, S - 3000:S]
  want = em.unwrap_batch(xd[rows].cpu().numpy(), np.pi, 2 * np.pi)[0]
  assert bits(y[rows].cpu().numpy()) == bits(want)
  sample = torch.randint(0, S, (20000,), device="cuda", generator=g)
  assert bits(y[sample].cpu().numpy()) == bits(em.unwrap_batch(xd[sample].cpu().numpy(), np.pi, 2 * np.pi)[0])


def test_clip_both_dtypes(torch):
  rng = np.random.default_rng(8)
  x = rng.uniform(-3, 3, (33, 4099))
  x[0, :6] = [np.nan, -0., 0., np.inf, -np.inf, 1.0000000001]
  for low, high in ((-1., 1.), (None, .1), (-.3, None), (-0., 0.), (math.nan, 1.)):
    for dt in (np.float64, np.float32):
      xd = torch.from_numpy(x.astype(dt)).cuda()
      want = em.clip(x.astype(dt), low, high)
      got = ab.Clip(low, high).apply(xd)
      assert got.dtype == xd.dtype and bits(got.cpu().numpy()) == bits(want.astype(dt)), (low, high, dt)
      got64 = ab.Clip(low, high).apply(xd, out_dtype=torch.float64).cpu().numpy()
      assert bits(got64) == bits(want), (low, high, dt)


def test_inf_in_one_stream_leaves_the_others_untouched(torch):
  rng = np.random.default_rng(6)
  x = rng.uniform(-7, 7, (4, 3 * TILE + 7))
  x[2, TILE + 3] = np.inf
  y = ab.Unwrap().apply(torch.from_numpy(x).cuda()).cpu().numpy()
  want = em.unwrap_batch(x, np.pi, 2 * np.pi)[0]
  assert bits(y) == bits(want)
  assert np.isnan(y[2, TILE + 3:]).all() and not np.isnan(y[[0, 1, 3]]).any()


def test_step_zero_index_and_lazy_error(torch):
  x = np.zeros((3, 3 * TILE), dtype=np.float64)
  x[0, 5000] = 10.
  x[1, 7] = 10.
  uw = ab.Unwrap(math.pi, 0.)
  state = uw.new_state(3)
  a = uw.apply(torch.from_numpy(x[:, :4000]).cuda(), state=state)
  assert state.failures().tolist() == [-1, 7, -1]
  b = uw.apply(torch.from_numpy(x[:, 4000:]).cuda(), state=state)
  assert state.failures().tolist() == [5000, 7, -1]
  y = torch.cat([a, b], dim=1).cpu().numpy()
  assert np.isnan(y[0, 5000:]).all() and not np.isnan(y[0, :5000]).any() and not np.isnan(y[2]).any()
  got = []
  with pytest.raises(ZeroDivisionError, match="float modulo"):
    for v in ab.unwrap(it.chain(x[0].tolist(), it.repeat(0.)), math.pi, 0):
      got.append(v)
  assert got == [0.0] * 5000
  assert list(ab.unwrap([1., 2., 3.], 5, 0)) == [1., 2., 3.]   # no jump: no error
  with pytest.raises(RuntimeError, match="StopIteration"):
    list(ab.unwrap([]))


def test_lazy_call_on_an_endless_iterator(torch, golden):
  x = make_unwrap.inputs()["tone"]
  case = next(c for c in golden["cases"] if c["input"] == "tone" and c["params"] == "(pi, 2 * pi)")
  got = list(it.islice(ab.unwrap(it.chain(x.tolist(), it.repeat(0.))), len(x)))
  check_case(case, got)


def test_one_unwrap_on_several_streams_and_threads(torch):
  rng = np.random.default_rng(12)
  xa = torch.from_numpy(rng.uniform(-9, 9, (64, 30000))).cuda()
  xb = torch.from_numpy(rng.uniform(-9, 9, (1, 500000)).astype(np.float32)).cuda()
  uw = ab.Unwrap()
  wa, wb = uw.apply(xa).cpu().numpy(), uw.apply(xb, out_dtype=torch.float32).cpu().numpy()
  torch.cuda.synchronize()
  results, errors = [], []

  def work(x, out_dtype, want):
    try:
      s = torch.cuda.Stream()
      with torch.cuda.stream(s):
        ys = [uw.apply(x, out_dtype=out_dtype) for _ in range(3)]
      s.synchronize()
      results.append(all(bits(y.cpu().numpy()) == bits(want) for y in ys))
    except Exception as exc:   # reported below
      errors.append(exc)

  threads = [threading.Thread(target=work, args=a) for a in ((xa, torch.float64, wa), (xb, torch.float32, wb)) * 2]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  assert not errors and results == [True] * 4


def test_state_checks(torch):
  uw = ab.Unwrap(1., 3.)
  x = torch.zeros((2, 100), dtype=torch.float64, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    uw.apply(x, state=uw.new_state(3))
  with pytest.raises(ValueError, match="max_delta or step"):
    uw.apply(x, state=ab.Unwrap(1., 4.).new_state(2))
  with pytest.raises(ValueError, match="Unwrap.new_state"):
    uw.apply(x, state=object())
  with pytest.raises(ValueError, match="float32 or float64"):
    uw.apply(x.to(torch.int32))
  with pytest.raises(ValueError, match="out_dtype"):
    uw.apply(x, out_dtype=torch.float16)
  with pytest.raises(ValueError, match="CUDA"):
    uw.apply(x.cpu())
  if torch.cuda.device_count() > 1:
    with torch.cuda.device(1):
      other = uw.new_state(2)
    with pytest.raises(ValueError, match="lives on"):
      uw.apply(x, state=other)
  nan = ab.Unwrap(math.nan, 2.)
  assert ab.Unwrap(math.nan, 2.).apply(x, state=nan.new_state(2)).shape == (2, 100)
  assert uw.apply(torch.zeros((0, 5), dtype=torch.float64, device="cuda")).shape == (0, 5)


def test_the_smoke_example(torch):
  assert list(ab.unwrap([0., 10., 20., 30., 2., 3., 4.], max_delta=8, step=10)) == [0.0, 0.0, 0.0, 0.0, 2.0, 3.0, 4.0]
  assert repr(list(ab.clip([-2., math.nan, -0., .5, 3.], low=-0., high=1.))) == "[-0.0, nan, -0.0, 0.5, 1.0]"


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((3, 5000), device="cuda", dtype=torch.float64) * 20
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for xd in (x, x.float()):
    for od in (torch.float32, torch.float64):
      ab.Unwrap().apply(xd, out_dtype=od)
      ab.Clip(-1., 1.).apply(xd, out_dtype=od)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_unwrap_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["unwrap"].path, _LAUNCH_PROBE)
