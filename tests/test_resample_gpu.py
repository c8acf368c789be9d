"""Resampler / resample on the GPU: every golden bit for bit in float64 and as its float32 rounding, streams cut into
blocks of any lengths, batch shapes, strided and misaligned buffers, the lazy API, concurrent use, state misuse, and
coverage of every kernel in libalz_b200_resample.so."""
import builtins
import sys
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, resampling
import resample_emulation as em
from conftest import GOLDEN
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
from test_resample import case_id, check_case, golden  # noqa: F401  (fixture)

sys.path.insert(0, GOLDEN)
import make_resample  # noqa: E402

pytestmark = pytest.mark.gpu

INPUTS = make_resample.inputs()


def same(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def resampler(c):
  return ab.Resampler(c["old"], c["new"], c["order"], make_resample.dec(c["zero"]))


def test_every_golden_bit_for_bit(torch, golden):
  for c in golden["cases"]:
    r = resampler(c)
    x = torch.from_numpy(INPUTS[c["input"]][None].copy()).cuda()
    y64 = r.apply(x, dtype=torch.float64)[0].cpu().numpy()
    try:
      check_case(c, y64)
    except AssertionError:
      raise AssertionError("case %s" % case_id(c))
    y32 = r.apply(x)[0].cpu().numpy()
    with np.errstate(over="ignore"):          # zero = 1e300 rounds to inf in float32, as the kernel's store does
      assert same(y32, y64.astype(np.float32)), case_id(c)


def _cuts(rng, T, order, pos):
  """Block lengths summing to T: 0, 1, fewer than order + 1, and cuts at the consumption points ``pos``."""
  cuts, at = [], 0
  points = set(int(p) for p in pos)
  while at < T:
    kind = rng.integers(0, 4)
    if kind == 0:
      n = 0
    elif kind == 1:
      n = 1
    elif kind == 2:
      n = int(rng.integers(1, order + 2))
    else:
      ahead = sorted(p for p in points if p > at)
      n = (ahead[0] - at) if ahead else T - at
    n = min(n, T - at)
    cuts.append(n)
    at += n
  return cuts + [0]


@pytest.mark.parametrize("order", [1, 3, 4, 8, 15, 64])
@pytest.mark.parametrize("old,new", [(44100, 48000), (48000, 16000), (1, 3), (50, 1)])
def test_blocks_give_the_bits_of_one_call(torch, order, old, new):
  rng = np.random.default_rng(order * 1000 + int(old / new * 100))
  x = torch.from_numpy(rng.uniform(-1, 1, (3, 700)).astype(np.float32)).cuda()
  r = ab.Resampler(old, new, order, zero=.25)
  want = r.apply(x, dtype=torch.float64).cpu().numpy()
  pos, _, _ = r.schedule(resampling.start_index(order), 700)
  state = r.new_state(3)
  parts, at = [], 0
  for n in _cuts(rng, 700, order, pos):
    parts.append(r.apply(x[:, at:at + n], state=state, dtype=torch.float64).cpu().numpy())
    at += n
  assert same(np.concatenate(parts, axis=1), want)
  assert same(want[0], em.resample(x[0].cpu().numpy(), old, new, order, .25))


def test_many_short_streams(torch):
  rng = np.random.default_rng(1)
  x = rng.uniform(-1, 1, (4096, 300)).astype(np.float32)
  x[17, 100] = np.nan
  x[2000, 5] = np.inf
  r = ab.Resampler(44100, 48000)
  got = r.apply(torch.from_numpy(x).cuda(), dtype=torch.float64).cpu().numpy()
  assert same(got, em.resample_batch(x, 44100, 48000))


@pytest.mark.parametrize("old,new,order", [(48000, 44100, 3), (1, 3, 5)])
def test_one_long_stream(torch, old, new, order):
  x = np.random.default_rng(2).uniform(-1, 1, (1, 2_000_000)).astype(np.float32)
  r = ab.Resampler(old, new, order)
  got = r.apply(torch.from_numpy(x).cuda(), dtype=torch.float64).cpu().numpy()
  assert same(got, em.resample_batch(x, old, new, order))


def test_strided_and_misaligned_buffers(torch):
  rng = np.random.default_rng(3)
  S, T, order = 5, 999, 3
  base = torch.from_numpy(rng.uniform(-1, 1, (S, T + 7)).astype(np.float32)).cuda()
  x = base[:, 1:T + 1]                               # rows 4 * (T + 7) bytes apart, 4 bytes past an alignment
  r = ab.Resampler(3, 4, order)
  want = em.resample_batch(x.cpu().numpy(), 3, 4, order)
  assert same(r.apply(x, dtype=torch.float64).cpu().numpy(), want)
  assert same(r.apply(x.t().contiguous().t()).cpu().numpy(), want.astype(np.float32))   # column-major input
  # through the ABI: output rows out_stride apart, starting one element past the allocation
  pos, idxs, _ = r.schedule(resampling.start_index(order), T)
  n = len(pos)
  for f64, dt in ((1, torch.float64), (0, torch.float32)):
    out = torch.full((S * (n + 3) + 1,), -7., dtype=dt, device="cuda")
    state = r.new_state(S)
    w = torch.empty((n, order + 1), dtype=torch.float64, device="cuda")
    pos_d, idx_d = torch.from_numpy(pos).cuda(), torch.from_numpy(idxs).cuda()
    resampling._check(resampling.lib().alz_resample_apply(
      x.data_ptr(), out.data_ptr() + out.element_size(), f64, state.tensor.data_ptr(), pos_d.data_ptr(),
      idx_d.data_ptr(), w.data_ptr(), n, S, T, x.stride(0), n + 3, order, torch.cuda.current_stream().cuda_stream))
    o = out.cpu().numpy()
    rows = o[1:].reshape(S, n + 3)
    assert same(rows[:, :n], want.astype(o.dtype))
    assert o[0] == -7 and np.all(rows[:, n:] == -7)


def test_lazy_api_equals_the_reference(torch, golden):
  for c in golden["cases"]:
    s = ab.resample(INPUTS[c["input"]].tolist(), c["old"], c["new"], c["order"], make_resample.dec(c["zero"]))
    out = []
    with pytest.raises(getattr(builtins, golden["end"][0]), match=golden["end"][1]):
      for v in s:
        out.append(v)
    check_case(c, out)
  # the Resampler's lazy form, on an iterator read ahead in growing blocks
  c = golden["cases"][0]
  it = iter(resampler(c)(iter(INPUTS[c["input"]].tolist())))
  want = ab.resample(INPUTS[c["input"]].tolist(), c["old"], c["new"], c["order"], make_resample.dec(c["zero"]))
  assert [next(it) for _ in range(50)] == want.take(50)


def test_concurrent_streams_and_threads(torch):
  rng = np.random.default_rng(11)
  r = ab.Resampler(44100, 48000, 7)
  xs = [torch.from_numpy(rng.uniform(-1, 1, (64, 20000)).astype(np.float32)).cuda() for _ in range(4)]
  want = []
  for x in xs:
    state = r.new_state(64)
    want.append(np.concatenate([r.apply(x[:, i:i + 5000], state=state).cpu().numpy() for i in range(0, 20000, 5000)],
                               axis=1))
  streams = [torch.cuda.Stream() for _ in range(4)]
  outs = [None] * 4

  def run(i):
    with torch.cuda.stream(streams[i]):
      state = r.new_state(64)
      parts = [r.apply(xs[i][:, j:j + 5000], state=state) for j in range(0, 20000, 5000)]
      outs[i] = torch.cat(parts, dim=1)
    streams[i].synchronize()

  threads = [threading.Thread(target=run, args=(i,)) for i in range(4)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for o, w in zip(outs, want):
    assert same(o.cpu().numpy(), w)


def test_state_checks(torch):
  r = ab.Resampler(1, 2, 3)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    r.apply(x, state=r.new_state(3))
  for other in (ab.Resampler(1, 2, 4), ab.Resampler(1, 3, 3)):
    with pytest.raises(ValueError, match="another"):
      r.apply(x, state=other.new_state(2))
  r.apply(x, state=ab.Resampler(2, 4, 3, zero=1.).new_state(2))     # the same order and step
  with pytest.raises(ValueError, match="Resampler.new_state"):
    r.apply(x, state=object())
  with pytest.raises(ValueError, match="dtype"):
    r.apply(x, dtype=torch.float16)
  with pytest.raises(ValueError, match="float32"):
    r.apply(x.double())


def test_smoke_example(torch):
  assert ab.resample([1., 2., 3., 4., 5.], 1, 2, order=1).take(8) == [1., 1.5, 2., 2.5, 3., 3.5, 4., 4.5]


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  r = ab.Resampler(44100, 48000)
  y = r.apply(x)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_resample_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["resample"].path, _LAUNCH_PROBE)
