"""dft / Dft / dft_frames on the GPU: every golden bit for bit in complex128 and as its complex64 rounding, tile edges
and batch shapes against the emulation, a sampled check at a full-machine shape, streams cut into blocks of any
lengths, strided and misaligned input, NaN isolation, concurrent use, state misuse, and coverage of every kernel in
libalz_b200_dft.so."""
import builtins
import re
import sys
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, fourier
import dft_emulation as em
from conftest import GOLDEN
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
from test_dft import case_id, check_values, framed_blocks, freqs_of, golden  # noqa: F401  (fixture)

sys.path.insert(0, GOLDEN)
import make_dft  # noqa: E402

pytestmark = pytest.mark.gpu


def same(a, b):
  """Equal complex arrays, each part NaN by NaN-ness."""
  a, b = np.asarray(a), np.asarray(b)
  return (a.shape == b.shape and np.array_equal(a.real, b.real, equal_nan=True) and
          np.array_equal(a.imag, b.imag, equal_nan=True))


def c64(v):
  """The complex64 rounding of each part of a complex128 array."""
  out = np.empty(v.shape, dtype=np.complex64)
  with np.errstate(over="ignore"):
    out.real, out.imag = v.real.astype(np.float32), v.imag.astype(np.float32)
  return out


def test_every_golden_through_dft(torch, golden):
  for c in golden["cases"]:
    x = make_dft.signal(c["input"], c["size"]).tolist()
    if "exception" in c:
      exc, msg = c["exception"]
      with pytest.raises(getattr(builtins, exc), match=re.escape(msg)):
        ab.dft(x, freqs_of(c), c["normalize"])
    else:
      check_values(c, ab.dft(x, freqs_of(c), c["normalize"]))


def test_every_golden_through_dft_frames_and_Dft(torch, golden):
  for c in golden["framed"]:
    x = make_dft.signal(c["input"], c["length"])
    w = make_dft.window(c["window"], c["size"])
    got = ab.dft_frames(x.tolist(), freqs_of(c), c["size"], c["hop"], w, c["normalize"])
    frames = list(got)
    assert len(frames) == c["frames"], case_id(c)
    check_values(c, [v for f in frames for v in f])
    if not c["freqs"]:
      continue
    xd = torch.from_numpy(x[None].copy()).cuda()
    for dtype in (torch.complex128, torch.complex64):
      d = ab.Dft(freqs_of(c), c["size"], c["hop"], w, c["normalize"], dtype=dtype)
      y = d.apply(xd, final=True)[0].cpu().numpy()
      if dtype == torch.complex128:
        check_values(c, y.reshape(-1).tolist())
        y128 = y
      else:
        assert same(y, c64(y128)), case_id(c)


@pytest.mark.parametrize("S,T,size,hop,nf", [(3, 700, 100, 37, 70), (1, 1000, 7, 3, 1), (5, 64, 64, 64, 65),
                                            (2, 2000, 33, 50, 129), (70, 300, 257, 100, 3), (1, 5, 8, 2, 64)])
def test_tile_edges_against_the_emulation(torch, S, T, size, hop, nf):
  rng = np.random.default_rng(S * 1000 + size)
  x = rng.uniform(-1, 1, (S, T)).astype(np.float32)
  freqs = rng.uniform(-4, 4, nf).tolist()
  w = rng.uniform(0, 1, size).tolist()
  d = ab.Dft(freqs, size, hop, w)
  got = d.apply(torch.from_numpy(x).cuda(), final=True).cpu().numpy()
  for s in range(S):
    want = em.dft_batch(em.frames(x[s], size, hop, w), d.table)
    assert same(got[s], want), s
  d64 = ab.Dft(freqs, size, hop, w, normalize=False, dtype=torch.complex64)
  got = d64.apply(torch.from_numpy(x).cuda(), final=True).cpu().numpy()
  assert same(got[0], c64(em.dft_batch(em.frames(x[0], size, hop, w), d.table, normalize=False)))


def test_benchmark_shape_sampled(torch):
  gen = torch.Generator("cuda").manual_seed(3)
  x = torch.rand((4096, 16384), device="cuda", generator=gen) * 2 - 1
  freqs = [2 * np.pi * 440 * 2 ** ((m - 69) / 12) / 48000 for m in range(36, 100)]
  w = ab.window.hann(1024)
  d = ab.Dft(freqs, 1024, 512, w)
  y = d.apply(x)
  assert y.shape == (4096, 31, 64)
  rng = np.random.default_rng(4)
  for s in rng.choice(4096, 12, replace=False):
    ks = rng.choice(31, 25, replace=False)
    b = em.frames(x[s].cpu().numpy(), 1024, 512, w, final=False)[ks]
    assert same(y[s, ks].cpu().numpy(), em.dft_batch(b, d.table)), s


def _cuts(rng, T, size):
  cuts, at = [], 0
  while at < T:
    n = int(min(T - at, rng.choice([0, 1, 2, size // 2, size - 1, size + 3, 3 * size])))
    cuts.append(n)
    at += n
  return cuts + [0]


@pytest.mark.parametrize("size,hop", [(64, 16), (64, 64), (50, 80), (1, 1), (300, 7)])
def test_blocks_give_the_bits_of_one_call(torch, size, hop):
  rng = np.random.default_rng(size * 100 + hop)
  x = torch.from_numpy(rng.uniform(-1, 1, (3, 2000)).astype(np.float32)).cuda()
  d = ab.Dft(rng.uniform(-3, 3, 20).tolist(), size, hop, ab.window.hann)
  want = d.apply(x, final=True).cpu().numpy()
  state = d.new_state(3)
  parts, at = [], 0
  cuts = _cuts(rng, 2000, size)
  for i, n in enumerate(cuts):
    parts.append(d.apply(x[:, at:at + n], state=state, final=i == len(cuts) - 1).cpu().numpy())
    at += n
  assert same(np.concatenate(parts, axis=1), want)


def test_strided_and_misaligned_input(torch):
  rng = np.random.default_rng(8)
  S, T = 5, 999
  base = torch.from_numpy(rng.uniform(-1, 1, (S, T + 7)).astype(np.float32)).cuda()
  x = base[:, 1:T + 1]                               # rows 4 * (T + 7) bytes apart, 4 bytes past an alignment
  d = ab.Dft(rng.uniform(-3, 3, 9).tolist(), 100, 45)
  want = d.apply(x.contiguous(), final=True).cpu().numpy()
  assert same(d.apply(x, final=True).cpu().numpy(), want)
  assert same(d.apply(x.t().contiguous().t(), final=True).cpu().numpy(), want)   # column-major input
  xn = x.cpu().numpy()
  assert same(want[2], em.dft_batch(em.frames(xn[2], 100, 45), d.table))


def test_nan_sample_touches_only_its_frames(torch):
  rng = np.random.default_rng(9)
  x = rng.uniform(-1, 1, (2, 1000)).astype(np.float32)
  x[1, 500] = np.nan
  d = ab.Dft(rng.uniform(-3, 3, 5).tolist(), 64, 32)
  y = d.apply(torch.from_numpy(x).cuda()).cpu().numpy()
  bad = np.isnan(y.real).any(-1) | np.isnan(y.imag).any(-1)
  want = np.zeros_like(bad)
  want[1, [k for k in range(y.shape[1]) if k * 32 <= 500 < k * 32 + 64]] = True
  assert (bad == want).all()
  assert np.isnan(y[1, 15].real).all() and np.isnan(y[1, 15].imag).all()


def test_concurrent_streams_and_threads(torch):
  """Two Dfts whose launches need different shared-memory sizes above 48 KB (frames of 24 and of 1024 samples), each
  on two CUDA streams from its own host threads, give the bits of serial runs."""
  rng = np.random.default_rng(11)
  dfts = [ab.Dft(rng.uniform(-3, 3, 40).tolist(), 24, 8), ab.Dft(rng.uniform(-3, 3, 40).tolist(), 1024, 256)]
  xs = [torch.from_numpy(rng.uniform(-1, 1, (64, 12000)).astype(np.float32)).cuda() for _ in range(4)]
  want = []
  for i, x in enumerate(xs):
    d = dfts[i % 2]
    state = d.new_state(64)
    want.append(np.concatenate([d.apply(x[:, j:j + 3000], state=state).cpu().numpy()
                                for j in range(0, 12000, 3000)], axis=1))
  streams = [torch.cuda.Stream() for _ in range(4)]
  outs = [None] * 4

  def run(i):
    d = dfts[i % 2]
    with torch.cuda.stream(streams[i]):
      state = d.new_state(64)
      parts = [d.apply(xs[i][:, j:j + 3000], state=state) for j in range(0, 12000, 3000)]
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
  d = ab.Dft([1., 2.], 16, 8)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    d.apply(x, state=d.new_state(3))
  for other in (ab.Dft([1., 3.], 16, 8), ab.Dft([1., 2.], 16, 4), ab.Dft([1., 2.], 16, 8, normalize=False),
                ab.Dft([1., 2.], 16, 8, ab.window.hann)):
    with pytest.raises(ValueError, match="another|other"):
      d.apply(x, state=other.new_state(2))
  d.apply(x, state=ab.Dft([1., 2.], 16, 8, dtype=torch.complex64).new_state(2))     # output type is not state
  with pytest.raises(ValueError, match="Dft.new_state"):
    d.apply(x, state=object())
  state = d.new_state(2)
  d.apply(x, state=state, final=True)
  with pytest.raises(ValueError, match="ended"):
    d.apply(x, state=state)
  with pytest.raises(ValueError, match="float32"):
    d.apply(x.double())
  with pytest.raises(ValueError, match="math domain error"):
    ab.Dft([1e308], 3)
  with pytest.raises(ValueError, match="frequencies"):
    ab.Dft([], 3)
  with pytest.raises(ValueError, match="Incompatible window size"):
    ab.Dft([1.], 3, wnd=[1., 2.])


def test_lazy_overflow_raises_at_the_first_frame(torch):
  s = ab.dft_frames([1., 2., 3., 4.], [1e308], 4)                # nothing raises at call time
  with pytest.raises(ValueError, match="math domain error"):
    s.take()


def test_smoke_example(torch):
  assert ab.dft([1., 2., 3., 4.], [0., np.pi / 2, np.pi]) == [
    (2.5+0j), (-0.5000000000000001+0.4999999999999999j), (-0.5-2.4492935982947064e-16j)]


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  d = ab.Dft([.1, .2, .3], 256, 128)
  y = d.apply(x)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_dft_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["dft"].path, _LAUNCH_PROBE)
