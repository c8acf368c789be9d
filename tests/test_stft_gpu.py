"""Stft / OverlapAdd / stft / overlap_add on the GPU: analysis against numpy's rfft of the same float64 frames, the
complex64 output as the rounded complex128 one, resynthesis with overlap-add against OverlapAdd of the same frames,
the overlap-add against the reference's arithmetic bit for bit, block splits, shapes, NaN, concurrent use, state
misuse, the lazy API, and coverage of every kernel in libalz_b200_stft.so."""
import json
import os
import sys
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
import stft_emulation as em
from conftest import GOLDEN
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
from test_stft import golden_stft_case

sys.path.insert(0, GOLDEN)
import make_stft  # noqa: E402

pytestmark = pytest.mark.gpu

SIZES = list(range(1, 65)) + [97, 1000, 1024, 4096, 8192]


def same(a, b):
  a, b = np.asarray(a), np.asarray(b)
  return a.shape == b.shape and np.array_equal(a, b, equal_nan=True)


def check_spectra(got, want):
  """complex128 spectra within 1e-12 of each frame's peak |X|, zero frames exactly zero."""
  assert got.shape == want.shape
  for g, w in zip(got, want):
    peak = np.max(np.abs(w)) if w.size else 0.
    if peak == 0:
      assert not np.any(g)
    else:
      assert np.max(np.abs(g - w)) <= 1e-12 * peak


@pytest.mark.parametrize("size", SIZES)
def test_analysis_against_numpy(torch, size):
  rng = np.random.default_rng(size)
  hop = max(1, size // 2 + (size % 3 == 0))
  T = 3 * size + 5
  x = rng.uniform(-1, 1, (3, T)).astype(np.float32)
  x[1, :size] = 0                                    # a zero frame
  w = ab.window.hann(size)
  st = ab.Stft(size, hop, wnd=w, dtype=torch.complex128)
  spec = st.analyze(torch.from_numpy(x).cuda(), final=True).cpu().numpy()
  for s in range(3):
    check_spectra(spec[s], em.analysis(x[s], size, hop, w))
  st32 = ab.Stft(size, hop, wnd=w)
  spec32 = st32.analyze(torch.from_numpy(x).cuda(), final=True).cpu().numpy()
  assert same(spec32, spec.astype(np.complex64))
  # no shift, no window
  st = ab.Stft(size, hop, before=False, dtype=torch.complex128)
  spec = st.analyze(torch.from_numpy(x).cuda(), final=True).cpu().numpy()
  check_spectra(spec[0], em.analysis(x[0], size, hop, None, before=False))


def test_analysis_large_batch_sampled(torch):
  rng = np.random.default_rng(7)
  S, T, size, hop = 4096, 16384, 1024, 512
  x = torch.rand((S, T), device="cuda", dtype=torch.float32) * 2 - 1
  st = ab.Stft(size, hop, wnd=ab.window.hann, dtype=torch.complex128)
  spec = st.analyze(x)
  assert spec.shape == (S, st.n_frames(0, T, False), size // 2 + 1)
  for s, k in zip(rng.integers(0, S, 12), rng.integers(0, spec.shape[1], 12)):
    row = x[s].cpu().numpy()
    want = em.analysis(row, size, hop, ab.window.hann(size))[k]
    check_spectra(spec[s, k].cpu().numpy()[None], want[None])


@pytest.mark.parametrize("size,hop", [(1, 1), (8, 2), (15, 4), (64, 64), (97, 30), (1000, 441), (1024, 512),
                                      (8192, 2048)])
@pytest.mark.parametrize("strategy", ["numpy", "list"])
def test_synthesis_equals_ola_of_frames(torch, size, hop, strategy):
  rng = np.random.default_rng(size + hop)
  x = torch.from_numpy(rng.uniform(-1, 1, (2, 3 * size + 7)).astype(np.float32)).cuda()
  kw = dict(wnd=ab.window.hann, ola_wnd=ab.window.hann)
  st = ab.Stft(size, hop, ola=strategy, **kw)
  frames_st = ab.Stft(size, hop, ola=None, **kw)
  spec = st.analyze(x, final=True)
  y = st.synthesize(spec, final=True)
  v = frames_st.synthesize(spec, final=True)
  ola = ab.OverlapAdd(size, hop, ab.window.hann, strategy=strategy)
  assert same(y.cpu().numpy(), ola.apply(v, final=True).cpu().numpy())
  # the overlap-add is the reference's float64 arithmetic, rounded once
  for s in range(2):
    want = em.ola(v[s].cpu().numpy(), size, hop, ola.window).astype(np.float32)
    assert same(y[s].cpu().numpy(), want)
  # the frames are numpy's irfft of the spectra
  want = em.synthesis_frames(spec[0].cpu().numpy().astype(np.complex128), size)
  got = v[0].cpu().numpy()
  assert np.max(np.abs(got - want)) <= 1e-12 * max(1., np.max(np.abs(want)))


def test_round_trip_complex64(torch):
  rng = np.random.default_rng(3)
  size, hop = 1024, 256
  x = rng.uniform(-1, 1, (3, 20000)).astype(np.float32)
  st = ab.Stft(size, hop, wnd=ab.window.hann, ola_wnd=ab.window.hann)
  y = st.apply(torch.from_numpy(x).cuda(), lambda s: s, final=True).cpu().numpy()
  w = ab.window.hann(size)
  for s in range(3):
    v = em.synthesis_frames(em.analysis(x[s], size, hop, w), size)
    want = em.ola(v, size, hop, ab.spectral.ola_window(size, hop, ab.window.hann))
    assert np.max(np.abs(y[s] - want)) <= 1e-6 * np.max(np.abs(want))


@pytest.mark.parametrize("size,hop", [(8, 2), (64, 64), (97, 13), (1024, 441)])
def test_blocks_of_any_length_give_the_bits_of_one_call(torch, size, hop):
  rng = np.random.default_rng(size)
  T = 6 * size + 3
  x = torch.from_numpy(rng.uniform(-1, 1, (2, T)).astype(np.float32)).cuda()
  st = ab.Stft(size, hop, wnd=ab.window.hann, ola_wnd=ab.window.hann)
  whole_spec = st.analyze(x, final=True)
  whole = st.synthesize(whole_spec, final=True)
  state = st.new_state(2)
  specs, outs, t = [], [], 0
  lengths = [0, 1, max(1, hop - 1), size + 3, 0]
  while t < T:
    n = lengths[len(specs) % len(lengths)] if len(specs) < 12 else T - t
    n = min(n, T - t)
    spec = st.analyze(x[:, t:t + n], state)
    specs.append(spec)
    outs.append(st.synthesize(spec, state))
    t += n
  spec = st.analyze(x[:, T:], state, final=True)
  specs.append(spec)
  outs.append(st.synthesize(spec, state, final=True))
  assert same(torch.cat(specs, 1).cpu().numpy(), whole_spec.cpu().numpy())
  assert same(torch.cat(outs, 1).cpu().numpy(), whole.cpu().numpy())


def test_shapes_and_strides(torch):
  st = ab.Stft(1, dtype=torch.complex128)
  x = torch.tensor([[.5]], device="cuda")
  assert same(st.analyze(x, final=True).cpu().numpy(), np.array([[[.5 + 0j]]]))
  rng = np.random.default_rng(5)
  base = torch.from_numpy(rng.uniform(-1, 1, (3, 1001)).astype(np.float32)).cuda()
  st = ab.Stft(64, 16, wnd=ab.window.hann)
  want = st.analyze(base[:, 1:].contiguous(), final=True)
  got = st.analyze(base[:, 1:], final=True)                      # strided, unaligned rows
  assert same(got.cpu().numpy(), want.cpu().numpy())
  wide = torch.zeros((3, want.shape[1], 40), dtype=want.dtype, device="cuda")
  wide[:, :, 3:36] = want
  a = st.synthesize(wide[:, :, 3:36], final=True)                 # non-contiguous spectra
  b = st.synthesize(want.contiguous(), final=True)
  assert same(a.cpu().numpy(), b.cpu().numpy())


def test_nan_touches_only_its_frames(torch):
  size, hop = 16, 4
  x = np.random.default_rng(2).uniform(-1, 1, 200).astype(np.float32)
  x[101] = np.nan
  st = ab.Stft(size, hop, wnd=ab.window.hann, ola_wnd=ab.window.hann, dtype=torch.complex128)
  spec = st.analyze(torch.from_numpy(x).cuda(), final=True)[0].cpu().numpy()
  bad = [k for k in range(spec.shape[0]) if k * hop <= 101 < k * hop + size]
  assert [k for k in range(spec.shape[0]) if not np.all(np.isfinite(spec[k]))] == bad
  y = st.synthesize(torch.from_numpy(spec[None]).cuda(), final=True)[0].cpu().numpy()
  assert np.flatnonzero(~np.isfinite(y)).tolist() == list(range(bad[0] * hop, bad[-1] * hop + size))


def test_concurrent_streams_and_threads(torch):
  rng = np.random.default_rng(11)
  st = ab.Stft(256, 64, wnd=ab.window.hann, ola_wnd=ab.window.hann)
  xs = [torch.from_numpy(rng.uniform(-1, 1, (8, 5000)).astype(np.float32)).cuda() for _ in range(2)]
  want = [st.apply(x, abs, final=True).cpu().numpy() for x in xs]
  streams = [torch.cuda.Stream() for _ in range(2)]
  outs = [None, None]

  def run(i):
    with torch.cuda.stream(streams[i]):
      for _ in range(3):
        outs[i] = st.apply(xs[i], abs, final=True)
    streams[i].synchronize()

  threads = [threading.Thread(target=run, args=(i,)) for i in range(2)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for o, w in zip(outs, want):
    assert same(o.cpu().numpy(), w)


def test_state_checks(torch):
  st = ab.Stft(32, 16)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    st.analyze(x, state=st.new_state(3))
  for other in (ab.Stft(33, 16), ab.Stft(32, 8), ab.Stft(32, 16, wnd=ab.window.hann), ab.Stft(32, 16, before=False)):
    with pytest.raises(ValueError, match="another"):
      st.analyze(x, state=other.new_state(2))
  with pytest.raises(ValueError, match="Stft.new_state"):
    st.analyze(x, state=object())
  state = st.new_state(2)
  spec = st.analyze(x, state=state, final=True)
  with pytest.raises(ValueError, match="final"):
    st.analyze(x, state=state)
  st.synthesize(spec, state=state, final=True)
  with pytest.raises(ValueError, match="final"):
    st.synthesize(spec, state=state)
  ola = ab.OverlapAdd(32, 16)
  with pytest.raises(ValueError, match="block size"):
    ola.apply(torch.zeros((1, 2, 31), dtype=torch.float64, device="cuda"))


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "stft_cases.json")) as fh:
    return json.load(fh)


def test_lazy_overlap_add_equals_the_reference(torch, golden):
  """Every overlap_add golden (both strategies, no window, callable and list windows, normalize on and off, hop ==
  size, hop | size, hop not dividing size, 0 / 1 / many blocks, -0.0, NaN, +-inf): the float32 of the reference's
  values, bit for bit."""
  for c in golden["ola"]:
    blocks = make_stft.ola_inputs(c["size"])[c["input"]]
    wnd = getattr(ab.window, c["wnd"]) if isinstance(c["wnd"], str) else c["wnd"]
    got = list(ab.overlap_add[c["strategy"]](blocks, size=c["size"], hop=c["hop"], wnd=wnd, normalize=c["normalize"]))
    want = np.array([float(v) for v in c["output"]]).astype(np.float32)
    assert same(np.float32(got), want), c


def gpu_func(name, size, torch):
  mask = torch.from_numpy(make_stft.mask(size)).cuda()
  return {"identity": lambda b: b, "abs": abs, "ifftshift": torch.fft.ifftshift, "mask": lambda b: b * mask}[name]


def test_lazy_stft_equals_the_reference(torch, golden):
  """Every stft golden through the lazy API: within 1e-7 of each output's peak (the float32 rounding of a float64
  pipeline), NaN where the reference has NaN."""
  arrays = np.load(os.path.join(GOLDEN, "stft_cases.npz"))
  for i, c in enumerate(golden["stft"]):
    x, size, hop, wnd, before, after, ola, ola_w = golden_stft_case(c)
    kws = dict(c["kwargs"])
    for k in ("wnd", "ola_wnd"):
      if isinstance(kws.get(k), str):
        kws[k] = getattr(ab.window, kws[k])
    if kws.get("ola") == "list":
      kws["ola"] = ab.overlap_add.list
    if c["hop"] is not None:
      kws["hop"] = c["hop"]
    out = list(ab.stft(gpu_func(c["func"], size, torch), size=size, **kws)(x.astype(np.float64).tolist()))
    got = np.array(out, dtype=np.float64).reshape(arrays["stft_%d" % i].shape)
    want = arrays["stft_%d" % i]
    assert np.array_equal(np.isnan(got), np.isnan(want)), c["name"]
    fin = np.isfinite(want)
    peak = np.max(np.abs(want[fin]), initial=0.)
    assert np.all(np.abs(got[fin] - want[fin]) <= 1e-7 * peak), (c["name"], np.max(np.abs(got[fin] - want[fin])), peak)


def test_lazy_overlap_add_matches_the_emulation(torch):
  rng = np.random.default_rng(4)
  for strategy in ("numpy", "list"):
    for size, hop in ((4, 2), (8, 8), (7, 3)):
      for n in (0, 1, 5):
        blocks = rng.standard_normal((n, size))
        if n:
          blocks[0, 0] = -0.0
        got = list(ab.overlap_add[strategy](list(blocks), size=size, hop=hop, wnd=ab.window.hann))
        w = ab.spectral.ola_window(size, hop, ab.window.hann, True, strategy)
        assert same(np.float32(got), em.ola(blocks, size, hop, w).astype(np.float32))
        assert all(type(v) is float for v in got)


def test_lazy_stft_docstring_examples(torch):
  analyzer = ab.stft(torch.fft.ifftshift, ola=None, size=8, hop=2)
  res = analyzer([1, 0, -1, 0] * 4)
  a, b = res.take(), res.take()
  assert np.allclose(a, .5, rtol=0, atol=1e-12) and np.allclose(b, -.5, rtol=0, atol=1e-12)
  assert list(ab.stft(abs, size=4, hop=2)([])) == [0.0, 0.0]
  stft64 = ab.stft(size=64)
  p1 = stft64(abs)([.1, .3, -.1, -.3, .5, .4, .3]).peek(200)
  p2 = ab.stft(abs, size=64)([.1, .3, -.1, -.3, .5, .4, .3]).peek(200)
  assert p1 == p2 and len(p1) == 64
  robot = ab.stft(abs, size=1024, hop=441, before=None, wnd=ab.window.hann, ola_wnd=ab.window.hann)
  sig = np.random.default_rng(0).uniform(-1, 1, 3000).astype(np.float32)
  got = np.array(list(robot(sig.tolist())))
  st = ab.Stft(1024, 441, wnd=ab.window.hann, before=False, ola_wnd=ab.window.hann, dtype=torch.complex128)
  want = st.apply(torch.from_numpy(sig).cuda(), abs, final=True)[0].cpu().numpy()
  assert same(np.float32(got), want)


def test_lazy_errors(torch):
  with pytest.raises(TypeError, match="Missing 'size'"):
    ab.stft(abs)([1, 2])
  with pytest.raises(ValueError, match="Hop value"):
    ab.stft(abs, size=4, hop=5)([1, 2])
  with pytest.raises(TypeError, match="no overlap-add"):
    ab.stft(abs, size=4, ola=None, ola_wnd=None)([1, 2])
  with pytest.raises(TypeError, match="Unknown"):
    ab.stft(abs, size=4, foo=1)([1, 2])
  with pytest.raises(TypeError, match="Window should be"):
    ab.stft(abs, size=4, wnd=3)([1, 2])
  with pytest.raises(ValueError, match="Incompatible window size"):
    ab.stft(abs, size=4, wnd=[1., 2.])([1, 2])
  with pytest.raises(TypeError, match="ola_foo|foo"):
    ab.stft(abs, size=4, ola_foo=1)([1, 2])
  for kw in ("transform", "inverse_transform"):
    with pytest.raises(NotImplementedError, match=kw):
      ab.stft(abs, size=4, **{kw: None})([1, 2])
  # the defaults given explicitly are the defaults
  want = list(ab.stft(abs, size=4, hop=2)([1., 2., 3., 4., 5.]))
  assert list(ab.stft(abs, size=4, hop=2, transform=np.fft.rfft, inverse_transform=np.fft.irfft,
                      before=np.fft.ifftshift, after=np.fft.fftshift)([1., 2., 3., 4., 5.])) == want
  for name in ("cfft", "cfftr"):
    with pytest.raises(NotImplementedError, match=name):
      ab.stft[name](abs, size=4)


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  st = ab.Stft(256, 128, wnd=ab.window.hann)
  y = st.apply(x, abs, final=True)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_stft_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["stft"].path, _LAUNCH_PROBE)
