"""LpcFrames / lpc_frames on the GPU: the lazy call against the reference's answers, the batched path against the
float64 emulation on sampled streams and frames, a long stream, strided and unaligned rows, block splits through an
LpcState, concurrent CUDA streams, state misuse, and coverage of every kernel in libalz_b200_lpc.so.  Every
comparison is of bits (NaN equal to NaN)."""
import json
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import GOLDEN
import lpc_emulation as em
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)

sys.path.insert(0, GOLDEN)
from make_lpc import inputs  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "lpc_cases.json")) as fh:
    return json.load(fh)


def same(a, b):
  a, b = em.canon(np.asarray(a)), em.canon(np.asarray(b))
  return a.shape == b.shape and a.tobytes() == b.tobytes()


def test_lazy_call_equals_the_reference(torch, golden):
  xs = inputs()
  for c in golden["cases"]:
    x = xs[c["input"]]
    key = (c["input"], c["order"], c["size"], c["hop"], c["window"])
    L = c["order"] + 1
    stream = iter(ab.lpc_frames(x.astype(np.float64).tolist(), c["order"], c["size"], c["hop"], c["window_values"]))
    coefs, errs = [], []
    n_ok = c["failed"][0] if c["failed"] else c["frames"]
    for k in range(n_ok):
      filt = next(stream)
      num = filt.numerator
      assert type(num[0]) is int and num[0] == 1 and len(num) == c["lengths"][k], (key, k)
      coefs.append([float(v) for v in num] + [0.] * (L - len(num)))
      errs.append(filt.error)
    if c["failed"]:
      with pytest.raises(ab.ParCorError):
        next(stream)
    else:
      assert next(stream, None) is None
    # the whole case through LpcFrames, failed frames included
    lp = ab.LpcFrames(c["order"], c["size"], c["hop"], c["window_values"])
    xd = torch.from_numpy(x).cuda()
    res = lp.apply(xd, final=True)
    r = lp.acorr(xd, final=True)
    coef, err, failed = (t[0].cpu().numpy() for t in res)
    assert np.flatnonzero(failed).tolist() == c["failed"], key
    assert em.digest(r[0].cpu().numpy()) == c["acorr"], key
    assert em.digest(coef) == c["coef"] and em.digest(err) == c["error"], key
    assert same(coef[:n_ok], np.array(coefs).reshape(-1, L)) and same(err[:n_ok], errs), key


def test_doctest(torch):
  (filt,) = list(ab.lpc_frames([-1, 0, 1, 0] * 4, 2, 16))
  assert filt.numerator == [1, 0.0, 0.875] and filt.error == 1.875


def check_sampled(x, lp, res, r, rng, n=12, final=True):
  """Compare sampled (stream, frame) pairs of a batched result with the emulation."""
  coef, err, failed = (t.cpu().numpy() for t in res)
  r = r.cpu().numpy()
  S, F = failed.shape
  assert F == lp.n_frames(0, x.shape[1], final)
  if F == 0:
    return
  for s, k in zip(rng.integers(0, S, n), rng.integers(0, F, n)):
    blk = em.frames(x[s, k * lp.hop:k * lp.hop + lp.size], lp.size, lp.hop, lp.window, final=True)[0]
    wr, wc, we, wf = em.kautocor(blk, lp.order)
    assert same(r[s, k], wr) and same(coef[s, k], wc) and same(err[s, k], we) and failed[s, k] == wf, (s, k)


@pytest.mark.parametrize("S,T,order,size,hop,win", [
    (1, 1000, 16, 128, 64, "hann"), (3, 777, 0, 50, 50, None), (33, 2000, 32, 96, 40, "hamming"),
    (7, 3001, 64, 100, 130, None), (5, 400, 40, 24, 16, "hann"), (4096, 2048, 16, 256, 128, "hann"),
    (4096, 16384, 16, 1024, 512, "hann"), (2, 20000, 12, 8192, 4096, None)])
def test_batched_against_the_emulation(torch, S, T, order, size, hop, win):
  rng = np.random.default_rng(S * 7 + order)
  x = rng.uniform(-1, 1, (S, T)).astype(np.float32)
  x[:, ::97] = 0
  w = None if win is None else (np.hanning(size) if win == "hann" else np.hamming(size))
  lp = ab.LpcFrames(order, size, hop, w)
  xd = torch.from_numpy(x).cuda()
  res = lp.apply(xd, final=True)
  r = lp.acorr(xd, final=True)
  check_sampled(x, lp, res, r, rng, n=6 if size >= 1024 else 12)


def test_one_long_stream(torch):
  T = 10 ** 7 + 37
  rng = np.random.default_rng(11)
  x = rng.standard_normal((1, T)).astype(np.float32)
  lp = ab.LpcFrames(16, 400, 160, np.hamming(400))
  xd = torch.from_numpy(x).cuda()
  res = lp.apply(xd, final=True)
  r = lp.acorr(xd, final=True)
  assert res.coef.shape == (1, lp.n_frames(0, T, True), 17)
  check_sampled(x, lp, res, r, rng, n=8)
  # the padded last frame
  F = res.coef.shape[1]
  blk = em.frames(x[0], 400, 160, lp.window)[-1]
  assert same(r[0, F - 1].cpu().numpy(), em.kautocor(blk, 16)[0])


def test_strided_and_unaligned_rows(torch):
  rng = np.random.default_rng(13)
  y = rng.uniform(-1, 1, (5, 2 * 3001 + 3)).astype(np.float32)
  yd = torch.from_numpy(y).cuda()
  lp = ab.LpcFrames(12, 64, 48, np.hanning(64))
  for o in (1, 2, 3):                             # rows starting 4, 8 and 12 bytes past a 16-byte boundary
    want = lp.apply(torch.from_numpy(np.ascontiguousarray(y[:, o:o + 3001])).cuda(), final=True)
    got = lp.apply(yd[:, o:o + 3001], final=True)
    assert all(torch.equal(a.nan_to_num(), b.nan_to_num()) for a, b in zip(got, want)), o
    check_sampled(y[:, o:o + 3001], lp, got, lp.acorr(yd[:, o:o + 3001], final=True), rng)
  got = lp.apply(yd[:, ::2], final=True)
  check_sampled(y[:, ::2], lp, got, lp.acorr(yd[:, ::2], final=True), rng)


@pytest.mark.parametrize("order,size,hop", [(16, 256, 100), (3, 7, 7), (12, 40, 90), (32, 64, 1)])
def test_block_splits_equal_one_call(torch, order, size, hop):
  S, T = 3, 30000
  rng = np.random.default_rng(order * 100 + size)
  x = rng.uniform(-1, 1, (S, T + 1)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()[:, 1:]
  lp = ab.LpcFrames(order, size, hop, np.hanning(size))
  whole = lp.apply(xd, final=True)
  whole_r = lp.acorr(xd, final=True)
  lengths = [0, 1, size - 1, 0, 1, 4096, size - 1, 5000] + [int(v) for v in rng.integers(0, 3000, 5)]
  lengths.append(T - sum(lengths))
  state, rstate = lp.new_state(S), lp.new_state(S)
  parts, rparts, t = [], [], 0
  for i, n in enumerate(lengths):
    last = i == len(lengths) - 1
    parts.append(lp.apply(xd[:, t:t + n], state=state, final=last))
    rparts.append(lp.acorr(xd[:, t:t + n], state=rstate, final=last))
    t += n
  assert t == T and state.consumed == T
  for j in range(3):
    got = torch.cat([p[j] for p in parts], dim=1)
    assert same(got.cpu().numpy(), whole[j].cpu().numpy()), j
  assert same(torch.cat(rparts, dim=1).cpu().numpy(), whole_r.cpu().numpy())


def test_two_cuda_streams_at_once(torch):
  rng = np.random.default_rng(17)
  xa, xb = rng.uniform(-1, 1, (256, 20000)).astype(np.float32), rng.uniform(-1, 1, (1, 2 * 10 ** 6)).astype(np.float32)
  da, db = torch.from_numpy(xa).cuda(), torch.from_numpy(xb).cuda()
  lp = ab.LpcFrames(16, 512, 256, np.hanning(512))
  wa, wb = lp.apply(da, final=True), lp.apply(db, final=True)
  sa, sb = torch.cuda.Stream(), torch.cuda.Stream()
  torch.cuda.synchronize()
  outs = []
  for _ in range(3):
    with torch.cuda.stream(sa):
      ra = lp.apply(da, final=True)
    with torch.cuda.stream(sb):
      rb = lp.apply(db, final=True)
    outs.append((ra, rb))
  torch.cuda.synchronize()
  for ra, rb in outs:
    for got, want in ((ra, wa), (rb, wb)):
      assert all(same(g.cpu().numpy(), w.cpu().numpy()) for g, w in zip(got, want))


def test_state_checks(torch):
  lp = ab.LpcFrames(4, 32, 16)
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    lp.apply(x, state=lp.new_state(3))
  for other in (ab.LpcFrames(5, 32, 16), ab.LpcFrames(4, 33, 16), ab.LpcFrames(4, 32, 8),
                ab.LpcFrames(4, 32, 16, [1.] * 32)):
    with pytest.raises(ValueError, match="order, size, hop or window"):
      lp.apply(x, state=other.new_state(2))
  with pytest.raises(ValueError, match="LpcFrames.new_state"):
    lp.apply(x, state=object())
  with pytest.raises(ValueError):
    lp.apply(x.double())
  if torch.cuda.device_count() > 1:
    with torch.cuda.device(1):
      other = lp.new_state(2)
    with pytest.raises(ValueError, match="lives on"):
      lp.apply(x, state=other)
  state = lp.new_state(2)
  lp.acorr(x, state=state, final=True)
  with pytest.raises(ValueError, match="final"):
    lp.apply(x, state=state)
  assert ab.LpcFrames(4, 32, 16).apply(x, state=ab.LpcFrames(4, 32, 16).new_state(2)).coef.shape == (2, 5, 5)


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  lp = ab.LpcFrames(8, 256, 128)
  state = lp.new_state(2)
  lp.apply(x, state=state, final=True)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_lpc" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_lpc_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["lpc"].path, _LAUNCH_PROBE)
