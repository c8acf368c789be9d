"""Covariance-method LPC on the GPU (LpcFrames(method="kcovar"), LpcFrames.lag_matrix, lpc_frames): the reference's
answers from the goldens, the batched path against the float64 emulation on sampled streams and frames across orders,
sizes, batch shapes and layouts, block splits through an LpcState, state misuse and ABI errors, and coverage of every
kernel in libalz_b200_lpc.so by both methods.  Every comparison is of bits (NaN equal to NaN)."""
import ctypes
import json
import os
import sys

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, linear_prediction as lpm
from conftest import GOLDEN
import lpc_covar_emulation as em
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)

sys.path.insert(0, GOLDEN)
from make_lpc_covar import inputs  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def golden():
  with open(os.path.join(GOLDEN, "lpc_covar_cases.json")) as fh:
    return json.load(fh)


def same(a, b):
  a, b = em.canon(np.asarray(a)), em.canon(np.asarray(b))
  return a.shape == b.shape and a.tobytes() == b.tobytes()


def test_every_golden_through_lpc_frames_and_lpc_frames_batched(torch, golden):
  xs = inputs()
  for c in golden["cases"]:
    x = xs[c["input"]]
    key = (c["input"], c["order"], c["size"], c["hop"], c["window"])
    L = c["order"] + 1
    stream = iter(ab.lpc_frames(x.astype(np.float64).tolist(), c["order"], c["size"], c["hop"], c["window_values"],
                                method="kcovar"))
    n_ok = c["failed"][0][0] if c["failed"] else c["frames"]
    coefs, errs = [], []
    for k in range(n_ok):
      filt = next(stream)
      num = filt.numerator
      assert type(num[0]) is int and num[0] == 1 and len(num) == c["lengths"][k], (key, k)
      coefs.append([float(v) for v in num] + [0.] * (L - len(num)))
      errs.append(filt.error)
    if c["failed"]:
      kind = c["failed"][0][1]
      with pytest.raises(ZeroDivisionError if kind == 1 else ValueError,
                         match="Can't find next coefficient" if kind == 1 else "Unstable filter"):
        next(stream)
    else:
      assert next(stream, None) is None
    lp = ab.LpcFrames(c["order"], c["size"], c["hop"], c["window_values"], method="kcov")
    xd = torch.from_numpy(x).cuda()
    coef, err, failed = (t[0].cpu().numpy() for t in lp.apply(xd, final=True))
    M = lp.lag_matrix(xd, final=True)[0].cpu().numpy()
    assert [[k, int(f)] for k, f in enumerate(failed) if f] == c["failed"], key
    assert em.digest(M) == c["lagm"], key
    assert em.digest(coef) == c["coef"] and em.digest(err) == c["error"], key
    assert same(coef[:n_ok], np.array(coefs).reshape(-1, L)) and same(err[:n_ok], errs), key


def test_order_zero_raises_index_error_at_the_first_frame(torch):
  stream = iter(ab.lpc_frames([.5, -1., 2., .25] * 8, 0, 8, method="kcovar"))
  with pytest.raises(IndexError):
    next(stream)
  assert list(ab.lpc_frames([], 0, 8, method="kcovar")) == []              # no frame, nothing raised
  # the lag matrix of order 0 is the frame's energy
  x = torch.tensor([[1., 2., 3., 4.]], device="cuda")
  assert ab.LpcFrames(0, 4).lag_matrix(x).tolist() == [[[[30.]]]]


def check_sampled(x, lp, res, M, rng, n=6, final=True):
  coef, err, failed = (t.cpu().numpy() for t in res)
  M = M.cpu().numpy()
  S, F = failed.shape
  assert F == lp.n_frames(0, x.shape[1], final) and M.shape == (S, F, lp.order + 1, lp.order + 1)
  if F == 0:
    return
  picks = list(zip(rng.integers(0, S, n), rng.integers(0, F, n))) + [(S - 1, F - 1)]
  for s, k in picks:
    blk = em.frames(x[s, k * lp.hop:k * lp.hop + lp.size], lp.size, lp.hop, lp.window, final=True)[0]
    phi = em.lag_matrix(blk, lp.order)
    wc, we, wf = em.kcovar(phi)
    assert same(M[s, k], phi), (s, k)
    assert same(coef[s, k], wc) and same(err[s, k], we) and failed[s, k] == wf, (s, k, failed[s, k], wf)


@pytest.mark.parametrize("order", [1, 2, 16, 21, 22, 32, 63, 64])
@pytest.mark.parametrize("size", ["order+1", 1024, 8192])
def test_orders_and_sizes_against_the_emulation(torch, order, size):
  size = order + 1 if size == "order+1" else size
  S, hop = 3, max(1, size // 2)
  T = 3 * size + hop // 3
  rng = np.random.default_rng(order * 31 + size)
  # noise, and an AR(2) resonance whose frames stay stable at high orders
  e = rng.standard_normal((S, T))
  x = np.zeros((S, T))
  for i in range(T):
    x[:, i] = e[:, i] + 1.8 * (x[:, i - 1] if i else 0.) - .9 * (x[:, i - 2] if i > 1 else 0.)
  x[0] = rng.uniform(-1, 1, T)
  x = (x / np.abs(x).max()).astype(np.float32)
  lp = ab.LpcFrames(order, size, hop, np.hanning(size) if size > 64 else None, method="kcovar")
  xd = torch.from_numpy(x).cuda()
  check_sampled(x, lp, lp.apply(xd, final=True), lp.lag_matrix(xd, final=True), rng, n=3)


@pytest.mark.parametrize("S,T,order,size,hop,win", [
    (1, 5000, 16, 256, 100, "hann"), (3, 777, 2, 50, 50, None), (37, 2000, 12, 96, 140, "hamming"),
    (1000, 2048, 16, 256, 128, "hann"), (5, 400, 8, 24, 16, None)])
def test_batch_shapes_against_the_emulation(torch, S, T, order, size, hop, win):
  rng = np.random.default_rng(S * 7 + order)
  x = rng.uniform(-1, 1, (S, T)).astype(np.float32)
  x[:, ::97] = 0
  w = None if win is None else (np.hanning(size) if win == "hann" else np.hamming(size))
  lp = ab.LpcFrames(order, size, hop, w, method="kcovar")
  xd = torch.from_numpy(x).cuda()
  check_sampled(x, lp, lp.apply(xd, final=True), lp.lag_matrix(xd, final=True), rng)
  # without final, the padded frame is left out and the others keep their bits
  res = lp.apply(xd)
  F = res.coef.shape[1]
  full = lp.apply(xd, final=True)
  assert same(res.coef.cpu().numpy(), full.coef[:, :F].cpu().numpy())


def test_strided_rows(torch):
  rng = np.random.default_rng(13)
  y = rng.uniform(-1, 1, (5, 2 * 3001 + 3)).astype(np.float32)
  yd = torch.from_numpy(y).cuda()
  lp = ab.LpcFrames(12, 64, 48, np.hanning(64), method="kcovar")
  for view in (yd[:, 1:3002], yd[:, ::2]):                # x_stride > T, and a copy of a strided view
    want = lp.apply(view.contiguous(), final=True)
    got = lp.apply(view, final=True)
    assert all(same(a.cpu().numpy(), b.cpu().numpy()) for a, b in zip(got, want))
    check_sampled(view.cpu().numpy(), lp, got, lp.lag_matrix(view, final=True), rng)


@pytest.mark.parametrize("order,size,hop", [(16, 256, 100), (3, 7, 7), (12, 40, 90), (32, 64, 1)])
def test_block_splits_equal_one_call(torch, order, size, hop):
  S, T = 3, 20000
  rng = np.random.default_rng(order * 100 + size)
  x = rng.uniform(-1, 1, (S, T + 1)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()[:, 1:]
  lp = ab.LpcFrames(order, size, hop, np.hanning(size), method="kcovar")
  whole = lp.apply(xd, final=True)
  whole_m = lp.lag_matrix(xd, final=True)
  lengths = [0, 1, size - 1, 0, 1, 4096, size - 1, 3000] + [int(v) for v in rng.integers(0, 3000, 3)]
  lengths.append(T - sum(lengths))
  state, mstate = lp.new_state(S), lp.new_state(S)
  parts, mparts, t = [], [], 0
  for i, n in enumerate(lengths):
    last = i == len(lengths) - 1
    parts.append(lp.apply(xd[:, t:t + n], state=state, final=last))
    mparts.append(lp.lag_matrix(xd[:, t:t + n], state=mstate, final=last))
    t += n
  for j in range(3):
    assert same(torch.cat([p[j] for p in parts], dim=1).cpu().numpy(), whole[j].cpu().numpy()), j
  assert same(torch.cat(mparts, dim=1).cpu().numpy(), whole_m.cpu().numpy())


def test_a_minute_of_audio_frame_for_frame(torch):
  """lpc_frames(x, 16, 1024, 512, hann, method="kcovar") on a minute at 48 kHz, sampled against the emulation."""
  rng = np.random.default_rng(21)
  T = 48000 * 60
  x = rng.standard_normal(T).astype(np.float32)
  w = np.hanning(1024)
  filts = list(ab.lpc_frames(x, 16, 1024, 512, w, method="kcovar"))
  frames = em.frames(x, 1024, 512, w)
  assert len(filts) == len(frames) == 5624
  for k in list(rng.integers(0, len(frames), 6)) + [len(frames) - 1]:
    coef, err, failed = em.kcovar(em.lag_matrix(frames[k], 16))
    assert not failed
    num = filts[k].numerator
    assert [float(v) for v in num] + [0.] * (17 - len(num)) == coef and filts[k].error == err, k


def test_state_checks_and_abi_errors(torch):
  lp = ab.LpcFrames(4, 32, 16, method="kcovar")
  x = torch.zeros((2, 100), dtype=torch.float32, device="cuda")
  with pytest.raises(ValueError, match="streams"):
    lp.apply(x, state=lp.new_state(3))
  for other in (ab.LpcFrames(4, 32, 16), ab.LpcFrames(5, 32, 16, method="kcovar"),
                ab.LpcFrames(4, 32, 8, method="kcovar"), ab.LpcFrames(4, 32, 16, [1.] * 32, method="kcovar")):
    with pytest.raises(ValueError, match="order, size, hop or window"):
      lp.apply(x, state=other.new_state(2))
    with pytest.raises(ValueError, match="order, size, hop or window"):
      other.apply(x, state=lp.new_state(2))
  state = lp.new_state(2)
  lp.lag_matrix(x, state=state, final=True)
  with pytest.raises(ValueError, match="final"):
    lp.apply(x, state=state)
  with pytest.raises(ValueError, match="Block length"):
    ab.LpcFrames(40, 32).lag_matrix(x)
  # the C ABI: too little scratch, a misaligned output, and a stride below the row length
  L = lpm.lib()
  st = lp.new_state(2)
  F = lp.n_frames(0, 100, False)
  coef = torch.empty((2, F, 5), dtype=torch.float64, device="cuda")
  need = L.alz_lpc_covar_scratch_bytes(2, F, 4)
  scratch = torch.empty(need, dtype=torch.uint8, device="cuda")
  args = (x.data_ptr(), 100, None)
  assert L.alz_lpc_covar_apply_f32(*args, None, coef.data_ptr(), None, None, F, st.tensor.data_ptr(), 2, 100, 4, 32,
                                   16, 0, scratch.data_ptr(), need - 8, None) == -1
  assert "scratch" in L.alz_lpc_last_error().decode()
  lagm = torch.empty(2 * F * 25 + 1, dtype=torch.float64, device="cuda")
  assert L.alz_lpc_covar_apply_f32(*args, ctypes.c_void_p(lagm.data_ptr() + 4), None, None, None, F,
                                   st.tensor.data_ptr(), 2, 100, 4, 32, 16, 0, None, 0, None) == -1
  assert "misaligned" in L.alz_lpc_last_error().decode()
  assert L.alz_lpc_covar_apply_f32(x.data_ptr(), 50, None, lagm.data_ptr(), None, None, None, F,
                                   st.tensor.data_ptr(), 2, 100, 4, 32, 16, 0, None, 0, None) == -1
  # none of the refused calls touched the state
  torch.cuda.synchronize()
  assert same(lp.apply(x, state=st).coef.cpu().numpy(), lp.apply(x).coef.cpu().numpy())


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
x = torch.rand((2, 5000), device="cuda") * 2 - 1
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for method in ("kautocor", "kcovar"):
    lp = ab.LpcFrames(8, 256, 128, method=method)
    state = lp.new_state(2)
    lp.apply(x, state=state, final=True)
  ab.LpcFrames(64, 256, 128, method="kcovar").apply(x, final=True)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_lpc" in e.name}):
  print("LAUNCHED", name)
"""


def test_both_methods_launch_exactly_the_library_kernels(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["lpc"].path, _LAUNCH_PROBE)
