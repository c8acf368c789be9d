"""Time-parallel ``LpcFilter`` synthesis on the GPU (include/alz_b200_lpcscan.h): forced and model-chosen chunk counts
against the sequential synthesis within the bar (per stream, max |y_tp - y_seq| <= 1e-9 max |y_seq|) for both sample
dtypes, stream counts, every order, strided and shared tables and the reference's golden rows; the sequential
fallback of non-finite streams, bit for bit; state mixing; P = 1 calls; concurrency; kernel coverage."""
import json
import os
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import ROOT
from lpc_filter_emulation import lpc_filter, same_bits
from lpc_scan_emulation import lpc_scan, max_chunks, within_bar
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "lpc_filter_cases.npz"))
META = json.loads(str(GOLDEN["meta"]))


def rand_rows(rng, S, F, order, scale):
  return np.concatenate([np.ones((S, F, 1)), rng.standard_normal((S, F, order)) * scale], axis=2)


def pair(torch, order, hop, tp, dtype=None):
  dtype = dtype or torch.float64
  return (ab.LpcFilter(order, hop, "synthesis", dtype),
          ab.LpcFilter(order, hop, "synthesis", dtype, time_parallel=tp))


def np64(t):
  return t.double().cpu().numpy()


@pytest.mark.parametrize("S", [1, 3, 64])
@pytest.mark.parametrize("tp", [True, 50])
def test_dtypes_and_stream_counts(torch, S, tp):
  """float32 and float64 in and out: the float64 output within the bar, the float32 output its rounding."""
  rng = np.random.default_rng(S)
  T, hop, order = 40000, 480, 16
  e = rng.standard_normal((S, T))
  coef = torch.tensor(rand_rows(rng, S, -(-T // hop), order, .04), device="cuda")
  for xt in (torch.float32, torch.float64):
    x = torch.tensor(e, dtype=xt, device="cuda")
    seq, par = pair(torch, order, hop, tp)
    par32 = ab.LpcFilter(order, hop, "synthesis", torch.float32, time_parallel=tp)
    assert par.chunks(S, T) > 1
    want, got = seq.apply(x, coef), par.apply(x, coef)
    assert within_bar(np64(got), np64(want))
    assert torch.equal(par32.apply(x, coef), got.float())


def test_every_order(torch):
  rng = np.random.default_rng(2)
  for order in range(1, 65):
    S, T = 3, 3000
    hop = int(rng.choice([1, 7, 160, 480, 5000]))
    x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
    coef = torch.tensor(rand_rows(rng, S, -(-T // hop), order, .5 / order), device="cuda")
    P = int(rng.integers(2, max_chunks(T, order) + 1))
    seq, par = pair(torch, order, hop, P)
    assert par.chunks(S, T) == P
    assert within_bar(np64(par.apply(x, coef)), np64(seq.apply(x, coef))), (order, hop, P)


def test_strided_and_shared_rows(torch):
  rng = np.random.default_rng(9)
  S, T, hop, order = 6, 7000, 50, 8
  x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
  rows = rand_rows(rng, S, T // hop, order, .1)
  seq, par = pair(torch, order, hop, 40)
  big = torch.full((S, 2 * (T // hop), 20), 7.0, dtype=torch.float64, device="cuda")
  big[:, ::2, 4:4 + order + 1] = torch.tensor(rows, device="cuda")
  strided = big[:, ::2, 4:4 + order + 1]
  assert within_bar(np64(par.apply(x, strided)), np64(seq.apply(x, strided)))          # row stride 40
  perm = torch.tensor(rows, device="cuda").permute(1, 0, 2).contiguous().permute(1, 0, 2)
  assert within_bar(np64(par.apply(x, perm)), np64(seq.apply(x, perm)))                # stream stride 9
  shared = torch.tensor(rows[:1], device="cuda").expand(S, -1, -1)                    # stream stride 0
  assert within_bar(np64(par.apply(x, shared)), np64(seq.apply(x, shared)))


def test_golden_rows(torch):
  """Each synthesis case at 2, 3 and the most chunks: against the reference's recorded outputs and the sequential
  call, bit for bit where the emulation falls back, within the bar elsewhere."""
  for i, m in enumerate(META):
    if m["kind"] != "synthesis" or m["order"] == 0:
      continue
    x, coef, y = GOLDEN["x_%d" % i], GOLDEN["coef_%d" % i], GOLDEN["y_%d" % i]
    xd = torch.tensor(x[None], dtype=torch.float64, device="cuda")
    c = torch.tensor(coef[None], dtype=torch.float64, device="cuda")
    top = max_chunks(len(x), m["order"])
    for P in sorted({min(2, top), min(3, top), top}):
      got = ab.LpcFilter(m["order"], m["hop"], "synthesis", torch.float64, time_parallel=P).apply(xd, c)[0]
      got = got.cpu().numpy()
      _, _, flagged = lpc_scan(x[None], coef[None], m["hop"], P)
      if flagged[0]:
        assert same_bits(got, y), (m["name"], P)
      else:
        assert within_bar(got[None], y[None]), (m["name"], P)


def test_fallback_streams_keep_their_bits(torch):
  """Streams with an inf sample, a NaN sample, a NaN row or overflowing unstable rows, batched with clean streams, give
  the sequential bits and state; only those streams do."""
  rng = np.random.default_rng(11)
  S, T, order, hop = 7, 20000, 8, 100
  coef = rand_rows(rng, S, T // hop, order, .05)
  for s in (0, 6):                                              # clean resonators: a memory longer than a chunk
    coef[s, :, 1:3] = [-2 * .9995 * np.cos(.1 * (s + 1)), .9995 ** 2]
    coef[s, :, 3:] *= 1e-3
  x = rng.standard_normal((S, T))
  x[1, 12345] = np.inf
  x[2, 77] = np.nan
  coef[3, 90, 4] = np.nan
  coef[4, 5:, 1] = -3.0
  x[5, -1] = -np.inf
  _, _, flagged = lpc_scan(x, coef, hop, 16)
  assert flagged.tolist() == [False, True, True, True, True, True, False]
  xt, ct = torch.tensor(x, device="cuda"), torch.tensor(coef, device="cuda")
  seq, par = pair(torch, order, hop, 64)
  s_seq, s_par = seq.new_state(S), par.new_state(S)
  want, got = np64(seq.apply(xt, ct, state=s_seq)), np64(par.apply(xt, ct, state=s_par))
  hist_seq = s_seq.tensor.view(torch.float64).view(S, order).cpu().numpy()
  hist_par = s_par.tensor.view(torch.float64).view(S, order).cpu().numpy()
  for s in range(S):
    if flagged[s]:
      assert same_bits(got[s], want[s]) and same_bits(hist_par[s], hist_seq[s]), s
    else:
      assert within_bar(got[s:s + 1], want[s:s + 1]), s
      assert not same_bits(got[s], want[s]), s                  # chunked: the scan's drift shows
  assert np.isnan(want[4]).any() and np.isinf(want[1]).any()


@pytest.mark.parametrize("order,hop", [(16, 480), (3, 1), (64, 160), (33, 7000)])
def test_block_splits_mix_both_paths(torch, order, hop):
  """Calls cut at random, alternating time-parallel and sequential calls on one state, stay within the bar of one
  sequential call."""
  rng = np.random.default_rng(order * 1000 + hop)
  S, T = 3, 60000
  x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
  coef = torch.tensor(rand_rows(rng, S, -(-T // hop) + 2, order, .3 / order), device="cuda")
  seq, par = pair(torch, order, hop, 37)
  want = seq.apply(x, coef)
  cuts = sorted(set(rng.integers(1, T, 9).tolist()) | {hop, hop + 1, T // 2})
  state = seq.new_state(S)
  parts = []
  for i, (a, b) in enumerate(zip([0] + cuts, cuts + [T])):
    parts.append((par if i % 2 == 0 else seq).apply(x[:, a:b], coef[:, a // hop:], state=state))
  assert state.consumed == T
  assert within_bar(np64(torch.cat(parts, dim=1)), np64(want))


def test_one_chunk_is_todays_path(torch):
  """Where the model picks 1 (many streams, short calls) or 1 is forced, the bits are the sequential call's."""
  rng = np.random.default_rng(4)
  for S, T, tp in ((4096, 2048, True), (2, 300, True), (3, 5000, 1)):
    x = torch.tensor(rng.standard_normal((S, T)).astype(np.float32), device="cuda")
    coef = torch.tensor(rand_rows(rng, S, -(-T // 512), 16, .04), device="cuda")
    seq, par = pair(torch, 16, 512, tp, torch.float32)
    assert par.chunks(S, T) == 1
    assert torch.equal(par.apply(x, coef).view(torch.int32), seq.apply(x, coef).view(torch.int32))


def test_streams_and_threads(torch):
  rng = np.random.default_rng(6)
  S, T = 4, 50000
  x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
  coef = torch.tensor(rand_rows(rng, S, T // 100, 16, .04), device="cuda")
  f = ab.LpcFilter(16, 100, "synthesis", torch.float64, time_parallel=True)
  assert f.chunks(S, T) > 1
  want = f.apply(x, coef)
  torch.cuda.synchronize()
  outs = {}
  streams = [torch.cuda.Stream() for _ in range(4)]

  def work(i, stream):
    with torch.cuda.stream(stream):
      for _ in range(3):
        state = f.new_state(S)
        parts = [f.apply(x[:, :23456], coef, state=state), f.apply(x[:, 23456:], coef[:, 234:], state=state)]
        outs[i] = (torch.cat(parts, dim=1), f.apply(x, coef))
      stream.synchronize()

  threads = [threading.Thread(target=work, args=(i, s)) for i, s in enumerate(streams)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for split, whole in outs.values():
    assert torch.equal(whole.view(torch.int64), want.view(torch.int64))
    assert within_bar(np64(split), np64(want))


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for order in list(range(1, 33)) + [40]:
    ab.LpcFilter(order, 10, "synthesis", time_parallel=4).apply(
      torch.rand((2, 400), device="cuda"), torch.rand((2, 40, order + 1), dtype=torch.float64, device="cuda") * .01)
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_lpcscan" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_lpcscan_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["lpcscan"].path, _LAUNCH_PROBE)
