"""``LpcFilter`` on the GPU: the reference's goldens, every order, block splits, stream counts, strided and shared
coefficient tables, NaN rows of failed LpcFrames frames, the flagship LpcFrames -> analysis -> synthesis chain,
concurrency and kernel coverage, all bit for bit against the reference or the CPU restatement
(tests/lpc_filter_emulation.py)."""
import json
import os
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import ROOT
from lpc_filter_emulation import lpc_filter, same_bits
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "lpc_filter_cases.npz"))
META = json.loads(str(GOLDEN["meta"]))
KINDS = ["analysis", "synthesis"]


def f32_of(y):
  with np.errstate(all="ignore"):
    return np.asarray(y, np.float64).astype(np.float32)


def same_f32(got, want64):
  got = np.asarray(got, np.float32)
  want = f32_of(want64)
  nan = np.isnan(want)
  return got.shape == want.shape and np.array_equal(np.isnan(got), nan) and \
      np.array_equal(got[~nan].view(np.uint32), want[~nan].view(np.uint32))


def rand_rows(rng, S, F, order, scale=.3):
  return np.concatenate([np.ones((S, F, 1)), rng.standard_normal((S, F, order)) * scale], axis=2)


def test_every_golden(torch):
  """Each case from float64 input (and from float32 input where its samples are float32), to float64 output bit for
  bit and to float32 output as its rounding."""
  for i, m in enumerate(META):
    x, coef, y = GOLDEN["x_%d" % i], GOLDEN["coef_%d" % i], GOLDEN["y_%d" % i]
    c = torch.tensor(coef[None], dtype=torch.float64, device="cuda")
    xd = torch.tensor(x[None], dtype=torch.float64, device="cuda")
    f64 = ab.LpcFilter(m["order"], m["hop"], m["kind"], torch.float64)
    f32 = ab.LpcFilter(m["order"], m["hop"], m["kind"], torch.float32)
    assert same_bits(f64.apply(xd, c)[0].cpu().numpy(), y), m["name"]
    assert same_f32(f32.apply(xd, c)[0].cpu().numpy(), y), m["name"]
    if m["x_f32"]:
      xf = torch.tensor(x[None], dtype=torch.float32, device="cuda")
      assert same_bits(f64.apply(xf, c)[0].cpu().numpy(), y), m["name"]


@pytest.mark.parametrize("kind", KINDS)
def test_every_order(torch, kind):
  rng = np.random.default_rng(5)
  for order in range(0, 65):
    hop = int(rng.choice([1, 3, 64, 200, 1500]))
    S, T = 5, 1100
    x = rng.standard_normal((S, T))
    x[1, 17] = np.inf
    coef = rand_rows(rng, S, -(-T // hop), order, .5 / max(order, 1) if kind == "synthesis" else .5)
    if order:
      coef[2, 0, order] = 0.0
      coef[3, -1, 1] = np.nan
    want, _ = lpc_filter(kind, x, coef, hop)
    got = ab.LpcFilter(order, hop, kind, torch.float64).apply(torch.tensor(x, device="cuda"),
                                                              torch.tensor(coef, device="cuda"))
    assert same_bits(got.cpu().numpy(), want), order


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("order,hop", [(16, 7), (3, 1), (64, 160), (1, 5000), (40, 33), (32, 512)])
def test_block_splits_equal_one_call(torch, kind, order, hop):
  """Random cuts, with 1-sample, empty, mid-row and shorter-than-order blocks, give the bits of one call."""
  rng = np.random.default_rng(order * 1000 + hop)
  S, T = 33, 3000
  x = torch.tensor(rng.standard_normal((S, T)).astype(np.float32), device="cuda")
  coef = torch.tensor(rand_rows(rng, S, -(-T // hop) + 2, order, .05), device="cuda")
  f = ab.LpcFilter(order, hop, kind, torch.float64)
  want = f.apply(x, coef)
  cuts = sorted(c for c in set(rng.integers(0, T, 12).tolist()) | {0, 1, 2, 3, hop, hop + 1, T - 1, T} if c <= T)
  state = f.new_state(S)
  parts = []
  for a, b in zip([0] + cuts, cuts + [T]):
    r0 = a // hop
    parts.append(f.apply(x[:, a:b], coef[:, r0:], state=state))
  assert state.consumed == T
  assert torch.equal(torch.cat(parts, dim=1).view(torch.int64), want.view(torch.int64))


@pytest.mark.parametrize("S", [1, 31, 33, 4096])
@pytest.mark.parametrize("kind", KINDS)
def test_stream_counts(torch, S, kind):
  rng = np.random.default_rng(S)
  T, hop, order = 1500, 160, 16
  x = rng.standard_normal((S, T)).astype(np.float32)
  coef = rand_rows(rng, S, 10, order, .04)
  got = ab.LpcFilter(order, hop, kind, torch.float32).apply(torch.tensor(x, device="cuda"),
                                                            torch.tensor(coef, device="cuda")).cpu().numpy()
  pick = np.unique(np.r_[0, S - 1, rng.integers(0, S, 6)])
  want, _ = lpc_filter(kind, x[pick].astype(np.float64), coef[pick], hop)
  assert same_f32(got[pick], want)


@pytest.mark.parametrize("kind", KINDS)
def test_strided_and_shared_coef(torch, kind):
  rng = np.random.default_rng(9)
  S, T, hop, order = 6, 700, 50, 8
  x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
  rows = rand_rows(rng, S, 14, order, .1)
  f = ab.LpcFilter(order, hop, kind, torch.float64)
  want = f.apply(x, torch.tensor(rows, device="cuda")).cpu().numpy()
  big = torch.full((S, 28, 20), 7.0, dtype=torch.float64, device="cuda")
  big[:, ::2, 4:4 + order + 1] = torch.tensor(rows, device="cuda")
  assert same_bits(f.apply(x, big[:, ::2, 4:4 + order + 1]).cpu().numpy(), want)       # row stride 40
  perm = torch.tensor(rows, device="cuda").permute(1, 0, 2).contiguous().permute(1, 0, 2)
  assert same_bits(f.apply(x, perm).cpu().numpy(), want)                                 # stream stride 9
  shared = torch.tensor(rows[:1], device="cuda").expand(S, -1, -1)                       # stream stride 0
  one, _ = lpc_filter(kind, x.cpu().numpy(), np.broadcast_to(rows[:1], rows.shape), hop)
  assert shared.stride(0) == 0 and same_bits(f.apply(x, shared).cpu().numpy(), one)
  tcol = torch.tensor(rows, device="cuda").transpose(1, 2).contiguous().transpose(1, 2)  # taps not contiguous: copied
  assert same_bits(f.apply(x, tcol).cpu().numpy(), want)
  extra = torch.tensor(np.concatenate([rows, np.full((S, 5, order + 1), np.nan)], axis=1), device="cuda")
  assert same_bits(f.apply(x, extra).cpu().numpy(), want)                                # rows past F not read
  with pytest.raises(ValueError):
    f.apply(x, torch.tensor(rows[:, :13], device="cuda"))
  with pytest.raises(ValueError):
    f.apply(x, torch.tensor(rows[:, :, :order], device="cuda"))
  with pytest.raises(ValueError):
    f.apply(x, torch.tensor(rows, device="cuda").float())
  with pytest.raises(ValueError):
    f.apply(x, torch.tensor(rows, device="cuda"), state=ab.LpcFilter(order, hop + 1, kind).new_state(S))
  with pytest.raises(ValueError):
    f.apply(x, torch.tensor(rows, device="cuda"), state=f.new_state(S + 1))
  empty = f.apply(x[:, :0], torch.empty((S, 0, order + 1), dtype=torch.float64, device="cuda"))
  assert empty.shape == (S, 0)


def test_nan_rows_stay_in_their_stream(torch):
  """LpcFrames' failed frames (silent streams) give NaN rows; their NaN stays in their own stream."""
  g = torch.Generator(device="cuda").manual_seed(3)
  x = torch.rand((40, 8192), device="cuda", generator=g) * 2 - 1
  x[7] = 0
  x[9, 3000:] = 0
  coef = ab.LpcFrames(16, 1024, 512).apply(x).coef
  assert torch.isnan(coef[7]).all() and torch.isnan(coef[9, -1]).all()
  coef = torch.cat([coef, coef[:, -1:]], dim=1)                 # 16 rows cover the 8192 samples
  for kind in KINDS:
    f = ab.LpcFilter(16, 512, kind, torch.float64)
    y = f.apply(x, coef).cpu().numpy()
    assert np.isnan(y[7]).all()
    ok = [s for s in range(40) if s not in (7, 9)]
    assert not np.isnan(y[ok]).any()
    want, _ = lpc_filter(kind, x[[0, 9]].double().cpu().numpy(), coef[[0, 9]].cpu().numpy(), 512)
    assert same_bits(y[[0, 9]], want)


def test_flagship_chain(torch):
  """LpcFrames(16, 1024, 512) of 4096 x 16384 samples, its rows (the last repeated to cover every sample) through the
  analysis and then the synthesis filter; sampled streams against the emulation, and the resynthesis against x."""
  g = torch.Generator(device="cuda").manual_seed(8)
  x = torch.rand((4096, 16384), device="cuda", generator=g) * 2 - 1
  coef = ab.LpcFrames(16, 1024, 512).apply(x).coef
  F = ab.LpcFilter(16, 512).n_rows(0, 16384)
  coef = torch.cat([coef, coef[:, -1:].expand(-1, F - coef.shape[1], -1)], dim=1)
  res = ab.LpcFilter(16, 512, "analysis", torch.float64).apply(x, coef)
  syn = ab.LpcFilter(16, 512, "synthesis", torch.float64).apply(res, coef)
  pick = [0, 1, 777, 2048, 4095]
  xs = x[pick].double().cpu().numpy()
  cs = coef[pick].cpu().numpy()
  want_res, _ = lpc_filter("analysis", xs, cs, 512)
  assert same_bits(res[pick].cpu().numpy(), want_res)
  want_syn, _ = lpc_filter("synthesis", want_res, cs, 512)
  assert same_bits(syn[pick].cpu().numpy(), want_syn)
  assert torch.allclose(syn, x.double(), rtol=0, atol=1e-9)


def test_streams_and_threads(torch):
  rng = np.random.default_rng(4)
  S, T = 300, 5000
  x = torch.tensor(rng.standard_normal((S, T)), device="cuda")
  coef = torch.tensor(rand_rows(rng, S, 50, 16, .04), device="cuda")
  filters = [ab.LpcFilter(16, 100, kind, torch.float64) for kind in KINDS]
  want = [f.apply(x, coef) for f in filters]
  torch.cuda.synchronize()
  outs = {}
  streams = [torch.cuda.Stream() for _ in range(4)]

  def work(i, stream):
    f = filters[i % 2]
    with torch.cuda.stream(stream):
      for _ in range(3):
        state = f.new_state(S)
        parts = [f.apply(x[:, :1234], coef, state=state), f.apply(x[:, 1234:], coef[:, 12:], state=state)]
        outs[i] = torch.cat(parts, dim=1)
      stream.synchronize()

  threads = [threading.Thread(target=work, args=(i, s)) for i, s in enumerate(streams)]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for i, y in outs.items():
    assert torch.equal(y.view(torch.int64), want[i % 2].view(torch.int64))


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for kind, order in (("analysis", 4), ("synthesis", 4), ("synthesis", 40)):
    for xt in (torch.float32, torch.float64):
      for ot in (torch.float32, torch.float64):
        x = torch.rand((3, 100), dtype=xt, device="cuda")
        c = torch.rand((3, 10, order + 1), dtype=torch.float64, device="cuda") * .01
        ab.LpcFilter(order, 10, kind, ot).apply(x, c)
  for order in range(1, 33):
    ab.LpcFilter(order, 10, "synthesis").apply(torch.rand((3, 100), device="cuda"),
                                               torch.rand((3, 10, order + 1), dtype=torch.float64, device="cuda"))
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_lpcfilt" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_lpcfilt_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["lpcfilt"].path, _LAUNCH_PROBE)
