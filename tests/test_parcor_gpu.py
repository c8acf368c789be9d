"""``parcor_batch`` on the GPU: the reference's goldens, LpcFrames output at the flagship shape, every row length, row
counts across grid edges, leading shapes, strided rows, NaN isolation, concurrency and kernel coverage, all bit for bit
against the CPU restatement (tests/parcor_emulation.py)."""
import json
import os
import threading

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build
from conftest import ROOT
from native_libs import check_every_kernel_is_launched, torch  # noqa: F401  (fixture)
from parcor_emulation import parcor_row

pytestmark = pytest.mark.gpu

CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "parcor_cases.json")))["cases"]
ERRORS = {None: 0, "ParCorError": 1, "OverflowError": 2}


def expected(rows, L):
  """(k [n, L - 1], count, failed, stable) of the emulation, k NaN past count."""
  n = len(rows)
  k = np.full((n, L - 1), np.nan)
  count = np.zeros(n, np.int32)
  failed = np.zeros(n, np.uint8)
  stable = np.zeros(n, bool)
  for i, row in enumerate(rows):
    ks, f, st = parcor_row(row)
    k[i, :len(ks)] = ks
    count[i], failed[i], stable[i] = len(ks), f, st
  return k, count, failed, stable


def same(got, want):
  got = np.asarray(got, np.float64)
  want = np.asarray(want, np.float64)
  nan = np.isnan(want)
  return got.shape == want.shape and np.array_equal(np.isnan(got), nan) and \
      np.array_equal(got[~nan].view(np.uint64), want[~nan].view(np.uint64))


def check(res, rows, L):
  k, count, failed, stable = expected(rows, L)
  assert same(res.k.cpu().numpy().reshape(len(rows), L - 1), k)
  assert np.array_equal(res.count.cpu().numpy().reshape(-1), count)
  assert np.array_equal(res.failed.cpu().numpy().reshape(-1), failed)
  assert np.array_equal(res.stable.cpu().numpy().reshape(-1), stable)


@pytest.mark.parametrize("pad", [False, True])
def test_every_golden(torch, pad):
  """Each golden row at its own length, and all of them in one batch padded with zeros to L = 65 (trailing zeros are
  dropped, so the results are the same)."""
  if pad:
    res = ab.parcor_batch(torch.tensor([c["row"] + [0.0] * (65 - len(c["row"])) for c in CASES],
                                       dtype=torch.float64, device="cuda"))
    outs = [tuple(t[i].cpu().numpy().reshape(-1) for t in res) for i in range(len(CASES))]
  else:
    outs = [tuple(t.cpu().numpy().reshape(-1)
                  for t in ab.parcor_batch(torch.tensor([c["row"]], dtype=torch.float64, device="cuda")))
            for c in CASES]
  for c, (k, count, failed, stable) in zip(CASES, outs):
    if not c["row"][0] == 1.0:
      assert failed[0] == 3 and count[0] == 0 and not stable[0] and np.isnan(k).all()
      continue
    n = len(c["k"])
    assert count[0] == n and failed[0] == ERRORS[c["error"]] and bool(stable[0]) == c["stable"], c["name"]
    assert same(k[:n], c["k"]) and np.isnan(k[n:]).all(), c["name"]


def test_lpc_frames_flagship(torch):
  """LpcFrames(16, 1024, 512) of 4096 x 16384 samples: a sample of rows and every failed row against the
  emulation."""
  g = torch.Generator(device="cuda").manual_seed(5)
  x = torch.rand((4096, 16384), device="cuda", generator=g) * 2 - 1
  x[7, :] = 0                                                   # silent streams: failed LPC frames, NaN rows
  x[9, 4000:] = 0.25
  coef = ab.LpcFrames(16, 1024, 512).apply(x).coef
  res = ab.parcor_batch(coef)
  flat = coef.reshape(-1, 17)
  n = flat.shape[0]
  pick = np.unique(np.r_[np.random.default_rng(0).choice(n, 3000, replace=False), np.arange(64), n - 1,
                         np.flatnonzero(res.failed.reshape(-1).cpu().numpy())])
  rows = flat[torch.from_numpy(pick).cuda()].cpu().numpy().tolist()
  k, count, failed, stable = expected(rows, 17)
  sel = torch.from_numpy(pick).cuda()
  assert same(res.k.reshape(-1, 16)[sel].cpu().numpy(), k)
  assert np.array_equal(res.count.reshape(-1)[sel].cpu().numpy(), count)
  assert np.array_equal(res.failed.reshape(-1)[sel].cpu().numpy(), failed)
  assert np.array_equal(res.stable.reshape(-1)[sel].cpu().numpy(), stable)
  assert res.k.shape == (4096, coef.shape[1], 16) and res.stable.shape == coef.shape[:2]


def _random_rows(rng, n, L):
  """Stable and unstable rows with zeros and a few specials."""
  rows = rng.standard_normal((n, L)) * rng.choice([.05, .3, 1.], (n, 1))
  rows[:, 0] = 1.0
  rows[rng.random((n, L)) < .05] = 0.0
  if L > 1:
    spec = rng.random(n) < .01
    rows[spec, rng.integers(1, L, spec.sum())] = rng.choice([np.nan, np.inf, -np.inf, 1.0, -1.0, 1e200], spec.sum())
  return rows


@pytest.mark.parametrize("L", range(1, 66))
def test_every_row_length(torch, L):
  rows = _random_rows(np.random.default_rng(L), 300, L)
  check(ab.parcor_batch(torch.tensor(rows, device="cuda")), rows.tolist(), L)


@pytest.mark.parametrize("n,L", [(1, 17), (31, 17), (32, 17), (33, 17), (15, 33), (16, 33), (17, 33), (7, 65),
                                 (8, 65), (9, 65), (262145, 17), (1_000_000, 17), (200_000, 65)])
def test_row_counts_across_grid_edges(torch, n, L):
  rng = np.random.default_rng(n)
  rows = torch.tensor(_random_rows(rng, n, L), device="cuda")
  res = ab.parcor_batch(rows)
  pick = np.unique(np.r_[np.arange(min(n, 40)), np.arange(max(0, n - 40), n),
                         rng.integers(0, n, 500)]) if n > 2000 else np.arange(n)
  sel = torch.from_numpy(pick).cuda()
  k, count, failed, stable = expected(rows[sel].cpu().numpy().tolist(), L)
  assert same(res.k[sel].cpu().numpy(), k)
  assert np.array_equal(res.count[sel].cpu().numpy(), count) and np.array_equal(res.failed[sel].cpu().numpy(), failed)
  assert np.array_equal(res.stable[sel].cpu().numpy(), stable)


def test_leading_shapes_and_strided_rows(torch):
  rows = _random_rows(np.random.default_rng(3), 2 * 3 * 5, 9)
  t = torch.tensor(rows, device="cuda")
  want = ab.parcor_batch(t)
  got = ab.parcor_batch(t.reshape(2, 3, 5, 9))
  assert got.k.shape == (2, 3, 5, 8) and got.count.shape == (2, 3, 5)
  assert same(got.k.reshape(-1, 8).cpu(), want.k.cpu()) and torch.equal(got.stable.reshape(-1), want.stable)
  wide = torch.full((30, 20), 7.0, dtype=torch.float64, device="cuda")
  wide[:, 3:12] = t                                             # rows of 9 inside rows of 20: stride 20
  strided = ab.parcor_batch(wide[:, 3:12])
  assert same(strided.k.cpu(), want.k.cpu()) and torch.equal(strided.failed, want.failed)
  transposed = t.t().contiguous().t()                           # last dimension not contiguous: copied
  assert same(ab.parcor_batch(transposed).k.cpu(), want.k.cpu())
  empty = ab.parcor_batch(torch.empty((0, 5), dtype=torch.float64, device="cuda"))
  assert empty.k.shape == (0, 4) and empty.count.shape == (0,)
  one = ab.parcor_batch(torch.ones((4, 1), dtype=torch.float64, device="cuda"))
  assert one.k.shape == (4, 0) and one.count.tolist() == [0] * 4 and one.stable.all()


def test_nan_rows_do_not_leak(torch):
  """A NaN, inf or failing row shares its warp with clean rows, which keep their values."""
  rng = np.random.default_rng(11)
  rows = _random_rows(rng, 64, 17)
  clean = ab.parcor_batch(torch.tensor(rows, device="cuda"))
  bad = rows.copy()
  bad[1::2, 5] = np.nan
  bad[2::4, 16] = 1e300
  bad[3::8, 0] = np.nan
  res = ab.parcor_batch(torch.tensor(bad, device="cuda"))
  even = slice(0, None, 4)
  assert same(res.k[even].cpu(), clean.k[even].cpu())
  check(res, bad.tolist(), 17)


def test_streams_and_threads(torch):
  rows = torch.tensor(_random_rows(np.random.default_rng(4), 50_000, 33), device="cuda")
  want = ab.parcor_batch(rows)
  torch.cuda.synchronize()
  outs = {}
  s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()

  def work(i, stream):
    with torch.cuda.stream(stream):
      for _ in range(3):
        outs[i] = ab.parcor_batch(rows)
      stream.synchronize()

  threads = [threading.Thread(target=work, args=(i, s)) for i, s in enumerate((s1, s2))]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for res in outs.values():
    assert same(res.k.cpu(), want.k.cpu()) and torch.equal(res.count, want.count)
    assert torch.equal(res.failed, want.failed) and torch.equal(res.stable, want.stable)


_LAUNCH_PROBE = r"""
import sys
sys.path.insert(0, sys.argv[1])
import torch
from torch.profiler import ProfilerActivity, profile
import audiolazy_b200 as ab
torch.cuda.set_device(0)
with profile(activities=[ProfilerActivity.CUDA]) as prof:
  for L in (9, 30, 65):
    ab.parcor_batch(torch.rand((100, L), dtype=torch.float64, device="cuda"))
  torch.cuda.synchronize()
for name in sorted({e.name.split("(")[0].strip() for e in prof.events() if e.name and "alz_parcor" in e.name}):
  print("LAUNCHED", name)
"""


def test_every_parcor_kernel_is_launched(torch):
  check_every_kernel_is_launched(_build.LIBRARIES["parcor"].path, _LAUNCH_PROBE)
