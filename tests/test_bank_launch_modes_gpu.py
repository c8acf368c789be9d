"""Launch modes of the TMA bank kernel at shapes too large or too ragged for the kernel matrix, on a representative set
of its instantiations: the ones whose register allocation the vector store path changed (DESIGN.md section 3) and the
extremes of cascade length, numerator taps and gain placement.

Tile groups are forced at plan creation (``ALZ_TILE_GROUP``), the store path of groups of 4 with ``ALZ_STORE_PATH``.
Every run must give the bits and the final state of the plan at tile group 1, whose output is checked against the
float64 oracle, and leave every output word it must not write as the NaN sentinel ``km.Gpu.run`` fills in.  Every bank
launch's ``ALZ_LOG_LAUNCH`` line must name the forced tile group and the store path that group takes."""
import numpy as np
import pytest

import oracle
import test_kernel_matrix as km
from test_segment_tail_gpu import LOG as GEOMETRY_LOG, expected_segments

pytestmark = pytest.mark.gpu

REPRESENTATIVES = [
  "biquad-K1-kmax1-nb1-monic0-small",
  "biquad-K4-kmax4-nb2-monic1-large",     # <4, 2, 1>: spills since the vector path
  "biquad-K3-kmax3-nb3-monic1-large",     # <3, 3, 1>: spills since the vector path
  "biquad-K4-kmax4-nb3-monic0-large",     # <4, 3, 0>: more spills
  "biquad-K8-kmax8-nb3-monic2-large",     # <8, 3, 2>: more spills; the longest cascade
  "klapuri-monic2-C30",                   # the zero-tap-mask <4, 3, 0> instantiation
  "headfir-K4-nb3-monic2-C30",            # head FIR: tile group 4 keeps TMA box stores
]

# S: one stream, ragged stream groups on both sides of 32, and more than two groups.  T: less than one tile; every
# remainder mod 4 (1, 2, 3: the lanes write the ragged last tile); last tile groups of 1 (129, 160, 4099), 2 (36),
# 3 (196) and 4 (98, 228) tiles, most of them with a partial last tile.
RAGGED_S = [1, 31, 33, 70]
RAGGED_T = [1, 3, 4, 31, 32, 36, 98, 129, 160, 196, 228, 4099]
SEGMENT_T = 2304

_PLANS = {}


@pytest.fixture(scope="module")
def gpu():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return km.Gpu()


def _plan(gpu, case, group, path="vec"):
  key = (case.id, group, path)
  if key not in _PLANS:
    _PLANS[key] = km._plan(gpu, case, ALZ_TILE_GROUP=group, ALZ_STORE_PATH=path)
  return _PLANS[key]


def _check_log(log, plan, group, path, what):
  assert log, "%s: no TMA bank launch logged" % what
  assert all(g == group and p == km.store_path(plan, group, path) for g, _, _, p, _ in log), (what, log)


@pytest.mark.parametrize("S", RAGGED_S)
@pytest.mark.parametrize("cid", REPRESENTATIVES)
def test_ragged_shapes(gpu, capfd, cid, S):
  """Group 4 on both store paths against group 1, at every ragged T.  Each T filters the first T samples of one signal:
  group 1 must give the first T samples of its output over the whole signal, which is checked against the oracle.  (The
  bars are set on rows of a few hundred samples and more: rows of 3 to 31 samples of the plans with the gain on the
  float32 input measured up to 7e-7 against 2.5e-7, relative to their small peaks.)"""
  case = km.BY_ID[cid]
  p1 = _plan(gpu, case, 1)
  xo, yo, xg, yg = km._seeds(case, p1)
  x_all = km._signal(case, S, max(RAGGED_T))
  y_all, log = km.logged(capfd, lambda: gpu.run(p1, x_all, xg, yg))
  _check_log(log, p1, 1, "vec", "%s S=%d, tile group 1" % (cid, S))
  km._check_rows(y_all, oracle.bank_apply(x_all, case.bank, xinit=xo, yinit=yo), km._row_tol(p1, case),
                 "%s S=%d T=%d" % (cid, S, x_all.shape[1]))
  for T in RAGGED_T:
    x = np.ascontiguousarray(x_all[:, :T])
    (y1, st1), log = km.logged(capfd, lambda: gpu.run(p1, x, xg, yg, state_out=True))
    _check_log(log, p1, 1, "vec", "%s S=%d T=%d, tile group 1" % (cid, S, T))
    assert np.array_equal(km.bits(y1), km.bits(y_all[:, :, :T])), "%s S=%d T=%d: not a prefix of the whole run" % (
      cid, S, T)
    for path in ("vec", "tma"):
      what = "%s S=%d T=%d, tile group 4, %s stores" % (cid, S, T, path)
      p4 = _plan(gpu, case, 4, path)
      (y, st), log = km.logged(capfd, lambda: gpu.run(p4, x, xg, yg, state_out=True))
      _check_log(log, p4, 4, path, what)
      assert np.array_equal(km.bits(y), km.bits(y1)), "%s: output differs from tile group 1" % what
      assert np.array_equal(km.bits(st), km.bits(st1)), "%s: final state differs from tile group 1" % what


@pytest.mark.parametrize("group", [2, 4])
@pytest.mark.parametrize("cid", REPRESENTATIVES)
def test_segmented(gpu, capfd, cid, group):
  """About 1.2 waves of warps at the group's occupancy: cut into time segments chained through the state, which give
  the bits of the unsegmented launch."""
  case = km.BY_ID[cid]
  plan = _plan(gpu, case, group)
  C = plan.n_channels
  _, log = km.logged(capfd, lambda: gpu.run(plan, km._signal(case, 32, 64)), GEOMETRY_LOG)
  slots = log[0][3]
  groups = -(-6 * slots // (5 * C))
  S, T = 32 * groups, SEGMENT_T
  warps = C * groups
  x = km._signal(case, S, T)
  xo, yo, xg, yg = km._seeds(case, plan)
  (y, st), log = km.logged(capfd, lambda: gpu.run(plan, x, xg, yg, state_out=True), GEOMETRY_LOG)
  assert len(log) == 1, log
  w, ng, _, sl, nseg, _ = log[0]
  assert (w, ng, sl) == (warps, group, slots), log
  assert nseg == expected_segments(warps, slots, groups, T, ng) > 1, log
  with km._env(ALZ_NO_SEGMENT=1):
    (y2, st2), log = km.logged(capfd, lambda: gpu.run(plan, x, xg, yg, state_out=True), GEOMETRY_LOG)
  assert len(log) == 1 and log[0][4] == 1, log
  assert np.array_equal(km.bits(y), km.bits(y2)), "%s, tile group %d: segments differ from one launch" % (cid, group)
  assert np.array_equal(km.bits(st), km.bits(st2)), "%s, tile group %d: segmented final state differs" % (cid, group)
  rows = [0, 31, 32, S // 2, S - 1]
  km._check_rows(y[rows], oracle.bank_apply(x[rows], case.bank, xinit=xo, yinit=yo), km._row_tol(plan, case),
                 "%s, tile group %d, %d segments" % (cid, group, nseg))


def _run_layout(gpu, plan, x, xg, yg, layout):
  """``x`` [S][T] (T a multiple of 4) into channel-major rows y[C][S][T + 8] (row stride S (T + 8), stream stride
  T + 8), or into channels 8 ... 8 + C of y[S][C + 16][T + 8]: (y as [S][C][T], final state); every word of the
  buffer outside the written rows keeps the sentinel."""
  torch = gpu.torch
  S, T = x.shape
  C, Tp = plan.n_channels, T + 8
  xd = torch.from_numpy(x).to(gpu.dev)
  if layout == "channel":
    shape, off, ys, ysS = (C, S, Tp), 0, S * Tp, Tp
  else:
    shape, off, ys, ysS = (S, C + 16, Tp), 8 * Tp, Tp, (C + 16) * Tp
  buf = torch.full((int(np.prod(shape)) + 4,), km.SENTINEL, dtype=torch.int32, device=gpu.dev)
  st = torch.empty(plan.state_doubles(S), dtype=torch.float64, device=gpu.dev)
  cur = gpu.stream()
  plan.state_init(st.data_ptr(), S, xg, yg, cur)
  plan.apply_ex(xd.data_ptr(), buf.data_ptr() + 4 * off, st.data_ptr(), S, T, T, ys, ysS, cur)
  torch.cuda.synchronize()
  rows = buf[:-4].view(*shape)
  written = torch.zeros_like(rows, dtype=torch.bool)
  if layout == "channel":
    written[:, :, :T] = True
    y = rows[:, :, :T].permute(1, 0, 2)
  else:
    written[:, 8:8 + C, :T] = True
    y = rows[:, 8:8 + C, :T]
  outside = torch.cat([rows[~written], buf[-4:]])
  assert bool((outside == km.SENTINEL).all()), "%d words outside the output rows were written" % int(
    (outside != km.SENTINEL).sum())
  assert not bool((rows[written] == km.SENTINEL).any()), "samples of the output rows were never written"
  return y.contiguous().view(torch.float32).cpu().numpy(), st.cpu().numpy()


@pytest.mark.parametrize("layout", ["channel", "slice"])
@pytest.mark.parametrize("cid", REPRESENTATIVES)
def test_layouts(gpu, capfd, cid, layout):
  """Channel-major output and a channel slice of a wider output at group 4 on the vector path: the bits of stream-major
  output at group 1."""
  case = km.BY_ID[cid]
  S, T = 70, 4100
  p1, p4 = _plan(gpu, case, 1), _plan(gpu, case, 4)
  xo, yo, xg, yg = km._seeds(case, p1)
  x = km._signal(case, S, T)
  y1, st1 = gpu.run(p1, x, xg, yg, state_out=True)
  km._check_rows(y1[::23], oracle.bank_apply(x[::23], case.bank, xinit=xo, yinit=yo), km._row_tol(p1, case), cid)
  (y, st), log = km.logged(capfd, lambda: _run_layout(gpu, p4, x, xg, yg, layout))
  what = "%s, %s layout, tile group 4" % (cid, layout)
  _check_log(log, p4, 4, "vec", what)
  assert np.array_equal(km.bits(y), km.bits(y1)), "%s: output differs from stream-major tile group 1" % what
  assert np.array_equal(km.bits(st), km.bits(st1)), "%s: final state differs from tile group 1" % what
