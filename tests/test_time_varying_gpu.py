"""The time-varying coefficient path on the GPU (``alz_apply_tv_f32``: the generic kernels with a per-sample coefficient
table), through the C ABI against ``oracle.tv_apply`` at 1e-7 of each row's peak, the kernel matrix's WINDOW bar.

The contract (include/alz_b200.h): every stream of a batch shares the table, tap ``i`` of sample ``j`` OF THE CALL reads
``table[i * coef_stride + j]``, and the histories are rings indexed by the absolute sample count.  So the tests cover
many streams, several sections, delays at and around the power-of-two ring sizes, ``coef_stride > T``, the three
load engines, block splits that advance the x, y and table pointers, seeded states, identical rows in every lane,
non-finite samples, the error codes, and every reference golden through the lazy API.
"""
import numpy as np
import pytest

import oracle
import test_kernel_matrix as km
from test_time_varying import CASES, check_golden_case, split_sections

pytestmark = pytest.mark.gpu

TOL = km.WINDOW                  # 1e-7 of each row's peak: float32 rounding of a float64 result is 6e-8
SHAPES_S = (1, 2, 31, 32, 33, 100, 1000)
SHAPES_T = (1, 31, 32, 33, 4097, 20000)
ORACLE_ROWS = (0, 1, 30, 31, 32, 33, 99, 511, 999)     # rows checked against the oracle (lane, warp and group edges)


def _section(num, den):
  """A (b, a) section with nonzero coefficients at the numerator delays ``num`` (delay 0 is always a tap) and feedback
  delays ``den``: the values only mark the taps, the table supplies the coefficients."""
  b = [0.0] * (max(num + [0]) + 1)
  a = [1.0] + [0.0] * max(den + [0])
  for d in num:
    b[d] = 1.0
  for d in den:
    a[d] = -0.5
  return b, a


#: name -> cascade of sections
TAP_SETS = {
  "d0": [_section([0], [])],
  "dense0-3": [_section([0, 1, 2, 3], [])],
  "sparse0-16-17": [_section([0, 16, 17], [])],
  "fb1-3": [_section([0], [1, 2, 3])],
  "three-sections": [_section([0, 1], [1]), _section([0, 3], [2, 17]), _section([0], [1, 16])],
  "two-sections": [_section([0, 2, 65], []), _section([0, 1], [1, 64])],
}
for _d in (15, 16, 17, 63, 64, 65, 255, 256, 257):
  TAP_SETS["max%d" % _d] = [_section([0, _d // 2, _d], [1, _d])]


def expected_taps(sections):
  """The documented table order: section by section, numerator then feedback taps, ascending delay."""
  out = []
  for b, a in sections:
    out += [(d, False) for d, v in enumerate(b) if v != 0 or d == 0]
    out += [(d, True) for d, v in enumerate(a) if d >= 1 and v != 0]
  return out


def make_table(taps, T, stride, seed):
  """Random per-sample coefficients with sign changes and exact zeros at some samples.  Every section stays stable:
  its feedback magnitudes sum to at most 0.9, its numerator magnitudes to at most 1.5."""
  rng = np.random.default_rng(seed)
  table = np.zeros((len(taps), stride))
  sections = split_sections(taps)
  row = 0
  for sec in sections:
    nnum = sum(1 for _, den in sec if not den)
    nden = len(sec) - nnum
    for d, den in sec:
      scale = 0.9 / nden if den else 1.5 / nnum
      vals = rng.uniform(-scale, scale, T)
      vals[rng.random(T) < 0.05] = 0.0
      table[row, :T] = vals
      row += 1
  table[:, T:] = np.nan              # beyond the call: read by mistake, it poisons the output
  return table


class Tv(object):
  """Plans and calls of ``alz_apply_tv_f32`` on device buffers."""

  def __init__(self):
    self.g = km.Gpu()
    self.torch, self.capi = self.g.torch, self.g.capi

  def plan(self, sections):
    plan = self.capi.Plan([sections], force_generic=True)
    assert plan.kind == self.capi.KIND_GENERIC and plan.n_channels == 1 and plan.n_sections == len(sections)
    return plan

  def seeds(self, plan, seed):
    """Random float32-valued histories: ``(oracle xinit [K][xd], yinit [K][yd], plan xinit, plan yinit)``."""
    rng = np.random.default_rng(seed)
    K = plan.n_sections
    xi = rng.uniform(-.5, .5, (K, plan.xd)).astype(np.float32).astype(np.float64)
    yi = rng.uniform(-.5, .5, (K, plan.yd)).astype(np.float32).astype(np.float64)
    return xi, yi, xi[None] if plan.xd else None, yi[None] if plan.yd else None

  def run(self, plan, x, table, xinit=None, yinit=None, splits=None, engine="tma"):
    """``x`` [S][T] with ``table`` [ntaps][coef_stride] (host) through ``plan``: rows padded to a multiple of 4 samples;
    engine "tma" (16-byte aligned rows), "cpasync" (ALZ_NO_TMA=1) or "unaligned" (base pointers one float off 16 bytes);
    ``splits``: lengths of the leading calls, the last call takes the rest.  Returns ``(y [S][T], launches)``."""
    torch = self.torch
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    S, T = x.shape
    stride = (T + 3) // 4 * 4
    off = 1 if engine == "unaligned" else 0
    dev = self.g.dev
    xb = torch.zeros(S * stride + 4, dtype=torch.float32, device=dev)
    xb[off:off + S * stride].view(S, stride)[:, :T] = torch.from_numpy(x).to(dev)
    yb = torch.full((S * stride + 4,), float("nan"), dtype=torch.float32, device=dev)
    tb = torch.from_numpy(np.ascontiguousarray(table)).to(dev)
    st = torch.empty(max(1, plan.state_doubles(S)), dtype=torch.float64, device=dev)
    cur = self.g.stream()
    plan.state_init(st.data_ptr(), S, xinit, yinit, cur)
    before = self.capi.launch_count()
    with km._env(ALZ_NO_TMA=1 if engine == "cpasync" else 0):
      t0 = 0
      for n in list(splits or []) + [T - sum(splits or [])]:
        plan.apply_tv(xb.data_ptr() + 4 * (off + t0), yb.data_ptr() + 4 * (off + t0), st.data_ptr(), S, n, stride,
                      stride, tb.data_ptr() + 8 * t0, table.shape[1], cur)
        t0 += n
      torch.cuda.synchronize()
    launches = self.capi.launch_count() - before
    return yb[off:off + S * stride].view(S, stride)[:, :T].cpu().numpy(), launches


@pytest.fixture(scope="module")
def tv():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return Tv()


def row_errors(y, ref):
  den = np.max(np.abs(ref), axis=-1)
  return np.max(np.abs(y.astype(np.float64) - ref), axis=-1) / np.where(den == 0, 1.0, den)


def check_oracle(plan, x, y, table, xi=None, yi=None, what=""):
  """Rows ORACLE_ROWS of ``y`` against ``oracle.tv_apply`` at TOL of each row's peak."""
  S, T = x.shape
  rows = sorted({r for r in ORACLE_ROWS if r < S} | {S - 1})
  ref = oracle.tv_apply(x[rows], split_sections(plan.taps()), table[:, :T], xi, yi)
  err = row_errors(y[rows], ref)
  print("%-40s worst row %.3g of its peak" % (what, err.max()))
  assert np.all(np.isfinite(y[rows])), what
  assert err.max() <= TOL, (what, rows[int(np.argmax(err))], float(err.max()))
  return err.max()


def _signal(seed, S, T):
  return np.random.default_rng(seed).uniform(-1, 1, (S, T)).astype(np.float32)


# ---- shapes x tap sets ----------------------------------------------------------------------------------------------
NAMES = sorted(TAP_SETS)
SHAPE_CASES = [(S, T, NAMES[(i * len(SHAPES_T) + j) % len(NAMES)])
               for i, S in enumerate(SHAPES_S) for j, T in enumerate(SHAPES_T)]


@pytest.mark.parametrize("S, T, name", SHAPE_CASES)
def test_shapes_against_the_oracle(tv, S, T, name):
  """Every (S, T) pair with one of the tap sets (each set meets several shapes); a coefficient stride 5 samples longer
  than T; one launch per call, also above the time-parallel threshold (time-varying calls are always sequential)."""
  sections = TAP_SETS[name]
  plan = tv.plan(sections)
  taps = plan.taps()
  assert taps == expected_taps(sections)
  table = make_table(taps, T, T + 5, seed=S * 100003 + T)
  x = _signal(S + 7 * T, S, T)
  y, launches = tv.run(plan, x, table)
  assert launches == 1
  check_oracle(plan, x, y, table, what="S=%d T=%d %s" % (S, T, name))


@pytest.mark.parametrize("name", NAMES)
def test_tap_sets_seeded_against_the_oracle(tv, name):
  """Each tap set on 33 streams x 4097 samples from seeded ``memory=`` / ``zero=`` histories."""
  sections = TAP_SETS[name]
  plan = tv.plan(sections)
  taps = plan.taps()
  assert taps == expected_taps(sections)
  S, T = 33, 4097
  table = make_table(taps, T, T, seed=NAMES.index(name))
  x = _signal(500 + NAMES.index(name), S, T)
  xi, yi, xg, yg = tv.seeds(plan, NAMES.index(name))
  y, _ = tv.run(plan, x, table, xg, yg)
  check_oracle(plan, x, y, table, xi, yi, what="seeded %s" % name)
  if plan.xd or plan.yd:                  # the seeds matter: the unseeded run differs near the start
    y0, _ = tv.run(plan, x, table)
    assert not np.array_equal(y0[:, :300], y[:, :300])


# ---- bit-level invariants -------------------------------------------------------------------------------------------
INVARIANT_SETS = ["three-sections", "max16", "max64", "max256", "sparse0-16-17"]


@pytest.mark.parametrize("name", INVARIANT_SETS)
def test_engines_and_block_splits_give_the_same_bits(tv, name):
  """The TMA, cp.async and unaligned-row engines agree; block splits of 0, 1, 31, 32, 33 and 1000 samples (x, y and
  table pointers advanced by the samples done) give the bits of one call; seeded, against the oracle."""
  sections = TAP_SETS[name]
  plan = tv.plan(sections)
  S, T = 37, 3001
  table = make_table(plan.taps(), T, T + 3, seed=7 + INVARIANT_SETS.index(name))
  x = _signal(900 + INVARIANT_SETS.index(name), S, T)
  xi, yi, xg, yg = tv.seeds(plan, 11)
  y, _ = tv.run(plan, x, table, xg, yg)
  check_oracle(plan, x, y, table, xi, yi, what="engines %s" % name)
  assert np.array_equal(tv.run(plan, x, table, xg, yg, engine="cpasync")[0], y), "cp.async engine differs from TMA"
  assert np.array_equal(tv.run(plan, x, table, xg, yg, engine="unaligned")[0], y), "unaligned rows differ from TMA"
  split, launches = tv.run(plan, x, table, xg, yg, splits=[0, 1, 31, 32, 33, 1000])
  assert launches == 6                          # the empty call launches nothing
  assert np.array_equal(split, y), "block splits are not bit-exact"


@pytest.mark.parametrize("name", ["three-sections", "max65"])
def test_identical_rows_in_every_lane_and_warp(tv, name):
  """1000 copies of one row give the one-stream result in every lane of every warp, bit for bit."""
  plan = tv.plan(TAP_SETS[name])
  T = 2049
  table = make_table(plan.taps(), T, T, seed=3)
  x1 = _signal(4, 1, T)
  xi, yi, xg, yg = tv.seeds(plan, 5)
  y1, _ = tv.run(plan, x1, table, xg, yg)
  check_oracle(plan, x1, y1, table, xi, yi, what="one row %s" % name)
  y, _ = tv.run(plan, np.repeat(x1, 1000, axis=0), table, xg, yg)
  assert np.array_equal(y, np.repeat(y1, 1000, axis=0))


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf])
def test_nonfinite_samples_stay_in_their_stream(tv, value):
  """A NaN or inf sample in one stream leaves every other stream, and that stream's earlier outputs, bit-identical
  (the streams share only the coefficient table)."""
  plan = tv.plan(TAP_SETS["three-sections"])
  S, T, s_bad, t_bad = 70, 1500, 33, 700
  table = make_table(plan.taps(), T, T, seed=9)
  x = _signal(10, S, T)
  clean, _ = tv.run(plan, x, table)
  x[s_bad, t_bad] = value
  for engine in ("tma", "cpasync", "unaligned"):
    y, _ = tv.run(plan, x, table, engine=engine)
    others = np.arange(S) != s_bad
    assert np.array_equal(y[others], clean[others]), engine
    assert np.array_equal(y[s_bad, :t_bad], clean[s_bad, :t_bad]), engine
    assert not np.isfinite(y[s_bad, t_bad]), engine


# ---- error codes ----------------------------------------------------------------------------------------------------
def test_error_codes(tv):
  """Plans without a tap table refuse (ALZ_ERR_UNSUPPORTED); a coefficient stride shorter than the call or a null
  table is ALZ_ERR_INVALID."""
  torch, capi = tv.torch, tv.capi
  dev, cur = tv.g.dev, tv.g.stream()
  S, T = 2, 64
  x = torch.zeros((S, T), dtype=torch.float32, device=dev)
  y = torch.empty((S, T), dtype=torch.float32, device=dev)
  table = torch.zeros((8, T), dtype=torch.float64, device=dev)
  state = torch.zeros(4096, dtype=torch.float64, device=dev)
  biquad = capi.Plan([[([1., .5, .25], [1., -.5, .2])]])
  window = capi.Plan([[([1.] + [0.] * 19 + [.5], [1., -.3])]])
  multi = capi.Plan([[([1., .5], [1., -.3])], [([1., .25], [1., .2])]], force_generic=True)
  assert biquad.kind == capi.KIND_BIQUAD and window.kind == capi.KIND_GENERIC and multi.n_channels == 2
  for plan in (biquad, window, multi):
    with pytest.raises(capi.NativeError, match="error -6"):
      plan.apply_tv(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T, table.data_ptr(), T, cur)
  with pytest.raises(capi.NativeError, match="error -6"):
    window.taps()
  plan = tv.plan([_section([0, 1], [1])])
  with pytest.raises(ValueError):
    plan.apply_tv(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T, table.data_ptr(), T - 1, cur)
  with pytest.raises(ValueError):
    plan.apply_tv(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T, None, T, cur)
  plan.apply_tv(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T, table.data_ptr(), T, cur)
  torch.cuda.synchronize()


# ---- the reference's goldens through the lazy API -------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(CASES))
def test_golden_case_through_the_lazy_api(tv, monkeypatch, name):
  """At 1e-7 of the peak.  The LTI members of the cascade cases run without the float32 tier, whose bar is its own
  (2.5e-6, tests/test_tiers.py); the time-varying filters always run in float64."""
  import audiolazy_b200 as ab
  from audiolazy_b200 import _engine
  monkeypatch.setenv("ALZ_NO_FP32_TIER", "1")
  monkeypatch.setattr(_engine, "_cache", {})
  check_golden_case(ab, CASES[name])
