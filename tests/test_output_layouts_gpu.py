"""Every output layout the filter entry points accept, on the GPU: channel-major, padded channel-major, channel slices
of a wider tensor and stream-major rows with a gap between streams (``alz_apply_f32_ex``), the stream-split loop of
launches over more than 65535 x 32 streams, and the host staging pipeline with several chunks.

Each layout runs through the C ABI (and ``FilterBank.apply(..., channel_major=True)`` where the public API has it) on
the default engine (TMA where the strides allow it), with ``ALZ_NO_TMA=1`` and with x and y one float off 16 bytes.
Every row must be the bits of the same plan's dense ``alz_apply_f32`` output, every element outside the written rows
must keep the NaN the buffer was filled with, and rows 0, 1, 31, 32 and S - 1 must meet the float64 oracle at the
kernel matrix's per-tier bars.

16-byte vector stores need y, y_stride and y_stream_stride all aligned: the cp.async engine steps between the 32 rows of
a warp by y_stream_stride.  ``MISALIGNED_IF_UNCHECKED`` lists the cases whose y and y_stride are aligned while
y_stream_stride is not, and the module asserts that every plan has such cases on full and partial stream groups.
"""
import collections
import types

import numpy as np
import pytest

import oracle
import test_kernel_matrix as km
from design_space import BY_ID, kernel
from test_filter_designs_gpu import _SAMPLED, F32_RANGE
from test_time_varying import split_sections
from test_time_varying_gpu import _section, make_table

pytestmark = pytest.mark.gpu

#: a quiet NaN with a payload no kernel produces: written into every output buffer before a call, as int32 bits
SENTINEL = 0x7FC0DEAD


def _gammatone(strategy):
  import audiolazy_b200 as ab
  return ab.gammatone_bank(strategy=strategy)       # 64 channels, 48 kHz


def _filterbank(sections):
  """A FilterBank whose channels are the given sections (the public API over a design-space bank)."""
  import audiolazy_b200 as ab
  return ab.FilterBank([ab.CascadeFilter([ab.ZFilter(list(b), list(a)) for b, a in ch]) for ch in sections])


#: name -> FilterBank; each reaches its own store path
BANKS = collections.OrderedDict()
BANKS["slaney"] = _gammatone("slaney")                         # biquad K = 4, both precision tiers, gain mode 2
BANKS["sampled"] = _gammatone("sampled")                       # biquad K = 4 behind an 8-tap head FIR
for _id in ("sos-butter-N16",                                  # biquad K = 8
            "comb-fb-d15", "comb-fb-d100",                     # window kernel: near taps; a far-tap ring
            "cascade-comb48-biquad", "wide-comb-C113"):        # generic kernel
  BANKS[_id] = _filterbank(BY_ID[_id].bank)
  assert BANKS[_id].sections() == BY_ID[_id].bank

#: the oracle bar of a bank where a documented reason lifts it above the per-tier bar (test_filter_designs_gpu): the
#: sampled bank's float64-tier rows measured up to 1.1e-7 here (H100 80GB HBM3, 700 W), above their 6.5e-8
CEILING = {"sampled": (2.5e-7, _SAMPLED)}

SHAPES = [(S, T) for S in (4, 6, 33, 64) for T in (4096, 4097, 4098, 4099)] + [(1, 1), (1, 31)]
ENGINES = ("default", "notma", "offset")
ORACLE_ROWS = (0, 1, 31, 32)


def _round4(n):
  return (n + 3) // 4 * 4


def _layouts(S, C, T):
  """name -> (ys, ysS) of every layout at this shape; "slices" write one plan per channel range at ysS = C * ys."""
  out = collections.OrderedDict()
  out["cm"] = (S * T, T)
  for r in range(4):                                           # ysS mod 4 = r, ys mod 4 = 0, both padded
    ysS = T + 1 + (r - T - 1) % 4
    out["cmpad%d" % r] = (S * ysS + 1 + (-S * ysS - 1) % 4, ysS)
  out["slices-ysT"] = (T, C * T)
  out["slices-ys4"] = (_round4(T), C * _round4(T))
  for g in (1, 4):
    out["gap%d" % g] = (T, C * T + g)
  return out


def _ranges(C):
  """Three uneven channel ranges where the bank has three channels or more."""
  if C >= 38:
    cuts = [0, 5, 37, C]
  elif C >= 3:
    cuts = [0, 1, C // 2 + 1, C]
  else:
    cuts = [0, C]
  return list(zip(cuts, cuts[1:]))


CASES = [(name, S, T, lay, eng) for name in BANKS for S, T in SHAPES for lay in _layouts(S, 1, T) for eng in ENGINES]


def _case_id(c):
  return "%s-S%d-T%d-%s-%s" % c


def _misaligned_if_unchecked(name, S, T, lay, eng):
  """A case in which y and ys are 16-byte aligned, ysS is not, and a row holds a whole 16-byte group: without the ysS
  term in the store-alignment rule the cp.async engine would issue st.global.v4 at addresses 4 or 8 bytes off."""
  C = len(BANKS[name])
  ys, ysS = _layouts(S, C, T)[lay]
  return eng != "offset" and ys % 4 == 0 and ysS % 4 != 0 and T >= 4


MISALIGNED_IF_UNCHECKED = [_case_id(c) for c in CASES if _misaligned_if_unchecked(*c)]
for _name in BANKS:
  for _full in (True, False):                                  # the lean store path (32 streams) and the edge path
    assert any(_misaligned_if_unchecked(*c) and (c[1] >= 32) == _full for c in CASES if c[0] == _name), (_name, _full)
assert any("-cm-" in i and "-S64-T4097-" in i for i in MISALIGNED_IF_UNCHECKED)


# --------------------------------------------------------------------------------------------------------------------
# helpers
# --------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return km.Gpu()


_PLANS = {}


def _plan(gpu, name, lo=None, hi=None, **kw):
  key = (name, lo, hi, tuple(sorted(kw.items())))
  if key not in _PLANS:
    secs = BANKS[name].sections()
    _PLANS[key] = gpu.capi.Plan(secs if lo is None else secs[lo:hi], **kw)
  return _PLANS[key]


def _routing(plan):
  return (plan.kind, plan.n_sections, plan.num_taps, plan.monic_mode, kernel(plan))


class _X(object):
  """x [S][T] on the device: rows padded to a multiple of 4 samples, base ``off`` floats past a 16-byte boundary."""

  def __init__(self, gpu, x, off=0):
    torch = gpu.torch
    S, T = x.shape
    self.xs = max(_round4(T), 4)
    self.buf = torch.zeros(off + S * self.xs + 4, dtype=torch.float32, device=gpu.dev)
    self.rows = self.buf[off:off + S * self.xs].view(S, self.xs)[:, :T]
    self.rows.copy_(torch.from_numpy(x).to(gpu.dev))
    self.ptr = self.buf.data_ptr() + 4 * off


def _filled(gpu, n):
  """A float32 buffer of ``n`` elements holding SENTINEL bits."""
  torch = gpu.torch
  return torch.full((n,), SENTINEL, dtype=torch.int32, device=gpu.dev).view(torch.float32)


def _view(buf, off, S, C, T, ys, ysS):
  """The [S][C][T] rows at (ys, ysS) from element ``off`` of ``buf``, as int32 bits."""
  import torch
  return buf.view(torch.int32).as_strided((S, C, T), (ysS, ys, 1), off)


def _untouched(buf, written):
  """Every element of ``buf`` outside the ``written`` row sets ``(off, S, C, T, ys, ysS)`` still holds SENTINEL."""
  import torch
  mask = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
  for off, S, C, T, ys, ysS in written:
    mask.as_strided((S, C, T), (ysS, ys, 1), off).fill_(True)
  return bool((buf.view(torch.int32)[~mask] == SENTINEL).all())


def _zero_state(gpu, plan, S):
  return gpu.torch.zeros(max(1, plan.state_doubles(S)), dtype=gpu.torch.float64, device=gpu.dev)


def _signal(name, S, T):
  return np.random.default_rng([list(BANKS).index(name), S, T]).uniform(-1, 1, (S, T)).astype(np.float32)


_DENSE = collections.OrderedDict()


def _dense(gpu, plan, key, x):
  """The plan's dense ``alz_apply_f32`` output [S][C][T] (int32 bits, device) and final state, from a zero state."""
  S, T = x.shape
  k = (key, S, T)
  if k not in _DENSE:
    torch = gpu.torch
    X = _X(gpu, x)
    y = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device=gpu.dev)
    st = _zero_state(gpu, plan, S)
    plan.apply(X.ptr, y.data_ptr(), st.data_ptr(), S, T, X.xs, T, gpu.stream())
    torch.cuda.synchronize()
    _DENSE[k] = (y.view(torch.int32), st)
    while len(_DENSE) > 8:
      _DENSE.popitem(last=False)
  return _DENSE[k]


_ORACLE = {}


def _oracle_rows(name, x, rows):
  k = (name, x.shape)
  if k not in _ORACLE:
    _ORACLE.clear()
    _ORACLE[k] = oracle.bank_apply(x[rows], BANKS[name].sections())
  return _ORACLE[k]


def _check_oracle(plan, name, got, want, what):
  """Rows ``got`` [R][C][T] (float32) against ``want`` (float64) at the per-tier bars."""
  tol = km._row_tol(plan, types.SimpleNamespace(id=name))
  ceiling, _ = CEILING.get(name, (0.0, None))
  bar = np.maximum(tol, ceiling)
  err = km._row_err(got, want)
  err[np.max(np.abs(want), axis=-1) < F32_RANGE] = 0.0       # subnormal float32 rows (a lone first sample of a tiny gain)
  worst = np.unravel_index(np.argmax(err / tol[None, :]), err.shape)
  print("%s: worst row error %.3g (stream row %d, channel %d, per-tier bar %.3g, ceiling %.3g)" % (
    what, err[worst], worst[0], worst[1], tol[worst[1]], ceiling))
  assert not (err > bar[None, :]).any(), "%s: %d rows over the bar" % (what, int((err > bar[None, :]).sum()))


def _split(T):
  """Two blocks, the first of odd length (None when T is too short)."""
  return [T // 2 | 1, T - (T // 2 | 1)] if T >= 3 else None


# --------------------------------------------------------------------------------------------------------------------
# the layout grid
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=_case_id)
def test_output_layout(gpu, case):
  name, S, T, lay, eng = case
  torch = gpu.torch
  plan = _plan(gpu, name)
  C = plan.n_channels
  ys, ysS = _layouts(S, C, T)[lay]
  x = _signal(name, S, T)
  dense, dense_st = _dense(gpu, plan, name, x)
  off = 1 if eng == "offset" else 0
  X = _X(gpu, x, off)
  n = off + (S - 1) * ysS + (C - 1) * ys + T + 4
  rows = sorted({r for r in ORACLE_ROWS + (S - 1,) if r < S})
  want = _oracle_rows(name, x, rows)
  cur = gpu.stream()

  def run(ranges, blocks):
    """One plan per channel range writes its rows at base + lo * ys; checks the memory outside the rows written so far
    after each range.  -> (buffer, final states)."""
    buf = _filled(gpu, n)
    written, states = [], []
    for lo, hi in ranges:
      p = plan if (lo, hi) == (0, C) else _plan(gpu, name, lo, hi)
      st = _zero_state(gpu, p, S)
      t0 = 0
      for nb in blocks:
        p.apply_ex(X.ptr + 4 * t0, buf.data_ptr() + 4 * (off + lo * ys + t0), st.data_ptr(), S, nb, X.xs, ys, ysS, cur)
        t0 += nb
      torch.cuda.synchronize()
      written.append((off + lo * ys, S, hi - lo, T, ys, ysS))
      assert _untouched(buf, written), "%s: a write outside the rows of channels [%d, %d)" % (lay, lo, hi)
      states.append(st)
    return buf, states

  with km._env(ALZ_NO_TMA=1 if eng == "notma" else 0):
    ranges = _ranges(C) if lay.startswith("slices") else [(0, C)]
    buf, states = run(ranges, [T])
    for (lo, hi), st in zip(ranges, states):
      p = plan if (lo, hi) == (0, C) else _plan(gpu, name, lo, hi)
      got = _view(buf, off + lo * ys, S, hi - lo, T, ys, ysS)
      sub_dense, sub_st = (dense, dense_st) if p is plan else _dense(gpu, p, (name, lo, hi), x)
      assert torch.equal(got, sub_dense), "%s: channels [%d, %d) differ from the plan's dense output" % (lay, lo, hi)
      assert torch.equal(st, sub_st), "%s: channels [%d, %d): final state differs from the dense call's" % (lay, lo, hi)
      if p is not plan and _routing(p) == _routing(plan) and \
          np.array_equal(p.tiers()[0], plan.tiers()[0][lo:hi]):
        assert torch.equal(got, dense[:, lo:hi]), "%s: channels [%d, %d) differ from the full bank's" % (lay, lo, hi)
      _check_oracle(p, name, got[rows].view(torch.float32).cpu().numpy(), want[:, lo:hi],
                    "%s channels [%d, %d)" % (_case_id(case), lo, hi))
    if (lay == "cm" or lay.startswith("slices")) and _split(T):
      buf2, _ = run(ranges, _split(T))
      assert torch.equal(buf2.view(torch.int32), buf.view(torch.int32)), "two blocks differ from one call"
    if lay == "cm":                                            # the public API: FilterBank.apply(channel_major=True)
      pub = _filled(gpu, off + C * S * T + 4)
      out = pub[off:off + C * S * T].view(C, S, T)
      BANKS[name].apply(X.rows, out=out, channel_major=True)
      torch.cuda.synchronize()
      assert torch.equal(out.view(torch.int32).permute(1, 0, 2), dense), "FilterBank.apply(channel_major=True) differs"
      assert _untouched(pub, [(off, S, C, T, S * T, T)])


# --------------------------------------------------------------------------------------------------------------------
# launch paths at full scale
# --------------------------------------------------------------------------------------------------------------------
def _memsets(gpu, fn):
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    fn()
    gpu.torch.cuda.synchronize()
  return sum(1 for e in prof.events() if e.name and "memset" in e.name.lower())


@pytest.mark.parametrize("T", [4096, 4097])
def test_channel_major_full_scale(gpu, T):
  """The slaney bank, channel-major, 2048 streams: at T = 4096 the TMA engine segments the launch in time (it clears
  its segment flags with a memset); at T = 4097 the stream stride is odd, so the cp.async engine stores the rows with
  its lean path and scalar stores.  Both give the stream-major bits, with and without ALZ_NO_SEGMENT=1."""
  torch = gpu.torch
  plan = _plan(gpu, "slaney")
  S, C = 2048, plan.n_channels
  g = torch.Generator(device=gpu.dev)
  g.manual_seed(T)
  x = torch.rand((S, T), device=gpu.dev, generator=g) * 2 - 1
  sm = torch.empty((S, C, T), dtype=torch.float32, device=gpu.dev)
  plan.apply(x.data_ptr(), sm.data_ptr(), _zero_state(gpu, plan, S).data_ptr(), S, T, T, T, gpu.stream())
  outs, memsets = [], []
  for no_segment in (0, 1):
    cm = torch.empty((C, S, T), dtype=torch.float32, device=gpu.dev)
    st = _zero_state(gpu, plan, S)
    torch.cuda.synchronize()
    with km._env(ALZ_NO_SEGMENT=no_segment):
      memsets.append(_memsets(gpu, lambda: plan.apply_ex(x.data_ptr(), cm.data_ptr(), st.data_ptr(), S, T, T, S * T, T,
                                                        gpu.stream())))
    outs.append(cm)
  assert (memsets[0] > memsets[1]) == (T == 4096), "memsets with / without segmentation: %s" % memsets
  for cm in outs:
    assert torch.equal(cm.view(torch.int32).permute(1, 0, 2), sm.view(torch.int32))


# --------------------------------------------------------------------------------------------------------------------
# few long streams on the _ex entry
# --------------------------------------------------------------------------------------------------------------------
def test_ex_few_long_streams(gpu):
  """One stream of 200 077 samples: with the dense stream stride alz_apply_f32_ex is alz_apply_f32, time-parallel
  evaluation included (>= 4 launches); channel-major it is evaluated sequentially (< 4 launches) and gives the bits of
  a sequential plan."""
  torch = gpu.torch
  plan, seq = _plan(gpu, "slaney"), _plan(gpu, "slaney", sequential=True)
  assert plan.time_parallel
  S, T, C = 1, 200077, plan.n_channels
  X = _X(gpu, _signal("slaney", S, T))
  cur = gpu.stream()

  def launched(fn):
    y = torch.empty((C, T), dtype=torch.float32, device=gpu.dev)
    before = gpu.capi.launch_count()
    fn(y.data_ptr())
    torch.cuda.synchronize()
    return y.view(torch.int32), gpu.capi.launch_count() - before

  ref, n_ref = launched(lambda y: plan.apply(X.ptr, y, _zero_state(gpu, plan, S).data_ptr(), S, T, X.xs, T, cur))
  dense, n_dense = launched(lambda y: plan.apply_ex(X.ptr, y, _zero_state(gpu, plan, S).data_ptr(), S, T, X.xs, T,
                                                    C * T, cur))
  cm, n_cm = launched(lambda y: plan.apply_ex(X.ptr, y, _zero_state(gpu, plan, S).data_ptr(), S, T, X.xs, T, T, cur))
  sref, _ = launched(lambda y: seq.apply(X.ptr, y, _zero_state(gpu, seq, S).data_ptr(), S, T, X.xs, T, cur))
  assert n_ref >= 4 and n_dense >= 4, (n_ref, n_dense)
  assert torch.equal(dense, ref)
  assert n_cm < 4, n_cm
  assert torch.equal(cm, sref)


# --------------------------------------------------------------------------------------------------------------------
# more than 65535 x 32 streams: the stream-split loop
# --------------------------------------------------------------------------------------------------------------------
BIG_S = 65535 * 32 + 37
BIG_BLOCKS = (4, 37)                      # a block that leaves a per-stream state, then one tile plus a ragged tail
BIG_T = sum(BIG_BLOCKS)
BIG_XS = _round4(BIG_T)
BIG_ROWS = sorted(set([0, 31, 65535 * 32 - 1, 65535 * 32, 65535 * 32 + 1, BIG_S - 1] +
                      np.random.default_rng(65535).choice(BIG_S, 64, replace=False).tolist()))
TV_SECTIONS = [_section([0, 1, 3], [1, 2])]


def _big_plan(gpu, which):
  Plan = gpu.capi.Plan
  if which == "biquad":                  # the slaney bank's two widest channels: they ring up within the 41 samples
    return Plan(BANKS["slaney"].sections()[-2:])
  if which == "window":
    p = Plan(BY_ID["comb-fb-d15"].bank[:2])
    assert kernel(p) == "window"
    return p
  return Plan([TV_SECTIONS], force_generic=True)


@pytest.mark.parametrize("which,layout", [("biquad", "dense"), ("biquad", "cm"), ("window", "dense"),
                                          ("window", "cm"), ("tv", "dense")])
def test_more_streams_than_one_launch(gpu, which, layout):
  """BIG_S streams, two blocks (4 then 37 samples) with the state carried: the launches split at 65535 x 32 streams.
  Rows at both sides of the split, the last row and 64 random ones meet the oracle, and they and their final states
  are the bits of the same two calls over just those rows."""
  torch = gpu.torch
  plan = _big_plan(gpu, which)
  S, C = BIG_S, plan.n_channels
  g = torch.Generator(device=gpu.dev)
  g.manual_seed(17)
  x = torch.zeros((S, BIG_XS), dtype=torch.float32, device=gpu.dev)
  x[:, :BIG_T] = torch.rand((S, BIG_T), device=gpu.dev, generator=g) * 2 - 1
  table = coef = None
  if which == "tv":
    table = make_table(plan.taps(), BIG_T, BIG_T, 23)
    coef = torch.from_numpy(table).to(gpu.dev)
  cur = gpu.stream()

  def run(xd, n_streams, lay):
    """-> (y [n_streams][C][BIG_T] float32 view, final state [slot][C][n_streams])."""
    if lay == "dense":
      ys, ysS = BIG_XS, C * BIG_XS
      y = torch.full((n_streams, C, BIG_XS), float("nan"), dtype=torch.float32, device=gpu.dev)
    else:
      ys, ysS = n_streams * BIG_T, BIG_T
      y = torch.full((C, n_streams, BIG_T), float("nan"), dtype=torch.float32, device=gpu.dev)
    st = _zero_state(gpu, plan, n_streams)
    t0 = 0
    for n in BIG_BLOCKS:
      args = (xd.data_ptr() + 4 * t0, y.data_ptr() + 4 * t0, st.data_ptr(), n_streams, n, BIG_XS, ys)
      if which == "tv":
        plan.apply_tv(*args, coef.data_ptr() + 8 * t0, BIG_T, cur)
      else:
        plan.apply_ex(*args, ysS, cur)
      t0 += n
    torch.cuda.synchronize()
    slots = st.numel() // (C * n_streams)
    assert slots * C * n_streams == st.numel()
    yv = y.as_strided((n_streams, C, BIG_T), (ysS, ys, 1))
    return yv, st.view(slots, C, n_streams)

  idx = torch.tensor(BIG_ROWS, device=gpu.dev)
  y, st = run(x, S, layout)
  got = y.index_select(0, idx).contiguous()
  got_st = st.index_select(2, idx).contiguous()
  del y, st
  xr = x.index_select(0, idx).contiguous()
  small, small_st = run(xr, len(BIG_ROWS), "dense")
  assert torch.equal(got.view(torch.int32), small.contiguous().view(torch.int32)), "rows differ from a small launch"
  assert torch.equal(got_st, small_st), "final states differ from a small launch"
  xh = xr[:, :BIG_T].cpu().numpy()
  yh = got.cpu().numpy()
  if which == "tv":
    want = oracle.tv_apply(xh, split_sections(plan.taps()), table)[:, None, :]
    tol = np.full(1, km.WINDOW)
  else:
    bank = BANKS["slaney"].sections()[-2:] if which == "biquad" else BY_ID["comb-fb-d15"].bank[:2]
    want = oracle.bank_apply(xh, bank)
    tol = km._row_tol(plan, types.SimpleNamespace(id=which))
  err = km._row_err(yh, want)
  print("%s %s: worst row error %.3g" % (which, layout, err.max()))
  assert (err <= tol[None, :]).all(), err.max()


def test_entries_that_refuse_more_streams(gpu):
  """alz_apply_envelope_f32_ex and alz_apply_sum_f32 make one launch: they refuse BIG_S streams with
  ALZ_ERR_UNSUPPORTED before any work, and leave their output untouched."""
  torch, capi = gpu.torch, gpu.capi
  L = capi.lib()
  S, T, cur = BIG_S, 8, gpu.stream()
  x = torch.zeros((S, 8), dtype=torch.float32, device=gpu.dev)
  env_plan = _plan(gpu, "slaney")
  env = _filled(gpu, S * env_plan.n_channels)
  # states are refused before they are read: null ones turn a missing size check into ALZ_ERR_INVALID, not a launch
  rc = L.alz_apply_envelope_f32_ex(env_plan._h, x.data_ptr(), env.data_ptr(), None, None, S, T, 8, 1, 8, 0, 0, 0.02,
                                   0.98, cur)
  assert rc == capi.ALZ_ERR_UNSUPPORTED, rc
  psum = capi.Plan(BY_ID["psum-resonators-C8-bw1"].bank, parallel=True)
  out = _filled(gpu, S * 8)
  st = _zero_state(gpu, psum, S)
  rc = L.alz_apply_sum_f32(psum._h, x.data_ptr(), out.data_ptr(), st.data_ptr(), S, T, 8, 8, cur)
  assert rc == capi.ALZ_ERR_UNSUPPORTED, rc
  torch.cuda.synchronize()
  assert _untouched(env, []) and _untouched(out, [])


# --------------------------------------------------------------------------------------------------------------------
# host staging with several chunks (sequential plans: the bits do not depend on how time is cut)
# --------------------------------------------------------------------------------------------------------------------
def _device_run(gpu, plan, x, st):
  torch = gpu.torch
  S, T = x.shape
  X = _X(gpu, x)
  y = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device=gpu.dev)
  plan.apply(X.ptr, y.data_ptr(), st.data_ptr(), S, T, X.xs, T, gpu.stream())
  torch.cuda.synchronize()
  return y.cpu().numpy()


@pytest.mark.parametrize("carried", [False, True])
def test_host_staging_chunks(gpu, carried):
  """alz_apply_f32_host, 100 streams x 16384 samples: 128 MiB of output per chunk makes chunks of 32, 32, 32 and 4
  streams, through host rows of stride T + 3 (x) and T + 5 (y).  From a zero state, or from a device state a previous
  block left; the output and that state are the device path's bits, and the host padding keeps its NaN."""
  torch = gpu.torch
  plan = _plan(gpu, "slaney", sequential=True)
  S, T, C = 100, 16384, plan.n_channels
  assert (128 << 20) // (C * T * 4) == 32
  x = _signal("slaney", S, T)
  xh = np.zeros((S, T + 3), dtype=np.float32)
  xh[:, :T] = x
  yh = np.full((S * C, T + 5), SENTINEL, dtype=np.int32).view(np.float32)
  st_host = _zero_state(gpu, plan, S)
  st_dev = _zero_state(gpu, plan, S)
  if carried:
    _device_run(gpu, plan, _signal("slaney", S, 1001), st_dev)
    st_host.copy_(st_dev)
    torch.cuda.synchronize()
  rc = gpu.capi.lib().alz_apply_f32_host(plan._h, xh.ctypes.data, yh.ctypes.data, st_host.data_ptr() if carried else None,
                                         S, T, T + 3, T + 5)
  assert rc == gpu.capi.ALZ_OK, rc
  want = _device_run(gpu, plan, x, st_dev)
  assert np.array_equal(yh[:, :T].reshape(S, C, T).view(np.int32), want.view(np.int32))
  assert (yh[:, T:].view(np.int32) == SENTINEL).all(), "the host row padding was written"
  if carried:
    assert torch.equal(st_host, st_dev)


def test_host_staging_time_segments(gpu):
  """Three streams of 600 000 samples: each is cut into two time segments of its own chunk (state carried on the
  device between them); the result is the device path's bits."""
  plan = _plan(gpu, "slaney", sequential=True)
  S, T = 3, 600000
  assert plan.n_channels * T * 4 > (128 << 20)
  x = _signal("slaney", S, T)
  got = plan.apply_host(x)
  want = _device_run(gpu, plan, x, _zero_state(gpu, plan, S))
  assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_host_envelope_chunks(gpu):
  """alz_apply_envelope_f32_host_ex, 1100 streams x 16384 samples: chunks of 1024 and 76 streams, decimation 48 at
  phase 5, bank and lowpass states carried from a previous block; values and states are the bits of
  alz_apply_envelope_f32_ex on the device."""
  torch = gpu.torch
  plan = _plan(gpu, "slaney", sequential=True)
  S, T, C, decim, g, R = 1100, 16384, plan.n_channels, 48, 0.02, 0.98
  assert max(32, (64 << 20) // (T * 4) // 32 * 32) == 1024
  st = _zero_state(gpu, plan, S)
  es = torch.zeros(S * C, dtype=torch.float64, device=gpu.dev)
  prev = _X(gpu, _signal("slaney", S, 101))
  env_prev = torch.empty((S, C, 101 // decim), dtype=torch.float32, device=gpu.dev)
  plan.apply_envelope_ex(prev.ptr, env_prev.data_ptr(), st.data_ptr(), es.data_ptr(), S, 101, prev.xs, 101 // decim,
                         decim, 0, "abs", g, R, gpu.stream())
  phase = 101 % decim
  assert phase == 5
  st2, es2 = st.clone(), es.clone()
  torch.cuda.synchronize()
  x = _signal("slaney", S, T)
  got = plan.apply_envelope_host_ex(x, state_ptr=st.data_ptr(), env_state_ptr=es.data_ptr(), decim=decim, phase=phase,
                                    mode="abs", g=g, R=R)
  Td = (phase + T) // decim
  X = _X(gpu, x)
  env = torch.empty((S, C, Td), dtype=torch.float32, device=gpu.dev)
  plan.apply_envelope_ex(X.ptr, env.data_ptr(), st2.data_ptr(), es2.data_ptr(), S, T, X.xs, Td, decim, phase, "abs", g,
                         R, gpu.stream())
  torch.cuda.synchronize()
  assert np.array_equal(got.view(np.int32), env.cpu().numpy().view(np.int32))
  assert torch.equal(st, st2) and torch.equal(es, es2)


# --------------------------------------------------------------------------------------------------------------------
# argument checks of alz_apply_f32_ex
# --------------------------------------------------------------------------------------------------------------------
def test_ex_argument_checks(gpu):
  """A stream stride shorter than a row and overlapping stream-major rows are refused; S = 0 or T = 0 is a no-op.
  None of them writes or launches anything."""
  plan = _plan(gpu, "slaney")
  S, T, C = 4, 64, plan.n_channels
  X = _X(gpu, _signal("slaney", S, T))
  buf = _filled(gpu, S * C * T + 4)
  st = _zero_state(gpu, plan, S)
  cur = gpu.stream()
  before = gpu.capi.launch_count()
  with pytest.raises(ValueError):
    plan.apply_ex(X.ptr, buf.data_ptr(), st.data_ptr(), S, T, X.xs, S * T, T - 1, cur)       # ysS < T
  with pytest.raises(ValueError):
    plan.apply_ex(X.ptr, buf.data_ptr(), st.data_ptr(), S, T, X.xs, T, C * T - 1, cur)       # rows overlap
  plan.apply_ex(X.ptr, buf.data_ptr(), st.data_ptr(), 0, T, X.xs, T, C * T, cur)
  plan.apply_ex(X.ptr, buf.data_ptr(), st.data_ptr(), S, 0, X.xs, T, C * T, cur)
  gpu.torch.cuda.synchronize()
  assert gpu.capi.launch_count() == before
  assert _untouched(buf, [])
