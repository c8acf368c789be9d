"""The designs the public builders produce (``tests/design_space.py``) on the GPU: every row of every case over its whole
length against the float64 oracle at the kernel matrix's per-tier tolerances, plus the invariants the plan logic
promises for them; and the isolation of streams and of earlier samples from NaN, inf and extreme samples."""
import os
import types

import numpy as np
import pytest

import oracle
import test_kernel_matrix as km
from conftest import rel_err, signal
from design_space import BY_ID, CASES
from test_envelope_stream_gpu import _unfused

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1
TP_SEQ, TP_ORACLE = 3e-6, 1e-5           # time-parallel: against the sequential plan / the oracle (test_kernel_matrix)
#: powers of two: the oracle's output scales exactly, so a scaled row failing points at a range problem (the float32
#: input-side gain, flushed subnormals)
SCALES = (2.0 ** -30, 2.0 ** 30)


@pytest.fixture(scope="module")
def gpu():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return km.Gpu()


def _noise(case, S=None, T=None):
  S, T = S or case.S, T or case.T
  return np.stack([signal(1000 * CASES.index(case) + s, T) for s in range(S)])


def _reference_seeds(b, a, memory, zero):
  """The reference's seeding of one section (lazy_filters.py:181-195, restated as oracle.py_section does): trailing
  zero taps dropped; the output history is the first la - 1 items of ``memory``, padded with ``zero`` on the left; the
  input history is ``zero``.  -> (input history, output history), delay 1 first."""
  b, a = list(b), list(a)
  while len(b) > 1 and b[-1] == 0:
    b.pop()
  while len(a) > 1 and a[-1] == 0:
    a.pop()
  m = list(memory)[:len(a) - 1]
  return [zero] * (len(b) - 1), [zero] * (len(a) - 1 - len(m)) + m


def _seeds(case, plan):
  """memory= / zero= seeds: the oracle's histories [C][KM][h] from the reference's rule, the plan's
  [C][n_sections][depth] from the package's (what FilterBank.new_state(memory=, zero=) hands to the plan)."""
  if case.seed is None:
    return None, None, None, None
  from audiolazy_b200.filters import _seed_histories
  memory, zero = case.seed
  C, KM = len(case.bank), max(len(ch) for ch in case.bank)
  out = []
  for side, depth in ((0, plan.xd), (1, plan.yd)):
    ref = [[_reference_seeds(b, a, memory, zero)[side] for b, a in ch] for ch in case.bank]
    pkg = [_seed_histories(ch, memory, zero)[side] for ch in case.bank]
    o = np.zeros((C, KM, max([1] + [len(v) for ch in ref for v in ch])))
    g = np.zeros((C, plan.n_sections, depth))
    for c, ch in enumerate(case.bank):
      for k, (b, a) in enumerate(ch):
        v, w = ref[c][k], pkg[c][k]
        o[c, k, :len(v)] = v
        g[c, k, :min(len(w), depth)] = w[:depth]
        coef = b if side == 0 else a
        assert not any(coef[depth + 1:]), "a seeded history tap the plan does not keep has a nonzero coefficient"
    out += [o, g]
  xo, xg, yo, yg = out
  return xo, yo, xg, yg


def _oracle(x, bank, xo=None, yo=None):
  return oracle.bank_apply(x, bank, xinit=xo, yinit=yo, threads=THREADS)


def _launched(gpu, fn):
  before = gpu.capi.launch_count()
  out = fn()
  return out, gpu.capi.launch_count() - before


def _worst(y, ref):
  return float(np.max(km._row_err(y, ref))) if np.size(y) else 0.0


#: rows whose peak lies below this cannot keep 2^-24 of it in float32 (subnormal outputs): not compared
F32_RANGE = 2.0 ** -102


_SAMPLED = ("gammatone.sampled's head FIR cancels to ~(w)^3 of its input on the low channels: float64 evaluations in "
            "another order than the reference's differ by up to 1.2e-5 of the row peak at 44.1 to 192 kHz")
_SHORT = ("rows shorter than a narrow channel's ring-up: the float32 rounding of x * G is relative to the input, and the "
          "first 33 outputs peak far below it (up to 2.1e-5 of that peak)")
#: the cases measured over their per-tier bar although every bit-level invariant holds (DESIGN.md section 3): id ->
#: (the ceiling every oracle bar of the case is held to instead, why).  Each is an xfail that still fails above it.
KNOWN_MISS = dict(
  [(cid, (1.5e-5, _SAMPLED)) for cid in ("gammatone-sampled-r44100-n64", "gammatone-sampled-r96000-n13",
                                         "gammatone-sampled-r96000-n64", "gammatone-sampled-r192000-n13",
                                         "gammatone-sampled-r192000-n64", "long-gammatone-sampled-r192000-n64")] +
  [(cid, (2.5e-5, _SHORT)) for cid in
   ["gammatone-slaney-r%d-n100" % r for r in (8000, 16000, 44100, 96000, 192000)] +
   ["gammatone-klapuri-r%d-n13" % r for r in (8000, 22050, 44100, 96000, 192000)] +
   ["gammatone-klapuri-r%d-n100" % r for r in (16000, 22050, 44100, 96000, 192000)] +
   ["sos-butter-N8", "wide-resonator-C200"]])


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_design_vs_oracle(gpu, case):
  """Every row, full length, against the oracle: the sequential plan at the per-tier bars, the time-parallel result
  (when the plan takes that path) within 3e-6 of it and 1e-5 of the oracle; block splits of a sequential plan, the
  TMA / cp.async / unaligned engines and the float64 tier against an exact plan give the same bits; an impulse and the
  noise scaled by 2^-30 and 2^30 meet the same bars."""
  Plan = gpu.capi.Plan
  plan = Plan(case.bank, **case.plan_kw)
  seq = Plan(case.bank, sequential=True, **case.plan_kw)
  tol = km._row_tol(plan, types.SimpleNamespace(id=case.id))
  x = _noise(case)
  xo, yo, xg, yg = _seeds(case, plan)
  y, n_fast = _launched(gpu, lambda: gpu.run(plan, x, xg, yg))
  ys, n_seq = _launched(gpu, lambda: gpu.run(seq, x, xg, yg))
  tp = n_fast > n_seq
  if case.id.startswith("long-"):
    assert tp == plan.time_parallel, "the time-parallel path engaged: %s; the plan admits it: %s" % (tp, plan.time_parallel)
  if not tp:
    assert np.array_equal(y, ys), "a plan that does not go time-parallel differs from a sequential one"
  if case.splits:
    assert np.array_equal(gpu.run(seq, x, xg, yg, splits=case.splits), ys), "block splits are not bit-exact"
  assert np.array_equal(gpu.run(plan, x, xg, yg, engine="cpasync"), y), "cp.async engine differs from TMA"
  assert np.array_equal(gpu.run(plan, x, xg, yg, engine="unaligned"), y), "unaligned rows differ from TMA"
  if plan.kind == km.KIND_BIQUAD and plan.n_fp32_channels:
    tier = plan.tiers()[0]
    exact = gpu.run(Plan(case.bank, exact=True, **case.plan_kw), x, xg, yg)
    assert np.array_equal(exact[:, tier == 0], y[:, tier == 0]), "a float64-tier channel depends on the tiering"
  imp = np.zeros((1, case.T), dtype=np.float32)
  imp[0, 0] = 1.0
  yi, n_i = _launched(gpu, lambda: gpu.run(plan, imp))
  yis, n_is = _launched(gpu, lambda: gpu.run(seq, imp))
  if n_i == n_is:
    assert np.array_equal(yi, yis)
  ref = _oracle(x, case.bank, xo, yo)
  errs = {"seq": _worst(ys, ref)}
  if tp:
    errs["tp_vs_seq"], errs["tp"] = _worst(y, ys), _worst(y, ref)
  print("design %s [%s] S=%d T=%d tp=%d: %s" % (case.id, case.family, case.S, case.T, tp,
                                                 " ".join("%s %.3g" % kv for kv in sorted(errs.items()))))

  ceiling, reason = KNOWN_MISS.get(case.id, (0.0, None))
  bar = np.maximum(tol, ceiling)
  missed = []

  def check(got, want, rows, what):
    """Rows ``rows`` of got [S][C][T] within ``bar`` of want; notes a row over the per-tier bar ``tol``."""
    err = km._row_err(got, want)
    over = err[rows] > np.broadcast_to(bar, err.shape)[rows]
    assert not over.any(), "%s %s: %d rows over %s, worst %.3g" % (case.id, what, over.sum(),
                                                                   "its ceiling" if reason else "tolerance", err.max())
    missed.append(bool((err[rows] > np.broadcast_to(tol, err.shape)[rows]).any()))

  every = np.ones(ys.shape[:2], dtype=bool)
  check(ys, ref, every, "sequential")
  if tp:
    assert errs["tp_vs_seq"] <= TP_SEQ and errs["tp"] <= TP_ORACLE, errs
  if case.seed is None:
    for s in SCALES:
      ysc, want = gpu.run(plan, x * np.float32(s)), ref * s
      rows = np.max(np.abs(want), axis=-1) >= F32_RANGE
      if tp:
        assert _worst(ysc[rows], want[rows]) <= TP_ORACLE, s
      else:
        check(ysc, want, rows, "x %g" % s)
  refi = _oracle(imp, case.bank)
  check(yis, refi, np.ones(yis.shape[:2], dtype=bool), "impulse")
  if n_i > n_is:
    assert _worst(yi, refi) <= TP_ORACLE
  if reason and any(missed):
    pytest.xfail(reason)


PSUM_CASES = [c for c in CASES if c.family == "psum"]


@pytest.mark.parametrize("case", PSUM_CASES, ids=lambda c: c.id)
def test_parallel_sum_vs_oracle(gpu, case):
  """ParallelFilter of resonators through apply_sum against the oracle's left-to-right float64 sum of the channels;
  a carried state over blocks of 0, 4, 32, ... samples gives the same bits."""
  torch = gpu.torch
  plan = gpu.capi.Plan(case.bank, parallel=True)
  x = _noise(case)
  S, T = x.shape
  ch = _oracle(x, case.bank)
  want = ch[:, 0].copy()
  for c in range(1, len(case.bank)):
    want = want + ch[:, c]
  Tp = (T + 3) // 4 * 4                                     # the fused kernel moves 16-byte aligned rows
  xd = torch.zeros((S, Tp), dtype=torch.float32, device=gpu.dev)
  xd[:, :T] = torch.from_numpy(x).to(gpu.dev)

  def run(blocks):
    out = torch.full((S, Tp), float("nan"), dtype=torch.float32, device=gpu.dev)
    st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device=gpu.dev)
    t0 = 0
    for n in blocks:
      if n:
        plan.apply_sum(xd.data_ptr() + 4 * t0, out.data_ptr() + 4 * t0, st.data_ptr(), S, n, Tp, Tp, gpu.stream())
      t0 += n
    torch.cuda.synchronize()
    return out[:, :T].cpu().numpy()

  out = run([T])
  err = rel_err(out, want)
  print("psum %s: %.3g" % (case.id, err))
  assert err <= km.TIER0_GAIN_IN
  # the fused kernel takes 16-byte aligned block starts: lengths that are multiples of 4, and 0
  assert np.array_equal(run([0, 4, 32, 0, T - 36] if T > 36 else [0, T]), out)


ENVELOPE_CASES = [c for c in CASES if c.family == "gammatone" and c.meta["rate"] in (8000, 192000)
                  and len(c.bank) >= 64 and not c.id.startswith("long-")]


@pytest.mark.parametrize("case", ENVELOPE_CASES, ids=lambda c: c.id)
def test_envelope_vs_unfused(gpu, case):
  """FilterBank.envelope of the 8 kHz and 192 kHz banks against the bank output rectified and lowpassed in float64 on
  the host; a carried EnvelopeState over two blocks gives the bits of one call.  At 192 kHz also one long stream,
  which the time-parallel envelope evaluates."""
  import audiolazy_b200 as ab
  torch = gpu.torch
  bank = ab.gammatone_bank(case.meta["freqs"], case.meta["rate"], case.meta["strategy"])
  g, R = bank._envelope_pole(np.pi / 512)
  mode = ("abs", "squared", "rms")[ENVELOPE_CASES.index(case) % 3]
  shapes = [(37, 4800)] + ([(1, 200077)] if case.meta["rate"] == 192000 else [])
  for S, T in shapes:
    decim = 48
    x = _noise(case, S, T)
    xd = torch.from_numpy(x).to(gpu.dev)
    st = bank.new_envelope_state(S, decim=decim, mode=mode)
    parts = [bank.envelope(xd[:, :1001], decim=decim, mode=mode, state=st),
             bank.envelope(xd[:, 1001:], decim=decim, mode=mode, state=st)]
    env = torch.cat(parts, dim=2).cpu().numpy()
    if T % decim == 0:
      assert np.array_equal(bank.envelope(xd, decim=decim, mode=mode).cpu().numpy(), env)
    y = bank.apply(xd).cpu().numpy()
    want, _ = _unfused(y, g, R, np.zeros((S, len(bank))), decim, 0, mode)
    err = rel_err(env.reshape(-1, env.shape[-1]), want.reshape(-1, want.shape[-1]))
    print("envelope %s %s S=%d T=%d: %.3g" % (case.id, mode, S, T, err))
    assert err <= (1e-7 if S > 1 else TP_ORACLE)


# --------------------------------------------------------------------------------------------------------------------
# isolation from non-finite and extreme samples
# --------------------------------------------------------------------------------------------------------------------
BAD = [float("nan"), float("inf"), -float("inf"), 3e38, -3e38]


def _slaney():
  import audiolazy_b200 as ab
  return ab.gammatone_bank(strategy="slaney").sections()


class _Path(object):
  """One launch path: ``run(x)`` maps a device batch x[S, T] (rows padded to 16 bytes) to the output, whose first
  axis is the stream and last axis is time at ``rate`` outputs per input sample (1, or 1 / decim)."""

  def __init__(self, gpu, name):
    torch, Plan = gpu.torch, gpu.capi.Plan
    self.gpu, self.decim = gpu, 1
    if name == "plain":
      self.S, self.T, self.plan, self.kind = 37, 4096, Plan(_slaney()), "apply"
    elif name == "segmented":                       # cfg 4: 8192 warps = 2.3 waves, the launch is time-segmented
      self.S, self.T, self.plan, self.kind = 4096, 16384, Plan(_slaney()), "apply"
    elif name.startswith("timepar"):
      self.S, self.T, self.plan, self.kind = int(name[-1]), 200077, Plan(_slaney()), "apply"
    elif name == "window":
      self.S, self.T, self.plan, self.kind = 37, 4096, Plan(BY_ID["comb-fb-d100"].bank), "apply"
    elif name == "generic":
      self.S, self.T, self.plan, self.kind = 37, 4096, Plan(BY_ID["cascade-comb48-biquad"].bank), "apply"
    elif name == "psum":
      self.S, self.T, self.plan, self.kind = 37, 4096, Plan(BY_ID["psum-resonators-C8-bw1"].bank, parallel=True), "sum"
    elif name == "envelope":
      import audiolazy_b200 as ab
      self.S, self.T, self.kind, self.decim = 3, 200077, "envelope", 48
      self.bank = ab.gammatone_bank(strategy="slaney")
    self.Tp = (self.T + 3) // 4 * 4

  def run(self, xd):
    torch, gpu = self.gpu.torch, self.gpu
    S, T, Tp = self.S, self.T, self.Tp
    if self.kind == "envelope":                     # a carried state: a 5-sample block, then the rest (time-parallel)
      st = self.bank.new_envelope_state(S, decim=self.decim)
      parts = [self.bank.envelope(xd[:, :5], decim=self.decim, state=st),
               self.bank.envelope(xd[:, 5:T], decim=self.decim, state=st)]
      return torch.cat(parts, dim=2)
    plan = self.plan
    st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device=gpu.dev)
    if self.kind == "sum":
      out = torch.empty((S, Tp), dtype=torch.float32, device=gpu.dev)
      plan.apply_sum(xd.data_ptr(), out.data_ptr(), st.data_ptr(), S, T, Tp, Tp, gpu.stream())
      return out[:, :T]
    out = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device=gpu.dev)
    plan.apply(xd.data_ptr(), out.data_ptr(), st.data_ptr(), S, T, Tp, T, gpu.stream())
    return out


@pytest.mark.parametrize("path", ["plain", "segmented", "timepar-S1", "timepar-S3", "window", "generic", "psum",
                                  "envelope"])
def test_nonfinite_samples_stay_in_their_stream(gpu, path):
  """NaN, +-inf and +-3e38 at one sample of one stream: every other stream's output, and the affected stream's
  outputs before that sample, are the bits of the same batch without it.  What the affected stream shows after the
  sample is not asserted (the reference turns most IIR states into NaN)."""
  torch = gpu.torch
  p = _Path(gpu, path)
  S, T = p.S, p.T
  g = torch.Generator(device=gpu.dev)
  g.manual_seed(5)
  xd = torch.zeros((S, p.Tp), dtype=torch.float32, device=gpu.dev)
  xd[:, :T] = torch.rand((S, T), device=gpu.dev, generator=g) * 2 - 1
  s0, t0 = S // 2, T // 2 + 3
  clean, launches = _launched(gpu, lambda: p.run(xd))
  torch.cuda.synchronize()
  assert bool(torch.isfinite(clean).all())
  # the path is the one the test is named for: the time-parallel passes launch zero-state, scan and replay kernels
  # (the envelope two scans); a segmented launch clears its segment flags, which the unsegmented one does not
  if path.startswith("timepar") or path == "envelope":
    assert launches >= 4, "%s: %d launches, not time-parallel" % (path, launches)
  else:
    assert launches < 4, "%s: %d launches, time-parallel passes" % (path, launches)
  if path in ("plain", "segmented"):
    from torch.profiler import ProfilerActivity, profile
    memsets = []
    for no_segment in (0, 1):
      with km._env(ALZ_NO_SEGMENT=no_segment), profile(activities=[ProfilerActivity.CUDA]) as prof:
        p.run(xd)
        torch.cuda.synchronize()
      memsets.append(sum(1 for e in prof.events() if e.name and "memset" in e.name.lower()))
    assert (memsets[0] > memsets[1]) == (path == "segmented"), "%s: memsets %s" % (path, memsets)
  keep = t0 // p.decim                               # outputs computed from samples before t0 only
  for v in BAD:
    xb = xd.clone()
    xb[s0, t0] = v
    dirty = p.run(xb)
    torch.cuda.synchronize()
    assert torch.equal(dirty[:s0], clean[:s0]) and torch.equal(dirty[s0 + 1:], clean[s0 + 1:]), \
      "%s: a sample %r in stream %d changed another stream" % (path, v, s0)
    assert torch.equal(dirty[s0, ..., :keep], clean[s0, ..., :keep]), "%s: a sample %r changed earlier outputs" % (path, v)
    del dirty, xb
