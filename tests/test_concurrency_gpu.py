"""Every library under concurrent use: one plan (or bank object) driven from several CUDA streams and host threads at
once.  Each case first runs its calls alone on the default stream; every concurrent result, and every state it carries
out, must equal that serial result bit for bit (the plans fix tiers, segments, engines, P and L from the shape, so a
call is deterministic).  A few rows of each serial result are checked against the float64 oracles as well, so that a
result that is wrong in the same way twice is still caught.

Races are provoked by construction, never by repetition: a low-priority stream holds a long bank launch (the
"blocker") while a high-priority stream's work overtakes it, and the time-parallel chunk-transition cache (8 entries per
plan) is churned with more than 8 chunk lengths so that an entry another stream still uses is evicted."""
import gc
import math
import threading
import types

import numpy as np
import pytest
from scipy.signal import lfilter

import audiolazy_b200 as ab
import lpc_emulation as em
import oracle
import test_kernel_matrix as km
import test_time_varying_gpu as tvm
from amdf_emulation import amdf_bank as amdf_emulate
from audiolazy_b200 import _capi, _engine, analysis, crossing, linear_prediction
from conftest import rel_err
from native_libs import torch  # noqa: F401  (fixture)
from zcross_emulation import block_sums, zcross as zcross_emulate

pytestmark = pytest.mark.gpu

ROUNDS = 3


# ---------------------------------------------------------------------------------------------------------------------
# helpers
# ---------------------------------------------------------------------------------------------------------------------
def torch_mod():
  import torch
  return torch


def _bits(t):
  torch = torch_mod()
  if t.is_complex():
    t = torch.view_as_real(t)
  return t.detach().contiguous().reshape(-1).view(torch.uint8)


def _same(got, want, what):
  """Every tensor of the dict ``want`` (a serial result) equals the one of ``got`` bit for bit (NaNs included)."""
  torch = torch_mod()
  assert got.keys() == want.keys(), what
  for k in want:
    assert got[k].shape == want[k].shape, (what, k)
    assert torch.equal(_bits(got[k]), _bits(want[k])), "%s: %s differs from the serial run" % (what, k)


def _kernels(fn, *names):
  """fn() and, for each name, the number of kernel launches whose name contains it (CUDA events of every stream)."""
  torch = torch_mod()
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    out = fn()
    torch.cuda.synchronize()
  return out, [sum(1 for e in prof.events() if e.name and n in e.name) for n in names]


def _run_threads(fns):
  """Runs every fn in a thread of its own, all released at once; re-raises the first failure."""
  barrier = threading.Barrier(len(fns))
  errors = [None] * len(fns)
  results = [None] * len(fns)

  def body(i):
    try:
      barrier.wait()
      results[i] = fns[i]()
    except BaseException as exc:  # noqa: BLE001  (re-raised below, in the test's thread)
      errors[i] = exc
  threads = [threading.Thread(target=body, args=(i,)) for i in range(len(fns))]
  for t in threads:
    t.start()
  for t in threads:
    t.join()
  for e in errors:
    if e is not None:
      raise e
  return results


def _on(stream, fn):
  """fn() with ``stream`` as torch's current stream of this thread (None: the stream already current)."""
  torch = torch_mod()
  if stream is None:
    return fn()
  with torch.cuda.stream(stream):
    return fn()


def _in_stream_thread(stream, fn):
  """A thread body: fn() on ``stream``, synchronised before it returns."""
  def body():
    out = _on(stream, fn)
    stream.synchronize()
    return out
  return body


def chunk_geometry(plan, S, T, passes=2, sm_count=132):
  """``(P, L)`` the time-parallel evaluation of ``alz_capi.cu`` picks for S streams of T samples (its cost model,
  term for term), or None when the call is evaluated sequentially."""
  C, d = plan.n_channels, plan.state_doubles_per_recurrence
  if not plan.time_parallel or T < 16384 or d > 32 or S > 65535:
    return None
  slots = sm_count * 24
  if C * ((S + 31) // 32) * 2 > slots:
    return None
  work = max(1, plan.fp64_ops) / 12.0
  t_seq = T * 36e-9 * work
  P, best = 0, 1e30
  for q in range(32, 1025, 32):
    if q * 256 > T:
      break
    waves = float(C) * S * q / 32.0 / slots
    occ = min(waves, 1.0)
    Lq = T // q // 32 * 32
    tail = T - q * Lq
    t_sample = max(36e-9, 92e-9 * occ) * work
    t_state = 6.0 * d * 8.0 * C * float(S) * float(q) / 4e12
    t = passes * math.ceil(waves) * (Lq * t_sample + 1e-5) + t_state + tail * 36e-9 * work + q * 1e-7
    if t < best:
      best, P = t, q
  if P == 0 or 1.25 * best + 5e-5 > 0.8 * t_seq:
    return None
  L = T // P // 32 * 32
  return None if L < 256 else (P, L)


def chunk_lengths(plan, S, T, sm_count):
  """Every chunk length a call of S x T samples uses (the tail left over by one time-parallel pass is decided again)."""
  out = []
  while True:
    g = chunk_geometry(plan, S, T, sm_count=sm_count)
    if g is None:
      return out
    out.append(g[1])
    T -= g[0] * g[1]


def pick_lengths(plan, n, exclude, start, sm_count):
  """``n`` single-stream block lengths T >= start, each of whose calls uses exactly one chunk length, all different and
  not in ``exclude``; returns ``[(T, L)]``."""
  out, seen = [], set(exclude)
  T = start
  while len(out) < n:
    ls = chunk_lengths(plan, 1, T, sm_count)
    if len(ls) == 1 and ls[0] not in seen:
      seen.add(ls[0])
      out.append((T, ls[0]))
    T += 997
  return out


def _apply(plan, x, y, st):
  """``alz_apply_f32`` of rows x [S][T] into y [S][C][T] with state st, on torch's current stream."""
  torch = torch_mod()
  S, T = x.shape
  plan.apply(x.data_ptr(), y.data_ptr(), st.data_ptr(), S, T, x.stride(0), T, torch.cuda.current_stream().cuda_stream)


# ---------------------------------------------------------------------------------------------------------------------
# the jobs: one call each, on torch's current stream, with outputs and states of its own
# ---------------------------------------------------------------------------------------------------------------------
class Job(object):
  """``run()`` -> dict of result tensors (outputs and carried states); ``check(result)`` compares a few rows of a
  serial result with the float64 oracle."""

  def __init__(self, name, run, check=None):
    self.name, self.run, self.check = name, run, check


def _bank_job(name, bank, x, channel_rows=(0, 1)):
  def run():
    st = bank.new_state(x.shape[0])
    y = bank.apply(x, state=st)
    return {"y": y, "state": st.tensor}

  def check(res):
    rows = list(channel_rows)
    xh = x[rows].cpu().numpy()
    plan = bank.device_bank().plan
    km._check_rows(res["y"][rows].cpu().numpy(), oracle.bank_apply(xh, bank.sections()),
                   km._row_tol(plan, types.SimpleNamespace(id=name)), name)
  return Job(name, run, check)


def _plan_job(name, plan, bank, x, tol=None):
  """A raw plan through alz_apply_f32."""
  torch = torch_mod()
  S, T = x.shape

  def run():
    y = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device="cuda")
    st = torch.zeros(max(1, plan.state_doubles(S)), dtype=torch.float64, device="cuda")
    _apply(plan, x, y, st)
    return {"y": y, "state": st}

  def check(res):
    rows = [0, S - 1]
    want = oracle.bank_apply(x[rows].cpu().numpy(), bank)
    t = km._row_tol(plan, types.SimpleNamespace(id=name)) if tol is None else np.full(plan.n_channels, tol)
    km._check_rows(res["y"][rows].cpu().numpy(), want, t, name)
  return Job(name, run, check)


def _envelope_job(name, bank, x, decim, mode):
  def run():
    st = bank.new_envelope_state(x.shape[0], decim=decim, mode=mode)
    env = bank.envelope(x, decim=decim, mode=mode, state=st)
    return {"env": env, "bank_state": st.bank_state.tensor, "env_state": st.env_tensor}

  def check(res):
    g, R = bank._envelope_pole(np.pi / 512)
    y = bank.apply(x[:1]).cpu().numpy().astype(np.float64)
    r = np.abs(y) if mode == "abs" else y ** 2
    e = lfilter([g], [1.0, -R], r, axis=-1)[:, :, decim - 1::decim]
    want = np.sqrt(e) if mode == "rms" else e
    assert rel_err(res["env"][:1].cpu().numpy().reshape(-1, want.shape[-1]), want.reshape(-1, want.shape[-1])) <= 1e-5
  return Job(name, run, check)


def _tv_job(x):
  torch = torch_mod()
  sections = tvm.TAP_SETS["three-sections"]
  plan = _capi.Plan([sections], force_generic=True)
  S, T = x.shape
  table = tvm.make_table(plan.taps(), T, T, 5)
  tdev = torch.from_numpy(table).cuda()

  def run():
    y = torch.empty((S, T), dtype=torch.float32, device="cuda")
    st = torch.zeros(max(1, plan.state_doubles(S)), dtype=torch.float64, device="cuda")
    plan.apply_tv(x.data_ptr(), y.data_ptr(), st.data_ptr(), S, T, T, T, tdev.data_ptr(), T,
                  torch.cuda.current_stream().cuda_stream)
    return {"y": y, "state": st}

  def check(res):
    rows = [0, 31, 32, S - 1]
    ref = oracle.tv_apply(x[rows].cpu().numpy(), tvm.split_sections(plan.taps()), table)
    assert tvm.row_errors(res["y"][rows].cpu().numpy(), ref).max() <= tvm.TOL
  return Job("time-varying", run, check), plan


def _psum_job(x):
  torch = torch_mod()
  bank = km.biquad_bank(704, 3, 4, 3, 2)
  plan = _capi.Plan(bank, parallel=True)
  S, T = x.shape

  def run():
    out = torch.empty((S, T), dtype=torch.float32, device="cuda")
    st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device="cuda")
    plan.apply_sum(x.data_ptr(), out.data_ptr(), st.data_ptr(), S, T, T, T, torch.cuda.current_stream().cuda_stream)
    return {"out": out, "state": st}

  def check(res):
    ch = oracle.bank_apply(x[:2].cpu().numpy(), bank)
    want = ch[:, 0].copy()
    for c in range(1, len(bank)):
      want = want + ch[:, c]
    assert rel_err(res["out"][:2].cpu().numpy(), want) <= km.TIER0_GAIN_IN
  return Job("parallel-sum", run, check), plan


def _freq_job(bank):
  torch = torch_mod()
  db = bank.device_bank()
  w = torch.linspace(0, np.pi, 4099, dtype=torch.float64, device="cuda")

  def run():
    return {"h": db.freq_response(w)}

  def check(res):
    from scipy.signal import freqz
    h = res["h"].cpu().numpy()
    for c in (0, 31, 63):
      want = np.ones(w.numel(), dtype=complex)
      for b, a in bank.sections()[c]:
        want *= freqz(b, a, worN=w.cpu().numpy())[1]
      assert np.max(np.abs(h[c] - want)) <= 1e-9 * np.max(np.abs(want)), c
  return Job("freq-response", run, check)


def _amdf_job(name, bank, x, decim, zero, lag_rows):
  def run():
    st = bank.new_state(x.shape[0], decim=decim, zero=zero)
    out = bank.apply(x, decim=decim, state=st)
    return {"out": out, "state": st.tensor}

  def check(res):
    if bank.sequential:
      rows = [0, x.shape[0] - 1]
      want = amdf_emulate(x[rows].cpu().numpy(), [bank.taps[l] for l in lag_rows], bank.size, zero)
      want = want[:, :, decim - 1::decim].astype(np.float32)
      assert np.array_equal(res["out"][rows][:, lag_rows].cpu().numpy(), want)
    else:                                          # time-parallel: its float64 drift, <= 1e-5 of the row's peak
      xs = x[:1, :200000].cpu().numpy()
      want = amdf_emulate(xs, [bank.taps[l] for l in lag_rows], bank.size, zero)[:, :, decim - 1::decim]
      got = res["out"][:1, lag_rows, :want.shape[-1]].cpu().numpy()
      assert rel_err(got.reshape(-1, want.shape[-1]), want.reshape(-1, want.shape[-1])) <= 1e-5
  return Job(name, run, check)


def _zcross_job(name, x):
  zc = ab.Zcross(.01, 0)

  def run():
    st = zc.new_state(x.shape[0], size=2048, hop=1024)
    flags = zc.apply(x)
    counts = zc.counts(x, 2048, 1024, state=st)
    return {"flags": flags, "counts": counts, "state": st.tensor}

  def check(res):
    xh = x[:1].cpu().numpy()
    want = zcross_emulate(xh, .01)
    assert np.array_equal(res["flags"][:1].cpu().numpy(), want)
  return Job(name, run, check)


def _lpc_job(name, x):
  lp = ab.LpcFrames(16, 512, 256, np.hanning(512))

  def run():
    st = lp.new_state(x.shape[0])
    res = lp.apply(x, state=st, final=True)
    return {"coef": res[0], "error": res[1], "failed": res[2], "state": st.tensor}

  def check(res):
    xh = x[:1].cpu().numpy()[0]
    for k in (0, 7, res["coef"].shape[1] - 1):
      blk = em.frames(xh[k * lp.hop:k * lp.hop + lp.size], lp.size, lp.hop, lp.window, final=True)[0]
      _, wc, we, wf = em.kautocor(blk, lp.order)
      got = res["coef"][0, k].cpu().numpy()
      assert em.canon(got).tobytes() == em.canon(np.asarray(wc)).tobytes() and res["failed"][0, k].item() == wf, k
  return Job(name, run, check)


class World(object):
  """Inputs, objects and serial results shared by the cases."""

  def __init__(self, torch):
    self.torch = torch
    self.sm_count = torch.cuda.get_device_properties(0).multi_processor_count
    rng = np.random.default_rng(2024)

    def dev(*shape):
      return torch.from_numpy(rng.uniform(-1, 1, shape).astype(np.float32)).cuda()
    self.slaney = ab.gammatone_bank(strategy="slaney")
    self.x_seg = dev(2048, 4096)         # 64 x 64 warps: between 1 and 8 waves, cut into time segments
    self.x_tp = dev(2, 10 ** 6 + 37)     # few long streams: time-parallel
    self.x_env = dev(256, 48 * 200)
    self.x_env_tp = dev(1, 10 ** 6 + 37)
    rng_w = km._rng(21, 8, 1)            # near windows of 16 taps and far taps on both sides
    self.window_bank = [km.window_channel(rng_w, km.NEAR[16], km.NEAR_Y[16], [16, 49], [17, 48], 1.0 if c == 0 else 0.6)
                        for c in range(40)]
    self.window_plan = _capi.Plan(self.window_bank)
    assert self.window_plan.kind == _capi.KIND_GENERIC and self.window_plan.n_sections == 1
    self.generic_bank = km.CASES[[c.id for c in km.CASES].index("generic-fir10-biquad-order3-C5")].bank
    self.generic_plan = _capi.Plan(self.generic_bank)
    self.x_window = dev(256, 8192)
    self.x_tv = dev(100, 20000)
    self.x_psum = dev(512, 8192)
    self.amdf_seq = ab.AmdfBank([0, 0.4] + list(np.linspace(3.25, 800, 208)), 333, sequential=True)
    self.amdf_tp = ab.AmdfBank(list(np.linspace(48, 800, 256)), 1024)
    self.x_amdf = dev(64, 20000)
    self.x_amdf_tp = dev(1, 10 ** 6 + 37)
    self.x_zc = [dev(64, 300000), dev(1, 5 * 10 ** 6)]
    self.x_lpc = [dev(256, 20000), dev(1, 2 * 10 ** 6)]
    tv, self.tv_plan = _tv_job(self.x_tv)
    psum, self.psum_plan = _psum_job(self.x_psum)
    self.filter_jobs = [
      _bank_job("bank-segmented", self.slaney, self.x_seg),
      _bank_job("bank-time-parallel", self.slaney, self.x_tp, channel_rows=(0,)),
      _envelope_job("envelope", self.slaney, self.x_env, 48, "rms"),
      _envelope_job("envelope-time-parallel", self.slaney, self.x_env_tp, 48, "abs"),
      _plan_job("window-far-taps", self.window_plan, self.window_bank, self.x_window, tol=km.WINDOW),
      _plan_job("generic", self.generic_plan, self.generic_bank, self.x_window[:64, :3000], tol=km.WINDOW),
      tv, psum, _freq_job(self.slaney)]
    self.amdf_jobs = [_amdf_job("amdf-sequential", self.amdf_seq, self.x_amdf, 1, .25, [0, 1, 100, 209]),
                      _amdf_job("amdf-time-parallel", self.amdf_tp, self.x_amdf_tp, 7, .25, [0, 255])]
    self.other_jobs = [_zcross_job("zcross-many", self.x_zc[0]), _zcross_job("zcross-long", self.x_zc[1]),
                       _lpc_job("lpc-many", self.x_lpc[0]), _lpc_job("lpc-long", self.x_lpc[1])]
    self.jobs = {j.name: j for j in self.filter_jobs + self.amdf_jobs + self.other_jobs}
    torch.cuda.synchronize()
    self.serial = {}
    for name, job in self.jobs.items():
      if "time-parallel" in name and "amdf" not in name:
        res, (scans,) = _kernels(job.run, "alz_chunk_scan_kernel")
        assert scans >= 1, "%s: the time-parallel path did not engage" % name
      else:
        res = job.run()
      torch.cuda.synchronize()
      self.serial[name] = res
    assert self.amdf_seq.chunks(64, 20000) == 1 and self.amdf_tp.chunks(1, 10 ** 6 + 37) > 1

  def check_serial(self, name):
    self.jobs[name].check(self.serial[name])


@pytest.fixture(scope="module")
def world(torch):
  w = World(torch)
  yield w
  del w
  gc.collect()
  torch.cuda.synchronize()
  torch.cuda.empty_cache()


def test_serial_results_against_the_oracles(world):
  """The serial results every other case compares with are right: a few rows of each against the float64 oracles at
  the kernel matrix's per-tier tolerances (the AMDF and zero-crossing emulations and the LPC frames exactly)."""
  for name in world.jobs:
    world.check_serial(name)


# ---------------------------------------------------------------------------------------------------------------------
# (a) two CUDA streams, one plan, three rounds issued interleaved
# ---------------------------------------------------------------------------------------------------------------------
def test_two_streams_all_libraries_interleaved(world, torch):
  """Every job on a low-priority and a high-priority stream at once, issued job by job alternately, with all four
  libraries in flight together: three rounds, each stream's outputs and states equal the serial bits."""
  lo, hi = torch.cuda.Stream(), torch.cuda.Stream(priority=-1)
  names = list(world.jobs)
  for r in range(ROUNDS):
    torch.cuda.synchronize()
    got = {lo: {}, hi: {}}
    for name in names:
      for s in ((lo, hi) if r % 2 == 0 else (hi, lo)):
        got[s][name] = _on(s, world.jobs[name].run)
    torch.cuda.synchronize()
    for s, tag in ((lo, "low"), (hi, "high")):
      for name in names:
        _same(got[s][name], world.serial[name], "round %d, %s-priority stream, %s" % (r, tag, name))
    del got


# ---------------------------------------------------------------------------------------------------------------------
# (b) the chunk-transition cache under churn
# ---------------------------------------------------------------------------------------------------------------------
class Churn(object):
  """A slaney plan for the time-parallel calls, a twin plan (same bank) that computes their serial results, and a
  blocker: two full-machine bank launches on another plan, a few milliseconds of device time."""

  def __init__(self, world):
    torch = world.torch
    self.world = world
    self.sections = world.slaney.sections()
    self.twin = _capi.Plan(self.sections)
    self.serial = {}
    self.x = torch.from_numpy(np.random.default_rng(77).uniform(-1, 1, (1, 400000)).astype(np.float32)).cuda()
    kl = ab.gammatone_bank(strategy="klapuri")
    self.blocker_bank = kl.device_bank()
    self.xb = torch.from_numpy(np.random.default_rng(78).uniform(-1, 1, (2048, 8192)).astype(np.float32)).cuda()
    self.yb = torch.empty((2048, 64, 8192), dtype=torch.float32, device="cuda")
    self.sb = self.blocker_bank.new_state(2048)

  def block(self):
    for _ in range(2):
      self.blocker_bank.apply(self.xb, self.sb, out=self.yb)

  def call(self, plan, T):
    torch = self.world.torch
    x = self.x[:, :T]
    y = torch.empty((1, 64, T), dtype=torch.float32, device="cuda")
    st = torch.zeros(plan.state_doubles(1), dtype=torch.float64, device="cuda")
    _apply(plan, x, y, st)
    return {"y": y, "state": st}

  def serial_of(self, T):
    if T not in self.serial:
      self.serial[T] = self.call(self.twin, T)
      self.world.torch.cuda.synchronize()
    return self.serial[T]

  def lengths(self, n, exclude=(), start=20000):
    return pick_lengths(self.twin, n, exclude, start, self.world.sm_count)


@pytest.fixture(scope="module")
def churn(world):
  return Churn(world)


def test_cache_eviction_while_another_stream_still_uses_the_entry(world, churn, torch):
  """One cached chunk length L0; the low-priority stream queues the blocker and a call that hits L0; the high-priority
  stream then runs 8 calls with new chunk lengths, the last of which evicts L0 while the first call's scan is queued.
  Every output equals its serial bits; the profiler shows a chunk scan per call and a basis run per new length."""
  plan = _capi.Plan(churn.sections)
  (T0, L0), *new = churn.lengths(9)
  for T, _ in [(T0, L0)] + new:
    churn.serial_of(T)
  first = churn.call(plan, T0)                        # L0 is computed and cached
  torch.cuda.synchronize()
  _same(first, churn.serial_of(T0), "first L0 call")
  lo, hi = torch.cuda.Stream(), torch.cuda.Stream(priority=-1)

  def issue():
    with torch.cuda.stream(lo):
      churn.block()
      held = churn.call(plan, T0)
    outs = []
    with torch.cuda.stream(hi):
      for T, _ in new:
        outs.append((T, churn.call(plan, T)))
    return held, outs
  torch.cuda.synchronize()
  (held, outs), (scans, basis) = _kernels(issue, "alz_chunk_scan_kernel", "alz_unit_state_kernel")
  assert scans >= 1 + len(new) and basis == len(new), (scans, basis)
  _same(held, churn.serial_of(T0), "L0 call behind the blocker, its entry evicted")
  for T, out in outs:
    _same(out, churn.serial_of(T), "high-priority call, T=%d" % T)


def test_cache_churn_from_two_threads(world, churn, torch):
  """Two host threads, each with its own stream and its own 9 chunk lengths, on one plan (the cache holds 8): every
  output equals its serial bits."""
  plan = _capi.Plan(churn.sections)
  sets = churn.lengths(18, start=30011)
  mine = [sets[0::2], sets[1::2]]
  for T, _ in sets:
    churn.serial_of(T)
  streams = [torch.cuda.Stream(), torch.cuda.Stream(priority=-1)]

  def worker(i):
    def body():
      out = []
      for T, _ in mine[i]:
        out.append((T, churn.call(plan, T)))
      return out
    return _in_stream_thread(streams[i], body)
  torch.cuda.synchronize()
  for outs in _run_threads([worker(0), worker(1)]):
    for T, out in outs:
      _same(out, churn.serial_of(T), "thread call, T=%d" % T)


def test_cache_hit_waits_for_an_entry_still_being_computed(world, churn, torch):
  """A new chunk length L1 is computed for the first time on the low-priority stream, behind the blocker; a call on
  the high-priority stream hits L1 right away, before its transition matrix exists: it must wait for it."""
  plan = _capi.Plan(churn.sections)
  (T1, L1), = churn.lengths(1, start=50021)
  want = churn.serial_of(T1)
  lo, hi = torch.cuda.Stream(), torch.cuda.Stream(priority=-1)
  torch.cuda.synchronize()

  def issue():
    with torch.cuda.stream(lo):
      churn.block()
      first = churn.call(plan, T1)
    with torch.cuda.stream(hi):
      second = churn.call(plan, T1)
    return first, second
  (first, second), (basis, scans) = _kernels(issue, "alz_unit_state_kernel", "alz_chunk_scan_kernel")
  assert basis == 1 and scans >= 2, (basis, scans)
  _same(first, want, "L1 computed behind the blocker")
  _same(second, want, "L1 hit on the high-priority stream")


def test_two_threads_miss_the_same_length_at_once(world, churn, torch):
  """Two threads call with a chunk length the plan has not cached, at the same moment: both outputs are the serial
  bits."""
  plan = _capi.Plan(churn.sections)
  (T2, _), = churn.lengths(1, start=70001)
  want = churn.serial_of(T2)
  streams = [torch.cuda.Stream(), torch.cuda.Stream(priority=-1)]
  torch.cuda.synchronize()
  outs = _run_threads([_in_stream_thread(s, lambda: churn.call(plan, T2)) for s in streams])
  for out in outs:
    _same(out, want, "simultaneous miss")


# ---------------------------------------------------------------------------------------------------------------------
# (c) host threads on the same objects
# ---------------------------------------------------------------------------------------------------------------------
def test_four_threads_share_the_same_objects(world, torch):
  """Four threads, each on its own stream, call the same FilterBank (apply, envelope), AmdfBank, Zcross and LpcFrames
  objects at once; every result equals the serial one."""
  names = ["bank-segmented", "envelope", "amdf-sequential", "zcross-many", "lpc-many", "bank-time-parallel"]
  streams = [torch.cuda.Stream(priority=-1 if i % 2 else 0) for i in range(4)]

  def worker(i):
    def body():                                    # each result is compared (and dropped) in its thread
      for n in names[i:] + names[:i]:
        got = _on(streams[i], world.jobs[n].run)
        streams[i].synchronize()
        _same(got, world.serial[n], "thread %d, %s" % (i, n))
    return body
  torch.cuda.synchronize()
  _run_threads([worker(i) for i in range(4)])


def test_device_bank_is_one_object_per_key(world, torch):
  """Four threads ask for the DeviceBank of a bank nobody has used yet, at once: they all get the same object."""
  bank = ab.gammatone_bank(freqs=ab.erb_space(n=24), strategy="slaney")
  got = _run_threads([bank.device_bank] * 4)
  assert all(db is got[0] for db in got)
  assert bank.device_bank() is got[0]


def test_host_entries_from_two_threads(world, torch):
  """apply_host / envelope_host on one plan from two threads, then on two plans (equal banks, separate plans): each
  result equals the serial one."""
  bank = world.slaney
  x = world.x_env[:64].cpu().numpy()                 # 48 x 200 samples: whole decimation windows
  want_y = bank.apply_host(x)
  want_e = bank.envelope_host(x, decim=48, mode="rms")
  other_plan = _capi.Plan(bank.sections())
  assert other_plan is not bank.device_bank().plan
  g, R = bank._envelope_pole(np.pi / 512)

  def one_plan(i):
    return lambda: bank.apply_host(x) if i == 0 else bank.envelope_host(x, decim=48, mode="rms")

  got = _run_threads([one_plan(0), one_plan(1), one_plan(0), one_plan(1)])
  for i, v in enumerate(got):
    assert np.array_equal(v, want_y if i % 2 == 0 else want_e), i
  got = _run_threads([lambda: bank.device_bank().plan.apply_host(x), lambda: other_plan.apply_host(x),
                      lambda: other_plan.apply_envelope_host(x, decim=48, mode="rms", g=g, R=R)])
  assert np.array_equal(got[0], want_y) and np.array_equal(got[1], want_y) and np.array_equal(got[2], want_e)


# ---------------------------------------------------------------------------------------------------------------------
# (d) plans created while another thread launches
# ---------------------------------------------------------------------------------------------------------------------
def test_plan_creation_while_another_thread_launches(world, torch):
  """Thread A launches the segmented bank and the AMDF bank three times; meanwhile thread B creates an AmdfBank with a
  delay over 990 samples (more than 48 KB of shared memory: the kernel's shared-memory limit is raised) and a gammatone
  bank at 44.1 kHz (the tier probe runs on the host), and uses both at once.  A's results are unchanged, and B's new
  plans give the same bits on both threads and agree with the oracles."""
  names = ["bank-segmented", "amdf-sequential"]
  sa, sb = torch.cuda.Stream(), torch.cuda.Stream(priority=-1)
  x = world.x_amdf[:3, :5000]
  created = {}

  def a():
    for r in range(ROUNDS):
      for n in names:
        got = _on(sa, world.jobs[n].run)
        sa.synchronize()
        _same(got, world.serial[n], "round %d, %s" % (r, n))

  def b():
    long_bank = ab.AmdfBank([1500, 1200.5, 48], 64)
    bank = ab.gammatone_bank(rate=44100, strategy="slaney")
    created["amdf"], created["bank"] = long_bank, bank
    return {"amdf": long_bank.apply(x, state=long_bank.new_state(3, zero=.25)), "bank": bank.apply(x)}
  torch.cuda.synchronize()
  _, got_b = _run_threads([a, _in_stream_thread(sb, b)])
  long_bank, bank = created["amdf"], created["bank"]
  again = _on(sa, lambda: {"amdf": long_bank.apply(x, state=long_bank.new_state(3, zero=.25)), "bank": bank.apply(x)})
  torch.cuda.synchronize()
  _same(again, got_b, "B's plans on thread A")
  xh = x.cpu().numpy()
  want = amdf_emulate(xh, long_bank.taps, 64, .25).astype(np.float32)
  assert np.array_equal(got_b["amdf"].cpu().numpy(), want)
  km._check_rows(got_b["bank"][:2].cpu().numpy(), oracle.bank_apply(xh[:2], bank.sections()),
                 km._row_tol(bank.device_bank().plan, types.SimpleNamespace(id="44k")), "44.1 kHz bank")


# ---------------------------------------------------------------------------------------------------------------------
# (e) errors stay in their thread
# ---------------------------------------------------------------------------------------------------------------------
def test_errors_stay_in_their_thread(world, torch):
  """Two threads make different invalid calls through every library's binding, 200 times each, at once; each
  exception carries its own call's message (every library keeps its last error per thread)."""
  y = torch.empty((4, 64, 16), dtype=torch.float32, device="cuda")
  xs = torch.zeros((4, 16), dtype=torch.float32, device="cuda")
  st = torch.zeros(world.slaney.device_bank().plan.state_doubles(4), dtype=torch.float64, device="cuda")
  plan = world.slaney.device_bank().plan
  amdf = world.amdf_seq._plan()
  lp = ab.LpcFrames(4, 32, 16)
  lp_other = ab.LpcFrames(5, 32, 16)
  lp_state = lp_other.new_state(4)
  cur = torch.cuda.current_stream().cuda_stream
  nan = float("nan")
  calls = [
    [(lambda: _capi.Plan([[([1.0, nan], [1.0, -0.5])]]), "non-finite coefficient"),
     (lambda: amdf.apply(xs.data_ptr(), y.data_ptr(), st.data_ptr(), 4, 16, 16, 16, 0, 0, cur), "need decim >= 1"),
     (lambda: linear_prediction._check(linear_prediction.lib().alz_lpc_state_bytes(-1, 16)), "1 <= size"),
     (lambda: crossing._check(crossing.lib().alz_zcross_state_bytes(-1, 0, 1)), "size >= 0, hop >= 1"),
     (lambda: lp.apply(xs, state=lp_state), "another order")],
    [(lambda: plan.apply_ex(xs.data_ptr(), y.data_ptr(), st.data_ptr(), 4, 16, 16, 16, 16, cur), "output rows overlap"),
     (lambda: analysis._Plan([[(1, 1.0)]], 0), "size must be >= 1 (got 0)"),
     (lambda: linear_prediction._check(linear_prediction.lib().alz_lpc_frames(-1, 10, 4, 2, 0)), "need consumed >= 0"),
     (lambda: crossing._check(crossing.lib().alz_zcross_scratch_bytes(-1, 10, 0, 1)), "bad shape"),
     (lambda: _capi.Plan([[([1.0], [0.0, 1.0])]]), "Invalid filter gain")],
  ]

  def worker(i):
    def body():
      for _ in range(200):
        for fn, msg in calls[i]:
          try:
            fn()
          except Exception as exc:  # noqa: BLE001
            assert msg in str(exc), "thread %d expected %r, got %r" % (i, msg, str(exc))
          else:
            raise AssertionError("thread %d: %r did not raise" % (i, msg))
    return body
  _run_threads([worker(0), worker(1)])
  torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------------------
# (f) a green-context partition alongside the full device
# ---------------------------------------------------------------------------------------------------------------------
def test_partition_stream_alongside_the_full_device(world, torch):
  """The segmented bank and the time-parallel call on a stream confined to half of the SMs, AMDF on an ordinary stream,
  at once: every result equals the serial bits."""
  try:
    part = _capi.PartitionStream(world.sm_count // 2 // 8 * 8)
  except _capi.NativeError as exc:
    pytest.skip("no green contexts here: %s" % exc)
  try:
    ext = torch.cuda.ExternalStream(part.handle, device=torch.device("cuda", 0))
    other = torch.cuda.Stream(priority=-1)
    torch.cuda.synchronize()
    on_part = ["bank-segmented", "bank-time-parallel"]
    on_other = ["amdf-sequential", "amdf-time-parallel"]
    got = {}
    for a, b in zip(on_part, on_other):
      got[a] = _on(ext, world.jobs[a].run)
      got[b] = _on(other, world.jobs[b].run)
    ext.synchronize()
    other.synchronize()
    for n in on_part + on_other:
      _same(got[n], world.serial[n], n)
  finally:
    torch.cuda.synchronize()
    part.close()


# ---------------------------------------------------------------------------------------------------------------------
# (g) plans dropped while their launches are queued
# ---------------------------------------------------------------------------------------------------------------------
def test_plans_dropped_while_their_launches_are_queued(world, churn, torch):
  """A window plan, a generic plan and an AmdfBank are dropped (del, gc.collect()) right after their launches are
  queued behind the blocker on a side stream: destroying a plan waits for the device, so the outputs are the serial
  bits."""
  side = torch.cuda.Stream()
  x_amdf = world.x_amdf[:8, :4000]
  lags = [3, 48.5, 1200]
  ref_amdf = ab.AmdfBank(lags, 64)
  want_amdf = ref_amdf.apply(x_amdf, state=ref_amdf.new_state(8, zero=.25))
  want_w = world.serial["window-far-taps"]
  xg = world.x_window[:64, :3000]
  want_g = world.serial["generic"]
  torch.cuda.synchronize()
  with torch.cuda.stream(side):
    churn.block()
    wplan = _capi.Plan(world.window_bank)
    gplan = _capi.Plan(world.generic_bank)
    amdf = ab.AmdfBank(lags, 64)
    state = amdf.new_state(8, zero=.25)
    out = {}
    for name, plan, x in (("window", wplan, world.x_window), ("generic", gplan, xg)):
      S, T = x.shape
      y = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device="cuda")
      st = torch.zeros(max(1, plan.state_doubles(S)), dtype=torch.float64, device="cuda")
      _apply(plan, x, y, st)
      out[name] = {"y": y, "state": st}
    out["amdf"] = amdf.apply(x_amdf, state=state)
    del wplan, gplan, amdf, state, plan
    gc.collect()
  side.synchronize()
  _same(out["window"], want_w, "window plan dropped")
  _same(out["generic"], want_g, "generic plan dropped")
  _same({"out": out["amdf"]}, {"out": want_amdf}, "AmdfBank dropped")


# ---------------------------------------------------------------------------------------------------------------------
# (h) launches above the 48 KB shared-memory default, of different sizes, from two threads
# ---------------------------------------------------------------------------------------------------------------------
def _frames_job(lp, x):
  def run():
    st = lp.new_state(x.shape[0])
    res = lp.apply(x, state=st, final=True)
    return {"coef": res[0], "error": res[1], "failed": res[2], "state": st.tensor}
  return run


def _stft_job(stft, x):
  def run():
    st = stft.new_state(x.shape[0])
    spec = stft.analyze(x, st, final=True)
    y = stft.synthesize(spec, st, final=True)
    return {"spec": spec, "y": y, "state": st.tensor, "ola_state": st.ola.tensor}
  return run


def test_two_threads_launch_one_kernel_with_different_sizes_above_48_kb(torch):
  """Thread A runs LPC frames of 8192 samples (64 KiB of dynamic shared memory for a frame) and an STFT of size 8192
  (128 KiB); thread B LPC frames of 7000 samples (about 55 KiB), an STFT of size 4096 (64 KiB) and kcovar at order 64
  (68 KiB a warp in the recursion).  Each job makes launches above the 48 KB default, and the two threads launch the
  same kernels with different sizes at once: each launch must find the kernel's limit at least as high as its own
  size, whatever the other thread launched last.  Three calls of each job per thread, each result equal to the serial
  one."""
  rng = np.random.default_rng(31)

  def dev(*shape):
    return torch.from_numpy(rng.uniform(-1, 1, shape).astype(np.float32)).cuda()
  jobs = [
    {"lpc-8192": _frames_job(ab.LpcFrames(16, 8192, 4096, np.hanning(8192)), dev(4, 3 * 8192)),
     "stft-8192": _stft_job(ab.Stft(8192, 2048, wnd=ab.window.hann, dtype=torch.complex128), dev(4, 3 * 8192))},
    {"lpc-7000": _frames_job(ab.LpcFrames(12, 7000, 3000), dev(4, 3 * 7000)),
     "stft-4096": _stft_job(ab.Stft(4096, 1024, wnd=ab.window.hann, dtype=torch.complex128), dev(4, 3 * 4096)),
     "kcovar-64": _frames_job(ab.LpcFrames(64, 512, 256, method="kcovar"), dev(4, 8192))}]
  serial = {}
  for mine in jobs:
    for name, run in mine.items():
      serial[name] = run()
  torch.cuda.synchronize()
  streams = [torch.cuda.Stream(), torch.cuda.Stream(priority=-1)]

  def worker(i):
    def body():
      for r in range(ROUNDS):
        for name, run in jobs[i].items():
          got = _on(streams[i], run)
          streams[i].synchronize()
          _same(got, serial[name], "thread %d, round %d, %s" % (i, r, name))
    return body
  _run_threads([worker(0), worker(1)])
