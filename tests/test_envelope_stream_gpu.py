"""The streamed filterbank envelope on the GPU: blocks of any length with a carried ``EnvelopeState``, the decimation
phase, the time-parallel evaluation of few long streams, and ``FilterBank.envelope_streams`` against the reference."""
import os

import numpy as np
import pytest
from scipy.signal import lfilter

import audiolazy_b200 as ab
from conftest import GOLDEN, rel_err, signal
from native_libs import torch  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

STRATEGIES = ["slaney", "klapuri", "sampled"]
MODES = ["abs", "squared", "rms"]


_BANKS = {}


def _bank(name):
  if name not in _BANKS:
    _BANKS[name] = ab.gammatone_bank(strategy=name)
  return _BANKS[name]


def _split(T, decim):
  """Block lengths 0, 1, decim - 1, lengths that are not multiples of 4 (so later blocks start at unaligned offsets),
  then the rest."""
  lengths = [0, 1, decim - 1, 5, 0, 301, 2, 1027]
  return lengths + [T - sum(lengths)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", STRATEGIES)
def test_any_block_split_is_bit_exact(torch, name, mode):
  """S = 37 streams (the time-parallel path does not engage): successive envelope(..., state=) calls on blocks of any
  length give exactly the values of one call over the whole input, of the stateless call, and of envelope_host with a
  state of its own."""
  bank = _bank(name)
  S, T = 37, 48 * 100
  x = np.random.default_rng(7).uniform(-1, 1, (S, T)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()
  for decim in (1, 7, 48):
    whole = bank.envelope(xd, decim=decim, mode=mode, state=bank.new_envelope_state(S, decim=decim, mode=mode))
    if T % decim == 0:
      assert torch.equal(whole, bank.envelope(xd, decim=decim, mode=mode))     # the stateless (phase 0) call
    st = bank.new_envelope_state(S, decim=decim, mode=mode)
    sh = bank.new_envelope_state(S, decim=decim, mode=mode)
    dev, host, t0 = [], [], 0
    for n in _split(T, decim):
      dev.append(bank.envelope(xd[:, t0:t0 + n], decim=decim, mode=mode, state=st))
      host.append(bank.envelope_host(x[:, t0:t0 + n], decim=decim, mode=mode, state=sh))
      t0 += n
    got = torch.cat(dev, dim=2)
    assert got.shape == (S, 64, T // decim)
    assert torch.equal(got, whole), "block split differs (decim %d)" % decim
    assert np.array_equal(np.concatenate(host, axis=2), whole.cpu().numpy()), "host entry differs (decim %d)" % decim
    assert st.phase == sh.phase == T % decim
    assert torch.equal(st.env_tensor, sh.env_tensor) and torch.equal(st.bank_state.tensor, sh.bank_state.tensor)


def test_ex_entry_with_phase_zero_is_the_old_entry(torch):
  """alz_apply_envelope_f32_ex with phase 0 and whole decimation windows is alz_apply_envelope_f32, bit for bit."""
  for name in STRATEGIES:
    plan = _bank(name).device_bank().plan
    S, T, decim = 37, 48 * 40, 48
    x = torch.from_numpy(np.random.default_rng(8).uniform(-1, 1, (S, T)).astype(np.float32)).cuda()
    outs = []
    for entry in (plan.apply_envelope, plan.apply_envelope_ex):
      env = torch.full((S, 64, T // decim), float("nan"), dtype=torch.float32, device="cuda")
      st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device="cuda")
      es = torch.zeros(S * 64, dtype=torch.float64, device="cuda")
      args = (x.data_ptr(), env.data_ptr(), st.data_ptr(), es.data_ptr(), S, T, T, T // decim, decim)
      if entry == plan.apply_envelope_ex:
        args += (0,)
      entry(*args, "rms", 0.01, 0.99, torch.cuda.current_stream().cuda_stream)
      torch.cuda.synchronize()
      outs.append((env.cpu(), st.cpu(), es.cpu()))
    for a, b in zip(*outs):
      assert torch.equal(a, b), name


def _unfused(y, g, R, e0, decim, phase, mode):
  """float64 lowpass e = g r + R e of the float32 bank output y [S][C][T] from state e0 [S][C], kept on the caller's
  decimation grid -> (values [S][C][n_out], final state)."""
  r = np.abs(y.astype(np.float64)) if mode == "abs" else y.astype(np.float64) ** 2
  e, zf = lfilter([g], [1.0, -R], r, axis=-1, zi=(R * e0)[..., None])
  kept = e[:, :, decim - 1 - phase::decim]
  return (np.sqrt(kept) if mode == "rms" else kept), zf[..., 0] / R


def _row_err(got, want):
  """max |got - want| / max |want| per output row, the worst row."""
  return rel_err(got.reshape(-1, got.shape[-1]), want.reshape(-1, want.shape[-1]))


def _scans(torch, fn):
  """fn() and the number of chunk-scan launches it made (the time-parallel envelope scans the bank states and then the
  lowpass states: two; a sequential call: none)."""
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    out = fn()
    torch.cuda.synchronize()
  return out, sum(1 for e in prof.events() if e.name and "alz_chunk_scan_kernel" in e.name)


@pytest.mark.parametrize("S", [1, 3])
def test_time_parallel_envelope(torch, S):
  """Few long streams: T = 10^6 + 37 samples after a 5-sample block (nonzero phase, a tail that is not a multiple of
  decim) against a plan created with ALZ_PLAN_SEQUENTIAL and against the unfused pipeline; then a state carried out of
  the time-parallel call into a short sequential call against one call over both parts."""
  from audiolazy_b200 import _capi
  bank = _bank("slaney")
  db = bank.device_bank()
  seq = _capi.Plan(bank.sections(), sequential=True)
  decim, mode, T = 48, "abs", 10 ** 6 + 37
  g, R = bank._envelope_pole(np.pi / 512)
  rng = np.random.default_rng(9)
  x = rng.uniform(-1, 1, (S, 5 + T + 1000)).astype(np.float32)
  xd = torch.from_numpy(x).cuda()
  st = bank.new_envelope_state(S, decim=decim, mode=mode)
  head = bank.envelope(xd[:, :5], decim=decim, mode=mode, state=st)
  assert head.shape[2] == 0 and st.phase == 5
  e_before = st.env_tensor.clone()
  s_before = st.bank_state.tensor.clone()
  fast, scans = _scans(torch, lambda: bank.envelope(xd[:, 5:5 + T], decim=decim, mode=mode, state=st))
  assert scans >= 2, "the time-parallel path did not engage"
  n_out = (5 + T) // decim
  assert fast.shape == (S, 64, n_out) and st.phase == (5 + T) % decim
  # the same block through the sequential plan, from the same states
  xs = torch.zeros((S, (T + 3) // 4 * 4), dtype=torch.float32, device="cuda")
  xs[:, :T] = xd[:, 5:5 + T]
  slow = torch.empty((S, 64, n_out), dtype=torch.float32, device="cuda")
  sst, ses = s_before.clone(), e_before.clone()
  _, scans = _scans(torch, lambda: seq.apply_envelope_ex(xs.data_ptr(), slow.data_ptr(), sst.data_ptr(), ses.data_ptr(), S, T,
                                                            xs.stride(0), n_out, decim, 5, mode, g, R,
                                                            torch.cuda.current_stream().cuda_stream))
  assert scans == 0
  fast_np, slow_np = fast.cpu().numpy(), slow.cpu().numpy()
  err_seq = _row_err(fast_np, slow_np)
  # the unfused pipeline: the bank (its own state carried over the 5-sample head), then the float64 lowpass on the host
  e0 = e_before.cpu().numpy().reshape(64, S).T
  want, e_final = [], []
  for s in range(S):                               # one stream at a time: the float64 host copies stay near 1 GB
    y = bank.apply(xd[s:s + 1, :5 + T]).cpu().numpy()[:, :, 5:]
    w, ef = _unfused(y, g, R, e0[s:s + 1], decim, 5, mode)
    want.append(w[0])
    e_final.append(ef[0])
  want, e_final = np.stack(want), np.stack(e_final)
  err_ref = _row_err(fast_np, want)
  print("time-parallel envelope, S=%d: max row error %.3g vs sequential plan, %.3g vs unfused pipeline" % (S, err_seq, err_ref))
  assert err_seq <= 1e-5 and err_ref <= 1e-5
  assert rel_err(st.env_tensor.cpu().numpy().reshape(64, S).T, e_final) <= 1e-5
  # carry the state into a short (sequential) call: one call over both parts from the 5-sample state
  tail = bank.envelope(xd[:, 5 + T:], decim=decim, mode=mode, state=st)
  st2 = bank.new_envelope_state(S, decim=decim, mode=mode)
  bank.envelope(xd[:, :5], decim=decim, mode=mode, state=st2)
  both = bank.envelope(xd[:, 5:], decim=decim, mode=mode, state=st2).cpu().numpy()
  assert rel_err(np.concatenate([fast_np, tail.cpu().numpy()], axis=2).reshape(-1, both.shape[2]),
                 both.reshape(-1, both.shape[2])) <= 1e-5


def test_envelope_streams_vs_reference(torch):
  """envelope_streams with decim 1 on a generator input against the reference's own envelope.abs / .rms / .squared of six
  slaney channels, the lowest included (tests/golden/envelope_streams.npz, made by make_envelope_streams.py from a
  reference checkout; every 40th value of 12000); with decim 48 the Streams equal one batch
  envelope call bit for bit; an endless input yields values lazily."""
  bank = _bank("slaney")
  ref = np.load(os.path.join(GOLDEN, "envelope_streams.npz"))
  chans = [int(c) for c in ref["channels"]]
  assert 0 in chans
  x = signal(77, 12000)
  for mode in MODES:
    streams = bank.envelope_streams((float(v) for v in x), decim=1, mode=mode)
    got = np.array([list(streams[c]) for c in chans])
    assert got.shape == (6, 12000)
    assert rel_err(got[:, ref["index"]], ref[mode]) <= 1e-5, mode
  streams = bank.envelope_streams((float(v) for v in x), decim=48, mode="rms")
  got = np.array([list(s) for s in streams], dtype=np.float32)
  batch = bank.envelope(torch.from_numpy(x).cuda()[None], decim=48, mode="rms").cpu().numpy()[0]
  assert np.array_equal(got, batch)
  first = bank.envelope_streams(ab.white_noise(), decim=48)[0].take(8)
  assert len(first) == 8 and all(v >= 0 for v in first)


@pytest.mark.parametrize("variant", ["nb2", "headfir-nb3"])
def test_time_parallel_envelope_kernel_variants(torch, variant):
  """The envelope kernel's time-parallel passes on the 2-tap and head-FIR instantiations (designs of the kernel matrix:
  poles at radius 0.99 ... 0.995, a lowpass pole of 0.999, so that both chunk scans carry visible state): one stream,
  a 5-sample block, then T - 5 samples from phase 5, against a plan created with ALZ_PLAN_SEQUENTIAL at the matrix's
  per-tier tolerances."""
  import types
  import test_kernel_matrix as km
  from audiolazy_b200 import _capi
  nb, hf, mode = (2, False, "abs") if variant == "nb2" else (3, True, "rms")
  bank = km.biquad_bank(850 + nb, 64, 4, nb, 2, counts="full", head_fir=8 if hf else 0, radius=(0.99, 0.995))
  S, T, C, decim, g, R = 1, 100077, 64, 48, 0.001, 0.999
  x = np.random.default_rng([51, nb]).uniform(-1, 1, (S, T)).astype(np.float32)
  outs = []
  for sequential in (False, True):
    plan = _capi.Plan(bank, sequential=sequential)
    st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device="cuda")
    es = torch.zeros(S * C, dtype=torch.float64, device="cuda")
    rows = []
    for t0, n in ((0, 5), (5, T - 5)):
      xb = torch.zeros((S, (n + 3) // 4 * 4), dtype=torch.float32, device="cuda")      # 16-byte aligned rows
      xb[:, :n] = torch.from_numpy(x[:, t0:t0 + n]).cuda()
      n_out = (t0 % decim + n) // decim
      env = torch.full((S, C, max(n_out, 1)), float("nan"), dtype=torch.float32, device="cuda")
      _, scans = _scans(torch, lambda: plan.apply_envelope_ex(xb.data_ptr(), env.data_ptr(), st.data_ptr(), es.data_ptr(), S, n,
                                                              xb.stride(0), env.shape[2], decim, t0 % decim, mode, g, R,
                                                              torch.cuda.current_stream().cuda_stream))
      if n > 5:
        assert (scans >= 2) != sequential, "time-parallel path engaged: %s" % (scans >= 2)
      rows.append(env.cpu().numpy()[:, :, :n_out])
    outs.append(np.concatenate(rows, axis=2))
  assert outs[0].shape == (S, C, T // decim)
  case = types.SimpleNamespace(id="envelope-timepar-" + variant)
  km._check_rows(outs[0], outs[1].astype(np.float64), km._row_tol(plan, case), case.id)
