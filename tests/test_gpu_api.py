"""The reference-facing Python API on a GPU: filters are callables that take an iterable and
return a Stream (reference lazy_filters.py:975-978); known answers are the reference's own
doctests / tests and the golden vectors."""
import itertools as it

import numpy as np
import pytest

import oracle
from conftest import rel_err, signal

pytestmark = pytest.mark.gpu
TOL = 1e-5


@pytest.fixture(scope="module")
def ab():
  import torch
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  import audiolazy_b200
  return audiolazy_b200


def test_reference_doctests(ab):
  z, ZFilter, Stream = ab.z, ab.ZFilter, ab.Stream
  filt = (1 + z ** -1) / (1 - z ** -1)                        # lazy_filters.py:722-726
  res = filt([1, 5, -4, -7, 9])
  assert isinstance(res, Stream)
  assert list(res) == [1.0, 7.0, 8.0, -3.0, -1.0]
  filt = ZFilter([1, 1], [1, -1])                             # :731-742
  result = list(filt([1, 5, -4, -7, 9], memory=[3], zero=0))
  assert result == [4, 10, 11, 0, 2]
  assert list((filt * z ** -1)(result, zero=0)) == [0, 4, 18, 39, 50]
  assert list((1 + z ** -1)([1.0, 2.0, 3.0])) == [1.0, 3.0, 5.0]      # :877-882
  casc = ab.CascadeFilter(z ** -1, 2 * (1 - z ** -3))                   # :982-985
  data = Stream(1, 3, 5, 3, 1, -1, -3, -5, -3, -1)                      # endless
  assert casc(data, zero=0).take(15) == [0, 2, 6, 10, 4, -4, -12, -12, -12, -4, 4, 12, 12, 12, 4]
  filt = 1 + z ** -1 - z ** -2                                          # :1040-1045
  pfilt = ab.ParallelFilter(1 + z ** -1, -z ** -2)
  assert list(filt(range(100))) == list(pfilt(range(100)))
  assert list(filt(range(10), zero=0)) == [0, 1, 3, 4, 5, 6, 7, 8, 9, 10]
  acc = 1 / (1 - z ** -1)                                               # __init__.py:27-30 (accumulator)
  assert acc(Stream(it.count())).take(6) == [0.0, 1.0, 3.0, 6.0, 10.0, 15.0]


def test_lfilter_grid(ab):
  """reference tests/test_filters_extdep.py:41-47 (ZFilter vs scipy.signal.lfilter)."""
  from scipy.signal import lfilter
  for a in [[1.], [3.], [1., 3.], [15., -17.2], [-18., 9.8, 0., 14.3]]:
    for b in [[1.], [-1.], [1., 0., -1.], [1., 3.]]:
      for data in [list(range(5)), list(range(5, 0, -1)), [7, 22, -5], [8., 3., 15.]]:
        got = list(ab.ZFilter(b, a)(data))
        want = lfilter(b, a, data).tolist()
        assert np.allclose(got, want, rtol=2e-6, atol=1e-30), (a, b, data, got, want)


def test_identity_gain_delay_empty_lists(ab):
  z, Stream = ab.z, ab.Stream                                    # reference tests/test_filters.py:47-114, :557-566
  data = [1.5, -2.0, 0.25, 8.0]
  assert list(ab.ZFilter(1)(data)) == data
  assert list((0.5 * z ** 0)(data)) == [v * 0.5 for v in data]
  assert list((z ** -2)(data)) == [0.0, 0.0, 1.5, -2.0]
  assert list((z ** -2)(data, zero=7.0)) == [7.0, 7.0, 1.5, -2.0]
  assert list(ab.CascadeFilter()(data)) == data
  assert list(ab.ParallelFilter()(data)) == [0.0] * 4
  assert list(ab.ParallelFilter()(data, zero=2.5)) == [2.5] * 4
  assert list(ab.ZFilter([1, 1])(Stream(data))) == [1.5, -0.5, -1.75, 8.25]
  one_pole = 1 / (1 - 0.5 * z ** -1)
  want, m = [], 0.0
  for v in data:
    m = v + 0.5 * m
    want.append(m)
  assert list(one_pole(data)) == want
  assert list(ab.CascadeFilter(2.0, z ** -1)(data)) == [0.0, 3.0, -4.0, 0.5]     # bare numbers are gains
  mixed = ab.CascadeFilter(z ** -1, lambda s: Stream(s) * 2)                      # non-linear member: generic path
  assert list(mixed(data)) == [0.0, 3.0, -4.0, 0.5]
  with pytest.raises(ValueError, match="Non-causal"):
    (z + 1)(data)


def test_configs_through_the_python_api(ab, designs, vectors):
  y = np.array(list(ab.ZFilter([1, 7, 2], [1, 0.5, 0.2])(signal(1, 48000).tolist())))      # cfg 1
  assert rel_err(y, vectors["cfg1_y"]) <= TOL
  casc = ab.CascadeFilter([ab.ZFilter(r[:3], r[3:]) for r in designs["cfg2_sos"]])          # cfg 2
  y = np.array(list(casc(ab.Stream(signal(2, 50000).tolist()))))
  assert rel_err(y, vectors["cfg2_y"]) <= TOL
  f = ab.ZFilter([0.5, -0.25, 2.0], [2.0, 0.5, -0.3])
  xs = signal(3, 64).tolist()
  assert rel_err(list(f(xs, memory=[0.75, -1.5], zero=0.125)), vectors["seed_single_y"]) <= TOL
  assert rel_err(list(f(xs, memory=[0.75], zero=-0.5)), vectors["seed_short_memory_y"]) <= TOL
  assert rel_err(list(f(xs, memory=lambda n: [0.75, -1.5, 9.0][:n], zero=0.125)), vectors["seed_single_y"]) <= TOL
  casc3 = ab.CascadeFilter(ab.ZFilter([1, 0.5], [1, -0.9]), ab.ZFilter([0.3, 0.2, 0.1], [1, 0.4, 0.2]),
                           ab.ZFilter([2.0], [1, 0, 0.81]))
  assert rel_err(list(casc3(xs, memory=[0.3, -0.2], zero=0.25)), vectors["seed_cascade_y"]) <= TOL
  par = ab.ParallelFilter(ab.ZFilter([1, 1], [1, -0.5]), ab.ZFilter([0.5], [1, 0.3, 0.1]), ab.ZFilter([0, 0, 2.0]))
  assert rel_err(list(par(xs)), vectors["parallel_y"]) <= TOL
  xg = signal(4, 4000).tolist()
  assert rel_err(list(ab.comb.fb(37, 0.8)(xg)), vectors["comb_fb_y"]) <= TOL
  assert rel_err(list(ab.comb.ff(100, -0.5)(xg)), vectors["comb_ff_y"]) <= TOL


@pytest.mark.parametrize("strategy", ["slaney", "klapuri", "sampled"])
def test_gammatone_channels_and_bank(ab, vectors, strategy):
  s, Hz = ab.sHz(48000)
  x = signal(0, 8000)
  bank = ab.gammatone_bank(strategy=strategy)
  chans = vectors["bank_channels"]
  c = int(chans[3])
  bw = ab.gammatone_erb_constants(4)[0] * ab.erb(bank.freqs[c] * Hz, Hz)       # examples/gammatone_plots.py:47,64
  single = ab.gammatone[strategy](bank.freqs[c] * Hz, bw)
  assert rel_err(list(single(x.tolist())), vectors["bank_%s_y" % strategy][3]) <= TOL
  streams = bank(x.tolist())                                                   # one input fanned out to 64 Streams
  assert len(streams) == 64 and all(isinstance(st, ab.Stream) for st in streams)
  got = np.array([list(streams[int(i)]) for i in chans])
  assert rel_err(got, vectors["bank_%s_y" % strategy]) <= TOL
  y = bank.apply_host(np.stack([x, signal(7, 8000)]))                          # batch API, host buffers
  assert y.shape == (2, 64, 8000)
  assert rel_err(y[0][chans], vectors["bank_%s_y" % strategy]) <= TOL


def test_lazy_pump_and_batch_state(ab):
  import torch
  z = ab.z
  filt = 1 / (1 - 0.999 * z ** -1)
  pulled = []

  def source():
    for i in it.count():
      pulled.append(i)
      yield 1.0

  out = filt(source())
  first = out.take(10)
  assert len(first) == 10 and len(pulled) <= 2048           # read-ahead is bounded, the input is endless
  more = out.take(5000)
  want, m = [], 0.0
  for _ in range(5010):
    m = 1.0 + 0.999 * m
    want.append(m)
  assert rel_err(first + more, want) <= TOL
  bank = ab.gammatone_bank(freqs=ab.erb_space(n=8), strategy="slaney")
  x = torch.from_numpy(np.stack([signal(40 + i, 4096) for i in range(70)])).cuda()
  whole = bank.apply(x)
  state = bank.new_state(70)
  parts = [bank.apply(x[:, a:b].contiguous(), state=state) for a, b in [(0, 1000), (1000, 1001), (1001, 4096)]]
  assert torch.equal(torch.cat(parts, dim=2), whole)
  assert rel_err(whole.cpu().numpy(), oracle.bank_apply(x.cpu().numpy(), bank.sections())) <= TOL


def test_nccl_sharding_parity_under_torchrun(ab):
  """Both multi-GPU partitionings on real NCCL, launched the way the driver launches bench.py: channel-sharded
  (overlapped broadcast pipeline, in-place all-gather, fused peer-memory store) and stream-sharded (scatter), every
  result bit-identical to the single-GPU bank (tools/nccl_check.py). Needs >= 2 GPUs."""
  import subprocess
  import sys
  import torch
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  from conftest import ROOT
  import os
  env = dict(os.environ, ALZ_CHECK_S="256", ALZ_CHECK_T="4096")
  out = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
                        "--master-addr", "127.0.0.1", "--master-port", "29533", os.path.join(ROOT, "tools", "nccl_check.py")],
                       capture_output=True, text=True, timeout=600, env=env)
  assert out.returncode == 0 and "PARITY OK" in out.stdout, out.stdout[-2000:] + out.stderr[-2000:]


def test_channel_major_output(ab):
  """``bank.apply(x, channel_major=True)`` writes y[C][S][T] (alz_apply_f32_ex with swapped strides): same values."""
  import torch
  bank = ab.gammatone_bank(freqs=ab.erb_space(n=12), strategy="klapuri")
  x = torch.from_numpy(np.stack([signal(80 + i, 4099) for i in range(70)])).cuda()
  y = bank.apply(x)
  ycm = bank.apply(x, channel_major=True)
  assert ycm.shape == (12, 70, 4099) and torch.equal(ycm.permute(1, 0, 2), y)
  x4 = x[:, :4096].contiguous()                      # 16-byte aligned rows: the TMA engine
  assert torch.equal(bank.apply(x4, channel_major=True).permute(1, 0, 2), bank.apply(x4))


def test_partition_stream(ab):
  """alz_stream_create_partition: a stream whose kernels run on a subset of the SMs (green context); the bank gives the
  same bits there (what BroadcastPipeline(compute_sms=...) relies on to leave SMs to NCCL)."""
  import torch
  from audiolazy_b200 import _capi
  try:
    part = _capi.PartitionStream(128)
  except _capi.NativeError as exc:
    pytest.skip("no green contexts here: %s" % exc)
  try:
    assert 8 <= part.sm_count <= torch.cuda.get_device_properties(0).multi_processor_count and part.sm_count % 8 == 0
    bank = ab.gammatone_bank(freqs=ab.erb_space(n=8), strategy="slaney")
    x = torch.from_numpy(np.stack([signal(90 + i, 4096) for i in range(40)])).cuda()
    want = bank.apply(x)
    ext = torch.cuda.ExternalStream(part.handle, device=x.device)
    ext.wait_stream(torch.cuda.current_stream())
    state = bank.new_state(40)
    out = torch.empty_like(want)
    torch.cuda.synchronize()
    with torch.cuda.stream(ext):
      bank.apply(x, state=state, out=out)
    ext.synchronize()
    assert torch.equal(out, want)
  finally:
    torch.cuda.synchronize()
    part.close()
  with pytest.raises(ValueError):
    _capi.PartitionStream(4)                            # fewer than the architecture's minimum of 8 SMs


def test_sharded_bank_single_process(ab):
  """world size 1 (no process group): the sharded wrapper degenerates to the bank itself; state=None is a fresh
  state on every call, as FilterBank.apply."""
  import torch
  from audiolazy_b200.parallel import ShardedBank
  bank = ab.gammatone_bank(freqs=ab.erb_space(n=8), strategy="slaney")
  x = torch.from_numpy(np.stack([signal(60 + i, 2048) for i in range(33)])).cuda()
  want = bank.apply(x)
  for mode in ("streams", "channels"):
    sb = ShardedBank(bank, mode=mode)
    assert torch.equal(sb.apply(x), want) and torch.equal(sb.apply(x), want)
    assert torch.equal(sb.gather_output(sb.apply(x)), want)
  sb = ShardedBank(bank, mode="channels")
  buf = sb.alloc_gather(33, 2048)
  sb.gather_output_into(want, buf)
  assert torch.equal(buf[0], want)
  st = bank.new_state(33)
  a = sb.apply(x[:, :1000].contiguous(), state=st)
  b = sb.apply(x[:, 1000:].contiguous(), state=st)
  assert torch.equal(torch.cat([a, b], dim=2), want)
  with pytest.raises(ValueError):                      # a state of another bank must not reach the kernel
    bank.apply(x, state=ab.gammatone_bank(freqs=ab.erb_space(n=4), strategy="slaney").new_state(33))


def test_callers_of_the_path(ab, vectors):
  """SURVEY.md 8f item 2: envelope / maverage / karplus_strong / accumulate, against outputs
  of the reference's own implementations (tests/golden/make_golden.py)."""
  xc = signal(5, 3000).tolist()
  assert rel_err(list(ab.envelope.rms(xc, cutoff=np.pi / 64)), vectors["envelope_rms_y"]) <= TOL
  assert rel_err(list(ab.envelope.abs(xc)), vectors["envelope_abs_y"]) <= TOL
  assert rel_err(list(ab.envelope.squared(xc, cutoff=0.2)), vectors["envelope_squared_y"]) <= TOL
  assert rel_err(list(ab.maverage.recursive(16)(xc)), vectors["maverage_recursive_y"]) <= TOL
  assert rel_err(list(ab.maverage.fir(5)(xc)), vectors["maverage_fir_y"]) <= TOL
  mem = signal(6, 400).astype(np.float64).tolist()
  ks = ab.karplus_strong(2 * np.pi * 220.5 / 44100, tau=5e3, memory=mem)      # endless silence in, seeded comb
  assert rel_err(ks.take(3000), vectors["karplus_strong_y"]) <= TOL
  assert rel_err(list(ab.accumulate_z(signal(8, 500).tolist())), vectors["accumulate_z_y"]) <= TOL


def test_time_varying_coefficients(ab, vectors):
  """SURVEY.md 8f item 4 / reference lazy_filters.py:169-176, 200-216: Stream-valued b_k, a_k, a_0;
  golden outputs from the reference (tests/golden/make_golden.py)."""
  z, St = ab.z, ab.Stream
  xt = signal(9, 300).tolist()
  filters = {
    "tv_gain_delay": lambda: St(0.5, -1.0, 2.0) * z ** -2,
    "tv_fir_div": lambda: (2 + St(1, 2, 3) * z ** -1) / St(1, 5),
    "tv_a0": lambda: 1 / (St(1, 2, 3) - z ** -1),
    "tv_iir": lambda: (0.5 + St(.3, -.2) * z ** -1) / (1 - St(.1, .7, -.5, -1e-3) * z ** -1 + 0.2 * z ** -2),
  }
  for key, make in filters.items():
    filt = make()
    assert not filt.is_lti()
    out = filt(xt)
    assert isinstance(out, St)
    assert rel_err(list(out), vectors[key + "_y"]) <= TOL, key
  assert rel_err(list(filters["tv_iir"]()(xt, memory=[0.4, -0.3], zero=0.2)), vectors["tv_iir_seeded_y"]) <= TOL
  short = St([1., 2., 3., 4., 5.]) * z ** -1 + 1
  assert rel_err(list(short(xt[:5])), vectors["tv_short_coef_y"]) <= TOL
  # copies keep both filters usable (reference tests/test_filters.py::test_copy)
  f1 = (2 + St(1, 2, 3) * z ** -1) / St(1, 5)
  f2 = f1.copy()
  assert list(f1(xt[:40])) == list(f2(xt[:40]))
  # a long lazy input crosses several pump blocks
  gain = St(1.0, 0.5)
  out = (gain * z ** -1)(St(xt * 20)).take(3000)
  want = [0.0] + [(1.0 if i % 2 == 0 else 0.5) * (xt * 20)[i - 1] for i in range(1, 3000)]
  assert np.allclose(out, want, rtol=1e-6, atol=1e-7)


def test_array_api_of_single_filters(ab, designs, vectors):
  import torch
  casc = ab.CascadeFilter([ab.ZFilter(r[:3], r[3:]) for r in designs["cfg2_sos"]])
  x = signal(2, 50000)
  y = casc.apply_host(x)
  assert y.shape == (50000,) and rel_err(y, vectors["cfg2_y"]) <= TOL
  xs = np.stack([x[:4000], signal(3, 4000)])
  yt = casc.apply(torch.from_numpy(xs).cuda())
  assert yt.shape == (2, 4000) and rel_err(yt[0].cpu().numpy(), vectors["cfg2_y"][:4000]) <= TOL
  f = ab.ZFilter([1, 7, 2], [1, 0.5, 0.2])
  assert rel_err(f.apply_host(signal(1, 48000)), vectors["cfg1_y"]) <= TOL


def test_bank_freq_response_on_device(ab, vectors):
  """FilterBank.freq_response (alz_freq_response_f64) against the reference's own
  freq_response values (golden) and the host evaluation of the same filters."""
  grid = vectors["freq_grid"]
  chans = vectors["bank_channels"]
  for name in ["slaney", "klapuri", "sampled"]:
    bank = ab.gammatone_bank(strategy=name)
    got = bank.freq_response(grid)
    assert got.shape == (64, len(grid)) and got.dtype == np.complex128
    want = vectors["bank_%s_freq_response" % name]
    scale = np.abs(want).max(axis=1, keepdims=True)
    # Horner on normalised sections vs the reference's Poly evaluation: rounding only; the 8-tap
    # numerator of "sampled" cancels heavily in the lowest channels (SURVEY 8c: 3.5e-8 vs lfilter)
    tol = 5e-8 if name == "sampled" else 1e-10
    assert (np.abs(got[chans] - want) / scale).max() <= tol
    host = np.array([[complex(bank[c].freq_response(float(w))) for w in grid[::16]] for c in (0, 31, 63)])
    assert (np.abs(got[[0, 31, 63]][:, ::16] - host) / np.abs(host).max(axis=1, keepdims=True)).max() <= tol
  # unit gain at each channel's own centre frequency (the designs are normalised there)
  peak = np.abs(ab.gammatone_bank(strategy="slaney").freq_response(grid[193:]))[chans, np.arange(len(chans))]
  assert np.abs(peak - 1).max() <= 1e-9
  # a pole on the grid is NaN, as the reference returns nan for den == 0
  acc = ab.FilterBank([1 / (1 - ab.z ** -1)])
  r = acc.freq_response([0.0, 1.0])
  assert np.isnan(r[0, 0]) and abs(r[0, 1] - 1 / (1 - np.exp(-1j))) < 1e-14


def test_stream_valued_design_parameters_filter(ab, vectors):
  """Builders called with Stream parameters (swept resonator / cutoff / decay) run through the
  time-varying kernel path; outputs against the reference's (golden)."""
  from test_designs import _tv_builders
  xb = signal(10, 2500).tolist()
  for key, make in _tv_builders(ab).items():
    out = list(make()(xb))
    assert len(out) == 2500
    assert rel_err(out, vectors[key + "_y"]) <= TOL, key
