#!/usr/bin/env python
"""Generate the golden fixtures of tests/golden/ by RUNNING THE REFERENCE ITSELF.

Run it with a checkout of the reference (danilobellini/audiolazy) at hand:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_golden.py

The reference (pure Python) is imported unmodified from that checkout; nothing of it
is copied.  The fixtures pin
  * the filter *designs* (coefficient lists of every builder on the hot path),
  * the *outputs* of the reference's sample-by-sample evaluator on seeded inputs, and
  * the answers tests/test_reference_live.py and tests/test_callers_io.py compare with
    (reference_cases.json),
so that oracle/ (and, through it, the CUDA path) is checked without the reference.

Inputs are float32 samples ``numpy.random.default_rng(seed).uniform(-1, 1, n)`` widened
to Python floats, exactly as SURVEY.md section 8(d) prescribes; they are regenerated from
the seed by the tests, not stored.
"""
import hashlib
import json
import os
import sys
import warnings

import numpy as np

REF = os.environ["ALZ_REFERENCE"]
sys.path.insert(0, REF)
sys.dont_write_bytecode = True
warnings.simplefilter("ignore")
import audiolazy as al  # noqa: E402  (the reference)

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
RATE = 48000
s, Hz = al.sHz(RATE)


def signal(seed, n):
  return np.random.default_rng(seed).uniform(-1, 1, n).astype(np.float32)


def erb_space(lo=50.0, hi=20000.0, n=64):
  """ERB-rate (Glasberg & Moore) spaced centre frequencies, SURVEY.md section 8(d)."""
  E = lambda f: 21.4 * np.log10(1 + 0.00437 * f)
  Einv = lambda e: (10 ** (e / 21.4) - 1) / 0.00437
  return [float(Einv(E(lo) + i * (E(hi) - E(lo)) / (n - 1))) for i in range(n)]


def sections_of(filt):
  """[(numlist, denlist), ...] of a reference ZFilter / CascadeFilter."""
  if isinstance(filt, al.CascadeFilter):
    return [(list(map(float, f.numlist)), list(map(float, f.denlist))) for f in filt]
  return [(list(map(float, filt.numlist)), list(map(float, filt.denlist)))]


def run(filt, x, **kw):
  return np.array(list(filt(x.astype(np.float64).tolist(), **kw)), dtype=np.float64)


def main():
  designs = {}
  vectors = {}

  # ---------------------------------------------------------------- bank designs
  fcs = erb_space()
  designs["bank_fc_hz"] = fcs
  bank_channels = [0, 1, 8, 16, 24, 32, 48, 63]
  x_bank = signal(0, 8000)
  for name in ["slaney", "klapuri", "sampled"]:
    strat = al.gammatone[name]
    chans = []
    for fc in fcs:
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fc * Hz, Hz)
      chans.append(sections_of(strat(fc * Hz, bw)))
    designs["bank_" + name] = chans
    outs = []
    for c in bank_channels:
      fc = fcs[c]
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fc * Hz, Hz)
      outs.append(run(strat(fc * Hz, bw), x_bank))
    vectors["bank_%s_y" % name] = np.stack(outs)
  vectors["bank_channels"] = np.array(bank_channels)
  # impulse responses (examples/gammatone_plots.py:71) of two channels, all strategies
  imp = np.zeros(2000, dtype=np.float32)
  imp[0] = 1
  for name in ["slaney", "klapuri", "sampled"]:
    outs = []
    for c in (4, 40):
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fcs[c] * Hz, Hz)
      outs.append(run(al.gammatone[name](fcs[c] * Hz, bw), imp))
    vectors["bank_%s_impulse" % name] = np.stack(outs)

  # frequency responses of the same channels (lazy_filters.py:267-301 via CascadeFilter, :1007)
  grid = np.concatenate([np.linspace(0.0, np.pi, 193), 2 * np.pi * np.array(fcs)[bank_channels] / 48000.0])
  vectors["freq_grid"] = grid
  for name in ["slaney", "klapuri", "sampled"]:
    rows = []
    for c in bank_channels:
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fcs[c] * Hz, Hz)
      filt = al.gammatone[name](fcs[c] * Hz, bw)
      rows.append([complex(filt.freq_response(float(w))) for w in grid])
    vectors["bank_%s_freq_response" % name] = np.array(rows, dtype=np.complex128)

  # ---------------------------------------------------------------- cfg 1
  x1 = signal(1, 48000)
  vectors["cfg1_y"] = run(al.ZFilter([1, 7, 2], [1, 0.5, 0.2]), x1)

  # ---------------------------------------------------------------- cfg 2 (first 50 000 samples)
  from scipy.signal import butter
  sos = butter(8, 0.25, output="sos")
  designs["cfg2_sos"] = sos.tolist()
  casc = al.CascadeFilter([al.ZFilter(r[:3].tolist(), r[3:].tolist()) for r in sos])
  vectors["cfg2_y"] = run(casc, signal(2, 50000))

  # ---------------------------------------------------------------- memory= / zero= seeding
  xs = signal(3, 64)
  f = al.ZFilter([0.5, -0.25, 2.0], [2.0, 0.5, -0.3])
  vectors["seed_single_y"] = run(f, xs, memory=[0.75, -1.5], zero=0.125)
  vectors["seed_short_memory_y"] = run(f, xs, memory=[0.75], zero=-0.5)
  casc3 = al.CascadeFilter(al.ZFilter([1, 0.5], [1, -0.9]), al.ZFilter([0.3, 0.2, 0.1], [1, 0.4, 0.2]),
                           al.ZFilter([2.0], [1, 0, 0.81]))
  designs["seed_cascade"] = sections_of(casc3)
  vectors["seed_cascade_y"] = run(casc3, xs, memory=[0.3, -0.2], zero=0.25)
  vectors["a0_not_one_y"] = run(al.ZFilter([1.0, 3.0], [-18.0, 9.8, 0.0, 14.3]), xs)
  vectors["a0_minus_one_y"] = run(al.ZFilter([1.0, 0.0, -1.0], [-1.0, 0.5]), xs)

  # ---------------------------------------------------------------- high order / sparse (generic kernel)
  b8 = [0.2, -0.1, 0.05, 0.3, 0.0, -0.2, 0.1, 0.07]
  a5 = [1.0, -0.5, 0.25, 0.0, -0.1]
  designs["generic_b"] = b8
  designs["generic_a"] = a5
  xg = signal(4, 4000)
  vectors["generic_y"] = run(al.ZFilter(b8, a5), xg)
  vectors["comb_fb_y"] = run(al.comb.fb(37, 0.8), xg)
  vectors["comb_ff_y"] = run(al.comb.ff(100, -0.5), xg)
  designs["comb_fb_37_0.8"] = sections_of(al.comb.fb(37, 0.8))
  designs["comb_tau_20_50"] = sections_of(al.comb.tau(20, 50.0))
  designs["comb_ff_100_-0.5"] = sections_of(al.comb.ff(100, -0.5))

  # ---------------------------------------------------------------- ParallelFilter
  par = al.ParallelFilter(al.ZFilter([1, 1], [1, -0.5]), al.ZFilter([0.5], [1, 0.3, 0.1]), al.ZFilter([0, 0, 2.0]))
  vectors["parallel_y"] = run(par, xs)
  designs["parallel"] = [sections_of(f) for f in par]

  # ---------------------------------------------------------------- callers of the path (SURVEY 8f)
  xc = signal(5, 3000)
  xl = xc.astype(np.float64).tolist()
  vectors["envelope_rms_y"] = np.array(list(al.envelope.rms(xl, cutoff=np.pi / 64)))
  vectors["envelope_abs_y"] = np.array(list(al.envelope.abs(xl)))
  vectors["envelope_squared_y"] = np.array(list(al.envelope.squared(xl, cutoff=0.2)))
  vectors["maverage_recursive_y"] = run(al.maverage.recursive(16), xc)
  vectors["maverage_fir_y"] = run(al.maverage.fir(5), xc)
  mem = signal(6, 400).astype(np.float64).tolist()
  ks = al.karplus_strong(2 * np.pi * 220.5 / 44100, tau=5e3, memory=mem)
  vectors["karplus_strong_y"] = np.array(ks.take(3000))
  vectors["accumulate_z_y"] = run(al.accumulate.z, signal(8, 500))

  # ---------------------------------------------------------------- time-varying coefficients (SURVEY 8f item 4)
  xt = signal(9, 300)
  St = al.Stream
  tv = {
    "tv_gain_delay": lambda: St(0.5, -1.0, 2.0) * al.z ** -2,
    "tv_fir_div": lambda: (2 + St(1, 2, 3) * al.z ** -1) / St(1, 5),
    "tv_a0": lambda: 1 / (St(1, 2, 3) - al.z ** -1),
    "tv_iir": lambda: (0.5 + St(.3, -.2) * al.z ** -1) / (1 - St(.1, .7, -.5, -1e-3) * al.z ** -1 + 0.2 * al.z ** -2),
  }
  for key, make in tv.items():
    vectors[key + "_y"] = run(make(), xt)
  vectors["tv_iir_seeded_y"] = run(tv["tv_iir"](), xt, memory=[0.4, -0.3], zero=0.2)
  vectors["tv_short_coef_y"] = run(al.Stream([1., 2., 3., 4., 5.]) * al.z ** -1 + 1, xt[:5])

  # Stream-valued DESIGN parameters (lazy_filters.py:1202-1206, examples/lptv.py:28-38): the builder
  # returns a filter whose coefficients are Streams
  sweep = lambda: al.Stream(0.1 + 0.001 * k for k in range(100000))
  tvb = {
    "tvb_resonator_poles_exp": lambda: al.resonator.poles_exp(sweep(), 0.05),
    "tvb_resonator_z_exp_bw": lambda: al.resonator.z_exp(0.3, sweep() * 0.1),
    "tvb_resonator_freq_z_exp_both": lambda: al.resonator.freq_z_exp(sweep(), sweep() * 0.1),
    "tvb_lowpass_pole": lambda: al.lowpass.pole(sweep()),
    "tvb_highpass_z": lambda: al.highpass.z(sweep()),
    "tvb_comb_tau": lambda: al.comb.tau(7, sweep() * 100),
  }
  xb = signal(10, 2500)
  for key, make in tvb.items():
    vectors[key + "_y"] = run(make(), xb)
    filt = make()
    rows = [np.array(c.take(40) if hasattr(c, "take") else [c] * 40, dtype=np.float64)
            for poly in (filt.numpoly, filt.denpoly) for _, c in poly.terms()]
    vectors[key + "_coefs"] = np.stack(rows)

  # ---------------------------------------------------------------- LPC (lazy_lpc.py) -- SURVEY 8f item 2
  np.mat = np.asmatrix          # the reference's elementwise() still looks numpy.mat up (removed in NumPy 2)
  rng = np.random.default_rng(5)
  n = np.arange(240)
  blk = (np.sin(0.3 * n) + 0.5 * np.sin(1.1 * n + 1) + 0.05 * rng.standard_normal(240)).astype(np.float32)
  blk_list = blk.astype(np.float64).tolist()
  lpc_cases = []
  for name in ["autocor", "nautocor", "kautocor", "covar", "kcovar"]:
    for order in [1, 2, 6, 14]:
      filt = al.lpc[name](blk_list, order)
      lpc_cases.append({"strategy": name, "order": order, "numerator": [float(c) for c in filt.numerator],
                        "error": float(filt.error)})
  filt8 = al.lpc.kautocor(blk_list, 8)
  designs["lpc"] = {"cases": lpc_cases, "parcor8": [float(k) for k in al.parcor(filt8)],
                    "lsf8": [float(w) for w in al.lsf(filt8)],
                    "acorr9": [float(v) for v in al.acorr(blk_list, 9)],
                    "lag_matrix3": [[float(v) for v in row] for row in al.lag_matrix(blk_list, 3)]}
  vectors["lpc_blk"] = blk
  filt12 = al.lpc.kautocor(blk_list, 12)
  resid = run(filt12, blk)                                   # analysis (whitening) FIR of order 12
  vectors["lpc_residual_y"] = resid
  vectors["lpc_synth_y"] = run(1 / filt12, resid.astype(np.float32))   # all-pole synthesis from the float32 residual

  # ---------------------------------------------------------------- builders (designs only)
  grid = []
  for name in ["poles_exp", "freq_poles_exp", "z_exp", "freq_z_exp"]:
    for freq in [0.01, 0.3, np.pi / 5, 1.7, 3.0]:
      for bw in [1e-3, 0.02, np.pi / 19, 0.5]:
        grid.append(("resonator." + name, [float(freq), float(bw)], sections_of(al.resonator[name](freq, bw))))
  for kind in ["lowpass", "highpass"]:
    for name in ["pole", "z", "pole_exp", "z_exp"]:
      for cutoff in [1e-3, 0.05, np.pi / 6, 1.0, np.pi / 2, 2.5, 3.1]:
        filt = getattr(al, kind)[name](cutoff)
        grid.append((kind + "." + name, [float(cutoff)], sections_of(filt)))
  for name in ["slaney", "klapuri", "sampled"]:
    for freq, bw in [(np.pi / 5, np.pi / 19), (0.05, 0.004), (2.0, 0.3)]:
      grid.append(("gammatone." + name, [float(freq), float(bw)], sections_of(al.gammatone[name](freq, bw))))
  grid.append(("gammatone.sampled", [0.7, 0.05, 0.6, 3], sections_of(al.gammatone.sampled(0.7, 0.05, phase=0.6, eta=3))))
  designs["builder_grid"] = grid
  designs["erb_gm90_hz"] = [[f, float(al.erb["gm90"](f))] for f in [20, 50, 440, 1000, 3000, 2e4]]
  designs["erb_mg83_hz"] = [[f, float(al.erb["mg83"](f))] for f in [20, 50, 440, 1000, 3000, 2e4]]
  designs["erb_gm90_rad"] = [[f, float(al.erb["gm90"](f * Hz, Hz))] for f in [20, 50, 440, 1000, 3000, 2e4]]
  designs["gammatone_erb_constants"] = [[n, list(map(float, al.gammatone_erb_constants(n)))] for n in range(1, 10)]
  designs["sHz_48000"] = [float(s), float(Hz)]
  # z algebra known answers
  zz = al.z
  alg = {
    "(1+z^-1)/(1-z^-1)": sections_of((1 + zz ** -1) / (1 - zz ** -1)),
    "1-2*0.9*cos(.3)z^-1+.81z^-2": sections_of(1 - 2 * 0.9 * np.cos(0.3) * zz ** -1 + 0.81 * zz ** -2),
    "(0.5*z^-1 + 1)*(1 - 0.25*z^-2)/ (1 + 0.1*z^-1)**2": sections_of(
      (0.5 * zz ** -1 + 1) * (1 - 0.25 * zz ** -2) / (1 + 0.1 * zz ** -1) ** 2),
    "sum of two": sections_of(1 / (1 - 0.5 * zz ** -1) + 2 / (1 + 0.25 * zz ** -1)),
    "diff": sections_of(((1 + 2 * zz ** -1) / (1 - 0.5 * zz ** -1)).diff()),
  }
  designs["z_algebra"] = alg
  # freq_response known answers
  fr = al.ZFilter([1, 7, 2], [1, 0.5, 0.2])
  designs["freq_response"] = [[w, [complex(fr.freq_response(w)).real, complex(fr.freq_response(w)).imag]]
                              for w in [0.0, 0.1, 1.0, np.pi / 2, 3.0]]

  with open(os.path.join(HERE, "designs.json"), "w") as fh:
    json.dump(designs, fh)
  np.savez_compressed(os.path.join(HERE, "vectors.npz"), **vectors)
  print("wrote", os.path.join(HERE, "designs.json"), os.path.getsize(os.path.join(HERE, "designs.json")), "bytes")
  print("wrote", os.path.join(HERE, "vectors.npz"), os.path.getsize(os.path.join(HERE, "vectors.npz")), "bytes")
  reference_cases()


def digest(y):
  """SHA-256 of a float64 array's little-endian bytes: bit-exact equality without storing the array."""
  return hashlib.sha256(np.ascontiguousarray(y, dtype="<f8").tobytes()).hexdigest()


def reference_cases():
  """reference_cases.json: what the reference answers in tests/test_reference_live.py and
  tests/test_callers_io.py (long outputs as digests of their float64 bytes)."""
  import audiolazy_b200 as ab
  from test_callers_io import make_wav
  cases = {}
  # test_oracle_vs_reference_all_64_channels: channels 0, 7, ..., 63 on signal(123, 3000)
  x = signal(123, 3000)
  cases["bank_digests"] = {}
  for name in ("slaney", "klapuri", "sampled"):
    bank = ab.gammatone_bank(strategy=name)
    rows = []
    for c in range(0, 64, 7):
      fc = bank.freqs[c]
      bw = al.gammatone_erb_constants(4)[0] * al.erb(fc * Hz, Hz)
      rows.append(digest(run(al.gammatone[name](fc * Hz, bw), x)))
    cases["bank_digests"][name] = rows
  # test_lfilter_grid_like_reference_test: reference tests/test_filters_extdep.py:41-47
  grid = []
  for a in [[1.], [3.], [1., 3.], [15., -17.2], [-18., 9.8, 0., 14.3]]:
    for b in [[1.], [-1.], [1., 0., -1.], [1., 3.]]:
      for data in [list(range(5)), list(range(5, 0, -1)), [7, 22, -5], [8., 3., 15.]]:
        grid.append([b, a, data, run(al.ZFilter(b, a), np.asarray(data, dtype=np.float32)).tolist()])
  cases["lfilter_grid"] = grid
  # test_random_designs_match_reference_bit_for_bit: the same draws as the test; per draw the digest of the
  # repr() of its seven filters' [(numlist, denlist), ...] (repr round-trips every float exactly)
  rng = np.random.default_rng(5)
  draws = []
  for _ in range(40):
    freq, bw, cutoff = rng.uniform(0.01, 3.0), rng.uniform(1e-3, 0.6), rng.uniform(0.01, 3.1)
    rng.integers(1, 50), rng.integers(1, 50)
    filts = [al.gammatone.slaney(freq, bw), al.gammatone.klapuri(freq, bw), al.gammatone.sampled(freq, bw),
             al.gammatone.sampled(freq, bw, phase=0.4, eta=5), al.lowpass.z(cutoff), al.highpass.pole(cutoff),
             al.resonator.z_exp(freq, bw)]
    draws.append(hashlib.sha256(repr([sections_of(f) for f in filts]).encode()).hexdigest())
  cases["random_designs"] = draws
  # test_memory_semantics_vs_reference
  xm = signal(9, 50)
  b, a = [0.3, 0.2, -0.4], [1.5, -0.2, 0.1, 0.05]
  cases["memory_semantics"] = [[memory, zero, run(al.ZFilter(b, a), xm, memory=memory, zero=zero).tolist()]
                               for memory, zero in [([0.1, 0.2, 0.3], 0.0), ([0.1], 0.25), ([0.1, 0.2, 0.3, 0.4, 0.5], -1.0),
                                                    (None, 0.5)]]
  # test_callers_io: WavStream, chunks, maverage / comb designs
  values = [0, 100, -100, 32767, -32768, 12345]
  cases["wavstream_16"] = list(al.WavStream(make_wav(16, 1, values)))
  wav = {}
  for bits in (8, 16, 24, 32):
    top = 1 << (bits - 1)
    vals = [0, 1, -1, top - 1, -top, top // 3, -(top // 7), 12345 % top, -(54321 % top)]
    for channels in (1, 2):
      v = vals if channels == 1 else vals + vals[::-1]
      wav["%d_%d" % (bits, channels)] = [list(al.WavStream(make_wav(bits, channels, v))),
                                         list(al.WavStream(make_wav(bits, channels, v), keep=True))]
  cases["wavstream_every_width"] = wav
  data = [0.5, -0.25, 1.0, 0.125, -1.0]
  cases["chunks"] = [[c.hex() for c in al.chunks(data, size=4)],
                     [c.hex() for c in al.chunks(data, size=2, dfmt="d", padval=9.)]]
  cases["maverage"] = {"%s_%d" % (name, size): [list(map(float, al.maverage[name](size).numlist)),
                                                list(map(float, al.maverage[name](size).denlist))]
                       for size in (1, 3, 8) for name in ("recursive", "fir")}
  kr = al.comb.tau(2 * np.pi / 0.05, 2e4).linearize()
  cases["comb_tau_linearized"] = [list(map(float, kr.numlist)), list(map(float, kr.denlist))]
  path = os.path.join(HERE, "reference_cases.json")
  with open(path, "w") as fh:
    json.dump(cases, fh, indent=0)
  print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
  main()
