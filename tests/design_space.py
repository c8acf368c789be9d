"""The filter designs users actually get, as test cases: every coefficient comes out of the package's public builders
(``gammatone_bank``, ``resonator``, ``lowpass`` / ``highpass``, ``comb``, ``maverage``, ``ZFilter`` algebra,
``CascadeFilter`` / ``ParallelFilter``) or, for the Butterworth cascades, out of ``scipy.signal.butter``.

Deterministic: no randomness at all; the shapes, block splits and seeds of a case follow from its position in the list.
``tests/test_design_space.py`` checks the routing of every case on any machine (``tests/golden/design_routing.json``)
and ``tests/test_filter_designs_gpu.py`` runs them against the float64 oracle.
"""
from functools import partial
from math import log

import numpy as np

import audiolazy_b200 as ab

RATES = [8000, 16000, 22050, 44100, 96000, 192000]
STRATEGIES = ["slaney", "klapuri", "sampled"]
BANK_SIZES = [1, 13, 64, 100]
COMB_DELAYS = [1, 15, 16, 17, 48, 49, 100, 1000, 4800]    # near / far taps (16) and ring sizes pow2(delay + 16) of the window kernel
COMB_ALPHAS = [0.9, -0.9, 0.999, -0.999, 0.9999, -0.9999]
#: (S, T) around the routing thresholds: a warp holds 32 streams; 16384 samples start the time-parallel evaluation
SHAPES = [(1, 1), (3, 33), (32, 16383), (33, 16384), (3, 200077), (4097, 33), (1, 200077), (33, 33), (4097, 1),
          (1, 16384), (3, 16383), (32, 200077)]
LONG_T = 10 ** 6 + 37
#: block lengths of the split runs (0, 1 and 31 included); the last block takes what is left
SPLITS = [0, 1, 31, 0, 33, 1000, 1, 16384]
#: S x C x T above which a case takes the next shape of the list (keeps the float64 oracle to about a second a case)
BUDGET = 4e7
#: the memory= / zero= seeds of the seeded cases (float32 values: the kernels round the seeded input history as they
#: round the input)
MEMORY, ZERO = [0.5, -0.25, 0.125], 0.125


class Case(object):
  """``bank``: channels -> sections -> ``(b, a)``; ``plan_kw``: for ``_capi.Plan``; ``seed``: ``(memory, zero)`` or
  None; ``meta``: what the design came from (``rate``, ``freqs``, ``strategy``, ``parallel``, ...)."""

  def __init__(self, cid, family, bank, S, T, splits, seed=None, plan_kw=None, **meta):
    self.id, self.family, self.bank = cid, family, bank
    self.S, self.T, self.splits, self.seed = S, T, splits, seed
    self.plan_kw = plan_kw or {}
    self.meta = meta

  def __repr__(self):
    return self.id


def _sections(filt):
  """Channel sections of one public filter object (what ``FilterBank.sections`` hands to the plan)."""
  return ab.FilterBank([filt]).sections()[0]


def _splits(T):
  out, left = [], T
  for n in SPLITS:
    if n > left:
      break
    out.append(n)
    left -= n
  return out


def _rad(hz, rate=48000):
  return hz * ab.sHz(rate)[1]


def _designs():
  """(id, family, bank, meta) in a fixed order."""
  out = []
  for rate in RATES:
    for strategy in STRATEGIES:
      for n in BANK_SIZES:
        freqs = ab.erb_space(50, 0.45 * rate, n)
        bank = ab.gammatone_bank(freqs, rate, strategy)
        out.append(("gammatone-%s-r%d-n%d" % (strategy, rate, n), "gammatone", bank.sections(),
                    dict(rate=rate, freqs=freqs, strategy=strategy)))
  # the sampled strategy is the one whose section count follows the gammatone order (eta)
  for order in (2, 6):
    freqs = ab.erb_space(50, 0.45 * 48000, 13)
    bank = ab.gammatone_bank(freqs, 48000, partial(ab.gammatone.sampled, eta=order), order=order)
    out.append(("gammatone-sampled-order%d-r48000-n13" % order, "gammatone", bank.sections(),
                dict(rate=48000, freqs=freqs, strategy="sampled")))
  # narrow single filters at 48 kHz, from near DC to near Nyquist
  for strategy in ("poles_exp", "freq_poles_exp", "z_exp", "freq_z_exp"):
    for f in (20, 1000, 23980):
      for bw in (1, 100):
        out.append(("resonator-%s-f%d-bw%d" % (strategy, f, bw), "resonator",
                    [_sections(ab.resonator[strategy](_rad(f), _rad(bw)))], {}))
  for kind, builder in (("lowpass", ab.lowpass), ("highpass", ab.highpass)):
    for strategy in ("pole", "z", "pole_exp", "z_exp"):
      for f in (1, 1000, 23000):
        out.append(("%s-%s-c%d" % (kind, strategy, f), "onepole", [_sections(builder[strategy](_rad(f)))], {}))
  # combs: one bank per strategy and delay, a channel per alpha
  for d in COMB_DELAYS:
    out.append(("comb-fb-d%d" % d, "comb", [_sections(ab.comb.fb(d, a)) for a in COMB_ALPHAS], {}))
    out.append(("comb-tau-d%d" % d, "comb",
                [_sections(ab.comb.tau(d, -d / log(a))) for a in COMB_ALPHAS if a > 0], {}))
    out.append(("comb-ff-d%d" % d, "comb", [_sections(ab.comb.ff(d, a)) for a in COMB_ALPHAS], {}))
  for strategy in ("recursive", "fir"):            # maverage.deque is a host generator, not a linear filter
    for size in (1, 16, 17, 1024):
      out.append(("maverage-%s-%d" % (strategy, size), "maverage", [_sections(ab.maverage[strategy](size))], {}))
  # Butterworth cascades: K = ceil(N / 2) sections, across the biquad kernel's K <= 8
  from scipy.signal import butter
  for N in range(2, 25):
    wn, btype = [(0.002, "lowpass"), (0.05, "highpass"), (0.3, "lowpass"), (0.9, "highpass")][N % 4]
    sos = butter(N, wn, btype=btype, output="sos")
    casc = ab.CascadeFilter([ab.ZFilter(list(r[:3]), list(r[3:])) for r in sos])
    out.append(("sos-butter-N%d" % N, "sos", [_sections(casc)], dict(wn=wn, btype=btype)))
  # compositions
  sos4 = butter(4, 0.05, output="sos")
  biquad = ab.ZFilter(list(sos4[0, :3]), list(sos4[0, 3:]))
  out.append(("cascade-biquad-comb16", "cascade", [_sections(ab.CascadeFilter([biquad, ab.comb.fb(16, 0.9)]))], {}))
  out.append(("cascade-comb48-biquad", "cascade", [_sections(ab.CascadeFilter([ab.comb.fb(48, -0.999), biquad]))], {}))
  out.append(("zfilter-resonator-times-comb", "cascade",
              [_sections(ab.resonator.poles_exp(_rad(440), _rad(20)) * ab.comb.ff(17, 0.5))], {}))
  out.append(("zfilter-lowpass-plus-highpass", "cascade",
              [_sections(ab.lowpass.pole(_rad(300)) + ab.highpass.z(_rad(8000)))], {}))
  out.append(("zfilter-resonator-over-comb", "cascade",
              [_sections(ab.resonator.z_exp(_rad(2000), _rad(50)) / (1 - 0.5 * ab.z ** -20))], {}))
  for C, bw in ((8, 1), (24, 30)):
    freqs = ab.erb_space(30, 23000, C)
    par = ab.ParallelFilter([ab.resonator.poles_exp(_rad(f), _rad(bw)) for f in freqs])
    out.append(("psum-resonators-C%d-bw%d" % (C, bw), "psum", par._flat_sections(), dict(parallel=True)))
  # 112 single-section channels fill the window kernel's parameter block; 113 and 200 go to the generic kernel.
  # The biquad kernel takes 73 one-section channels per small block and 512 per large one.
  for C in (111, 112, 113, 200):
    out.append(("wide-comb-C%d" % C, "wide",
                [_sections(ab.comb.fb(1 + c % 40, COMB_ALPHAS[c % 6])) for c in range(C)], {}))
    freqs = ab.erb_space(20, 23900, C)
    out.append(("wide-resonator-C%d" % C, "wide",
                [_sections(ab.resonator.freq_poles_exp(_rad(f), _rad(1 + c % 50))) for c, f in enumerate(freqs)], {}))
  return out


def _cases():
  cases = []
  for i, (cid, family, bank, meta) in enumerate(_designs()):
    C = len(bank)
    j = i % len(SHAPES)
    while SHAPES[j][0] * C * SHAPES[j][1] > BUDGET:
      j = (j + 1) % len(SHAPES)
    S, T = SHAPES[j]
    seed = (MEMORY, ZERO) if i % 5 == 2 and family != "psum" else None
    plan_kw = dict(parallel=True) if meta.get("parallel") else {}
    cases.append(Case(cid, family, bank, S, T, _splits(T), seed=seed, plan_kw=plan_kw, **meta))
  # few long streams: the time-parallel evaluation over a whole stream of a million samples
  by_id = {c.id: c for c in cases}
  # maverage.recursive(1) once ran on the float32 tier: its pole on the unit circle (cancelled by a zero) let the
  # float32 error random-walk to 4e-5 of the row peak over these samples
  long = ["gammatone-%s-r192000-n64" % s for s in STRATEGIES] + ["sos-butter-N16", "resonator-poles_exp-f20-bw1",
                                                                   "resonator-poles_exp-f1000-bw100", "maverage-recursive-1"]
  for base in long:
    c = by_id[base]
    cases.append(Case("long-" + base, c.family, c.bank, 1, LONG_T, [], **c.meta))
  return cases


CASES = _cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


#: what tests/golden/design_routing.json records of a plan, besides the kernel it runs on
ROUTING_FIELDS = ("kind", "n_sections", "monic_mode", "fp64_ops", "n_fp32_channels", "state_doubles_per_recurrence",
                  "time_parallel")


def kernel(plan):
  """"biquad", "window" or "generic" (a window plan has no tap table to report)."""
  from audiolazy_b200 import _capi
  if plan.kind == _capi.KIND_BIQUAD:
    return "biquad"
  try:
    plan.taps()
  except _capi.NativeError:
    return "window"
  return "generic"


def routing(plan):
  return dict({f: getattr(plan, f) for f in ROUTING_FIELDS}, kernel=kernel(plan))


def pole_radius(channel):
  """Largest pole radius of a channel (every section's denominator roots)."""
  r = 0.0
  for _, a in channel:
    a = np.trim_zeros(np.asarray(a, dtype=np.float64), "b")
    taps = np.flatnonzero(a[1:]) + 1
    if len(taps) == 1:                                   # 1 - alpha z^-d: d poles of radius |alpha / a0|^(1/d)
      r = max(r, abs(a[taps[0]] / a[0]) ** (1.0 / taps[0]))
    elif len(taps):
      r = max(r, float(np.max(np.abs(np.roots(a)))))
  return r
