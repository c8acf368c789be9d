"""The plan-time precision-tier decision (host logic, no GPU): a design-only plan runs every channel
through the kernel's own arithmetic in float64 and float32 on the CPU.  Here the float32 error it reports
is re-derived with an independent numpy emulation of the same recurrence on the same probe noise."""
import numpy as np
import pytest

from audiolazy_b200 import _capi

f32 = np.float32


def lcg_noise(n, seed=12345):
  out = np.empty(n, dtype=f32)
  s = seed
  for i in range(n):
    s = (s * 1664525 + 1013904223) & 0xFFFFFFFF
    out[i] = f32((s >> 8) * (2.0 / 16777216.0) - 1.0)
  return out


def fma32(a, b, c):
  return (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(f32)


def monic_emulation(bank, x, dtype):
  """Monic cascade of csrc/alz_biquad.cuh (gain on the float32 input), vectorised over channels."""
  C, K = len(bank), max(len(ch) for ch in bank)
  c1 = np.zeros((C, K)); na1 = np.zeros((C, K)); na2 = np.zeros((C, K)); G = np.ones(C)
  for c, ch in enumerate(bank):
    for k, (b, a) in enumerate(ch):
      assert len(b) <= 2 and a[0] == 1.0
      G[c] *= b[0]
      c1[c, k] = (b[1] if len(b) > 1 else 0.0) / b[0]
      na1[c, k], na2[c, k] = -a[1], -a[2]
  Gf = G.astype(f32)
  fma = fma32 if dtype is f32 else (lambda a, b, c: a * b + c)     # float64: fused vs. separate rounding is far below what is compared
  u = np.zeros((K + 1, 2, C), dtype=dtype)
  y = np.empty((C, len(x)), dtype=f32)
  cf = lambda v: v.astype(dtype)
  for n in range(len(x)):
    inp = (x[n] * Gf).astype(f32).astype(dtype)
    in1 = u[0, 0].copy()
    u[0, 1] = in1
    u[0, 0] = inp
    for k in range(K):
      y1, y2 = u[k + 1, 0].copy(), u[k + 1, 1].copy()
      t = fma(cf(c1[:, k]), in1, inp)
      t = fma(cf(na2[:, k]), y2, t)
      o = fma(cf(na1[:, k]), y1, t)
      u[k + 1, 1] = y1
      u[k + 1, 0] = o
      inp, in1 = o, y1
    y[:, n] = inp.astype(f32)
  return y


def test_tier_probe_matches_an_independent_emulation(designs):
  bank = designs["bank_slaney"]
  plan = _capi.Plan(bank, design_only=True)
  assert plan.kind == _capi.KIND_BIQUAD and plan.device == -1
  tier, probe = plan.tiers()
  assert plan.n_fp32_channels == int(tier.sum()) > 0
  # probe > tol on every float64 channel holds here because no slaney channel has a pole beyond radius 0.99; elsewhere
  # such a channel stays on float64 whatever it measures (tests/test_design_space.py)
  assert np.all(probe[tier == 1] <= plan.tier_tol) and np.all(probe[tier == 0] > plan.tier_tol)
  x = lcg_noise(8192)
  y64 = monic_emulation(bank, x, np.float64).astype(np.float64)
  y32 = monic_emulation(bank, x, f32).astype(np.float64)
  err = np.max(np.abs(y32 - y64), axis=1) / np.max(np.abs(y64), axis=1)
  # the probe also runs a step, an impulse, noise + a Nyquist tone and the Nyquist sequence, so it may only be larger; on most channels noise dominates
  assert np.all(probe >= err * 0.98)
  assert np.median(probe / err) < 1.25
  # monotone picture: the 16 lowest channels are orders of magnitude outside, the top 16 well inside
  assert probe[:16].min() > 2e-5 and probe[-16:].max() < 1.5e-6


def test_design_only_plans_cannot_compute(designs):
  plan = _capi.Plan(designs["bank_klapuri"], design_only=True)
  with pytest.raises(_capi.NativeError):
    plan.apply(0, 0, 0, 1, 1, 1, 1)
  exact = _capi.Plan(designs["bank_klapuri"], design_only=True, exact=True)
  assert exact.n_fp32_channels == 0 and plan.n_fp32_channels > 0
  assert plan.state_doubles(3) == exact.state_doubles(3)


def test_generic_plans_have_no_tiers(designs):
  plan = _capi.Plan([designs["comb_fb_37_0.8"]], design_only=True)
  assert plan.kind == _capi.KIND_GENERIC and plan.n_fp32_channels == 0
  tier, probe = plan.tiers()
  assert not tier.any() and np.all(probe < 0)
