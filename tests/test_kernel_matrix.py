"""The kernel matrix: every CUDA kernel instantiation of the library, run through the C ABI on small deterministic
cases and compared with the float64 oracle, plus a check that the matrix really launches every kernel the library
contains.

Each case is a bank (seeded pole / zero designs, never random denominators), a shape, optional ``memory=`` / ``zero=``
seeds and block splits, and the plan shape it was written for.  ``test_plan_routing`` checks that shape on any machine
(``design_only`` plans): a change to the plan logic that moves a case onto another kernel fails there first.

Tolerances (max |y - oracle| / max |oracle| per output row):
  * biquad, float64 tier: 2.5e-7 with the gain on the float32 input (MONIC 2: the input and the gain are rounded to
    float32 before the recurrence), 6.5e-8 otherwise (the float32 rounding of the float64 result, 2**-24, plus 10 %);
  * biquad, float32 tier: 1e-5 / 3 (what the plan-time probe admits, with a 3x margin on signals it has not seen);
  * window and generic kernels: 1e-7 (float32 rounding plus the reassociated float64 sum);
  * time-parallel evaluation: 3e-6 against the sequential one and 1e-5 against the oracle (the chunk states are
    rounded in float64 along a different path; the error grows with the chunk count, not with the precision tier).
"""
import contextlib
import os
import re

import numpy as np
import pytest

import oracle
from conftest import rel_err
from native_libs import compiled_kernels

TIER0_GAIN_IN = 2.5e-7
TIER0 = 6.5e-8
TIER1 = 1e-5 / 3
WINDOW = 1e-7
KIND_BIQUAD, KIND_GENERIC = 1, 2


def _rng(*key):
  return np.random.default_rng([int(k) for k in key])


def _pow2(n):
  q = 1
  while q < n:
    q <<= 1
  return q


# --------------------------------------------------------------------------------------------------------------------
# designs
# --------------------------------------------------------------------------------------------------------------------
def _gain_at(b, a, w):
  z = np.exp(-1j * w * np.arange(max(len(b), len(a))))
  return abs(np.dot(b, z[:len(b)]) / np.dot(a, z[:len(a)]))


def _section(rng, w, r, nb, fir=0):
  """A pole pair of radius r at angle w; nb numerator taps (1: constant, 2: one real zero, 3: a zero pair away from w;
  ``fir`` > 3: a head FIR of that many taps).  Scaled to unit gain at w."""
  a = [1.0, -2.0 * r * np.cos(w), r * r]
  if fir:
    b = [1.0] + list(rng.uniform(-0.6, 0.6, fir - 1))
  elif nb == 1:
    b = [1.0]
  elif nb == 2:
    b = [1.0, -rng.uniform(-0.9, 0.9)]
  else:
    rho, phi = rng.uniform(0.3, 1.0), (w + np.pi / 2 + rng.uniform(-0.5, 0.5)) % np.pi
    b = [1.0, -2.0 * rho * np.cos(phi), rho * rho]
  g = _gain_at(b, a, w)
  return [float(v / g) for v in b], [float(v) for v in a]


def _scale_gain(ch, target):
  """Scale the first section so that the product of the b0 of the cascade is ``target``."""
  prod = float(np.prod([s[0][0] for s in ch]))
  b, a = ch[0]
  ch[0] = ([v * target / prod for v in b], a)


def biquad_bank(key, C, kmax, nb, monic, counts="mixed", head_fir=0, radius=(0.9, 0.995)):
  """C channels; channel 0 has ``kmax`` sections of ``nb`` taps, the others (``counts="mixed"``) fewer sections and
  fewer taps.  Two channels in three have poles at radius 0.9 ... 0.995 (float64 tier), the third 0.3 ... 0.7 (usually
  the float32 tier).  monic 0: one channel's first b0 is 0; 1: one channel's gain product is 1e-33 (below a normal
  float32: the gain goes on the float64 output); 2: every product is near 1.  ``head_fir``: the first section of every
  channel is a 4 ... 8-tap FIR over the pole pair (channel 0: ``head_fir`` taps).  ``radius``: the pole radii of the
  float64-tier channels."""
  rng = _rng(11, key, C, kmax, nb, monic, head_fir)
  bank = []
  for c in range(C):
    sensitive = c % 3 != 2
    n = kmax if (c == 0 or counts != "mixed") else int(rng.integers(1, kmax + 1))
    w = rng.uniform(0.2, 2.9)
    rlo, rhi = radius if sensitive else (0.3, 0.7)
    ch = []
    for k in range(n):
      taps = nb if (c == 0 or counts != "mixed") else int(rng.integers(1, nb + 1))
      fir = 0
      if head_fir and k == 0:
        fir = head_fir if c == 0 else int(rng.integers(4, 9))
      ch.append(_section(rng, w * (1 + rng.uniform(-0.02, 0.02)), rng.uniform(rlo, rhi), taps, fir))
    _scale_gain(ch, 10.0 ** rng.uniform(-2, 2))
    bank.append(ch)
  if monic == 0:
    b, a = bank[-1][0]
    bank[-1][0] = ([0.0] + b[1:], a)
  elif monic == 1:
    _scale_gain(bank[0], 1e-33)
  return bank


def klapuri_bank(key, C):
  """gammatone.klapuri's structure: [1 - rho^2 z^-2, const, 1 - rho^2 z^-2, const] over pole pairs."""
  rng = _rng(12, key, C)
  bank = []
  for c in range(C):
    w, r = rng.uniform(0.2, 2.9), rng.uniform(0.9, 0.995) if c % 3 else rng.uniform(0.3, 0.7)
    ch = []
    for k in range(4):
      a = [1.0, -2.0 * r * np.cos(w), r * r]
      b = [1.0, 0.0, -rng.uniform(0.3, 1.0) ** 2] if k % 2 == 0 else [1.0]
      g = _gain_at(b, a, w)
      ch.append(([v / g for v in b], a))
    bank.append(ch)
  return bank


def window_channel(rng, near_x, near_y, far_x, far_y, keep=1.0):
  """One section: taps at the given delays (each kept with probability ``keep``); the feedback taps' magnitudes sum to
  0.95, so the filter is stable whatever the signs, and one dominant tap makes it ring."""
  xs = [d for d in near_x + far_x if rng.uniform() < keep]
  ys = [d for d in near_y + far_y if rng.uniform() < keep]
  b = np.zeros(max(xs + [0]) + 1)
  b[0] = rng.uniform(0.5, 1.0)
  for d in xs:
    b[d] = rng.uniform(-1, 1)
  a = np.zeros(max(ys + [0]) + 1)
  a[0] = 1.0
  if ys:
    mag = rng.uniform(0.1, 1.0, len(ys))
    mag[int(rng.integers(len(ys)))] += 3.0
    mag *= 0.95 / mag.sum()
    for d, m in zip(ys, mag):
      a[d] = m * rng.choice([-1.0, 1.0])
  return [(b.tolist(), a.tolist())]


# --------------------------------------------------------------------------------------------------------------------
# cases
# --------------------------------------------------------------------------------------------------------------------
class Case(object):
  def __init__(self, cid, family, bank, expect=None, S=37, T=301, seed=False, splits=None, plan_kw=None, **extra):
    self.id, self.family, self.bank, self.expect = cid, family, bank, expect
    self.S, self.T, self.seed, self.splits = S, T, seed, splits
    self.plan_kw = plan_kw or {}
    self.extra = extra

  def __repr__(self):
    return self.id


def _biquad_expect(K, nb, monic, head_fir=False, klapuri=False):
  NB0 = 8 if head_fir else 0
  h0 = 7 if head_fir else 2
  ops = K * (nb + 1) + (1 if monic == 1 else 0) if monic else K * (nb + 2)
  ops += (8 - nb) if head_fir else 0
  ops -= 6 if klapuri else 0
  return dict(kind=KIND_BIQUAD, n_sections=K, num_taps=NB0 or nb, monic=monic, state=h0 + 2 + 4 * (K - 1), fp64_ops=ops)


def _stride(K, head_fir=False):
  return 5 * K + 2 + (5 if head_fir else 0)


def _biquad_cases():
  out = []
  for K, kmax_small in ((1, 1), (2, 2), (3, 3), (4, 4), (6, 5), (8, 7)):
    for nb in (1, 2, 3):
      for monic in (0, 1, 2):
        for size in ("small", "large"):
          kmax = kmax_small if size == "small" else K          # Kmax = 5 / 7 run padded on the K = 6 / 8 kernels
          C = 5 if size == "small" else 512 // _stride(K) + 2   # one 512-double parameter block / one 3584-double block
          i = len(out)
          out.append(Case("biquad-K%d-kmax%d-nb%d-monic%d-%s" % (K, kmax, nb, monic, size), "biquad",
                          biquad_bank(i, C, kmax, nb, monic), _biquad_expect(K, nb, monic),
                          T=301 + (i % 4) * 33, seed=i % 2 == 0, splits=[1, 1, 30, 33, 100] if i % 3 == 0 else None,
                          coef="small" if size == "small" else "large"))
  for monic in (0, 1, 2):
    for C in (5, 30):
      bank = klapuri_bank(monic * 100 + C, C)
      if monic == 0:
        bank[-1][0] = ([0.0] + bank[-1][0][0][1:], bank[-1][0][1])
      elif monic == 1:
        _scale_gain(bank[0], 1e-33)
      out.append(Case("klapuri-monic%d-C%d" % (monic, C), "biquad", bank, _biquad_expect(4, 3, monic, klapuri=True),
                      seed=C == 5, splits=[7, 50]))
  for monic in (0, 1, 2):
    for C in (5, 50):
      out.append(Case("headfir-K1-monic%d-C%d" % (monic, C), "biquad",
                      biquad_bank(300 + C, C, 1, 1, monic, head_fir=4 if C == 5 else 7), _biquad_expect(1, 1, monic, head_fir=True),
                      seed=True, splits=[3]))
      for nb in (1, 3):
        C4 = 5 if C == 5 else 30
        out.append(Case("headfir-K4-nb%d-monic%d-C%d" % (nb, monic, C4), "biquad",
                        biquad_bank(400 + C4, C4, 4, nb, monic, head_fir=8), _biquad_expect(4, nb, monic, head_fir=True),
                        seed=C4 == 5, splits=[3]))
  # both sides of the small block, above one large chunk (two launches)
  for K, C in ((8, 12), (8, 13), (8, 90), (4, 170)):
    out.append(Case("biquad-K%d-C%d" % (K, C), "biquad", biquad_bank(500 + C, C, K, 3, 2, counts="full"),
                    _biquad_expect(K, 3, 2), S=40, T=260, seed=True, splits=[130]))
  return out


WINDOW_SHAPES = [(mx, my) for mx in (0, 4, 16) for my in (0, 4, 16)]
NEAR = {0: [], 4: [1, 3], 16: [2, 4, 15]}           # 3 / 4: the window size switches; 15: last near delay
NEAR_Y = {0: [], 4: [1, 3], 16: [1, 4, 15]}
FAR_X = [[16], [48], [16, 49], []]                   # 16: first far delay; 48: ring pow2(48 + 16) exactly full; 49: just over
FAR_Y = [[49], [], [17, 48], [16]]
WINDOW_LARGE_C = [3, 17, 112, 40, 5, 64, 9, 100, 33]


def _window_expect(mx, my, far_x, far_y, nb):
  xr = _pow2(max(far_x) + 16) if far_x else 0
  yr = _pow2(max(far_y) + 16) if far_y else 0
  near = (mx - 1 if mx else 0) + (my - 1 if my else 0)
  return dict(kind=KIND_GENERIC, n_sections=1, num_taps=nb, monic=0, state=1 + near + xr + yr,
              fp64_ops=1 + near + len(far_x) + len(far_y), taps_raise=True)


def _window_cases():
  out = []
  for i, (mx, my) in enumerate(WINDOW_SHAPES):
    for v in (0, 1):
      C = 1 + i % 2 if v == 0 else WINDOW_LARGE_C[i]
      far_x, far_y = FAR_X[(i + v) % 4], FAR_Y[(i + 2 * v) % 4]
      rng = _rng(21, i, v)
      bank = [window_channel(rng, NEAR[mx], NEAR_Y[my], far_x, far_y, 1.0 if c == 0 else 0.6) for c in range(C)]
      nb = max(len(ch[0][0]) for ch in bank)
      out.append(Case("window-mx%d-my%d-C%d" % (mx, my, C), "window", bank, _window_expect(mx, my, far_x, far_y, nb),
                      S=37 if v else 40, T=301, seed=True, splits=[5, 13, 1, 77], coef="small" if v == 0 else "large"))
  # 112 channels run on the window kernel; 113 do not fit its parameter block and fall back to the generic kernel
  for C in (112, 113):
    rng = _rng(22, C)
    bank = [window_channel(rng, [1, 2], [1, 2, 3], [], [], 1.0 if c == 0 else 0.7) for c in range(C)]
    if C == 112:
      exp = _window_expect(4, 4, [], [], 3)
    else:
      exp = dict(kind=KIND_GENERIC, n_sections=1, num_taps=3, monic=0, state=1 + 2 + 4, fp64_ops=3 + 3, taps_raise=False)
    out.append(Case("window-boundary-C%d" % C, "window" if C == 112 else "generic", bank, exp, S=5, T=203, seed=True,
                    splits=[9]))
  return out


def _generic_cases():
  out = []
  rng = _rng(31)
  # two sections: an order-4 all-pole section (two pole pairs at radius 0.95) with 2 numerator taps, then a biquad
  bank = []
  for c in range(3):
    p = [0.95 * np.exp(1j * rng.uniform(0.3, 2.5)) for _ in range(2)]
    a = np.real(np.poly(p + [np.conj(q) for q in p])).tolist()
    bank.append([([0.05, 0.02 * (c + 1)], a), _section(rng, rng.uniform(0.3, 2.5), 0.9, 3)])
  out.append(Case("generic-order4-biquad-C3", "generic", bank,
                  dict(kind=KIND_GENERIC, n_sections=2, num_taps=3, monic=0, state=1 + 1 + 4 + 2 + 2, fp64_ops=2 + 4 + 3 + 2,
                       taps_raise=False), seed=True, splits=[1, 15, 17]))
  # three sections of different shapes per channel, a 10-tap FIR first; channel 3 has only the first section
  bank = []
  for c in range(5):
    fir = ([1.0] + rng.uniform(-0.4, 0.4, 9).tolist(), [1.0, -0.5])
    rest = [_section(rng, rng.uniform(0.3, 2.5), 0.97, 3), ([0.3], [1.0, -0.6, 0.2, -0.1])]
    bank.append([fir] if c == 3 else [fir] + rest)
  out.append(Case("generic-fir10-biquad-order3-C5", "generic", bank,
                  dict(kind=KIND_GENERIC, n_sections=3, num_taps=10, monic=0, state=1 + 16 + 1 + 2 + 2 + 4,
                       fp64_ops=10 + 1 + 3 + 2 + 1 + 3, taps_raise=False), S=33, T=300, seed=True, splits=[4, 4, 31]))
  return out


def _tp_cases():
  """Poles at radius 0.99 ... 0.995: 8 % ... 28 % of a state survives a 256-sample chunk, so every state slot the chunk
  scan carries shows in the output."""
  out = []
  for K in (1, 2, 3, 6, 8):
    out.append(Case("timepar-K%d" % K, "timepar", biquad_bank(600 + K, 3, K, 3, 2, counts="full", radius=(0.99, 0.995)), _biquad_expect(K, 3, 2),
                    S=2, T=100077))
  out.append(Case("timepar-headfir-K1", "timepar", biquad_bank(607, 3, 1, 1, 2, counts="full", head_fir=8, radius=(0.99, 0.995)),
                  _biquad_expect(1, 1, 2, head_fir=True), S=2, T=100077))
  return out


def _psum_cases():
  out = []
  for K in (1, 2, 3, 4, 6, 8):
    for size in ("small", "large"):
      C = 3 if size == "small" else 512 // _stride(K) + 2
      out.append(Case("psum-K%d-%s" % (K, size), "psum", biquad_bank(700 + K, C, K, 3, 2), _biquad_expect(K, 3, 0),
                      S=70, T=1000, plan_kw=dict(parallel=True)))
  return out


ENVELOPE_VARIANTS = [("nb2", 2, False, False), ("nb3", 3, False, False), ("klapuri", 3, False, True),
                     ("headfir-nb1", 1, True, False), ("headfir-nb3", 3, True, False)]


def _envelope_cases():
  out = []
  for j, (name, nb, hf, kl) in enumerate(ENVELOPE_VARIANTS):
    for monic in (0, 1, 2):
      if kl:
        bank = klapuri_bank(800 + monic, 64)
        if monic == 0:
          bank[-1][0] = ([0.0] + bank[-1][0][0][1:], bank[-1][0][1])
        elif monic == 1:
          _scale_gain(bank[0], 1e-33)
      else:
        bank = biquad_bank(800 + 10 * j + monic, 64, 4, nb, monic, counts="full", head_fir=8 if hf else 0)
      mode = ("abs", "squared", "rms")[(j + monic) % 3]
      if monic == 1 and mode == "squared":
        mode = "rms"                                     # the 1e-33 channel's squares are below float32's range
      out.append(Case("envelope-%s-monic%d" % (name, monic), "envelope", bank,
                      _biquad_expect(4, nb, monic, head_fir=hf, klapuri=kl), S=1600, T=336, mode=mode))
  return out


def _launch_mode_cases():
  bank16 = biquad_bank(900, 16, 4, 3, 2, counts="full")
  return [
    Case("tilegroups-K4-C16", "tilegroup", bank16, _biquad_expect(4, 3, 2), S=6400, T=512),
    Case("segmented-K4-C16", "segment", bank16, _biquad_expect(4, 3, 2), S=6400, T=2100),
    Case("tierorder-K4-C16", "tierorder", bank16, _biquad_expect(4, 3, 2), S=37, T=301),
    Case("window-paired-C16", "wpaired", [window_channel(_rng(41, c), [1, 3], [1, 2, 3], [16], [48]) for c in range(16)],
         _window_expect(4, 4, [16], [48], 17), S=3200, T=256),
    Case("freqresp-sumchannels-K4-C5", "misc", biquad_bank(901, 5, 4, 3, 2), _biquad_expect(4, 3, 2), S=7, T=200),
  ]


CASES = _biquad_cases() + _window_cases() + _generic_cases() + _tp_cases() + _psum_cases() + _envelope_cases() + \
        _launch_mode_cases()
BY_ID = {c.id: c for c in CASES}
assert len(BY_ID) == len(CASES)


# --------------------------------------------------------------------------------------------------------------------
# 3. plan routing, on any machine
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_plan_routing(case):
  from audiolazy_b200 import _capi
  plan = _capi.Plan(case.bank, design_only=True, **case.plan_kw)
  e = case.expect
  got = dict(kind=plan.kind, n_sections=plan.n_sections, num_taps=plan.num_taps, monic=plan.monic_mode,
             state=plan.state_doubles_per_recurrence, fp64_ops=plan.fp64_ops)
  assert got == {k: e[k] for k in got}, case.id
  if plan.kind == KIND_GENERIC:
    if e["taps_raise"]:
      with pytest.raises(_capi.NativeError):
        plan.taps()
    else:
      assert len(plan.taps()) == e["fp64_ops"]
  if case.id == "timepar-K8":
    assert plan.state_doubles_per_recurrence == 32      # every slot of the chunk scan's warp
  if "coef" in case.extra and plan.kind == KIND_BIQUAD:
    assert (case.extra["coef"] == "small") == (len(case.bank) * _stride(plan.n_sections) <= 512)


# --------------------------------------------------------------------------------------------------------------------
# GPU side
# --------------------------------------------------------------------------------------------------------------------
@contextlib.contextmanager
def _env(**kv):
  old = {k: os.environ.get(k) for k in kv}
  os.environ.update({k: str(v) for k, v in kv.items()})
  try:
    yield
  finally:
    for k, v in old.items():
      if v is None:
        os.environ.pop(k, None)
      else:
        os.environ[k] = v


class Gpu(object):
  def __init__(self):
    import torch
    from audiolazy_b200 import _capi
    self.torch, self.capi, self.dev = torch, _capi, torch.device("cuda:0")

  def stream(self):
    return self.torch.cuda.current_stream().cuda_stream

  def run(self, plan, x, xinit=None, yinit=None, splits=None, engine="tma", state_out=False):
    """``x`` [S][T] through ``plan``; rows padded to a multiple of 4 samples, plus 8.  engine "tma": 16-byte aligned
    rows (the TMA engine); "cpasync": the same rows with ALZ_NO_TMA=1; "unaligned": base pointers one float off 16
    bytes.  The output buffer starts out as SENTINEL words: every word outside y[S][C][:T] must keep it, and none inside
    may (the 8 extra samples of each row are where a store past the row's end would land; the stride stays a multiple
    of 4, so the TMA and vector store paths stay eligible)."""
    torch = self.torch
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    S, T = x.shape
    C = plan.n_channels
    stride = (T + 3) // 4 * 4 + 8
    off = 1 if engine == "unaligned" else 0
    xb = torch.zeros(S * stride + 4, dtype=torch.float32, device=self.dev)
    xb[off:off + S * stride].view(S, stride)[:, :T] = torch.from_numpy(x).to(self.dev)
    yb = torch.full((S * C * stride + 4,), SENTINEL, dtype=torch.int32, device=self.dev).view(torch.float32)
    st = torch.empty(max(1, plan.state_doubles(S)), dtype=torch.float64, device=self.dev)
    cur = self.stream()
    plan.state_init(st.data_ptr(), S, xinit, yinit, cur)
    with _env(ALZ_NO_TMA=1 if engine == "cpasync" else 0):
      t0 = 0
      for n in list(splits or []) + [T - sum(splits or [])]:      # the last block takes what the splits leave
        plan.apply(xb.data_ptr() + 4 * (off + t0), yb.data_ptr() + 4 * (off + t0), st.data_ptr(), S, n, stride, stride, cur)
        t0 += n
      self.torch.cuda.synchronize()
    check_sentinels(yb, off, (S, C, stride), T)
    y = yb[off:off + S * C * stride].view(S, C, stride)[:, :, :T].cpu().numpy()
    return (y, st.cpu().numpy()) if state_out else y


SENTINEL = 0x7FC0DEAD                                 # a NaN no kernel produces


def check_sentinels(buf, off, shape, T):
  """``buf``: the whole float32 output buffer; ``shape`` rows of it from word ``off`` on, of which ``[..., :T]`` were
  written.  Every other word of the buffer must hold SENTINEL, and no written one may."""
  import torch
  w = buf.view(torch.int32)
  n = int(np.prod(shape))
  rows = w[off:off + n].view(*shape)
  outside = torch.cat([w[:off], w[off + n:], rows[..., T:].reshape(-1)])
  bad = int((outside != SENTINEL).sum())
  assert bad == 0, "%d words outside the output rows were written" % bad
  left = int((rows[..., :T] == SENTINEL).sum())
  assert left == 0, "%d samples of the output rows were never written" % left


def _signal(case, S=None, T=None):
  return _rng(51, CASES.index(case)).uniform(-1, 1, (S or case.S, T or case.T)).astype(np.float32)


def _seeds(case, plan):
  """float32-representable histories: oracle layout [C][KM][h] and the plan's [C][n_sections][depth]."""
  if not case.seed:
    return None, None, None, None
  C = len(case.bank)
  KM = max(len(ch) for ch in case.bank)
  rng = _rng(52, CASES.index(case))
  xo = np.zeros((C, KM, max(plan.xd, 1)))
  yo = np.zeros((C, KM, max(plan.yd, 1)))
  xo[:, :, :plan.xd] = rng.uniform(-0.5, 0.5, (C, KM, plan.xd)).astype(np.float32)
  yo[:, :, :plan.yd] = rng.uniform(-0.5, 0.5, (C, KM, plan.yd)).astype(np.float32)
  xg = np.zeros((C, plan.n_sections, plan.xd))
  yg = np.zeros((C, plan.n_sections, plan.yd))
  xg[:, :KM] = xo[:, :, :plan.xd]
  yg[:, :KM] = yo[:, :, :plan.yd]
  return xo, yo, xg, yg


#: cases that need more than the default bar, and why
WIDER = {
  # narrowband cascades (8 near-equal pole pairs; klapuri's four equal ones): rounding x * G to float32 before a float64
  # filter on the host already gives 2.6e-7 ... 2.8e-7 on some rows, so the input-side gain itself exceeds 2.5e-7
  "klapuri-monic2-C30": dict(gain_in=3.5e-7), "biquad-K8-C12": dict(gain_in=3.5e-7),
  "biquad-K8-C90": dict(gain_in=3.5e-7),
  # one float32-tier channel measured 3.4e-6 here (its probe: <= 2.5e-6): the tier keeps the 1e-5 bar, not a 3x margin
  "biquad-K6-kmax5-nb2-monic0-small": dict(tier1=1e-5),
}


def _row_tol(plan, case):
  """Per-channel tolerance from the plan's precision tiers."""
  if plan.kind != KIND_BIQUAD:
    return np.full(plan.n_channels, WINDOW)
  tier, _ = plan.tiers()
  wide = WIDER.get(case.id, {})
  t0 = wide.get("gain_in", TIER0_GAIN_IN) if plan.monic_mode == 2 else TIER0
  return np.where(tier == 1, wide.get("tier1", TIER1), t0)


def _row_err(y, ref):
  y = np.asarray(y, dtype=np.float64)
  num = np.max(np.abs(y - ref), axis=-1)
  den = np.max(np.abs(ref), axis=-1)
  return num / np.where(den == 0, 1.0, den)


def _check_rows(y, ref, tol, what):
  err = _row_err(y, ref)                                   # [S][C]
  bad = np.argwhere(err > tol[None, :])
  s, c = np.unravel_index(np.argmax(err / tol[None, :]), err.shape)
  assert bad.size == 0, "%s: %d rows over tolerance, worst: stream %d channel %d at %.3g (its bar %.3g)" % (
    what, len(bad), s, c, err[s, c], tol[c])


def _plan(gpu, case, **env):
  with _env(**env):
    return gpu.capi.Plan(case.bank, **case.plan_kw)


#: ALZ_LOG_LAUNCH lines: (tile group, segments, segment length, store path, chunks per stream) of a TMA bank launch;
#: (warps, tiles moved together) of a TMA window launch
BANK_LOG = re.compile(r"alz bank launch: \d+ warps, tile group (\d+), .* (\d+) segment\(s\) of (\d+) samples, "
                      r"(vector|TMA) stores, (\d+) chunks per stream")
WINDOW_LOG = re.compile(r"alz window launch: (\d+) warps, paired (\d+)")


def logged(capfd, fn, pattern=BANK_LOG):
  """``fn()`` under ALZ_LOG_LAUNCH=1: (its result, the fields of every launch line ``pattern`` matches).  Launches on
  the cp.async engine log nothing."""
  capfd.readouterr()
  with _env(ALZ_LOG_LAUNCH=1):
    out = fn()
  fields = [pattern.search(l) for l in capfd.readouterr().err.splitlines()]
  return out, [tuple(v if v in ("vector", "TMA") else int(v) for v in m.groups()) for m in fields if m]


def bits(a):
  """float32 / float64 array -> its words, for bit-for-bit comparisons (NaN included)."""
  a = np.ascontiguousarray(a)
  return a.view(np.int32 if a.dtype == np.float32 else np.int64)


#: tile group forced at plan creation (ALZ_TILE_GROUP) and ALZ_STORE_PATH: the launch modes of full-machine launches
TILE_GROUP_RUNS = [(2, "vec"), (4, "vec"), (4, "tma")]


def store_path(plan, group, path):
  """The store path a TMA bank launch of ``plan`` takes at tile group ``group``: warp-wide vector stores at group 4 on
  the default path, except in the head-FIR instantiations (NB0 = 8), which leave the vector path out."""
  return "vector" if group == 4 and path == "vec" and plan.num_taps != 8 else "TMA"


def run_tile_groups(gpu, case, x, xg, yg, want, capfd):
  """The case at tile groups 2 and 4 and on both store paths of group 4, whole and in its block splits: the bits and
  the final state of the group-1 run ``want``, and every logged launch at the forced group and on its store path."""
  y1, st1 = want
  for group, path in TILE_GROUP_RUNS:
    plan = _plan(gpu, case, ALZ_TILE_GROUP=group, ALZ_STORE_PATH=path)
    for splits in [None] + ([case.splits] if case.splits else []):
      what = "%s, tile group %d, %s stores, splits %s" % (case.id, group, path, splits)
      (y, st), log = logged(capfd, lambda: gpu.run(plan, x, xg, yg, splits=splits, state_out=True))
      assert log, "%s: no TMA bank launch logged" % what
      assert all(g == group and p == store_path(plan, group, path) for g, _, _, p, _ in log), (what, log)
      assert np.array_equal(bits(y), bits(y1)), "%s: output differs from tile group 1" % what
      assert np.array_equal(bits(st), bits(st1)), "%s: final state differs from tile group 1" % what


#: warps per SM of the window kernel (kWinWarpsPerSm): a launch of at least this many warps per SM moves tiles in pairs
WINDOW_WARPS_PER_SM = 12


def run_window_paired(gpu, plan, case, x, xg, yg, want, capfd):
  """The case's rows tiled up to a launch big enough for paired tiles: every replica row gives the small run's bits
  and final state."""
  y1, st1 = want
  C, d = plan.n_channels, plan.state_doubles_per_recurrence
  sm = gpu.torch.cuda.get_device_properties(gpu.dev).multi_processor_count
  S = -(-sm * WINDOW_WARPS_PER_SM // C) * 32 + 5
  rows = np.arange(S) % case.S
  (y, st), log = logged(capfd, lambda: gpu.run(plan, x[rows], xg, yg, state_out=True), WINDOW_LOG)
  assert log and all(p == 2 for _, p in log), "%s: %d streams not paired: %s" % (case.id, S, log)
  assert np.array_equal(bits(y), bits(y1)[rows]), "%s: paired rows differ from the small run" % case.id
  assert np.array_equal(bits(st).reshape(d, C, S), bits(st1).reshape(d, C, case.S)[:, :, rows]), \
    "%s: paired final states differ from the small run" % case.id


def run_filter_case(gpu, case, capfd):
  """biquad / window / generic: three engines agree bit for bit, block splits are bit-exact, the oracle agrees.  The
  biquad kernels give the same bits at tile groups 2 and 4 on both store paths, the window kernels in paired mode."""
  plan = _plan(gpu, case)
  assert (plan.kind, plan.n_sections, plan.state_doubles_per_recurrence) == \
         (case.expect["kind"], case.expect["n_sections"], case.expect["state"])
  x = _signal(case)
  xo, yo, xg, yg = _seeds(case, plan)
  (y, st), log = logged(capfd, lambda: gpu.run(plan, x, xg, yg, state_out=True),
                        WINDOW_LOG if case.family == "window" else BANK_LOG)
  assert np.array_equal(gpu.run(plan, x, xg, yg, engine="cpasync"), y), "cp.async engine differs from TMA"
  assert np.array_equal(gpu.run(plan, x, xg, yg, engine="unaligned"), y), "unaligned rows differ from TMA"
  if case.splits:
    assert np.array_equal(gpu.run(plan, x, xg, yg, splits=case.splits), y), "block splits are not bit-exact"
  if case.family == "biquad":
    assert log and all(l[0] == 1 for l in log), log      # the reference of the tile-group runs: one tile at a time
    run_tile_groups(gpu, case, x, xg, yg, (y, st), capfd)
  elif case.family == "window":
    assert log and all(p == 1 for _, p in log), log
    run_window_paired(gpu, plan, case, x, xg, yg, (y, st), capfd)
  _check_rows(y, oracle.bank_apply(x, case.bank, xinit=xo, yinit=yo), _row_tol(plan, case), case.id)


def run_timepar_case(gpu, case, capfd):
  """Time-parallel against sequential evaluation and the oracle; then at tile group 4 on both store paths, which must
  give the default run's bits: the chunked launch (virtual streams) on the group's store path, and the T - P L samples
  left over (1 mod 4: a lane-written ragged tile) in a sequential launch of their own."""
  plan = _plan(gpu, case)
  x = _signal(case)
  before = gpu.capi.launch_count()
  fast = gpu.run(plan, x)
  assert gpu.capi.launch_count() - before >= 4            # zero-state pass, scan, replay (+ the basis run): time-parallel
  with _env(ALZ_NO_TIME_PARALLEL=1):
    slow = gpu.run(plan, x)
  assert rel_err(fast, slow) <= 3e-6
  assert rel_err(fast[:1], oracle.bank_apply(x[:1], case.bank)) <= 1e-5
  for path in ("vec", "tma"):
    p4 = _plan(gpu, case, ALZ_TILE_GROUP=4, ALZ_STORE_PATH=path)
    y, log = logged(capfd, lambda: gpu.run(p4, x))
    what = "%s, tile group 4, %s stores" % (case.id, path)
    assert log and all(g == 4 and p == store_path(p4, 4, path) for g, _, _, p, _ in log), (what, log)
    chunked = [l for l in log if l[4] > 1]
    assert chunked, (what, log)
    _, _, L, _, P = chunked[-1]
    tail = log[-1]
    assert tail[4] == 1 and tail[2] == case.T - P * L and tail[2] % 4 == case.T % 4 == 1, (what, log)
    assert np.array_equal(bits(y), bits(fast)), "%s: output differs from the default tile group" % what


def run_psum_case(gpu, case, capfd):
  torch = gpu.torch
  plan = _plan(gpu, case)
  assert plan.kind == KIND_BIQUAD and plan.n_fp32_channels == 0 and plan.monic_mode == 0
  x = _signal(case)
  S, T = x.shape
  ch = oracle.bank_apply(x, case.bank)
  want = ch[:, 0].copy()
  for c in range(1, len(case.bank)):
    want = want + ch[:, c]
  xd = torch.from_numpy(x).to(gpu.dev)
  out = torch.full((S, T), float("nan"), dtype=torch.float32, device=gpu.dev)
  st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device=gpu.dev)
  plan.apply_sum(xd.data_ptr(), out.data_ptr(), st.data_ptr(), S, T, T, T, gpu.stream())
  torch.cuda.synchronize()
  assert rel_err(out.cpu().numpy(), want) <= TIER0_GAIN_IN
  out2 = torch.empty_like(out)
  st.zero_()
  for t0, n in ((0, 8), (8, 92), (100, T - 100)):
    plan.apply_sum(xd.data_ptr() + 4 * t0, out2.data_ptr() + 4 * t0, st.data_ptr(), S, n, T, T, gpu.stream())
  torch.cuda.synchronize()
  assert torch.equal(out, out2)


def run_envelope_case(gpu, case, capfd):
  """The fused envelope consumer in paired mode (64 channels x 1600 streams >= 132 SMs x 24 warps) against the plan's own
  float32 bank output, rectified, lowpassed in float64 and decimated by torch; state carried over two calls."""
  torch = gpu.torch
  plan = _plan(gpu, case)
  S, T, C = case.S, case.T, plan.n_channels
  x = _signal(case)
  xd = torch.from_numpy(x).to(gpu.dev)
  y = torch.empty((S, C, T), dtype=torch.float32, device=gpu.dev)
  st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device=gpu.dev)
  plan.apply(xd.data_ptr(), y.data_ptr(), st.data_ptr(), S, T, T, T, gpu.stream())
  rows = [0, 31, 32, 799, S - 1]
  _check_rows(y[rows].cpu().numpy(), oracle.bank_apply(x[rows], case.bank), _row_tol(plan, case), case.id + " bank")
  g, R = 0.02, 0.98
  y64 = y.double()
  r = y64.abs() if case.extra["mode"] == "abs" else y64 * y64
  e = torch.empty_like(r)
  acc = torch.zeros_like(r[:, :, 0])
  for n in range(T):
    acc = g * r[:, :, n] + R * acc
    e[:, :, n] = acc
  if case.extra["mode"] == "rms":
    e = e.sqrt()
  del y, y64, r
  for decim in (1, 7, 48):
    Td = T // decim
    want = e[:, :, decim - 1::decim].cpu().numpy()
    outs = []
    for split in (None, (T // 2) // decim * decim):
      env = torch.full((S, C, Td), float("nan"), dtype=torch.float32, device=gpu.dev)
      st.zero_()
      es = torch.zeros(S * C, dtype=torch.float64, device=gpu.dev)
      # decim 48: the second block's env pointer is 12 bytes past a 16-byte boundary, which the call once refused
      parts = [(0, T)] if split is None else [(0, split), (split, T - split)]
      for t0, n in parts:
        plan.apply_envelope(xd.data_ptr() + 4 * t0, env.data_ptr() + 4 * (t0 // decim), st.data_ptr(), es.data_ptr(), S, n,
                            T, Td, decim, case.extra["mode"], g, R, gpu.stream())
      torch.cuda.synchronize()
      outs.append(env.cpu().numpy())
    assert np.array_equal(outs[0], outs[1]), "envelope state carry is not bit-exact (decim %d)" % decim
    assert rel_err(outs[0], want) <= 1e-7, decim


def run_tilegroup_case(gpu, case, capfd):
  x = _signal(case)
  ys = []
  for grp in (1, 2, 4):
    plan = _plan(gpu, case, ALZ_TILE_GROUP=grp)
    ys.append(gpu.run(plan, x))
  ys.append(gpu.run(plan, x, engine="cpasync"))
  for y in ys[1:]:
    assert np.array_equal(y, ys[0])
  rows = [0, 31, 32, 3200, case.S - 1]
  _check_rows(ys[0][rows], oracle.bank_apply(x[rows], case.bank), _row_tol(plan, case), case.id)


def run_segment_case(gpu, case, capfd):
  plan = _plan(gpu, case)
  x = _signal(case)
  y, st = gpu.run(plan, x, state_out=True)
  with _env(ALZ_NO_SEGMENT=1):
    y2, st2 = gpu.run(plan, x, state_out=True)
  assert np.array_equal(y, y2) and np.array_equal(st, st2)
  rows = [0, 33, 4001, case.S - 1]
  _check_rows(y[rows], oracle.bank_apply(x[rows], case.bank), _row_tol(plan, case), case.id)


def run_tierorder_case(gpu, case, capfd):
  x = _signal(case)
  ys = []
  for order in (0, 1, 2):
    plan = _plan(gpu, case, ALZ_TIER_ORDER=order)
    assert 0 < plan.n_fp32_channels < plan.n_channels         # both tiers present: the orders differ
    ys.append(gpu.run(plan, x))
  assert np.array_equal(ys[0], ys[1]) and np.array_equal(ys[0], ys[2])
  _check_rows(ys[0], oracle.bank_apply(x, case.bank), _row_tol(plan, case), case.id)


def run_wpaired_case(gpu, case, capfd):
  """16 channels x 3200 streams = 1600 warps >= 132 SMs x 12: the window TMA kernel in paired mode."""
  plan = _plan(gpu, case)
  x = _signal(case)
  y = gpu.run(plan, x)
  rows = [0, 31, 32, 1601, case.S - 1]
  _check_rows(y[rows], oracle.bank_apply(x[rows], case.bank), _row_tol(plan, case), case.id)


def run_misc_case(gpu, case, capfd):
  """alz_freq_response_f64 against numpy in float64; alz_sum_channels_f32 against a left-to-right float64 sum."""
  torch = gpu.torch
  plan = _plan(gpu, case)
  w = np.linspace(0.0, np.pi, 257)
  wd = torch.from_numpy(w).to(gpu.dev)
  out = torch.empty((plan.n_channels, len(w), 2), dtype=torch.float64, device=gpu.dev)
  plan.freq_response(wd.data_ptr(), out.data_ptr(), len(w), gpu.stream())
  torch.cuda.synchronize()
  H = out.cpu().numpy()
  got = H[..., 0] + 1j * H[..., 1]
  for c, ch in enumerate(case.bank):
    want = np.ones(len(w), dtype=complex)
    for b, a in ch:
      z = np.exp(-1j * np.outer(w, np.arange(max(len(b), len(a)))))
      want *= (z[:, :len(b)] @ np.asarray(b)) / (z[:, :len(a)] @ np.asarray(a))
    assert np.max(np.abs(got[c] - want)) <= 1e-12 * np.max(np.abs(want))
  x = _signal(case)
  y = gpu.run(plan, x)
  yd = torch.from_numpy(y).to(gpu.dev)
  S, C, T = y.shape
  s = torch.empty((S, T), dtype=torch.float32, device=gpu.dev)
  gpu.capi.sum_channels(yd.data_ptr(), s.data_ptr(), S, C, T, T, T, gpu.stream())
  torch.cuda.synchronize()
  acc = y[:, 0].astype(np.float64)
  for c in range(1, C):
    acc = acc + y[:, c]
  assert np.array_equal(s.cpu().numpy(), acc.astype(np.float32))


RUNNERS = {"biquad": run_filter_case, "window": run_filter_case, "generic": run_filter_case, "timepar": run_timepar_case,
           "psum": run_psum_case, "envelope": run_envelope_case, "tilegroup": run_tilegroup_case,
           "segment": run_segment_case, "tierorder": run_tierorder_case, "wpaired": run_wpaired_case, "misc": run_misc_case}

_RAN = set()


@pytest.fixture(scope="module")
def gpu():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return Gpu()


@pytest.fixture(scope="module")
def launches(gpu):
  """One profiler session over the whole matrix: the kernels it launches, by name (CUDA activity records)."""
  from torch.profiler import ProfilerActivity, profile
  prof = profile(activities=[ProfilerActivity.CUDA], acc_events=True)
  prof.start()
  rec = {"prof": prof, "names": None}
  yield rec
  if rec["names"] is None:
    prof.stop()


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_kernel_matrix(gpu, launches, capfd, case):
  _RAN.add(case.id)
  RUNNERS[case.family](gpu, case, capfd)


# --------------------------------------------------------------------------------------------------------------------
# 2. launch coverage
# --------------------------------------------------------------------------------------------------------------------
#: kernels of the library the matrix is allowed not to launch, with the reason (kept empty: every kernel is reached)
NOT_LAUNCHED = {}


def kernel_key(name):
  """Demangled kernel name -> ``name<template args>`` without spaces (None if it is not one of the library's)."""
  name = name.strip()
  if name.startswith("void "):
    name = name[5:]
  m = re.match(r"(alz_\w+)(<[^()]*>)?", name)
  return m.group(1) + (m.group(2) or "").replace(" ", "") if m else None


def library_kernels():
  from audiolazy_b200 import _build
  keys = {kernel_key(n) for n in compiled_kernels(_build.LIB_PATH)}
  assert None not in keys
  return keys


@pytest.mark.gpu
def test_every_kernel_is_launched(gpu, launches, capfd):
  """Runs whatever part of the matrix did not run in this session, then compares the kernels the profiler saw launch
  with the kernels compiled into the library."""
  built = library_kernels()
  for case in CASES:
    if case.id not in _RAN:
      _RAN.add(case.id)
      try:
        RUNNERS[case.family](gpu, case, capfd)
      except AssertionError:
        pass                       # reported by test_kernel_matrix; only the launches matter here
  gpu.torch.cuda.synchronize()
  launches["prof"].stop()
  names = {kernel_key(e.name) for e in launches["prof"].events() if e.name}
  launches["names"] = names - {None}
  assert launches["names"], "the profiler recorded no kernel of the library"
  unknown = launches["names"] - built
  assert not unknown, "launched kernels not found in the library: %s" % sorted(unknown)
  missing = sorted(built - launches["names"] - set(NOT_LAUNCHED))
  assert not missing, "%d of %d kernels never launched by the matrix:\n  %s" % (len(missing), len(built), "\n  ".join(missing))
