"""The oracle and the host-side designs against the reference on inputs beyond the golden
vectors: what the reference answered is stored in tests/golden/reference_cases.json
(tests/golden/make_golden.py; long outputs as SHA-256 digests of their float64 bytes)."""
import hashlib
import json
import os

import numpy as np
import pytest

import oracle
from conftest import GOLDEN, signal


@pytest.fixture(scope="module")
def cases():
  with open(os.path.join(GOLDEN, "reference_cases.json")) as fh:
    return json.load(fh)


def digest(y):
  return hashlib.sha256(np.ascontiguousarray(y, dtype="<f8").tobytes()).hexdigest()


def test_oracle_vs_reference_all_64_channels(cases):
  import audiolazy_b200 as ab
  x = signal(123, 3000)
  for name in ("slaney", "klapuri", "sampled"):
    bank = ab.gammatone_bank(strategy=name)
    got = oracle.bank_apply(x, bank.sections())[0]
    for i, c in enumerate(range(0, 64, 7)):
      assert digest(got[c]) == cases["bank_digests"][name][i], (name, c)


def test_lfilter_grid_like_reference_test(cases):
  """reference tests/test_filters_extdep.py:41-47, through the oracle and the reference."""
  from scipy.signal import lfilter
  assert len(cases["lfilter_grid"]) == 80
  for b, a, data, want in cases["lfilter_grid"]:
    x = np.asarray(data, dtype=np.float32)
    got = oracle.bank_apply(x, [[(b, a)]])[0, 0]
    assert np.array_equal(got, np.asarray(want, dtype=np.float64))
    ref = lfilter(b, a, data)
    assert np.all(np.abs(got - ref) <= 2.0 ** -23 * np.abs(got + ref))   # the reference's almost_eq (32 bits, tol 1)


def test_random_designs_match_reference_bit_for_bit(cases):
  import audiolazy_b200 as ab
  rng = np.random.default_rng(5)
  for want in cases["random_designs"]:
    freq, bw, cutoff = rng.uniform(0.01, 3.0), rng.uniform(1e-3, 0.6), rng.uniform(0.01, 3.1)
    rng.integers(1, 50), rng.integers(1, 50)
    filts = [ab.gammatone.slaney(freq, bw), ab.gammatone.klapuri(freq, bw), ab.gammatone.sampled(freq, bw),
             ab.gammatone.sampled(freq, bw, phase=0.4, eta=5), ab.lowpass.z(cutoff), ab.highpass.pole(cutoff),
             ab.resonator.z_exp(freq, bw)]
    mine = [[(list(map(float, f.numlist)), list(map(float, f.denlist))) for f in
             (filt if isinstance(filt, ab.CascadeFilter) else [filt])] for filt in filts]
    assert hashlib.sha256(repr(mine).encode()).hexdigest() == want, (freq, bw, cutoff)


def test_memory_semantics_vs_reference(cases):
  x = signal(9, 50)
  b, a = [0.3, 0.2, -0.4], [1.5, -0.2, 0.1, 0.05]
  assert len(cases["memory_semantics"]) == 4
  for memory, zero, want in cases["memory_semantics"]:
    got = np.array(oracle.py_section(b, a, x.astype(np.float64).tolist(), memory=memory, zero=zero))
    assert np.array_equal(got, np.asarray(want, dtype=np.float64)), (memory, zero)
