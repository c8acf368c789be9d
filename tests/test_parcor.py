"""PARCOR on the CPU: the host ``parcor`` / ``parcor_stable`` and the batched form's restatement against the reference's
own outputs (tests/golden/make_parcor.py), the restatement of CPython's ``k ** 2`` against the live interpreter, the
argument checks of ``parcor_batch`` and of the PARCOR library, and the library's SASS."""
import ctypes
import json
import math
import os
import platform
import re
import shutil
import subprocess

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, linear_prediction as lp
from conftest import ROOT
from native_libs import cuobjdump
from parcor_emulation import parcor_row, same_float

CASES = json.load(open(os.path.join(ROOT, "tests", "golden", "parcor_cases.json")))["cases"]
ERRORS = {0: None, 1: "ParCorError", 2: "OverflowError"}


def test_goldens_cover_the_issue_rows():
  names = {c["name"].rsplit("_", 1)[0] for c in CASES}
  assert {"lpc_noise", "lpc_tone", "lpc_dc", "lpc_impulse", "stable", "unstable", "doctest", "unit_k", "overflow",
          "specials", "zeros", "one", "not_monic", "midpoint"} <= names
  assert sum(c["name"].startswith("midpoint") for c in CASES) >= 300
  assert {c["error"] for c in CASES} == {None, "ParCorError", "OverflowError"}


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_host_parcor_equals_the_reference(case):
  ks, err = [], None
  try:
    for k in ab.parcor(ab.ZFilter(case["row"])):
      ks.append(k)
  except (ab.ParCorError, OverflowError) as exc:
    err = type(exc).__name__
  assert err == case["error"]
  assert len(ks) == len(case["k"]) and all(map(same_float, ks, case["k"])), (ks, case["k"])
  assert ab.parcor_stable(1 / ab.ZFilter(case["row"])) == case["stable"]


@pytest.mark.parametrize("case", CASES, ids=[c["name"] for c in CASES])
def test_emulation_equals_the_reference(case):
  ks, failed, stable = parcor_row(case["row"])
  if failed == 3:
    assert not case["row"][0] == 1.0
    return
  assert ERRORS[failed] == case["error"] and stable == case["stable"]
  assert len(ks) == len(case["k"]) and all(map(same_float, ks, case["k"]))


#: the reference's levinson_durbin([1, 2, 3, 4, 5, 3, 2, 1]), the row of its parcor doctest
DOCTEST_ROW = [1.0, -0.2750000000000007, -0.27499999999999913, -0.4125000000000002, 1.5, -0.9125000000000005,
               -0.274999999999999, -0.27500000000000036]


def test_doctest_row():
  assert list(ab.parcor(ab.ZFilter(DOCTEST_ROW))) == [-0.27500000000000036, -0.3793103448275855, -1.4166666666666663,
                                   -0.2000000000000004, -0.25000000000000006, -0.3333333333333336, -2.0000000000000013]


def test_overflow_propagates_after_its_k():
  gen = ab.parcor(ab.ZFilter([1.0, 3.0, 1e200]))
  assert next(gen) == 1e200
  with pytest.raises(OverflowError):
    next(gen)
  assert ab.parcor_stable(1 / ab.ZFilter([1.0, 3.0, 1e200])) is False


# --- the pow restatement ---------------------------------------------------------------------------------------------

_SHIM = r"""
#include "alz_pow2.h"
void pow2_many(const double* k, double* out, unsigned char* ovf, long n) {
  for (long i = 0; i < n; ++i) { int o; out[i] = alz_py_pow2(k[i], &o); ovf[i] = (unsigned char)o; }
}
"""


def _glibc_fma_host():
  if platform.machine() != "x86_64" or platform.libc_ver() != ("glibc", "2.39"):
    return False
  try:
    flags = open("/proc/cpuinfo").read()
  except OSError:
    return False
  return re.search(r"\bfma\b", flags) is not None and re.search(r"\bavx2\b", flags) is not None


def _near_midpoint(rng, n):
  """Doubles in (-1, 1) whose exact square lies within 2**-8 ulp of a rounding midpoint."""
  out = []
  while len(out) < n:
    for k in rng.uniform(-1, 1, 4096).tolist():
      m, _ = math.frexp(abs(k))
      mi = int(m * 2 ** 53)
      sq = mi * mi
      drop = sq.bit_length() - 53
      if abs((sq & ((1 << drop) - 1)) - (1 << (drop - 1))) * 256 < (1 << drop):
        out.append(k)
  return np.array(out[:n])


def test_pow_restatement_equals_live_pow(tmp_path):
  """alz_pow2.h compiled for the host equals this interpreter's `k ** 2` (OverflowError included) on 10**7 values:
  uniform in (-1, 1), random bit patterns (every exponent, subnormals, NaN, inf) and squares near a midpoint."""
  if not _glibc_fma_host():
    pytest.skip("the host's libm is not glibc 2.39 with FMA: its pow may round differently; the goldens still hold")
  cc = shutil.which("cc") or shutil.which("gcc")
  if cc is None:
    pytest.skip("no C compiler")
  src = tmp_path / "shim.c"
  src.write_text(_SHIM)
  so = tmp_path / "shim.so"
  subprocess.check_call([cc, "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-I",
                         os.path.join(ROOT, "audiolazy_b200", "csrc_parcor"), "-o", str(so), str(src), "-lm"])
  shim = ctypes.CDLL(str(so))
  rng = np.random.default_rng(7)
  k = np.concatenate([rng.uniform(-1, 1, 5_000_000),
                      rng.integers(0, 2 ** 64, 4_990_000, dtype=np.uint64).view(np.float64),
                      _near_midpoint(rng, 10_000)])
  out = np.empty_like(k)
  ovf = np.empty(k.shape, np.uint8)
  shim.pow2_many(k.ctypes.data_as(ctypes.c_void_p), out.ctypes.data_as(ctypes.c_void_p),
                 ovf.ctypes.data_as(ctypes.c_void_p), ctypes.c_long(k.size))
  want = np.empty_like(k)
  want_ovf = np.zeros(k.shape, np.uint8)
  for i, x in enumerate(k.tolist()):
    try:
      want[i] = x ** 2
    except OverflowError:
      want[i] = math.inf
      want_ovf[i] = 1
  assert np.array_equal(ovf, want_ovf)
  nan = np.isnan(want)
  assert np.array_equal(np.isnan(out), nan)
  assert np.array_equal(out[~nan].view(np.uint64), want[~nan].view(np.uint64))
  assert np.count_nonzero(k[~nan] * k[~nan] != want[~nan]) > 1000       # the set does reach pow's misroundings


# --- arguments and the library ---------------------------------------------------------------------------------------

def test_parcor_batch_argument_errors():
  torch = pytest.importorskip("torch")
  with pytest.raises(TypeError):
    ab.parcor_batch([[1.0, .5]])
  with pytest.raises(TypeError):
    ab.parcor_batch(torch.zeros((2, 3), dtype=torch.float32))
  with pytest.raises(ValueError):
    ab.parcor_batch(torch.zeros((2, 0), dtype=torch.float64))
  with pytest.raises(ValueError):
    ab.parcor_batch(torch.zeros((2, 66), dtype=torch.float64))
  with pytest.raises(ValueError):
    ab.parcor_batch(torch.tensor(1.0, dtype=torch.float64))
  with pytest.raises(ValueError, match="CUDA"):
    ab.parcor_batch(torch.zeros((2, 3), dtype=torch.float64))


def test_library_checks_without_a_device():
  L = lp.PARCOR_LIB.load()
  assert L.alz_parcor_f64(None, 1, 1, 0, None, None, None, None, None) < 0
  assert "L must be" in L.alz_parcor_last_error().decode()
  assert L.alz_parcor_f64(None, 1, 1, 66, None, None, None, None, None) < 0
  assert L.alz_parcor_f64(None, 1, 1, 3, None, None, None, None, None) < 0
  assert "NULL" in L.alz_parcor_last_error().decode()
  assert L.alz_parcor_f64(8, 2, 2, 3, None, None, None, None, None) < 0
  assert "stride" in L.alz_parcor_last_error().decode()
  assert L.alz_parcor_f64(None, 1, 0, 3, None, None, None, None, None) == 0
  with pytest.raises(ValueError, match="L must be"):
    lp.PARCOR_LIB.check(L.alz_parcor_f64(None, 1, 1, 0, None, None, None, None, None))


def test_parcor_kernel_contracts_nothing():
  """Built with -fmad=false: the step-down's products are never contracted into an add.  Each instantiation holds
  the 21 DFMAs alz_pow2.h spells out (the ones glibc's compiled pow executes) and the Newton steps of the correctly
  rounded reciprocal 1 / d, and nothing else fused."""
  sass = subprocess.run([cuobjdump(), "-sass", _build.LIBRARIES["parcor"].path], capture_output=True, text=True).stdout
  functions = re.split(r"\n\s*Function : ", sass)[1:]
  assert len(functions) == 3
  counts = set()
  for body in functions:
    assert "alz_parcor_kernel" in body.split(None, 1)[0]
    assert "MUFU.RCP64H" in body and "DMUL" in body and "DADD" in body
    counts.add(len(re.findall(r"\bDFMA\b", body)))
  assert len(counts) == 1 and 21 <= counts.pop() <= 21 + 20
