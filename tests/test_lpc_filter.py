"""LpcFilter on the CPU: the kernels' float64 restatement (tests/lpc_filter_emulation.py) against the reference's own
outputs (tests/golden/make_lpc_filter.py), the argument and row-count checks, and the LPC filtering library's SASS."""
import json
import os
import re
import subprocess

import numpy as np
import pytest

import audiolazy_b200 as ab
from audiolazy_b200 import _build, _capi, linear_prediction as lp
from conftest import ROOT
from lpc_filter_emulation import lpc_filter, same_bits
from native_libs import cuobjdump

GOLDEN = np.load(os.path.join(ROOT, "tests", "golden", "lpc_filter_cases.npz"))
META = json.loads(str(GOLDEN["meta"]))


def test_goldens_cover_the_issue_grid():
  assert {m["order"] for m in META} >= {0, 1, 2, 3, 8, 16, 32, 64}
  assert {m["hop"] for m in META} >= {1, 7, 160, 512}
  assert any(m["hop"] > len(GOLDEN["x_%d" % i]) for i, m in enumerate(META))
  for kind in ("analysis", "synthesis"):
    assert {m["order"] for m in META if m["kind"] == kind} >= {0, 1, 2, 3, 8, 16, 32, 64}
  ys = np.concatenate([GOLDEN["y_%d" % i] for i in range(len(META))])
  assert np.isnan(ys).any() and np.isinf(ys).any()            # unstable synthesis overflows, then NaN
  coefs = np.concatenate([GOLDEN["coef_%d" % i].reshape(-1) for i in range(len(META))])
  assert np.isnan(coefs).any() and np.isposinf(coefs).any() and np.isneginf(coefs).any()
  assert (np.signbit(coefs) & (coefs == 0)).any()
  xs = np.concatenate([GOLDEN["x_%d" % i] for i in range(len(META))])
  assert np.isnan(xs).any() and np.isinf(xs).any() and (np.signbit(xs) & (xs == 0)).any()
  assert (np.abs(xs) == np.finfo(np.float32).max).any() and ((xs != 0) & (np.abs(xs) < 1.2e-38)).any()
  assert not all(m["x_f32"] for m in META) and sum(m["x_f32"] for m in META) > len(META) // 2


@pytest.mark.parametrize("i", range(len(META)), ids=[m["name"] for m in META])
def test_emulation_equals_the_reference(i):
  m = META[i]
  x, coef, y = GOLDEN["x_%d" % i], GOLDEN["coef_%d" % i], GOLDEN["y_%d" % i]
  got, _ = lpc_filter(m["kind"], x[None], coef[None], m["hop"])
  assert same_bits(got[0], y)


@pytest.mark.parametrize("kind", ["analysis", "synthesis"])
def test_emulation_blocks_equal_one_call(kind):
  rng = np.random.default_rng(1)
  x = rng.standard_normal((3, 100))
  coef = np.concatenate([np.ones((3, 15, 1)), rng.standard_normal((3, 15, 5)) * .3], axis=2)
  want, _ = lpc_filter(kind, x, coef, 7)
  got, hist, n = [], None, 0
  for cut in (0, 1, 3, 3, 10, 40, 43):
    r0 = n // 7
    y, hist = lpc_filter(kind, x[:, n:n + cut], coef[:, r0:], 7, n, hist)
    got.append(y)
    n += cut
  assert n == 100 and same_bits(np.concatenate(got, axis=1), want)


def test_readme_example():
  x = np.array([[-1., 0., 1., 0.] * 50])
  row = np.array([[[1., 0., .5, 0., -.5]]])
  res, _ = lpc_filter("analysis", x, row, 200)
  assert res[0, :6].tolist() == [-1.0, 0.0, 0.5, 0.0, 0.0, 0.0]
  back, _ = lpc_filter("synthesis", res, row, 200)
  assert same_bits(back, x)


# --- arguments ------------------------------------------------------------------------------------------------------

def test_constructor_errors():
  with pytest.raises(ValueError):
    ab.LpcFilter(65, 10)
  with pytest.raises(ValueError):
    ab.LpcFilter(-1, 10)
  with pytest.raises(TypeError):
    ab.LpcFilter(2.0, 10)
  with pytest.raises(ValueError):
    ab.LpcFilter(2, 0)
  with pytest.raises(ValueError):
    ab.LpcFilter(2, 10, kind="lattice")
  with pytest.raises(ValueError):
    ab.LpcFilter(2, 10, dtype="float16")
  f = ab.LpcFilter(64, 10, "synthesis")
  assert (f.order, f.hop, f.kind) == (64, 10, "synthesis")
  assert ab.LpcFilter(0, 1).order == 0


def test_n_rows():
  f = ab.LpcFilter(4, 10)
  assert f.n_rows(0, 0) == 0 and f.n_rows(7, 0) == 0
  assert f.n_rows(0, 1) == 1 and f.n_rows(0, 10) == 1 and f.n_rows(0, 11) == 2
  assert f.n_rows(9, 1) == 1 and f.n_rows(9, 2) == 2 and f.n_rows(10, 10) == 1 and f.n_rows(5, 30) == 4
  L = lp.LPCFILT_LIB.load()
  for consumed in range(0, 25):
    for T in range(0, 25):
      assert L.alz_lpcfilt_rows(consumed, T, 10) == f.n_rows(consumed, T)
  assert L.alz_lpcfilt_rows(0, 5, 0) < 0 and "hop" in L.alz_lpcfilt_last_error().decode()


def test_apply_needs_a_device():
  torch = pytest.importorskip("torch")
  if torch.cuda.is_available():
    pytest.skip("a CUDA device is present")
  with pytest.raises(_capi.NativeError):
    ab.LpcFilter(2, 4).apply(torch.zeros((1, 8)), torch.zeros((1, 2, 3), dtype=torch.float64))


def test_library_checks_without_a_device():
  L = lp.LPCFILT_LIB.load()
  args = dict(x=None, xt=0, xs=8, out=None, ot=1, os=8, coef=None, crs=3, ccs=3, F=2, state=None, S=1, T=8, C=0,
              order=2, hop=4, kind=0, stream=None)

  def call(**kw):
    a = dict(args, **kw)
    return L.alz_lpcfilt_apply(*a.values())

  assert call(kind=2) < 0 and "kind" in L.alz_lpcfilt_last_error().decode()
  assert call(order=65) < 0 and "order" in L.alz_lpcfilt_last_error().decode()
  assert call(hop=0) < 0 and "hop" in L.alz_lpcfilt_last_error().decode()
  assert call(xt=3) < 0 and "dtype" in L.alz_lpcfilt_last_error().decode()
  assert call(F=1) < 0 and "needs 2" in L.alz_lpcfilt_last_error().decode()
  assert call(C=3, F=2) < 0 and "needs 3" in L.alz_lpcfilt_last_error().decode()
  assert call() < 0 and "NULL" in L.alz_lpcfilt_last_error().decode()
  assert call(x=8, out=8, coef=8, state=8, crs=2) < 0 and "row stride" in L.alz_lpcfilt_last_error().decode()
  assert call(x=8, out=8, coef=8, state=8, S=2, xs=4) < 0 and "stride" in L.alz_lpcfilt_last_error().decode()
  assert call(x=8, out=8, coef=8, state=8, ccs=-1) < 0 and "stream stride" in L.alz_lpcfilt_last_error().decode()
  assert call(x=4, out=8, coef=8, state=8, xt=1) < 0 and "misaligned" in L.alz_lpcfilt_last_error().decode()
  assert call(T=0, F=0) == 0 and call(S=0) == 0
  assert L.alz_lpcfilt_state_bytes(3, 16) == 3 * 8 * 16 and L.alz_lpcfilt_state_bytes(3, 0) == 0
  assert L.alz_lpcfilt_state_bytes(-1, 2) < 0 and L.alz_lpcfilt_state_bytes(1, 65) < 0
  assert L.alz_lpcfilt_state_init(None, 1, 0, None) == 0
  assert L.alz_lpcfilt_state_init(None, 1, 2, None) < 0 and "NULL" in L.alz_lpcfilt_last_error().decode()
  with pytest.raises(ValueError, match="kind"):
    lp.LPCFILT_LIB.check(call(kind=2))


# --- the library ----------------------------------------------------------------------------------------------------

def test_lpcfilt_kernels_contract_nothing():
  """Built with -fmad=false: no product is fused into an addition, in any of the 42 kernels (analysis and the
  ring-buffer synthesis for each input and output dtype, the register synthesis for each order 1 .. 32, and the
  analysis state commit for each input dtype)."""
  sass = subprocess.run([cuobjdump(), "-sass", _build.LIBRARIES["lpcfilt"].path], capture_output=True, text=True).stdout
  functions = re.split(r"\n\s*Function : ", sass)[1:]
  assert len(functions) == 42
  names = [body.split(None, 1)[0] for body in functions]
  assert sum("alz_lpcfilt_analysis_kernel" in n for n in names) == 4
  assert sum("alz_lpcfilt_synthesis_kernel" in n for n in names) == 4
  assert sum("alz_lpcfilt_synthesis_reg_kernel" in n for n in names) == 32
  assert sum("alz_lpcfilt_commit_kernel" in n for n in names) == 2
  for name, body in zip(names, functions):
    assert not re.search(r"\bDFMA\b", body), name
    if "commit" not in name:
      assert "DMUL" in body and "DADD" in body, name
