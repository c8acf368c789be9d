"""The C-ABI shared library: builds, loads, exports every symbol include/alz_b200.h
declares, and fails loudly (never silently falls back) without a CUDA device."""
import os
import re

import numpy as np
import pytest

from audiolazy_b200 import _build, _capi
from conftest import ROOT
from native_libs import check_exports, check_sm90a, cuobjdump, header_functions


def test_library_is_built_in_tree():
  assert os.path.exists(_build.LIB_PATH), "run `python -c 'import __graft_entry__ as g; g.build()'` first"
  assert os.path.dirname(_build.LIB_PATH).startswith(ROOT)


def test_exports_every_declared_symbol():
  assert len(header_functions("alz_b200.h")) >= 14
  assert _capi.lib().alz_abi_version() == 2
  check_exports(_capi.LIB, "alz_b200.h")


def test_sass_is_sm90a_with_fp64_and_uniform_operands():
  import subprocess
  check_sm90a(_build.LIB_PATH)
  # stream the SASS and stop as soon as both signatures have been seen
  proc = subprocess.Popen([cuobjdump(), "-sass", _build.LIB_PATH], stdout=subprocess.PIPE, text=True)
  seen_ur = seen_cp = seen_tma_ld = seen_tma_st = False
  for line in proc.stdout:
    seen_ur = seen_ur or re.search(r"DFMA R\d+, R\d+(\.reuse)?, UR\d+, R\d+", line) is not None
    seen_cp = seen_cp or "LDGSTS" in line          # cp.async staging (fallback engine)
    seen_tma_ld = seen_tma_ld or "UTMALDG" in line  # TMA tile load
    seen_tma_st = seen_tma_st or "UTMASTG" in line  # TMA tile store
    if seen_ur and seen_cp and seen_tma_ld and seen_tma_st:
      break
  proc.kill()
  assert seen_ur, "coefficients are not in uniform registers"
  assert seen_cp, "no cp.async (LDGSTS) in the kernels"
  assert seen_tma_ld and seen_tma_st, "no TMA tile load/store (UTMALDG/UTMASTG) in the kernels"


def test_pack_sections_layout():
  coef, desc, C, KM = _capi.pack_sections([[([1, 2], [1, .5]), ([3], [1])], [([4, 5, 6], [2, 0, 1])]])
  assert (C, KM) == (2, 2)
  d = desc.reshape(C, KM, 3)
  assert d[0, 0].tolist() == [2, 2, 0] and d[0, 1].tolist() == [1, 1, 4] and d[1, 0].tolist() == [3, 3, 6]
  assert d[1, 1].tolist() == [0, 0, 0]               # absent section
  assert coef.tolist() == [1, 2, 1, .5, 3, 1, 4, 5, 6, 2, 0, 1]


def test_no_silent_cpu_fallback():
  """On a box without a GPU every compute entry fails with an error; nothing is computed."""
  import torch
  if torch.cuda.is_available():
    pytest.skip("GPU present: covered by the gpu tests")
  assert _capi.device_count() == 0
  with pytest.raises(_capi.NativeError):
    _capi.Plan([[([1.0, 0.5], [1.0, -0.5])]])
  import audiolazy_b200 as ab
  with pytest.raises(_capi.NativeError):
    ab.ZFilter([1, 1], [1, -0.5])([1.0, 2.0, 3.0])
  with pytest.raises(_capi.NativeError):
    ab.gammatone_bank(strategy="slaney").apply_host(np.zeros((1, 16), dtype=np.float32))


def test_missing_library_is_loud(monkeypatch):
  monkeypatch.setattr(_capi, "_lib", None)
  monkeypatch.setenv("ALZ_B200_LIB", "/nonexistent/libalz_b200.so")
  with pytest.raises(_capi.NativeError, match="no CPU fallback"):
    _capi.lib()


def test_header_is_plain_c(tmp_path):
  """include/alz_b200.h is the boundary: it must compile as C99 and as C++ on its own."""
  import shutil
  import subprocess
  inc = os.path.join(ROOT, "include")
  for compiler, std, ext in (("gcc", "-std=c99", "c"), ("g++", "-std=c++11", "cpp")):
    if shutil.which(compiler) is None:
      pytest.skip(compiler + " not available")
    src = tmp_path / ("use_header." + ext)
    src.write_text('#include "alz_b200.h"\nint main(void) { return ALZ_OK; }\n')
    subprocess.run([compiler, std, "-Wall", "-Wextra", "-Werror", "-pedantic", "-fsyntax-only", "-I", inc, str(src)],
                   check=True, capture_output=True)
