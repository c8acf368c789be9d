"""Every native library of ``_build.LIBRARIES``: it has a Python binding that binds exactly the functions its header
declares, the library exports them and targets sm_90a, the binding fails loudly when the library cannot be loaded
(there is no CPU fallback), the libraries are built in the table's order with the flags their bits depend on, and a
library is rebuilt when a source it depends on changes.  Each library's kernel launches are checked next to its GPU
tests (``native_libs.check_every_kernel_is_launched``)."""
import os
import shutil

import pytest

from audiolazy_b200 import _build, _capi, analysis, crossing, fourier, linear_prediction as lp, resampling, spectral
from audiolazy_b200 import unwrapping
from conftest import ROOT
from native_libs import check_exports, check_sm90a

NAMES = sorted(_build.LIBRARIES)
BINDINGS = {"filters": _capi.LIB, "amdf": analysis.LIB, "zcross": crossing.LIB, "lpc": lp.LIB, "stft": spectral.LIB,
            "resample": resampling.LIB, "dft": fourier.LIB, "unwrap": unwrapping.LIB, "parcor": lp.PARCOR_LIB,
            "lpcfilt": lp.LPCFILT_LIB, "lpcscan": lp.LPCSCAN_LIB}


def test_every_library_has_a_binding():
  assert sorted(BINDINGS) == NAMES


@pytest.mark.parametrize("name", NAMES)
def test_library_exports_exactly_its_header(name):
  check_exports(BINDINGS[name], _build.LIBRARIES[name].header)


@pytest.mark.parametrize("name", NAMES)
def test_library_is_sm90a(name):
  check_sm90a(_build.LIBRARIES[name].path)


@pytest.mark.parametrize("name", NAMES)
def test_unloadable_library_raises_native_error(name, tmp_path, monkeypatch):
  """A missing file and a file that is not a shared library both raise NativeError, never a silent fallback."""
  binding = BINDINGS[name]
  monkeypatch.delenv("ALZ_B200_LIB", raising=False)
  monkeypatch.setattr(binding, "cdll", None)
  monkeypatch.setattr(binding, "path", str(tmp_path / "missing.so"))
  with pytest.raises(_capi.NativeError, match="no CPU fallback"):
    binding.load()
  junk = tmp_path / "junk.so"
  junk.write_text("not an ELF file\n")
  monkeypatch.setattr(binding, "path", str(junk))
  with pytest.raises(_capi.NativeError, match="cannot load"):
    binding.load()


def test_build_native_builds_the_table_in_order(monkeypatch):
  built = []
  monkeypatch.setattr(_build, "build_library", lambda lib, force=False, verbose=False: built.append(lib.name) or lib.path)
  assert _build.build_native() == [lib.path for lib in _build.LIBRARIES.values()]
  assert built == list(_build.LIBRARIES) == ["filters", "amdf", "zcross", "lpc", "stft", "resample", "dft", "unwrap",
                                             "parcor", "lpcfilt", "lpcscan"]


def test_flags_and_dependencies_of_the_bit_exact_libraries():
  """Every library but the filter library shares csrc_common/alz_common.h and reproduces AudioLazy's bits, so nvcc
  must not fuse its products into additions (-fmad=false); the DFT library's host twiddles must not be contracted
  either.  Zero crossings only compare samples: there is nothing to contract."""
  for name, lib in _build.LIBRARIES.items():
    if name == "filters":
      continue
    assert lib.deps == ("csrc_common/alz_common.h",), name
    if name == "dft":
      assert lib.flags == ("-fmad=false", "-Xcompiler", "-ffp-contract=off")
    elif name == "zcross":
      assert lib.flags == ()
    else:
      assert lib.flags == ("-fmad=false",), name


def test_staleness_follows_the_dependencies(tmp_path, monkeypatch):
  """In a copy of the sources: touching the shared header marks exactly the libraries that include it stale, touching
  one library's unit, private header or public header marks only that library stale."""
  for d in ("include", "audiolazy_b200"):
    shutil.copytree(os.path.join(ROOT, d), str(tmp_path / d), ignore=shutil.ignore_patterns("_native", "__pycache__"))
  monkeypatch.setattr(_build, "ROOT", str(tmp_path))
  libs = list(_build.LIBRARIES.values())
  os.makedirs(str(tmp_path / _build.NATIVE))
  for lib in libs:
    open(lib.path, "w").close()

  def stale_after_touching(rel):
    for lib in libs:
      for src in lib.units() + lib.headers():
        os.utime(src, (1000, 1000))
      os.utime(lib.path, (2000, 2000))
    assert not any(_build.is_stale(lib) for lib in libs)
    os.utime(str(tmp_path / rel), (3000, 3000))
    return sorted(lib.name for lib in libs if _build.is_stale(lib))

  assert stale_after_touching("audiolazy_b200/csrc_common/alz_common.h") == sorted(set(_build.LIBRARIES) - {"filters"})
  assert stale_after_touching("audiolazy_b200/csrc_lpc/alz_lpc.cu") == ["lpc"]
  assert stale_after_touching("include/alz_b200_lpc.h") == ["lpc"]
  assert stale_after_touching("include/alz_b200_zcross.h") == ["zcross"]
  assert stale_after_touching("audiolazy_b200/csrc/alz_plan.h") == ["filters"]
  assert stale_after_touching("audiolazy_b200/csrc_stft/alz_stft.cu") == ["stft"]
  assert stale_after_touching("include/alz_b200_stft.h") == ["stft"]
  assert stale_after_touching("audiolazy_b200/csrc_resample/alz_resample.cu") == ["resample"]
  for name in ("dft", "unwrap", "parcor", "lpcfilt", "lpcscan"):
    assert stale_after_touching("audiolazy_b200/csrc_%s/alz_%s.cu" % (name, name)) == [name]
    assert stale_after_touching("include/alz_b200_%s.h" % name) == [name]
  assert stale_after_touching("audiolazy_b200/csrc_parcor/alz_pow2.h") == ["parcor"]
