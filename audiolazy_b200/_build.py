"""Build the native CUDA libraries in-tree (``audiolazy_b200/_native/``).

``nvcc`` cross-compiles for sm_90a (H100) without a GPU; the built ``.so`` files are git-ignored
but travel to the GPU box with the repository snapshot.

:data:`LIBRARIES` lists the eleven libraries, in build order.  Each one is the ``.cu`` units of its source directory,
compiled in parallel into ``_native/obj/<name>/`` (only the units that changed) and linked into one shared library.
Every library but the filter library also includes ``csrc_common/alz_common.h``.  ``-fmad=false`` keeps nvcc from
fusing a product into an addition, which would round once where AudioLazy rounds twice.

* ``filters``: ``libalz_b200.so``, ``csrc/*.cu`` behind ``include/alz_b200.h`` (the C ABI plus one unit of kernel
  instantiations per cascade length).
* ``amdf``: ``libalz_b200_amdf.so``, ``csrc_amdf/*.cu`` behind ``include/alz_b200_amdf.h``; ``-fmad=false``: its
  float64 arithmetic reproduces AudioLazy's bit for bit.
* ``zcross``: ``libalz_b200_zcross.so``, ``csrc_zcross/*.cu`` behind ``include/alz_b200_zcross.h``.
* ``lpc``: ``libalz_b200_lpc.so``, ``csrc_lpc/*.cu`` behind ``include/alz_b200_lpc.h``; ``-fmad=false``: its float64
  sums reproduce AudioLazy's bit for bit.
* ``stft``: ``libalz_b200_stft.so``, ``csrc_stft/*.cu`` behind ``include/alz_b200_stft.h``; ``-fmad=false``: its
  window products and overlap-add sums reproduce AudioLazy's bit for bit.
* ``resample``: ``libalz_b200_resample.so``, ``csrc_resample/*.cu`` behind ``include/alz_b200_resample.h``;
  ``-fmad=false``: its weights and compensated sums reproduce AudioLazy's bit for bit.
* ``dft``: ``libalz_b200_dft.so``, ``csrc_dft/*.cu`` behind ``include/alz_b200_dft.h``; ``-fmad=false`` and a host
  compiler told not to contract (``-ffp-contract=off``): its device sums and its host twiddles reproduce AudioLazy's
  ``dft`` bit for bit.
* ``unwrap``: ``libalz_b200_unwrap.so``, ``csrc_unwrap/*.cu`` behind ``include/alz_b200_unwrap.h``; ``-fmad=false``:
  its float64 running sums reproduce AudioLazy's ``unwrap`` bit for bit.
* ``parcor``: ``libalz_b200_parcor.so``, ``csrc_parcor/*.cu`` behind ``include/alz_b200_parcor.h``; ``-fmad=false``:
  its step-down and its restatement of glibc's ``pow`` reproduce AudioLazy's ``parcor`` bit for bit.
* ``lpcfilt``: ``libalz_b200_lpcfilt.so``, ``csrc_lpcfilt/*.cu`` behind ``include/alz_b200_lpcfilt.h``;
  ``-fmad=false``: its analysis and synthesis sums reproduce AudioLazy's time-varying ZFilters bit for bit.
* ``lpcscan``: ``libalz_b200_lpcscan.so``, ``csrc_lpcscan/*.cu`` behind ``include/alz_b200_lpcscan.h``;
  ``-fmad=false``: its walks of a flagged stream reproduce the LPC filtering library's synthesis bit for bit.

PARCOR and LPC filtering are libraries of their own rather than units of the LPC library, because that library's
kernel set is checked as it stands.
"""
from __future__ import annotations

import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor
from typing import NamedTuple

#: the repository root, which the paths of :data:`LIBRARIES` are resolved against when they are used
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = "audiolazy_b200"
NATIVE = os.path.join(PKG, "_native")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + [
  "-O3", "-lineinfo", "-std=c++17",
  "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",   # only the extern "C" ABI of the public header is exported
]


class Library(NamedTuple):
  """One shared library, ``_native/<file>``.  Every ``.cu`` of the package directory ``csrc`` is a unit; every
  ``.cuh`` / ``.h`` there, the public ``include/<header>`` and the private headers ``deps`` (package paths) are
  dependencies of all of them.  ``flags`` are added to the nvcc flags of its units."""
  name: str
  file: str
  csrc: str
  header: str
  flags: tuple = ()
  deps: tuple = ()

  @property
  def path(self):
    return os.path.join(ROOT, NATIVE, self.file)

  def units(self):
    d = os.path.join(ROOT, PKG, self.csrc)
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith(".cu"))

  def headers(self):
    d = os.path.join(ROOT, PKG, self.csrc)
    return sorted(os.path.join(d, f) for f in os.listdir(d) if f.endswith((".cuh", ".h"))) + \
           [os.path.join(ROOT, "include", self.header)] + [os.path.join(ROOT, PKG, h) for h in self.deps]


_COMMON = ("csrc_common/alz_common.h",)
LIBRARIES = {lib.name: lib for lib in (
  Library("filters", "libalz_b200.so", "csrc", "alz_b200.h"),
  Library("amdf", "libalz_b200_amdf.so", "csrc_amdf", "alz_b200_amdf.h", ("-fmad=false",), _COMMON),
  Library("zcross", "libalz_b200_zcross.so", "csrc_zcross", "alz_b200_zcross.h", (), _COMMON),
  Library("lpc", "libalz_b200_lpc.so", "csrc_lpc", "alz_b200_lpc.h", ("-fmad=false",), _COMMON),
  Library("stft", "libalz_b200_stft.so", "csrc_stft", "alz_b200_stft.h", ("-fmad=false",), _COMMON),
  Library("resample", "libalz_b200_resample.so", "csrc_resample", "alz_b200_resample.h", ("-fmad=false",), _COMMON),
  Library("dft", "libalz_b200_dft.so", "csrc_dft", "alz_b200_dft.h",
          ("-fmad=false", "-Xcompiler", "-ffp-contract=off"), _COMMON),
  Library("unwrap", "libalz_b200_unwrap.so", "csrc_unwrap", "alz_b200_unwrap.h", ("-fmad=false",), _COMMON),
  Library("parcor", "libalz_b200_parcor.so", "csrc_parcor", "alz_b200_parcor.h", ("-fmad=false",), _COMMON),
  Library("lpcfilt", "libalz_b200_lpcfilt.so", "csrc_lpcfilt", "alz_b200_lpcfilt.h", ("-fmad=false",), _COMMON),
  Library("lpcscan", "libalz_b200_lpcscan.so", "csrc_lpcscan", "alz_b200_lpcscan.h", ("-fmad=false",), _COMMON),
)}
#: the filter library (``_capi`` loads it from here unless ``ALZ_B200_LIB`` names another file)
LIB_PATH = LIBRARIES["filters"].path


def is_stale(lib: Library) -> bool:
  """The library is missing or older than one of its sources."""
  if not os.path.exists(lib.path):
    return True
  t = os.path.getmtime(lib.path)
  return any(os.path.getmtime(s) > t for s in lib.units() + lib.headers())


def find_nvcc():
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  return nvcc if os.path.exists(nvcc) else None


def build_native(force: bool = False, verbose: bool = False) -> list:
  """Build every library of :data:`LIBRARIES`, in order; returns their paths."""
  return [build_library(lib, force=force, verbose=verbose) for lib in LIBRARIES.values()]


def build_library(lib: Library, force: bool = False, verbose: bool = False) -> str:
  """Compile the units of ``lib`` that changed for sm_90a, in parallel, and link its shared library."""
  if not force and not is_stale(lib):
    return lib.path
  nvcc = find_nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found: cannot build audiolazy_b200's %s" % lib.file)
  obj_dir = os.path.join(ROOT, NATIVE, "obj", lib.name)
  os.makedirs(obj_dir, exist_ok=True)
  newest_header = max(os.path.getmtime(h) for h in lib.headers())
  units = lib.units()
  objs = [os.path.join(obj_dir, os.path.splitext(os.path.basename(src))[0] + ".o") for src in units]
  jobs = [(src, obj) for src, obj in zip(units, objs)
          if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), newest_header)]

  def compile_one(job):
    src, obj = job
    tmp = obj + ".tmp.%d" % os.getpid()
    cmd = [nvcc] + NVCC_FLAGS + list(lib.flags) + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", tmp, src]
    subprocess.check_call(cmd)
    os.replace(tmp, obj)

  with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as pool:
    list(pool.map(compile_one, jobs))
  tmp = lib.path + ".tmp.%d" % os.getpid()
  subprocess.check_call([nvcc] + ARCH_FLAGS + ["-shared", "-o", tmp] + objs)
  os.replace(tmp, lib.path)
  return lib.path
