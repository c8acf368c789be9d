"""Build the native CUDA libraries in-tree (``audiolazy_b200/_native/``).

``nvcc`` cross-compiles for sm_90a (H100) without a GPU; the built ``.so`` files are git-ignored
but travel to the GPU box with the repository snapshot.

* ``libalz_b200.so``, the filter library: the translation units ``csrc/*.cu`` (the C ABI plus
  one unit of kernel instantiations per cascade length) are compiled in parallel into
  ``_native/obj/`` and linked into ONE shared library.
* ``libalz_b200_amdf.so``, the AMDF library: ``csrc_amdf/*.cu`` behind ``include/alz_b200_amdf.h``,
  compiled with ``-fmad=false`` (its float64 arithmetic reproduces AudioLazy's bit for bit).
* ``libalz_b200_zcross.so``, the zero-crossing library: ``csrc_zcross/*.cu`` behind ``include/alz_b200_zcross.h``.
* ``libalz_b200_lpc.so``, the frame-wise LPC library: ``csrc_lpc/*.cu`` behind ``include/alz_b200_lpc.h``, compiled
  with ``-fmad=false`` (its float64 sums reproduce AudioLazy's bit for bit).
"""
from __future__ import annotations

import os
import shutil
import subprocess
from concurrent.futures import ThreadPoolExecutor

_PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_PKG, "csrc")
NATIVE_DIR = os.path.join(_PKG, "_native")
OBJ_DIR = os.path.join(NATIVE_DIR, "obj")
LIB_PATH = os.path.join(NATIVE_DIR, "libalz_b200.so")
INCLUDE = os.path.join(os.path.dirname(_PKG), "include")
AMDF_CSRC = os.path.join(_PKG, "csrc_amdf")
AMDF_LIB_PATH = os.path.join(NATIVE_DIR, "libalz_b200_amdf.so")
AMDF_HEADER = os.path.join(INCLUDE, "alz_b200_amdf.h")
ZCROSS_CSRC = os.path.join(_PKG, "csrc_zcross")
ZCROSS_LIB_PATH = os.path.join(NATIVE_DIR, "libalz_b200_zcross.so")
ZCROSS_HEADER = os.path.join(INCLUDE, "alz_b200_zcross.h")
LPC_CSRC = os.path.join(_PKG, "csrc_lpc")
LPC_LIB_PATH = os.path.join(NATIVE_DIR, "libalz_b200_lpc.so")
LPC_HEADER = os.path.join(INCLUDE, "alz_b200_lpc.h")

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH_FLAGS + [
  "-O3", "-lineinfo", "-std=c++17",
  "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",   # only the extern "C" ABI of include/alz_b200.h is exported
]


def _units():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers():
  return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + \
         [os.path.join(INCLUDE, "alz_b200.h")]


def _sources():
  return _units() + _headers()


def is_stale() -> bool:
  if not os.path.exists(LIB_PATH):
    return True
  t = os.path.getmtime(LIB_PATH)
  return any(os.path.getmtime(s) > t for s in _sources())


def find_nvcc():
  nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
  return nvcc if os.path.exists(nvcc) else None


def build_native(force: bool = False, verbose: bool = False) -> str:
  """Build the four libraries (see :func:`build_filters`, :func:`build_amdf`, :func:`build_zcross` and
  :func:`build_lpc`); returns the filter library's path."""
  path = build_filters(force=force, verbose=verbose)
  build_amdf(force=force, verbose=verbose)
  build_zcross(force=force, verbose=verbose)
  build_lpc(force=force, verbose=verbose)
  return path


def _amdf_sources():
  return sorted(os.path.join(AMDF_CSRC, f) for f in os.listdir(AMDF_CSRC) if f.endswith((".cu", ".cuh", ".h"))) + \
         [AMDF_HEADER]


def build_amdf(force: bool = False, verbose: bool = False) -> str:
  """Compile ``csrc_amdf/*.cu`` for sm_90a with ``-fmad=false`` and link ``libalz_b200_amdf.so``."""
  if not force and os.path.exists(AMDF_LIB_PATH) and \
     all(os.path.getmtime(s) <= os.path.getmtime(AMDF_LIB_PATH) for s in _amdf_sources()):
    return AMDF_LIB_PATH
  nvcc = find_nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found: cannot build audiolazy_b200's AMDF library")
  os.makedirs(NATIVE_DIR, exist_ok=True)
  units = sorted(os.path.join(AMDF_CSRC, f) for f in os.listdir(AMDF_CSRC) if f.endswith(".cu"))
  tmp = AMDF_LIB_PATH + ".tmp.%d" % os.getpid()
  cmd = [nvcc] + NVCC_FLAGS + ["-fmad=false"] + (["-Xptxas", "-v"] if verbose else []) + ["-shared", "-o", tmp] + units
  subprocess.check_call(cmd)
  os.replace(tmp, AMDF_LIB_PATH)
  return AMDF_LIB_PATH


def _zcross_sources():
  return sorted(os.path.join(ZCROSS_CSRC, f) for f in os.listdir(ZCROSS_CSRC) if f.endswith((".cu", ".cuh", ".h"))) + \
         [ZCROSS_HEADER]


def build_zcross(force: bool = False, verbose: bool = False) -> str:
  """Compile ``csrc_zcross/*.cu`` for sm_90a and link ``libalz_b200_zcross.so``."""
  if not force and os.path.exists(ZCROSS_LIB_PATH) and \
     all(os.path.getmtime(s) <= os.path.getmtime(ZCROSS_LIB_PATH) for s in _zcross_sources()):
    return ZCROSS_LIB_PATH
  nvcc = find_nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found: cannot build audiolazy_b200's zero-crossing library")
  os.makedirs(NATIVE_DIR, exist_ok=True)
  units = sorted(os.path.join(ZCROSS_CSRC, f) for f in os.listdir(ZCROSS_CSRC) if f.endswith(".cu"))
  tmp = ZCROSS_LIB_PATH + ".tmp.%d" % os.getpid()
  cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-shared", "-o", tmp] + units
  subprocess.check_call(cmd)
  os.replace(tmp, ZCROSS_LIB_PATH)
  return ZCROSS_LIB_PATH


def _lpc_sources():
  return sorted(os.path.join(LPC_CSRC, f) for f in os.listdir(LPC_CSRC) if f.endswith((".cu", ".cuh", ".h"))) + \
         [LPC_HEADER]


def build_lpc(force: bool = False, verbose: bool = False) -> str:
  """Compile ``csrc_lpc/*.cu`` for sm_90a with ``-fmad=false`` and link ``libalz_b200_lpc.so``."""
  if not force and os.path.exists(LPC_LIB_PATH) and \
     all(os.path.getmtime(s) <= os.path.getmtime(LPC_LIB_PATH) for s in _lpc_sources()):
    return LPC_LIB_PATH
  nvcc = find_nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found: cannot build audiolazy_b200's LPC library")
  os.makedirs(NATIVE_DIR, exist_ok=True)
  units = sorted(os.path.join(LPC_CSRC, f) for f in os.listdir(LPC_CSRC) if f.endswith(".cu"))
  tmp = LPC_LIB_PATH + ".tmp.%d" % os.getpid()
  cmd = [nvcc] + NVCC_FLAGS + ["-fmad=false"] + (["-Xptxas", "-v"] if verbose else []) + ["-shared", "-o", tmp] + units
  subprocess.check_call(cmd)
  os.replace(tmp, LPC_LIB_PATH)
  return LPC_LIB_PATH


def build_filters(force: bool = False, verbose: bool = False) -> str:
  """Compile ``csrc/*.cu`` for sm_90a (only the units that changed) and link the filter library."""
  if not force and not is_stale():
    return LIB_PATH
  nvcc = find_nvcc()
  if nvcc is None:
    raise RuntimeError("nvcc not found: cannot build audiolazy_b200's CUDA library")
  os.makedirs(OBJ_DIR, exist_ok=True)
  newest_header = max(os.path.getmtime(h) for h in _headers())
  jobs = []
  for src in _units():
    obj = os.path.join(OBJ_DIR, os.path.splitext(os.path.basename(src))[0] + ".o")
    if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), newest_header):
      jobs.append((src, obj))

  def compile_one(job):
    src, obj = job
    tmp = obj + ".tmp.%d" % os.getpid()
    cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", tmp, src]
    subprocess.check_call(cmd)
    os.replace(tmp, obj)

  with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as pool:
    list(pool.map(compile_one, jobs))
  objs = [os.path.join(OBJ_DIR, os.path.splitext(os.path.basename(s))[0] + ".o") for s in _units()]
  tmp = LIB_PATH + ".tmp.%d" % os.getpid()
  subprocess.check_call([nvcc] + ARCH_FLAGS + ["-shared", "-o", tmp] + objs)
  os.replace(tmp, LIB_PATH)
  return LIB_PATH
