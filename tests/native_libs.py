"""Helpers of the tests of the native libraries (``audiolazy_b200/_build.py``): what a header declares and a library
compiles, the checks every library takes (exports, target, kernel launches), and the GPU ``torch`` fixture."""
import os
import re
import shutil
import subprocess
import sys

import pytest

from conftest import ROOT


@pytest.fixture(scope="module")
def torch():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  return torch


def header_functions(header):
  """The functions ``include/<header>`` declares."""
  text = open(os.path.join(ROOT, "include", header)).read()
  text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
  return sorted(set(re.findall(r"\b(alz_[a-z0-9_]+)\s*\(", text)))


def cuobjdump():
  path = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
  if not os.path.exists(path):
    pytest.skip("cuobjdump not available")
  return path


def compiled_kernels(path):
  """The demangled names of the kernels compiled into the shared library ``path``."""
  filt = shutil.which("c++filt") or shutil.which("cu++filt") or "/usr/local/cuda/bin/cu++filt"
  if not os.path.exists(filt):
    pytest.skip("c++filt not available")
  elf = subprocess.run([cuobjdump(), "-elf", path], capture_output=True, text=True, check=True).stdout
  mangled = sorted(set(re.findall(r"\.text\.(_Z\w+)", elf)))
  assert mangled, "no kernels found in %s" % path
  names = subprocess.run([filt], input="\n".join(mangled), capture_output=True, text=True, check=True).stdout
  return [n for n in names.splitlines() if n.strip()]


def check_exports(binding, header):
  """The library of ``binding`` (an ``_capi.NativeLib``) is built, its binding binds exactly the functions
  ``include/<header>`` declares, and the library exports them and no other ``alz_`` function."""
  assert os.path.exists(binding.path), "run `python -c 'import __graft_entry__ as g; g.build()'` first"
  declared = header_functions(header)
  assert sorted(binding.symbols) == declared
  loaded = binding.load()
  for name in declared:
    assert hasattr(loaded, name), "library does not export %s" % name
  if not shutil.which("nm"):
    pytest.skip("nm not available")
  out = subprocess.run(["nm", "-D", "--defined-only", binding.path], capture_output=True, text=True).stdout
  assert sorted(line.split()[-1] for line in out.splitlines() if " T alz_" in line) == declared


def check_sm90a(path):
  out = subprocess.run([cuobjdump(), "-lelf", path], capture_output=True, text=True).stdout
  assert "sm_90a" in out


def check_every_kernel_is_launched(path, probe):
  """The kernels the script ``probe`` launches (it prints ``LAUNCHED <name>`` for each kernel its profiler saw) are the
  kernels compiled into the library ``path``.  The probe runs with the repository's root as its argument, in a process
  of its own, so that its profiling session leaves no profiler state behind in this one."""
  built = {n.split("(")[0].strip() for n in compiled_kernels(path)}
  run = subprocess.run([sys.executable, "-c", probe, ROOT], capture_output=True, text=True, timeout=300)
  assert run.returncode == 0, run.stderr[-2000:]
  launched = {line.split(None, 1)[1] for line in run.stdout.splitlines() if line.startswith("LAUNCHED ")}
  assert launched == built, (sorted(launched), sorted(built))
