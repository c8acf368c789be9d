"""The bank engine's L2 policy, read from the compiled sm_90a code (no GPU needed).

The TMA bank kernel writes 256 B for every 4 B it reads, and each input tile is read by every channel's warp of its
stream group, at different times.  Its tile stores therefore carry an evict-first L2 cache hint
(``cp.async.bulk.tensor...bulk_group.L2::cache_hint``), so the output stream takes the L2's first victims and the
input tiles stay for their later readers.  In SASS the hint is the store's third operand, the policy descriptor:
``UTMASTG.4D [URa], [URb], desc[URc]``; without it the store has two operands."""
import re
import subprocess

from audiolazy_b200 import _build
from native_libs import cuobjdump

K4_TMA_BANK = "_Z21alz_biquad_tma_kernelILi4E"   # alz_biquad_tma_kernel<4, ...>: the flagship slaney bank's kernel


def tma_stores(path, prefix):
  """{mangled kernel name: [its UTMASTG instructions]} for the kernels of ``path`` whose name starts with ``prefix``."""
  sass = subprocess.run([cuobjdump(), "-sass", path], capture_output=True, text=True, check=True).stdout
  stores, name = {}, None
  for line in sass.splitlines():
    m = re.match(r"\s*Function : (\S+)", line)
    if m:
      name = m.group(1) if m.group(1).startswith(prefix) else None
      if name:
        stores[name] = []
    elif name and "UTMASTG" in line:
      stores[name].append(re.sub(r"\s*/\*[^*]*\*/\s*", " ", line).strip())
  return stores


def test_k4_tma_bank_tile_stores_carry_an_l2_cache_hint():
  stores = tma_stores(_build.LIB_PATH, K4_TMA_BANK)
  assert stores, "no K = 4 TMA bank kernel in %s" % _build.LIB_PATH
  for name, ins in stores.items():
    assert ins, "%s has no TMA tile store" % name
    missing = [i for i in ins if "desc[" not in i]
    assert not missing, "%s: tile stores without an L2 cache hint: %s" % (name, missing)
