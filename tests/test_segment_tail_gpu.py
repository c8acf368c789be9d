"""Time segments of the TMA bank launch (``launch_biquad_chunk``, alz_launch.cuh).

A launch whose last wave of warps would leave more than 2 % of the warp slots idle is cut into the fewest time segments
that bring the idle share under that, and never into a count that idles no less than the whole launch: such a count
pays for the segment flags and the chained waits and gains nothing.  The geometry the library chose is read from its
``ALZ_LOG_LAUNCH`` line and checked against the rule recomputed here; a segmented launch gives the bits of the
unsegmented one."""
import json
import os
import re

import pytest

import test_kernel_matrix as km

HERE = os.path.dirname(os.path.abspath(__file__))
LOG = re.compile(r"alz bank launch: (\d+) warps, tile group (\d+), (\d+) CTAs per SM \((\d+) slots\), "
                 r"(\d+) segment\(s\) of (\d+) samples")
SEG_MIN, TAIL_IDLE = 1024, 0.02


def _idle(n, warps, slots):
  cap = -(-n * warps // slots) * slots
  return (cap - n * warps) / cap


def expected_segments(warps, slots, groups, T, ng):
  """The segment count of the launch rule for ``warps`` warps of ``groups`` stream groups on ``slots`` warp slots."""
  if warps <= slots or T < 2 * SEG_MIN or _idle(1, warps, slots) <= TAIL_IDLE:
    return 1
  best, nseg, quantum = _idle(1, warps, slots), 1, 32 * ng
  for n in range(2, T // SEG_MIN + 1):
    if groups * n > 65535:
      break
    ln = -(-(-(-T // n)) // quantum) * quantum
    if -(-T // ln) != n:
      continue
    f = _idle(n, warps, slots)
    if f < best:
      best, nseg = f, n
    if f <= TAIL_IDLE:
      break
  return nseg


@pytest.fixture(scope="module")
def slaney_plan():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  from audiolazy_b200 import _capi
  with open(os.path.join(HERE, "golden", "designs.json")) as fh:
    return torch, _capi.Plan(json.load(fh)["bank_slaney"][:64])


def _apply(torch, plan, x, capfd, **env):
  """``x`` [S][T] (device, 16-byte aligned rows) through ``plan`` from a zero state: (y, state, the launch's log)."""
  S, T = x.shape
  y = torch.empty((S, plan.n_channels, T), dtype=torch.float32, device=x.device)
  st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device=x.device)
  capfd.readouterr()
  with km._env(ALZ_LOG_LAUNCH=1, **env):
    plan.apply(x.data_ptr(), y.data_ptr(), st.data_ptr(), S, T, T, T, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
  lines = [LOG.search(l) for l in capfd.readouterr().err.splitlines()]
  lines = [tuple(int(v) for v in m.groups()) for m in lines if m]
  assert len(lines) == 1, "expected one bank launch, logged %r" % lines
  return y, st, lines[0]


# (S, T): 2048 warps of the 64-channel bank, 1.19 waves of an H100's 1716 slots at tile group 4: cut into 5 segments;
# 4352 warps, 2.54 waves, at T = 2048: two segments idle exactly as many slots as one launch, so it stays whole.
@pytest.mark.gpu
@pytest.mark.parametrize("S,T,segmented", [(1024, 5120, True), (2176, 2048, False)])
def test_segments_only_where_the_tail_shrinks(slaney_plan, capfd, S, T, segmented):
  torch, plan = slaney_plan
  g = torch.Generator(device="cuda")
  g.manual_seed(S + T)
  x = torch.rand((S, T), device="cuda", generator=g) * 2 - 1
  y, st, (warps, ng, per_sm, slots, nseg, seg_len) = _apply(torch, plan, x, capfd)
  groups = (S + 31) // 32
  assert warps == plan.n_channels * groups and slots % per_sm == 0
  assert nseg == expected_segments(warps, slots, groups, T, ng), (warps, ng, slots, nseg)
  if slots == 1716:                                   # H100 SXM: 132 SMs x 13 CTAs of 4 tiles
    assert ng == 4 and (nseg > 1) == segmented, (ng, nseg)
  if not segmented:
    assert _idle(1, warps, slots) > TAIL_IDLE         # the rule was consulted, and declined
  y1, st1, (_, _, _, _, nseg1, _) = _apply(torch, plan, x, capfd, ALZ_NO_SEGMENT=1)
  assert nseg1 == 1
  assert torch.equal(y, y1) and torch.equal(st, st1)
