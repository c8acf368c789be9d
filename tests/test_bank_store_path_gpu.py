"""The two store paths of the TMA bank kernel's tile groups of 4 (``alz_run_warp_tma``, alz_lane_tma.cuh): warp-wide
``st.global.v4`` of one row's 512 bytes per instruction (the default) and TMA box stores (``ALZ_STORE_PATH=tma``).

Each case runs one plan per path, at tile group 4 (``ALZ_TILE_GROUP=4``) unless it says otherwise, into output buffers
filled with a NaN sentinel, and asserts that both give the same bits everywhere -- the written rows, the rows and
samples they must not touch, and the final states -- and that the ``ALZ_LOG_LAUNCH`` line of every bank launch names
the store path the case expects."""
import json
import os
import re

import pytest

import test_kernel_matrix as km

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LOG = re.compile(r"alz bank launch: .*tile group (\d+), .* (\d+) segment\(s\) of \d+ samples, (vector|TMA) stores, "
                 r"(\d+) chunks per stream")
SENTINEL = 0x7FC0DEAD


@pytest.fixture(scope="module")
def env():
  torch = pytest.importorskip("torch")
  if not torch.cuda.is_available():
    pytest.skip("no CUDA device")
  torch.cuda.set_device(0)
  from audiolazy_b200 import _capi
  with open(os.path.join(HERE, "golden", "designs.json")) as fh:
    return torch, _capi, json.load(fh)["bank_slaney"][:64]


def _run(env, capfd, path, S, T, layout, group=4):
  """(y bits, state, [(tile group, segments, store path, chunks per stream) per bank launch]) of one call on a fresh
  plan; ``group`` None: the plan's own tile group."""
  torch, capi, bank = env
  with km._env(ALZ_STORE_PATH=path, **({} if group is None else {"ALZ_TILE_GROUP": group})):
    plan = capi.Plan(bank)
  C = plan.n_channels
  xs = (T + 3) // 4 * 4                                   # 16-byte aligned input rows: the TMA engine
  g = torch.Generator(device="cuda")
  g.manual_seed(S * 7 + T)
  x = (torch.rand((S, xs), device="cuda", generator=g) * 2 - 1).contiguous()
  if layout == "stream":                                  # y[S][C][ys], ys = T rounded up to 16 bytes
    ys = xs
    y = torch.full((S * C * ys,), 0, dtype=torch.int32, device="cuda")
    call = lambda yp, st: plan.apply(x.data_ptr(), yp, st, S, T, xs, ys, cur)
  elif layout == "channel":                               # y[C][S][ys]
    ys = xs
    y = torch.full((C * S * ys,), 0, dtype=torch.int32, device="cuda")
    call = lambda yp, st: plan.apply_ex(x.data_ptr(), yp, st, S, T, xs, S * ys, ys, cur)
  else:                                                   # channels 8 .. 8 + C of y[S][C + 16][T] plus a 16-byte gap
    ys, extra = xs, 16
    ysS = (C + extra) * ys + 4
    y = torch.full((S * ysS,), 0, dtype=torch.int32, device="cuda")
    call = lambda yp, st: plan.apply_ex(x.data_ptr(), yp + 4 * 8 * ys, st, S, T, xs, ys, ysS, cur)
  y.fill_(SENTINEL)
  st = torch.zeros(plan.state_doubles(S), dtype=torch.float64, device="cuda")
  cur = torch.cuda.current_stream().cuda_stream
  capfd.readouterr()
  with km._env(ALZ_LOG_LAUNCH=1):
    call(y.data_ptr(), st.data_ptr())
    torch.cuda.synchronize()
  logs = [LOG.search(l) for l in capfd.readouterr().err.splitlines()]
  return y, st, [(int(m.group(1)), int(m.group(2)), m.group(3), int(m.group(4))) for m in logs if m]


def _check(env, capfd, S, T, layout="stream", group=4, segmented=None, virtual=False):
  """The two paths give the same bits; the vector path was taken by every tile-group-4 launch and by no other."""
  torch = env[0]
  y_tma, st_tma, log_tma = _run(env, capfd, "tma", S, T, layout, group)
  y_vec, st_vec, log_vec = _run(env, capfd, "vec", S, T, layout, group)
  assert log_tma and log_vec, "no bank launch logged"
  assert all(p == "TMA" for _, _, p, _ in log_tma), log_tma
  assert all((p == "vector") == (g == 4) for g, _, p, _ in log_vec), log_vec
  if group is not None:
    assert any(g == group for g, _, _, _ in log_vec), log_vec
  if segmented is not None:
    assert any(n > 1 for _, n, _, _ in log_vec) == segmented, log_vec
  if virtual:                                           # virtual streams (chunks of a real stream) through vector stores
    assert any(p == "vector" and v > 1 for _, _, p, v in log_vec), log_vec
  assert torch.equal(y_vec, y_tma)
  assert torch.equal(st_vec.view(torch.int64), st_tma.view(torch.int64))
  assert (y_vec != SENTINEL).any()


# S and T whole stream groups and tiles; ragged S % 32; T % 32 != 0 with T % 4 == 0; T % 4 != 0 (the lanes store the
# ragged last tile); a last tile group of 1, 2 and 3 tiles
@pytest.mark.parametrize("S,T", [(64, 4096), (70, 4096), (64, 4100), (33, 4099), (96, 4097), (32, 4160), (32, 4192),
                                 (40, 4224)])
def test_shapes(env, capfd, S, T):
  _check(env, capfd, S, T)


@pytest.mark.parametrize("layout", ["channel", "slice"])
def test_layouts(env, capfd, layout):
  _check(env, capfd, 70, 4100, layout)


def test_segmented(env, capfd):
  """2048 warps, more than one wave of 13-CTA SMs: cut into time segments chained through the state."""
  _check(env, capfd, 1024, 5120, segmented=True)


def test_time_parallel(env, capfd):
  """One long stream: virtual streams, each a chunk of the real one, stored through the 4-D output map's geometry."""
  _check(env, capfd, 1, 1 << 18, virtual=True)


def test_group2_keeps_tma_stores(env, capfd):
  _check(env, capfd, 64, 4096, group=2)


def test_small_launch_keeps_tma_stores(env, capfd):
  """The plan's own tile group: 128 warps do not fill the machine, so the launch stays below group 4 by its size."""
  *_, log = _run(env, capfd, "vec", 64, 4096, "stream", group=None)
  assert log and all(g < 4 and p == "TMA" for g, _, p, _ in log), log
  _check(env, capfd, 64, 4096, group=None)
