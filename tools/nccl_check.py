"""Multi-GPU parity check on real NCCL (run under torchrun, >= 2 GPUs):

  python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29511 tools/nccl_check.py

channel-sharded bank = NCCL broadcast of the input block (overlapped pipeline) + local channels + the
in-place all-gather / the fused peer-memory store of the outputs; stream-sharded bank = scatter of the
input rows.  Every result is compared BIT FOR BIT with the single-GPU bank on the same inputs (the
kernels are the same, only the plumbing differs); rank 0 prints one line ending in "PARITY OK" and the
measured collective rates.  Exit code 1 on any mismatch."""
import os, sys
import numpy as np
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist
import audiolazy_b200 as ab
from audiolazy_b200.parallel import ShardedBank, PeerOutput

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
os.environ.setdefault("NCCL_DEBUG_FILE", "/dev/stderr")
try:
  dist.init_process_group("nccl", device_id=dev, pg_options=dist.ProcessGroupNCCL.Options(is_high_priority_stream=True))
except Exception:
  dist.init_process_group("nccl", device_id=dev)
bank = ab.gammatone_bank(strategy="slaney")
C = len(bank)
S, T = int(os.environ.get("ALZ_CHECK_S", 1024)), int(os.environ.get("ALZ_CHECK_T", 8192))
g = torch.Generator(device=dev); g.manual_seed(7)
blocks = [torch.rand((S, T), device=dev, generator=g) * 2 - 1 for _ in range(3)]          # same seed on every rank
# single-GPU truth: the three blocks are consecutive pieces of the same streams (state carried)
st = bank.new_state(S)
truth = [bank.apply(b, state=st).clone() for b in blocks]
fails = []

def check(name, ok):
  ok_t = torch.tensor([int(bool(ok))], device=dev)
  dist.all_reduce(ok_t, op=dist.ReduceOp.MIN)
  if not int(ok_t.item()):
    fails.append(name)

def timed(fn, n=5):
  fn(); torch.cuda.synchronize(); dist.barrier()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(n): fn()
  e1.record(); torch.cuda.synchronize()
  ms = torch.tensor([e0.elapsed_time(e1) / n], device=dev); dist.all_reduce(ms, op=dist.ReduceOp.MAX)
  return float(ms.item())

# ---- channels mode: overlapped broadcast pipeline ----------------------------------------------
sb = ShardedBank(bank, mode="channels")
Cl = sb.c_hi - sb.c_lo
xb = [torch.zeros((S, T), device=dev) for _ in range(2)]
y = sb.alloc_output(S, T)
state = sb.local.new_state(S)
pipe = sb.pipeline(xb, y, state)
if rank == 0:
  xb[0].copy_(blocks[0])        # rank 0 owns the input; the others receive it by broadcast only
for i, b in enumerate(blocks):
  if rank == 0 and i + 1 < len(blocks):
    xb[(i + 1) & 1].copy_(blocks[i + 1])     # the next block: broadcast under this block's kernel
  pipe.step()
  torch.cuda.synchronize()
  check("pipeline block %d" % i, torch.equal(y, truth[i][:, sb.c_lo:sb.c_hi]))
pipe.drain()
# the same pipeline with the bank kernel on an SM partition (green context): identical values
try:
  st_p = sb.local.new_state(S)
  pp = sb.pipeline(xb, y, st_p, compute_sms=128)
  if rank == 0:
    xb[0].copy_(blocks[0])
  for i, b in enumerate(blocks):
    if rank == 0 and i + 1 < len(blocks):
      xb[(i + 1) & 1].copy_(blocks[i + 1])
    pp.step()
    torch.cuda.synchronize()
    check("partitioned pipeline block %d" % i, torch.equal(y, truth[i][:, sb.c_lo:sb.c_hi]))
  pp.drain()
  pp.close()
except Exception as exc:
  if rank == 0:
    print("SM partition unavailable: %r" % (exc,), file=sys.stderr)
# ---- in-place gather ----------------------------------------------------------------------------
gbuf = sb.alloc_gather(S, T)
sb.gather_output_into(y, gbuf)
torch.cuda.synchronize()
check("gather_output_into", torch.equal(gbuf.permute(1, 0, 2, 3).reshape(S, C, T), truth[2]))
check("gather_output", torch.equal(sb.gather_output(y), truth[2]))
# ---- fused: kernels store straight into rank 0's y over NVLink peer memory ---------------------------
peer_ok = True
ms_peer = float("nan")
try:
  po = PeerOutput(S, C, T, dst=0)
  po.tensor.fill_(float("nan"))
  po.fence()
  x0 = blocks[0]
  st2 = sb.local.new_state(S)
  sb.apply_into(x0, po, state=st2)
  po.fence()
  torch.cuda.synchronize()
  if rank == 0:
    peer_ok = torch.equal(po.tensor, truth[0])
  check("apply_into (peer memory)", peer_ok)
  def fused():
    sb.apply_into(x0, po, state=st2)
    po.fence()
  ms_peer = timed(fused, n=3)
except Exception as exc:                       # symmetric memory needs P2P; report rather than fail the NCCL parity
  if rank == 0:
    print("peer-memory path unavailable: %r" % (exc,), file=sys.stderr)
ms_b = timed(lambda: sb.broadcast_input(xb[0], src=0))
ms_k = timed(lambda: pipe.compute_only())
ms_p = timed(lambda: pipe.step()); pipe.drain()
ms_g = timed(lambda: sb.gather_output_into(y, gbuf), n=3)
# ---- streams mode --------------------------------------------------------------------------------
ss = ShardedBank(bank, mode="streams")
lo, hi = ss.stream_range(S)
x_loc = torch.empty((hi - lo, T), device=dev)
ss.scatter_input_into(blocks[0] if rank == 0 else None, x_loc, src=0)
check("scatter_input_into", torch.equal(x_loc, blocks[0][lo:hi]))
y_loc = ss.apply(x_loc)
check("streams apply", torch.equal(y_loc, truth[0][lo:hi]))
check("state=None is a fresh state every call", torch.equal(ss.apply(x_loc), y_loc))
if rank == 0:
  in_bytes, recv = S * T * 4, S * (C - Cl) * T * 4
  print("nccl_check world=%d S=%d T=%d: broadcast %.3f ms (%.0f GB/s); kernel alone %.3f ms, with overlapped broadcast %.3f ms "
        "(%+.1f %%); in-place all-gather %.3f ms (%.0f GB/s received per GPU = %.2f of 450); fused peer-memory store to rank 0 "
        "%.3f ms (%.0f GB/s into rank 0); %s" % (
          world, S, T, ms_b, in_bytes / ms_b / 1e6, ms_k, ms_p, 100 * (ms_p / ms_k - 1), ms_g, recv / ms_g / 1e6,
          recv / ms_g / 1e6 / 450, ms_peer, recv / ms_peer / 1e6 if ms_peer == ms_peer else float("nan"),
          "PARITY OK" if not fails else "PARITY FAILED: " + ", ".join(fails)))
dist.barrier()
dist.destroy_process_group()
sys.exit(1 if fails else 0)
