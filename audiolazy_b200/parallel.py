"""Multi-GPU sharding of a filterbank: one process per GPU, ``torch.distributed`` (NCCL
over NVLink between H100s, gloo in CPU tests) for the plumbing.

Every (stream, channel) pair is an independent recurrence, so the path shards with no
data-path collective in steady state (SURVEY.md section 8e):

* ``mode="streams"`` -- rank ``r`` owns streams ``[lo, hi)`` and all channels. Inputs that
  already live on their rank need no communication at all (the benchmark's weak-scaling
  configuration); :meth:`ShardedBank.scatter_input_into` distributes a batch that starts on
  one rank (one NCCL scatter straight into the destination rows).
* ``mode="channels"`` -- the north-star shape: rank ``r`` owns channels ``[lo, hi)`` of every
  stream; the input block is broadcast (4 B per input sample per receiving GPU), outputs stay
  sharded. :class:`BroadcastPipeline` overlaps the broadcast of block ``i+1`` (side stream) with
  the kernel of block ``i``. Consumers that need all channels in one place have two ways:

  - :meth:`ShardedBank.gather_output_into` -- ONE in-place ``all_gather_into_tensor`` into a
    rank-major ``[world][S][C/world][T]`` buffer (no padding, no concatenation);
  - :meth:`ShardedBank.apply_into` with a :class:`PeerOutput` -- the fused form: every rank's
    kernel stores its channel rows (TMA) straight into the consumer GPU's ``y[S][C][T]`` over
    NVLink peer memory, so the transfer rides on the compute tile by tile and no gather runs.

  Both are NVLink-bound (224 B per input sample into one GPU) and are reported separately from
  the throughput path.

The compute callable is injectable so that the host-side logic is testable on CPU with
the gloo backend.
"""
from __future__ import annotations

__all__ = ["split_range", "ShardedBank", "BroadcastPipeline", "PeerOutput"]


def split_range(n, world, rank):
  """Contiguous, balanced partition of ``range(n)``: ``(lo, hi)`` of ``rank``."""
  if world < 1 or not 0 <= rank < world:
    raise ValueError("bad world/rank")
  base, extra = divmod(n, world)
  lo = rank * base + min(rank, extra)
  return lo, lo + base + (1 if rank < extra else 0)


class ShardedBank(object):
  """A :class:`~audiolazy_b200.bank.FilterBank` sharded over the ranks of a process group."""

  def __init__(self, bank, mode="streams", group=None, compute=None):
    import torch.distributed as dist
    if mode not in ("streams", "channels"):
      raise ValueError("mode must be 'streams' or 'channels'")
    self.mode = mode
    self.group = group
    self.dist = dist
    self.world = dist.get_world_size(group) if dist.is_initialized() else 1
    self.rank = dist.get_rank(group) if dist.is_initialized() else 0
    self.bank = bank
    self.n_channels = len(bank)
    if mode == "channels":
      self.c_lo, self.c_hi = split_range(self.n_channels, self.world, self.rank)
      from .bank import FilterBank
      self.local = FilterBank(list(bank)[self.c_lo:self.c_hi])
    else:
      self.c_lo, self.c_hi = 0, self.n_channels
      self.local = bank
    self._compute = compute

  # -- partitioning ----------------------------------------------------------------------
  def stream_range(self, n_streams):
    return split_range(n_streams, self.world, self.rank) if self.mode == "streams" else (0, n_streams)

  @property
  def even_channels(self):
    return self.n_channels % self.world == 0

  # -- communication ---------------------------------------------------------------------
  def broadcast_input(self, x, src=0):
    """channels mode: every rank needs the whole input block (in place broadcast)."""
    if self.world > 1:
      self.dist.broadcast(x, src=src, group=self.group)
    return x

  def scatter_input_into(self, x_full, out, src=0):
    """streams mode: rank ``src`` holds ``x_full[S_total, T]``; this rank's rows land in ``out[S_local, T]``.
    With equal shares (``S_total % world == 0``) this is ONE scatter whose send buffers are views of
    ``x_full`` -- no staging copies."""
    if self.world == 1:
      out.copy_(x_full[: out.shape[0]])
      return out
    n_total = out.shape[0] * self.world
    pieces = None
    if self.rank == src:
      if x_full.shape[0] != n_total:
        raise ValueError("scatter_input_into needs equal shares: %d rows for %d ranks x %d" % (x_full.shape[0], self.world, out.shape[0]))
      pieces = list(x_full.chunk(self.world, dim=0))
    self.dist.scatter(out, pieces, src=src, group=self.group)
    return out

  def scatter_input(self, x_full, n_streams, n_samples, src=0, device=None, dtype=None):
    """streams mode, any ``n_streams``: returns this rank's rows (ragged shares are padded to equal size)."""
    import torch
    lo, hi = self.stream_range(n_streams)
    if self.world == 1:
      return x_full[lo:hi]
    device = device or (x_full.device if x_full is not None else "cpu")
    dtype = dtype or (x_full.dtype if x_full is not None else torch.float32)
    if n_streams % self.world == 0:
      return self.scatter_input_into(x_full, torch.empty((hi - lo, n_samples), dtype=dtype, device=device), src=src)
    per = -(-n_streams // self.world)
    buf = torch.empty((per, n_samples), dtype=dtype, device=device)
    chunks = None
    if self.rank == src:
      chunks = []
      for r in range(self.world):
        a, b = split_range(n_streams, self.world, r)
        piece = torch.zeros((per, n_samples), dtype=dtype, device=device)
        piece[: b - a] = x_full[a:b]
        chunks.append(piece)
    self.dist.scatter(buf, chunks, src=src, group=self.group)
    return buf[: hi - lo].clone()

  def alloc_output(self, n_streams, n_samples, device=None):
    """This rank's output tensor ``y[S_local][C_local][T]``."""
    import torch
    dev = device or self.local.device_bank().device
    return torch.empty((n_streams, self.c_hi - self.c_lo, n_samples), dtype=torch.float32, device=dev)

  def alloc_gather(self, n_streams, n_samples, device=None):
    """Destination of :meth:`gather_output_into`: ``[world][S][C/world][T]`` (channels mode, even shares)."""
    import torch
    if self.mode != "channels" or not self.even_channels:
      raise ValueError("in-place gather needs channels mode with n_channels divisible by the world size")
    dev = device or self.local.device_bank().device
    return torch.empty((self.world, n_streams, self.n_channels // self.world, n_samples), dtype=torch.float32, device=dev)

  def gather_output_into(self, y_local, out):
    """ONE ``all_gather_into_tensor``: rank ``r``'s ``y[S][C/world][T]`` lands in ``out[r]``; channel ``c`` of stream
    ``s`` is ``out[c // (C/world), s, c % (C/world)]``. No padding, no concatenation: the collective moves exactly the
    payload. NVLink-bound; time it separately from the filtering."""
    if self.world == 1:
      out[0].copy_(y_local)
      return out
    self.dist.all_gather_into_tensor(out.view(-1), y_local.contiguous().view(-1), group=self.group)
    return out

  def gather_output(self, y_local):
    """Everything everywhere as ONE dense tensor: ``y[S, C, T]`` (channels mode) or ``y[S_total, C, T]`` (streams
    mode) on every rank. Channels mode with even shares = in-place gather + one permuting copy; the ragged cases
    pad. NVLink-bound; time it separately."""
    import torch
    if self.world == 1:
      return y_local
    if self.mode == "channels" and self.even_channels:
      S, Cl, T = y_local.shape
      buf = torch.empty((self.world, S, Cl, T), dtype=y_local.dtype, device=y_local.device)
      self.gather_output_into(y_local, buf)
      return buf.permute(1, 0, 2, 3).reshape(S, self.world * Cl, T)
    if self.mode == "channels":
      sizes = [split_range(self.n_channels, self.world, r) for r in range(self.world)]
      per = max(b - a for a, b in sizes)
      S, _, T = y_local.shape
      pad = torch.zeros((S, per, T), dtype=y_local.dtype, device=y_local.device)
      pad[:, : y_local.shape[1]] = y_local
      parts = [torch.empty_like(pad) for _ in range(self.world)]
      self.dist.all_gather(parts, pad, group=self.group)
      return torch.cat([p[:, : b - a] for p, (a, b) in zip(parts, sizes)], dim=1)
    counts = [torch.zeros(1, dtype=torch.int64, device=y_local.device) for _ in range(self.world)]
    self.dist.all_gather(counts, torch.tensor([y_local.shape[0]], dtype=torch.int64, device=y_local.device),
                         group=self.group)
    counts = [int(c.item()) for c in counts]
    per = max(counts)
    _, C, T = y_local.shape
    if min(counts) == per:
      buf = torch.empty((self.world * per, C, T), dtype=y_local.dtype, device=y_local.device)
      self.dist.all_gather_into_tensor(buf.view(-1), y_local.contiguous().view(-1), group=self.group)
      return buf
    pad = torch.zeros((per, C, T), dtype=y_local.dtype, device=y_local.device)
    pad[: y_local.shape[0]] = y_local
    parts = [torch.empty_like(pad) for _ in range(self.world)]
    self.dist.all_gather(parts, pad, group=self.group)
    return torch.cat([p[:n] for p, n in zip(parts, counts)], dim=0)

  # -- compute ---------------------------------------------------------------------------
  def apply(self, x_local, state=None, out=None):
    """Filter this rank's shard: ``x_local[S_local, T]`` -> ``y[S_local, C_local, T]``. No collective is issued
    here. As :meth:`FilterBank.apply`: ``state=None`` starts every stream from a zero state on EVERY call; pass
    ``state=sharded.local.new_state(S)`` to continue streams across calls."""
    if self._compute is not None:
      return self._compute(self.local, x_local)
    return self.local.apply(x_local, state=state, out=out)

  def apply_into(self, x, peer_out, state=None):
    """channels mode, fused compute + collective: filter ``x[S, T]`` and store this rank's channel rows straight into
    the destination GPU's ``y[S][C][T]`` (:class:`PeerOutput`) through NVLink peer memory -- the kernel's TMA tile
    stores ARE the transfer; nothing is gathered afterwards. Call :meth:`PeerOutput.fence` before the destination
    rank reads ``y``."""
    if self.mode != "channels":
      raise ValueError("apply_into is the channel-sharded path")
    db = self.local.device_bank()
    S, T = x.shape
    if state is None:
      state = self.local.new_state(S)
    import torch
    y_ptr = peer_out.dst_ptr + self.c_lo * T * 4
    db.plan.apply_ex(x.data_ptr(), y_ptr, state.tensor.data_ptr(), S, T, x.stride(0) if S > 1 else max(T, 1), T,
                     self.n_channels * T, torch.cuda.current_stream(x.device).cuda_stream)
    return peer_out

  def pipeline(self, x_blocks, y, state, compute_sms=None):
    return BroadcastPipeline(self, x_blocks, y, state, compute_sms=compute_sms)


class BroadcastPipeline(object):
  """channels mode: block ``i+1`` is broadcast from rank ``src`` on a side stream while block ``i`` is filtered.

  ``x_blocks``: two device tensors ``[S, T]`` per rank (on rank ``src`` they hold the data to send, alternately);
  ``y``: this rank's ``[S][C_local][T]``; ``state``: a :class:`~audiolazy_b200.bank.BankState` carried across blocks.
  ``step()`` issues, without any host synchronisation: (side stream) NCCL broadcast of the NEXT block once the
  kernel that last read that buffer is done; (main stream) wait for THIS block's broadcast, kernel."""

  def __init__(self, sharded, x_blocks, y, state, src=0, compute_sms=None):
    import torch
    self.sb, self.x, self.y, self.state, self.src = sharded, x_blocks, y, state, src
    self.torch = torch
    dev = y.device
    self.side = torch.cuda.Stream(device=dev, priority=-1)
    # ``compute_sms``: run the bank kernels on a green-context stream that owns only that many SMs. The kernel's
    # one-warp CTAs otherwise sit on EVERY SM for the whole kernel and an NCCL CTA (hundreds of threads x ~100
    # registers) needs a nearly empty SM: the side-stream broadcast then waits for the kernel to end.
    self.partition = None
    self.compute = None
    if compute_sms == "auto":
      # a partition is free of charge when the kernel under-fills the machine anyway (one-warp CTAs: 24 fit on an SM)
      n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
      ctas = len(sharded.local) * ((x_blocks[0].shape[0] + 31) // 32)
      compute_sms = (n_sm - 20) // 8 * 8 if (sharded.world > 1 and ctas <= 12 * n_sm) else None
    if compute_sms:
      from . import _capi
      self.partition = _capi.PartitionStream(compute_sms, dev.index)
      self.compute = torch.cuda.ExternalStream(self.partition.handle, device=dev)
    self.bc_done = [torch.cuda.Event(), torch.cuda.Event()]
    self.i = 0
    self.primed = False

  def _broadcast(self, j):
    torch = self.torch
    with torch.cuda.stream(self.side):
      self.sb.broadcast_input(self.x[j], src=self.src)
      self.bc_done[j].record(self.side)

  def step(self):
    """Filter block ``i`` (``x_blocks[i & 1]``) and, under its kernel, broadcast block ``i+1`` (``x_blocks[(i+1) & 1]``,
    which rank ``src`` must have filled on the current stream before this call)."""
    torch = self.torch
    main = torch.cuda.current_stream(self.y.device)
    j = self.i & 1
    # everything issued so far -- the kernel that last read the other buffer, the producer of the next block --
    # precedes the broadcast; the kernel issued below does not, so the two overlap
    self.side.wait_stream(main)
    if not self.primed:
      self._broadcast(j)
      self.primed = True
    self._broadcast(j ^ 1)
    if self.compute is None:
      main.wait_event(self.bc_done[j])
      self.sb.local.apply(self.x[j], state=self.state, out=self.y)
    else:
      self.compute.wait_stream(main)
      self.compute.wait_event(self.bc_done[j])
      with torch.cuda.stream(self.compute):
        self.sb.local.apply(self.x[j], state=self.state, out=self.y)
      main.wait_stream(self.compute)
    self.i += 1

  def compute_only(self, partition=False):
    """The same kernel on an already resident block (the no-collective reference time; ``partition=True``: on the
    SM partition, when there is one)."""
    if partition and self.compute is not None:
      torch = self.torch
      main = torch.cuda.current_stream(self.y.device)
      self.compute.wait_stream(main)
      with torch.cuda.stream(self.compute):
        self.sb.local.apply(self.x[0], state=self.state, out=self.y)
      main.wait_stream(self.compute)
    else:
      self.sb.local.apply(self.x[0], state=self.state, out=self.y)

  def close(self):
    if self.partition is not None:
      self.torch.cuda.synchronize(self.y.device)
      self.partition.close()
      self.partition = self.compute = None

  def drain(self):
    """Order the main stream after every outstanding broadcast (call before reusing the buffers by hand)."""
    main = self.torch.cuda.current_stream(self.y.device)
    main.wait_stream(self.side)
    self.primed = False
    self.i = 0


class PeerOutput(object):
  """``y[S][C][T]`` float32 in symmetric memory (``torch.distributed._symmetric_memory``): every rank holds one and
  knows the peer-mapped address of every other rank's. ``dst`` is the rank whose copy the kernels write."""

  def __init__(self, n_streams, n_channels, n_samples, dst=0, group=None, device=None):
    import torch
    import torch.distributed as dist
    import torch.distributed._symmetric_memory as symm
    self.dist, self.group = dist, group
    dev = device or torch.device("cuda", torch.cuda.current_device())
    self.tensor = symm.empty((n_streams, n_channels, n_samples), dtype=torch.float32, device=dev)
    self.handle = symm.rendezvous(self.tensor, group if group is not None else dist.group.WORLD)
    self.dst = dst
    self.dst_ptr = int(self.handle.buffer_ptrs[dst])

  def fence(self):
    """All ranks' kernels have finished writing into rank ``dst``'s tensor (stream-ordered barrier)."""
    self.handle.barrier(channel=0)
