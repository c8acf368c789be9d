"""Filterbank object: one input fanned out to many filters.

The reference has no bank class -- its only bank usage is a Python loop over centre
frequencies applying each cascade to a copy of the input
(``examples/gammatone_plots.py:42-73``; fan-out through ``thub``, reference
``audiolazy/lazy_stream.py:573-630``). :class:`FilterBank` is that loop as an object,
with each channel exactly the reference's filter, evaluated for all channels (and any
number of independent input streams) by ONE kernel launch per block.
"""
from __future__ import annotations

import numpy as np

from . import _engine
from .filters import CascadeFilter, FilterList, LinearFilter, _seed_histories

__all__ = ["FilterBank", "BankState", "EnvelopeState"]


class BankState(object):
  """Device state of a bank for ``n_streams`` input streams: carries every recurrence
  from one :meth:`FilterBank.apply` call to the next (endless inputs in blocks)."""

  def __init__(self, bank, n_streams, memory=None, zero=0.):
    self.bank = bank
    self.n_streams = int(n_streams)
    seeds = [_seed_histories(ch, memory, zero) for ch in bank.sections()]
    self.tensor = bank.device_bank().new_state(self.n_streams, [s[0] for s in seeds], [s[1] for s in seeds])


class EnvelopeState(object):
  """State of :meth:`FilterBank.envelope` over ``n_streams`` endless streams: the bank's state (a :class:`BankState`,
  seeded by ``memory`` / ``zero``), the float64 lowpass state of every (channel, stream) and the decimation ``phase``
  (samples of the current decimation window already consumed).  It is made for one ``cutoff``, ``decim`` and ``mode``."""

  def __init__(self, bank, n_streams, cutoff=np.pi / 512, decim=48, mode="abs", memory=None, zero=0.):
    if int(decim) < 1:
      raise ValueError("decim must be >= 1")
    if mode not in ("abs", "squared", "rms"):
      raise ValueError("mode must be 'abs', 'squared' or 'rms'")
    self.bank_state = BankState(bank, n_streams, memory=memory, zero=zero)
    self.bank = bank
    self.n_streams = self.bank_state.n_streams
    self.cutoff, self.decim, self.mode = float(cutoff), int(decim), mode
    self.phase = 0
    torch = _engine.torch_mod()
    self.env_tensor = torch.zeros(max(1, len(bank) * self.n_streams), dtype=torch.float64, device=self.bank_state.tensor.device)

  @property
  def device(self):
    return self.bank_state.tensor.device


class FilterBank(list):
  """List of LTI filters (``ZFilter`` / all-LTI ``CascadeFilter``) sharing one input.

  * ``bank(seq)`` -> list of Streams, one per channel (``[f(seq_copy) for f in bank]``).
  * ``bank.apply(x)`` -> CUDA tensor ``y[S, C, T]`` for a CUDA float32 tensor ``x[S, T]``
    of ``S`` independent streams (``channel_major=True``: ``y[C, S, T]``); pass
    ``state=bank.new_state(S)`` to continue streams across calls.
  * ``bank.apply_host(x)`` -> the same through numpy host buffers (copies inside).
  """

  def __init__(self, filters=()):
    list.__init__(self, filters)
    self._sections = None
    self._sections_of = None
    self.freqs = None
    self.rate = None

  def sections(self):
    """Channels -> sections -> ``(b, a)``: the table handed to ``alz_plan_create``."""
    ids = tuple(id(f) for f in self)                   # the cache follows any mutation of the list
    if self._sections is None or self._sections_of != ids:
      self._sections_of = ids
      table = []
      for f in self:
        if isinstance(f, CascadeFilter):
          secs = f._flat_sections()
          if secs is None:
            raise NotImplementedError("bank channels must be LTI filters")
        elif isinstance(f, LinearFilter):
          secs = f.sections()
        elif not callable(f):
          secs = LinearFilter(f).sections()
        else:
          raise NotImplementedError("bank channels must be LTI filters")
        table.append(secs)
      self._sections = table
    return self._sections

  def device_bank(self):
    return _engine.device_bank(self.sections())

  def new_state(self, n_streams, memory=None, zero=0.):
    return BankState(self, n_streams, memory=memory, zero=zero)

  def new_envelope_state(self, n_streams, cutoff=np.pi / 512, decim=48, mode="abs", memory=None, zero=0.):
    """State for :meth:`envelope` / :meth:`envelope_host` calls that continue ``n_streams`` streams block by block."""
    return EnvelopeState(self, n_streams, cutoff=cutoff, decim=decim, mode=mode, memory=memory, zero=zero)

  # -- lazy API ------------------------------------------------------------------------
  def __call__(self, seq, memory=None, zero=0.):
    secs = self.sections()
    seeds = [_seed_histories(ch, memory, zero) for ch in secs]
    return _engine.bank_streams(secs, seq, [s[0] for s in seeds], [s[1] for s in seeds])

  # -- batch API -----------------------------------------------------------------------
  def apply(self, x, state=None, out=None, channel_major=False):
    db = self.device_bank()
    if x.dim() == 1:
      x = x.unsqueeze(0)
    if state is None:
      state = self.new_state(x.shape[0])
    self._check_state(state, x.shape[0], db)
    return db.apply(x, state.tensor, out=out, channel_major=channel_major)

  def _check_state(self, state, n_streams, db):
    if state.n_streams != n_streams:
      raise ValueError("state was created for %d streams, x has %d" % (state.n_streams, n_streams))
    if state.tensor.numel() != max(1, db.plan.state_doubles(n_streams)) or state.tensor.device != db.device:
      raise ValueError("state belongs to another bank or device")

  def freq_response(self, freqs):
    """Complex128 ndarray ``[C, n]``: every channel's response on the grid ``freqs`` (rad/sample),
    evaluated on the device (the per-filter ``freq_response`` of reference
    ``lazy_filters.py:267-301``, batched over the bank)."""
    return self.device_bank().freq_response(np.asarray(freqs, dtype=np.float64)).cpu().numpy()

  # -- fused consumer --------------------------------------------------------------------
  @staticmethod
  def _envelope_pole(cutoff):
    from .filters import lowpass
    (b, a), = lowpass(cutoff).sections()      # the reference's envelope lowpass (lazy_analysis.py:440-520, lowpass.pole)
    if len(b) != 1 or len(a) != 2:
      raise NotImplementedError("the fused envelope uses a one-pole lowpass")
    return b[0] / a[0], -a[1] / a[0]

  def envelope(self, x, cutoff=np.pi / 512, decim=48, mode="abs", state=None):
    """Channel envelopes of a CUDA float32 batch ``x[S, T]`` -> ``[S, C, T // decim]``: ``envelope.<mode>`` (abs /
    squared / rms, reference ``lazy_analysis.py:440-520``) of every channel output, decimated by ``decim`` -- rectifier,
    lowpass and decimation run inside the bank kernel, the channel signals never reach memory.

    ``state`` (from :meth:`new_envelope_state`): ``x`` is the next block of the state's streams, of any length ``T``;
    returns ``[S, C, (state.phase + T) // decim]`` and advances the state, so that the outputs of successive blocks
    concatenate to the output of one call over the whole input.  ``cutoff`` / ``decim`` / ``mode`` must be the state's."""
    torch = _engine.torch_mod()
    db = self.device_bank()
    if state is not None:
      return self._envelope_block(db, x, cutoff, decim, mode, state)
    S, T = x.shape
    g, R = self._envelope_pole(cutoff)
    x = x.contiguous()
    env = torch.empty((S, len(self), T // decim), dtype=torch.float32, device=x.device)
    state = torch.zeros(max(1, db.plan.state_doubles(S)), dtype=torch.float64, device=x.device)
    env_state = torch.zeros(S * len(self), dtype=torch.float64, device=x.device)
    db.plan.apply_envelope(x.data_ptr(), env.data_ptr(), state.data_ptr(), env_state.data_ptr(), S, T, T, T // decim, decim,
                           mode, g, R, torch.cuda.current_stream(x.device).cuda_stream)
    return env

  def _check_envelope_state(self, state, n_streams, cutoff, decim, mode, db, device=None):
    if not isinstance(state, EnvelopeState):
      raise ValueError("state must come from FilterBank.new_envelope_state")
    if state.bank is not self and state.bank.sections() != self.sections():
      raise ValueError("state belongs to another bank")
    if (float(cutoff), int(decim), mode) != (state.cutoff, state.decim, state.mode):
      raise ValueError("state was created for cutoff=%r, decim=%d, mode=%r; the call asks for cutoff=%r, decim=%r, mode=%r"
                       % (state.cutoff, state.decim, state.mode, cutoff, decim, mode))
    if device is not None and state.device != device:
      raise ValueError("state lives on %s, x on %s" % (state.device, device))
    self._check_state(state.bank_state, n_streams, db)

  def _envelope_block(self, db, x, cutoff, decim, mode, state):
    torch = _engine.torch_mod()
    if x.dim() == 1:
      x = x.unsqueeze(0)
    if x.dtype != torch.float32 or x.dim() != 2:
      raise ValueError("x must be a float32 tensor [streams, samples]")
    S, T = x.shape
    self._check_envelope_state(state, S, cutoff, decim, mode, db, device=x.device)
    g, R = self._envelope_pole(cutoff)
    # the kernel moves x with TMA: 16-byte aligned rows; a block that is not is copied into a padded buffer
    xs = x.stride(0) if S > 1 else (T + 3) & ~3
    if x.stride(1) != 1 or x.data_ptr() % 16 or xs % 4:
      xp = torch.zeros((S, (T + 3) & ~3), dtype=torch.float32, device=x.device)
      xp[:, :T] = x
      x, xs = xp, xp.stride(0)
    n_out = (state.phase + T) // decim
    env = torch.empty((S, len(self), n_out), dtype=torch.float32, device=x.device)
    db.plan.apply_envelope_ex(x.data_ptr(), env.data_ptr(), state.bank_state.tensor.data_ptr(), state.env_tensor.data_ptr(),
                              S, T, max(xs, T, 1), max(n_out, 1), decim, state.phase, mode, g, R,
                              torch.cuda.current_stream(x.device).cuda_stream)
    state.phase = (state.phase + T) % decim
    return env

  def envelope_host(self, x, cutoff=np.pi / 512, decim=48, mode="abs", out=None, state=None):
    """:meth:`envelope` through host buffers (``alz_apply_envelope_f32_host``): a host caller receives ``256 / decim``
    bytes per input sample instead of the bank's 256.  ``state``: as for :meth:`envelope` (the same state object may
    serve both)."""
    g, R = self._envelope_pole(cutoff)
    db = self.device_bank()
    if state is None:
      return db.plan.apply_envelope_host(x, out, decim=decim, mode=mode, g=g, R=R)
    x = np.asarray(x, dtype=np.float32)
    S = 1 if x.ndim == 1 else x.shape[0]
    self._check_envelope_state(state, S, cutoff, decim, mode, db)
    # alz_apply_envelope_f32_host_ex runs on private streams ordered after the legacy default stream only: whatever
    # produced the state on torch's current stream must be complete
    _engine.torch_mod().cuda.current_stream(db.device).synchronize()
    env = db.plan.apply_envelope_host_ex(x, out, state.bank_state.tensor.data_ptr(), state.env_tensor.data_ptr(), decim=decim,
                                         phase=state.phase, mode=mode, g=g, R=R)
    state.phase = (state.phase + x.shape[-1]) % decim
    return env

  def envelope_streams(self, seq, cutoff=np.pi / 512, decim=48, mode="abs", memory=None, zero=0.):
    """One lazy Stream per channel of decimated envelope values of the input ``seq`` (any iterable, endless ones
    included), fed block by block through one :class:`EnvelopeState`; like :meth:`__call__`, a channel consumed far
    ahead of the others buffers their values.  With ``decim=1`` channel ``c`` is the reference's
    ``envelope.<mode>(bank(seq)[c], cutoff)``, except that the channel output is rounded to float32 (as every bank
    output is) before the rectifier."""
    db = self.device_bank()                 # errors (no device, non-LTI channel) raise at call time
    self._envelope_pole(cutoff)
    torch = _engine.torch_mod()
    state = self.new_envelope_state(1, cutoff=cutoff, decim=decim, mode=mode, memory=memory, zero=zero)

    def pump():
      for xb in _engine._blocks(seq):
        x_dev = torch.from_numpy(xb).to(db.device)
        yield self.envelope(x_dev, cutoff=cutoff, decim=decim, mode=mode, state=state)[0].cpu().numpy()

    return _engine.tee_streams(pump(), len(self))

  def apply_host(self, x, out=None, state=None):
    """``x``: float32 ndarray ``[S, T]`` (or ``[T]``) on the host; returns ndarray ``[S, C, T]``.
    Goes through ``alz_apply_f32_host`` (pipelined H2D / kernel / D2H)."""
    db = self.device_bank()
    x = np.asarray(x, dtype=np.float32)
    state_ptr = None
    if state is not None:
      self._check_state(state, 1 if x.ndim == 1 else x.shape[0], db)
      # alz_apply_f32_host runs on private streams ordered after the legacy default stream only: whatever
      # produced the state on torch's current stream (new_state, a previous apply) must be complete
      _engine.torch_mod().cuda.current_stream(db.device).synchronize()
      state_ptr = state.tensor.data_ptr()
    return db.plan.apply_host(x, out, state_ptr)
