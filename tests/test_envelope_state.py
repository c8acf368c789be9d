"""Bookkeeping of the streamed filterbank envelope (``EnvelopeState``, ``FilterBank.envelope(..., state=)``,
``envelope_host(..., state=)``, ``envelope_streams``) without a GPU: the native layer is tests/fake_envelope.py, whose
envelope is the oracle's bank output followed by a float64 lowpass on the caller's decimation grid.  The same properties
are checked against the kernels in tests/test_envelope_stream_gpu.py."""
import itertools as it

import numpy as np
import pytest

import audiolazy_b200 as ab
import fake_envelope
from conftest import signal


@pytest.fixture
def fake(monkeypatch):
  return fake_envelope.install(monkeypatch)


def _bank():
  return ab.FilterBank([ab.gammatone.slaney(0.3, 0.05), ab.gammatone.klapuri(0.6, 0.04), ab.gammatone.sampled(1.1, 0.08)])


def _blocks(bank, x, lengths, state, **kw):
  outs, t0 = [], 0
  for n in lengths:
    phase = state.phase
    out = bank.envelope(x[:, t0:t0 + n], state=state, **kw)
    assert out.shape == (x.shape[0], len(bank), (phase + n) // state.decim)
    assert state.phase == (phase + n) % state.decim
    outs.append(out.numpy())
    t0 += n
  return np.concatenate(outs, axis=2)


@pytest.mark.parametrize("decim", [1, 7, 48])
def test_blocks_of_any_length_concatenate(fake, decim):
  torch = fake
  bank = _bank()
  x = torch.from_numpy(np.stack([signal(40, 400), signal(41, 400)]))
  lengths = [0, 1, decim - 1, 5, 0, 13, 2, 400 - 20 - decim]
  st = bank.new_envelope_state(2, decim=decim, mode="rms")
  assert (st.phase, st.decim, st.mode, st.n_streams) == (0, decim, "rms", 2)
  got = _blocks(bank, x, lengths, st, decim=decim, mode="rms")
  whole = bank.envelope(x, decim=decim, mode="rms", state=bank.new_envelope_state(2, decim=decim, mode="rms")).numpy()
  assert got.shape == (2, 3, 400 // decim) and np.array_equal(got, whole)
  # the host entry with the same kind of state gives the same values
  sh = bank.new_envelope_state(2, decim=decim, mode="rms")
  xh = x.numpy()
  host, t0 = [], 0
  for n in lengths:
    host.append(bank.envelope_host(xh[:, t0:t0 + n], decim=decim, mode="rms", state=sh))
    t0 += n
  assert np.array_equal(np.concatenate(host, axis=2), whole)
  assert sh.phase == st.phase == 400 % decim


def test_zero_length_block_keeps_the_state(fake):
  torch = fake
  bank = _bank()
  st = bank.new_envelope_state(1, decim=4)
  bank.envelope(torch.from_numpy(signal(42, 6)), decim=4, state=st)
  before = (st.phase, st.env_tensor.clone())
  out = bank.envelope(torch.zeros((1, 0), dtype=torch.float32), decim=4, state=st)
  assert out.shape == (1, 3, 0)
  assert st.phase == before[0] == 2 and torch.equal(st.env_tensor, before[1])


def test_mismatched_state_raises(fake):
  torch = fake
  bank = _bank()
  x = torch.from_numpy(np.stack([signal(43, 50), signal(44, 50)]))
  st = bank.new_envelope_state(2, cutoff=0.05, decim=5, mode="squared")
  bank.envelope(x, cutoff=0.05, decim=5, mode="squared", state=st)
  with pytest.raises(ValueError, match="cutoff"):
    bank.envelope(x, cutoff=0.06, decim=5, mode="squared", state=st)
  with pytest.raises(ValueError, match="decim"):
    bank.envelope(x, cutoff=0.05, decim=6, mode="squared", state=st)
  with pytest.raises(ValueError, match="mode"):
    bank.envelope(x, cutoff=0.05, decim=5, mode="abs", state=st)
  with pytest.raises(ValueError, match="streams"):
    bank.envelope(x[:1], cutoff=0.05, decim=5, mode="squared", state=st)
  other = ab.FilterBank([ab.gammatone.slaney(0.2, 0.05)] * 3)
  with pytest.raises(ValueError, match="another bank"):
    other.envelope(x, cutoff=0.05, decim=5, mode="squared", state=st)
  with pytest.raises(ValueError, match="another bank"):
    other.envelope_host(x.numpy(), cutoff=0.05, decim=5, mode="squared", state=st)
  with pytest.raises(ValueError, match="new_envelope_state"):
    bank.envelope(x, cutoff=0.05, decim=5, mode="squared", state=bank.new_state(2))
  with pytest.raises(ValueError):
    bank.new_envelope_state(1, decim=0)
  with pytest.raises(ValueError):
    bank.new_envelope_state(1, mode="peak")
  # an equal bank (same sections) may use the state
  twin = _bank()
  assert twin.envelope(x, cutoff=0.05, decim=5, mode="squared", state=st).shape == (2, 3, 10)


def test_envelope_streams_end_to_end(fake):
  torch = fake
  bank = _bank()
  x = signal(45, 3000)
  streams = bank.envelope_streams(iter(x.tolist()), decim=5, mode="abs")   # an iterator: blocks of 256, 1024, ...
  assert len(streams) == 3 and all(isinstance(s, ab.Stream) for s in streams)
  first = streams[1].take(60)                                            # one channel ahead of the others
  outs = [list(s) for s in streams]
  want = bank.envelope(torch.from_numpy(x), decim=5, mode="abs", state=bank.new_envelope_state(1, decim=5)).numpy()[0]
  assert np.array_equal(np.asarray(first + outs[1], dtype=np.float32), want[1])
  assert np.array_equal(np.asarray(outs[0], dtype=np.float32), want[0])
  assert np.array_equal(np.asarray(outs[2], dtype=np.float32), want[2])
  # memory= / zero= seed the bank state as bank(seq, memory=, zero=) does
  seeded = bank.envelope_streams(x.tolist(), decim=1, mode="squared", zero=0.5)[0].take(3)
  plain = bank.envelope_streams(x.tolist(), decim=1, mode="squared")[0].take(3)
  assert seeded != plain
  # endless input, finite take
  assert len(bank.envelope_streams(ab.white_noise(), decim=48)[0].take(3)) == 3
  assert len(bank.envelope_streams(it.repeat(0.25), decim=1)[2].take(5)) == 5
