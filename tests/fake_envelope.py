"""The stand-in native layer of tests/fake_native.py plus the two streamed-envelope entries (``apply_envelope_ex``,
``apply_envelope_host_ex``), so that the host logic of ``EnvelopeState`` / ``envelope_streams`` runs without a GPU.

Test infrastructure only.  The envelope is the oracle's bank output rounded to float32, then the float64 one-pole
lowpass ``e = R e + g r`` and every ``decim``-th value on the caller's decimation grid (``phase`` samples of the current
window consumed before the block).
"""
import types

import numpy as np

import fake_native
import oracle
from fake_native import FakePlan, _f32, _f64


class FakeEnvelopePlan(FakePlan):

  def _envelope_rows(self, st, rows, env_state, decim, phase, mode, g, R):
    S, T = rows.shape
    C = self.n_channels
    st["x"] = np.concatenate([st["x"], rows], axis=1)
    full = oracle.bank_apply(st["x"], self._padded_bank(), xinit=st["xi"], yinit=st["yi"])
    y = full[:, :, full.shape[2] - T:].astype(np.float32).astype(np.float64)
    r = np.abs(y) if mode == "abs" else y * y
    e = env_state.reshape(C, S).T.copy()                  # [S][C]; the native layout is [C][S]
    out = np.empty((S, C, (phase + T) // decim), dtype=np.float32)
    k = 0
    for n in range(T):
      e = R * e + g * r[:, :, n]
      if (phase + n) % decim == decim - 1:
        out[:, :, k] = np.sqrt(e) if mode == "rms" else e
        k += 1
    env_state[:] = e.T.reshape(-1)
    return out

  def apply_envelope_ex(self, x_ptr, env_ptr, state_ptr, env_state_ptr, n_streams, n_samples, x_stride, env_stride, decim,
                        phase, mode, g, R, stream=0):
    S, T, C = int(n_streams), int(n_samples), self.n_channels
    if S == 0 or T == 0:
      return
    x = _f32(x_ptr, (S - 1) * x_stride + T).copy()
    rows = np.stack([x[s * x_stride:s * x_stride + T] for s in range(S)])
    out = self._envelope_rows(FakePlan.states[int(state_ptr)], rows, _f64(env_state_ptr, C * S), decim, phase, mode, g, R)
    n_out = out.shape[2]
    if n_out:
      env = _f32(env_ptr, (S * C - 1) * env_stride + n_out)
      for s in range(S):
        for c in range(C):
          off = (s * C + c) * env_stride
          env[off:off + n_out] = out[s, c]
    self.launches += 1

  def apply_envelope_host_ex(self, x, env=None, state_ptr=None, env_state_ptr=None, decim=48, phase=0, mode="abs", g=None,
                             R=None):
    x = np.atleast_2d(np.asarray(x, dtype=np.float32))
    S, C = x.shape[0], self.n_channels
    st = FakePlan.states[int(state_ptr)] if state_ptr else {"x": np.zeros((S, 0), dtype=np.float32), "xi": None, "yi": None}
    es = _f64(env_state_ptr, C * S) if env_state_ptr else np.zeros(C * S)
    out = self._envelope_rows(st, x, es, decim, phase, mode, g, R)
    if env is not None:
      env[...] = out
      return env
    return out


def install(monkeypatch):
  """fake_native.install with the envelope entries; the shim's stream can also be synchronised (the host entries order
  themselves after whatever produced the state on torch's current stream)."""
  from audiolazy_b200 import _capi
  shim = fake_native.install(monkeypatch)
  monkeypatch.setattr(_capi, "Plan", FakeEnvelopePlan)
  stream = types.SimpleNamespace(cuda_stream=0, synchronize=lambda: None)
  monkeypatch.setattr(shim.cuda, "current_stream", lambda *a, **k: stream)
  return shim
