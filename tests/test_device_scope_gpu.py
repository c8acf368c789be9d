"""Every entry point that takes a filter plan runs on the plan's device and returns with the caller's device current.

Plans are created on device 0, device 1 is made current, and each entry is called once on valid arguments; after each
call the thread's current device, read through the CUDA runtime, must still be 1.  Needs two devices."""
import ctypes

import numpy as np
import pytest

import test_kernel_matrix as km
import test_time_varying_gpu as tvm
from native_libs import torch  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def _cudart():
  """The CUDA runtime torch has loaded (already mapped under its soname), else the toolkit's."""
  for name in ("libcudart.so.12", "/usr/local/cuda/lib64/libcudart.so"):
    try:
      return ctypes.CDLL(name)
    except OSError:
      pass
  pytest.skip("no CUDA runtime library to query the current device")


def test_entries_keep_the_callers_device(torch):
  if torch.cuda.device_count() < 2:
    pytest.skip("needs 2 GPUs")
  import audiolazy_b200 as ab
  from audiolazy_b200 import _capi
  rt = _cudart()

  def current():
    dev = ctypes.c_int(-1)
    assert rt.cudaGetDevice(ctypes.byref(dev)) == 0
    return dev.value

  assert rt.cudaSetDevice(0) == 0
  bank = _capi.Plan(ab.gammatone_bank(strategy="slaney").sections())
  psum = _capi.Plan(km.biquad_bank(704, 3, 4, 3, 2), parallel=True)
  tv = _capi.Plan([tvm.TAP_SETS["three-sections"]], force_generic=True)
  assert (bank.device, psum.device, tv.device) == (0, 0, 0)

  S, T, decim, C = 2, 4096, 32, bank.n_channels
  rng = np.random.default_rng(5)
  xh = rng.uniform(-1, 1, (S, T)).astype(np.float32)
  d0 = torch.device("cuda", 0)
  x = torch.from_numpy(xh).to(d0)
  y = torch.empty((S, C, T), dtype=torch.float32, device=d0)
  out = torch.empty((S, T), dtype=torch.float32, device=d0)
  env = torch.empty((S, C, T // decim), dtype=torch.float32, device=d0)
  state = torch.zeros(bank.state_doubles(S), dtype=torch.float64, device=d0)
  env_state = torch.zeros(S * C, dtype=torch.float64, device=d0)
  psum_state = torch.zeros(psum.state_doubles(S), dtype=torch.float64, device=d0)
  tv_state = torch.zeros(max(1, tv.state_doubles(S)), dtype=torch.float64, device=d0)
  table = torch.from_numpy(tvm.make_table(tv.taps(), T, T, 5)).to(d0)
  w = torch.linspace(0, np.pi, 64, dtype=torch.float64, device=d0)
  fr = torch.empty((C, 64, 2), dtype=torch.float64, device=d0)
  torch.cuda.synchronize(d0)

  calls = [
      ("alz_state_init", lambda: bank.state_init(state.data_ptr(), S)),
      ("alz_apply_f32", lambda: bank.apply(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T)),
      ("alz_apply_f32_ex", lambda: bank.apply_ex(x.data_ptr(), y.data_ptr(), state.data_ptr(), S, T, T, T, C * T)),
      ("alz_apply_f32_host", lambda: bank.apply_host(xh)),
      ("alz_apply_envelope_f32", lambda: bank.apply_envelope(x.data_ptr(), env.data_ptr(), state.data_ptr(),
                                                             env_state.data_ptr(), S, T, T, T // decim, decim, "abs",
                                                             0.01, 0.99)),
      ("alz_apply_envelope_f32_ex", lambda: bank.apply_envelope_ex(x.data_ptr(), env.data_ptr(), state.data_ptr(),
                                                                   env_state.data_ptr(), S, T, T, T // decim, decim, 0,
                                                                   "abs", 0.01, 0.99)),
      ("alz_apply_envelope_f32_host", lambda: bank.apply_envelope_host(xh, decim=decim)),
      ("alz_apply_envelope_f32_host_ex", lambda: bank.apply_envelope_host_ex(xh, state_ptr=state.data_ptr(),
                                                                             env_state_ptr=env_state.data_ptr(),
                                                                             decim=decim)),
      ("alz_freq_response_f64", lambda: bank.freq_response(w.data_ptr(), fr.data_ptr(), 64)),
      ("alz_apply_sum_f32", lambda: psum.apply_sum(x.data_ptr(), out.data_ptr(), psum_state.data_ptr(), S, T, T, T)),
      ("alz_apply_tv_f32", lambda: tv.apply_tv(x.data_ptr(), out.data_ptr(), tv_state.data_ptr(), S, T, T, T,
                                               table.data_ptr(), T)),
  ]
  assert rt.cudaSetDevice(1) == 0
  try:
    for name, call in calls:
      call()
      assert current() == 1, "%s returned with device %d current" % (name, current())
    for name, plan in (("alz_plan_destroy", bank), ("alz_plan_destroy (parallel-sum)", psum),
                       ("alz_plan_destroy (generic)", tv)):
      _capi.lib().alz_plan_destroy(plan._h)
      plan._h = None
      assert current() == 1, "%s returned with device %d current" % (name, current())
  finally:
    assert rt.cudaSetDevice(0) == 0
  torch.cuda.synchronize(d0)
  assert torch.isfinite(y).all() and torch.isfinite(env).all() and torch.isfinite(fr).all()
