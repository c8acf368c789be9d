#!/usr/bin/env python
"""Generate tests/golden/stft_cases.json by RUNNING THE REFERENCE ITSELF, under CPython >= 3.12:

    ALZ_REFERENCE=<path of the checkout> python tests/golden/make_stft.py

It records the numpy version, the SHA-256 digests of the float64 bytes of every ``window`` / ``wsymm`` strategy (sizes
0, 1, 2, 3, 7, 8, 64, 1000, 1024, and alpha variants), the outputs of ``overlap_add.numpy`` and ``.list`` on the
blocks of ola_inputs() below (float64 values, NaN and +-inf as strings), and the outputs of ``stft`` for every case
of STFT_CASES on the inputs of stft_inputs() (float32 values widened to Python floats): the float64 samples, or the
float64 frames [F, size] with ``ola=None``, stored in stft_cases.npz under ``stft_<index>``.  numpy >= 2 refuses the generator that
``overlap_add.numpy`` hands ``np.vstack`` when it normalizes, so the script lets ``np.vstack`` take any iterable; the
values it stacks are unchanged.
"""
import hashlib
import json
import math
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
SIZES = [0, 1, 2, 3, 7, 8, 64, 1000, 1024]
ALPHAS = {"blackman": [.3, 2.0 * 1430 / 18608], "cos": [2, .5]}
#: (size, hop, window name or values or None, normalize)
OLA_CONFIGS = [(4, 2, None, True), (4, 2, None, False), (8, 8, "hann", True), (8, 3, "hann", True),
               (8, 4, [.5, 1., 2., -1., 0., .25, 3., 1.], True), (8, 4, [.5, 1., 2., -1., 0., .25, 3., 1.], False),
               (6, 4, "hamming", False), (5, 5, None, True), (7, 2, "bartlett", True)]


#: stft cases: name, input, size, hop, func (see reference_func), keywords (window names are strings)
STFT_CASES = (
  [("doc_abs64", "signal", 64, None, "abs", {}),
   ("doc_hann64", "signal", 64, None, "abs", {"wnd": "hann", "ola_wnd": "hann"}),
   ("doc_analyzer", "cos", 8, 2, "ifftshift", {"ola": None}),
   ("robotize", "noise", 1024, 441, "abs", {"before": None, "wnd": "hann", "ola_wnd": "hann"}),
   ("frames_abs", "noise", 64, 16, "abs", {"ola": None, "wnd": "hann"}),
   ("before_off", "noise", 64, 16, "identity", {"before": None, "wnd": "hamming", "ola_wnd": "hann"}),
   ("after_off", "noise", 64, 16, "abs", {"after": None, "wnd": "hann"}),
   ("list_ola", "noise", 64, 24, "mask", {"ola": "list", "ola_wnd": "hann", "ola_normalize": False}),
   ("empty", "empty", 4, 2, "abs", {}),
   ("short", "short", 64, 16, "abs", {"wnd": "hann", "ola_wnd": "hann"}),
   ("nan", "nan", 64, 16, "identity", {"wnd": "hann", "ola_wnd": "hann"})] +
  [("%s_%d" % (func, size), "noise", size, max(1, size // 2), func, {"wnd": "hann", "ola_wnd": "hann"} if size > 2 else {})
   for size in (1, 2, 8, 15, 64, 97, 1000, 1024, 4096, 8192)
   for func in (("identity", "mask", "abs") if size < 4096 else ("abs",))])


def stft_inputs():
  """name -> float32 samples: noise (a case of size N takes its first max(300, 2 N + N // 3 + 1) samples), the
  reference docstring's signal and cosine, an empty and a short input, and noise with one NaN sample."""
  rng = np.random.default_rng(2024)
  noise = rng.uniform(-1, 1, 20000).astype(np.float32)
  nan = rng.uniform(-1, 1, 300).astype(np.float32)
  nan[150] = np.nan
  return {"noise": noise, "signal": np.float32([.1, .3, -.1, -.3, .5, .4, .3]), "cos": np.float32([1, 0, -1, 0] * 4),
          "empty": np.zeros(0, np.float32), "short": rng.uniform(-1, 1, 10).astype(np.float32), "nan": nan}


def stft_input(name, size):
  x = stft_inputs()[name]
  return x[:max(300, 2 * size + size // 3 + 1)] if name == "noise" else x


def mask(size):
  """The bin mask of the "mask" cases: every third bin zeroed."""
  return (np.arange(size // 2 + 1) % 3 != 0).astype(np.float64)


def reference_func(name, size):
  return {"identity": lambda b: b, "abs": abs, "ifftshift": np.fft.ifftshift,
          "mask": lambda b: b * mask(size)}[name]


def digest(values):
  return hashlib.sha256(np.asarray(values, dtype=np.float64).tobytes()).hexdigest()


def ola_inputs(size):
  """name -> list of blocks: none, one, many, and blocks holding -0.0, NaN and +-inf."""
  rng = np.random.default_rng(size)
  many = rng.uniform(-1, 1, (9, size))
  special = rng.uniform(-1, 1, (4, size))
  special[0, 0] = -0.0
  special[1, size // 2] = np.nan
  special[2, -1] = np.inf
  special[3, 0] = -np.inf
  return {"none": [], "one": [list(many[0])], "many": [list(b) for b in many], "special": [list(b) for b in special]}


def encode(values):
  return [v if math.isfinite(v) else repr(v) for v in map(float, values)]


def main():
  ref = os.environ.get("ALZ_REFERENCE")
  if not ref:
    sys.exit("set ALZ_REFERENCE to a checkout of the reference")
  sys.path.insert(0, ref)
  warnings.simplefilter("ignore")
  vstack = np.vstack
  np.vstack = lambda tup, *a, **k: vstack(list(tup), *a, **k)
  import audiolazy as al
  out = {"python": sys.version.split()[0], "numpy": np.__version__, "windows": [], "ola": []}
  for sdict_name in ("window", "wsymm"):
    sdict = getattr(al, sdict_name)
    for names, func in sdict.items():
      for size in SIZES:
        for alpha in [None] + ALPHAS.get(names[0], []):
          vals = func(size) if alpha is None else func(size, alpha)
          out["windows"].append({"dict": sdict_name, "name": names[0], "size": size, "alpha": alpha,
                                 "digest": digest(vals)})
  for size, hop, wnd, normalize in OLA_CONFIGS:
    for strategy in ("numpy", "list"):
      for name, blocks in ola_inputs(size).items():
        w = getattr(al.window, wnd) if isinstance(wnd, str) else wnd
        got = list(al.overlap_add[strategy](blocks, size=size, hop=hop, wnd=w, normalize=normalize))
        out["ola"].append({"strategy": strategy, "size": size, "hop": hop, "wnd": wnd, "normalize": normalize,
                           "input": name, "output": encode(got)})
  out["stft"] = []
  arrays = {}
  for i, (name, inp, size, hop, func, kws) in enumerate(STFT_CASES):
    kw = {k: getattr(al.window, v) if k in ("wnd", "ola_wnd") and isinstance(v, str) else v for k, v in kws.items()}
    if kw.get("ola") == "list":
      kw["ola"] = al.overlap_add.list
    x = stft_input(inp, size)
    if hop is not None:
      kw["hop"] = hop
    res = list(al.stft(reference_func(func, size), size=size, **kw)(x.astype(np.float64).tolist()))
    arr = np.array(res, dtype=np.float64).reshape(-1, size) if kws.get("ola", 0) is None else np.array(res, np.float64)
    arrays["stft_%d" % i] = arr
    out["stft"].append({"name": name, "input": inp, "size": size, "hop": hop, "func": func, "kwargs": kws,
                        "shape": list(arr.shape)})
  with open(os.path.join(HERE, "stft_cases.json"), "w") as fh:
    json.dump(out, fh, indent=0)
  np.savez_compressed(os.path.join(HERE, "stft_cases.npz"), **arrays)
  print("wrote %d windows, %d overlap-add cases, %d stft cases" % (len(out["windows"]), len(out["ola"]),
                                                                  len(out["stft"])))


if __name__ == "__main__":
  main()
