"""Device-resident micro-benchmark of the contrast kernels (CUDA events on the ctx stream).

A 2048 x 2048 x 64 slab (the default task shape), uint8 and uint16: ign_histogram_dev,
ign_contrast_stretch_dev, ign_quantize_dev (float32 input of the same extent) and
ign_clahe_dev (clip 40, 8 x 8 tiles).  Per kernel: ms, GB/s of algorithmic bytes (histogram:
the input; the others: input + output; CLAHE's LUT writes and reads are reported
separately) and the fraction of 3.35 TB/s; beside it the host numpy / cv2 call on the same
slab.  Prints one JSON line per measurement, with the card's name and power limit."""
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402

PEAK = 3.35e12


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def timed(ctx, fn, reps):
  fn()
  fn()
  ctx.sync()
  ts = []
  for _ in range(reps):
    ctx.timer_start(0)
    fn()
    ctx.timer_stop(0)
    ts.append(ctx.timer_ms(0))
  return float(np.median(ts)), float(min(ts))


def host_ms(fn, reps=2):
  ts = []
  for _ in range(reps):
    t = time.perf_counter()
    fn()
    ts.append((time.perf_counter() - t) * 1e3)
  return round(min(ts), 1)


def main(reps=10, host=True):
  ctx = _shim.default_context()
  lib = ctx.lib
  gpu = card()
  sx, sy, sz = 2048, 2048, 64
  n = sx * sy * sz
  rng = np.random.default_rng(0)
  for dt, code, hs in ((np.uint8, _shim.IGN_U8, 256), (np.uint16, _shim.IGN_U16, 65536)):
    es = np.dtype(dt).itemsize
    img = rng.normal(hs * 0.4, hs * 0.1, size=(sx, sy, sz)).clip(0, hs - 1).astype(dt).T.copy().T  # F order
    d_in, d_out, d_hist = ctx.alloc(n * es), ctx.alloc(n * es), ctx.alloc(hs * 8)
    ctx.h2d(d_in, img)
    ctx.sync()
    common = {"shape": [sx, sy, sz], "dtype": np.dtype(dt).name, "gpu": gpu, "reps": reps}

    def report(op, ms, mn, algo_bytes, host=None, **extra):
      rec = dict(common, op=op, ms=round(ms, 3), min_ms=round(mn, 3), algo_GB=round(algo_bytes / 1e9, 3),
                 GBps=round(algo_bytes / (ms * 1e-3) / 1e9, 1), frac_peak=round(algo_bytes / (ms * 1e-3) / PEAK, 3),
                 **extra)
      if host is not None:
        rec["host_ms"] = host
      print(json.dumps(rec), flush=True)

    def hist():
      _shim.check(lib.ign_histogram_dev(ctx.handle, _shim.ptr(d_in), code, n, _shim.ptr(d_hist)))
    ms, mn = timed(ctx, hist, reps)
    report("ign_histogram_dev", ms, mn, n * es,
           host_ms(lambda: np.bincount(img.ravel(order="F"), minlength=hs)) if host else None)

    lower = np.full(sz, hs // 10, np.uint32)
    upper = np.full(sz, hs - hs // 5, np.uint32)

    def stretch():
      _shim.check(lib.ign_contrast_stretch_dev(ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, 1, _shim.ptr(lower),
                                               _shim.ptr(upper), 0.0, hs - 1.0, _shim.ptr(d_out), code))
    ms, mn = timed(ctx, stretch, reps)

    def np_stretch():
      f = img.astype(np.float32)
      f = (f - np.float32(hs // 10)) * np.float32((hs - 1) / float(upper[0] - lower[0]))
      return np.clip(np.round(f), 0, hs - 1).astype(dt)
    report("ign_contrast_stretch_dev", ms, mn, 2 * n * es, host_ms(np_stretch, 1) if host else None)

    def clahe():
      _shim.check(lib.ign_clahe_dev(ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, 40.0, 8, 8, _shim.ptr(d_out)))
    ms, mn = timed(ctx, clahe, reps)
    lut_bytes = sz * 64 * hs * es
    cv_ms = None
    if host:
      try:
        import cv2
        cl = cv2.createCLAHE(40.0, (8, 8))
        cv_ms = host_ms(lambda: [cl.apply(img[:, :, z]) for z in range(sz)], 1)
      except ImportError:
        pass
    report("ign_clahe_dev", ms, mn, 2 * n * es, cv_ms, lut_write_GB=round(lut_bytes / 1e9, 3),
           lut_reads_per_voxel=4)
    d_in.free(), d_out.free(), d_hist.free()

  f = rng.random((sx, sy, sz), dtype=np.float32)
  d_f, d_q = ctx.alloc(n * 4), ctx.alloc(n)
  ctx.h2d(d_f, f)
  ctx.sync()

  def quant():
    _shim.check(lib.ign_quantize_dev(ctx.handle, _shim.ptr(d_f), n, _shim.ptr(d_q)))
  ms, mn = timed(ctx, quant, reps)
  hq = host_ms(lambda: (f * 255.0).astype(np.uint8), 1) if host else None
  print(json.dumps({"shape": [sx, sy, sz], "dtype": "float32", "gpu": gpu, "reps": reps, "op": "ign_quantize_dev",
                    "ms": round(ms, 3), "min_ms": round(mn, 3), "algo_GB": round(5 * n / 1e9, 3),
                    "GBps": round(5 * n / (ms * 1e-3) / 1e9, 1), "frac_peak": round(5 * n / (ms * 1e-3) / PEAK, 3),
                    "host_ms": hq}), flush=True)


if __name__ == "__main__":
  main(host="--no-host" not in sys.argv)
