"""Device-resident micro-benchmark of ign_find_objects_dev (CUDA events on the ctx stream).

Workloads, all uint32 with the largest label passed in (one read of the volume):
  seg449      renumbered synthetic segmentation, 449^3 (SpatialIndexTask's 448^3 + 1 cutout)
  seg2k       renumbered synthetic segmentation, 2048 x 2048 x 256
  distinct    449^3, every voxel its own label (N = 90.5 M: one flush per voxel)
  one_label   449^3, one label filling the volume (every flush to one address)
Per workload: median and min ms over the timed reps after two warm-ups, GB/s of algorithmic bytes
(the labels read once; the 24 B per label written are reported apart) and the fraction of
3.35 TB/s; beside it, for the segmentations, scipy.ndimage.find_objects on one host core, on the
C-order transpose as the reference calls it.  Prints one JSON line per workload, with the card's name and power limit."""
import ctypes as c
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402

PEAK = 3.35e12
U32 = _shim.IGN_U32


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


def synth_renumbered(ctx, shape, pitch):
  """Synthetic segmentation made and renumbered on the device -> (device u32 labels, N)."""
  n = int(np.prod(shape))
  raw, out = ctx.alloc(n * 4), ctx.alloc(n * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(raw), U32, shape[0], shape[1], shape[2], 0, 0, 0, pitch,
                                        1 << 20, 0, 0))
  cap = 1 << 22
  uniq = ctx.alloc(cap * 8)
  k = c.c_uint64(0)
  _shim.check(ctx.lib.ign_renumber_dev(ctx.handle, _shim.ptr(raw), U32, n, _shim.ptr(out), _shim.ptr(uniq), cap,
                                       c.byref(k)))
  ctx.sync()
  raw.free()
  uniq.free()
  return out, int(k.value)


def main(reps=10, host=True):
  ctx = _shim.default_context()
  gpu = card()
  work = []
  for name, shape, pitch in (("seg449", (449, 449, 449), 16), ("seg2k", (2048, 2048, 256), 16)):
    d, N = synth_renumbered(ctx, shape, pitch)
    work.append((name, shape, d, N, "synthetic segmentation, pitch %d, renumbered" % pitch))
  shape = (449, 449, 449)
  n = int(np.prod(shape))
  work.append(("distinct", shape, ctx.to_device(np.arange(1, n + 1, dtype=np.uint32)), n, "every voxel its own label"))
  work.append(("one_label", shape, ctx.to_device(np.ones(n, dtype=np.uint32)), 1, "one label fills the volume"))

  for name, shape, d, N, what in work:
    n = int(np.prod(shape))
    boxes = ctx.alloc(N * 24)
    nn = c.c_uint64(N)

    def run():
      _shim.check(ctx.lib.ign_find_objects_dev(ctx.handle, _shim.ptr(d), U32, shape[0], shape[1], shape[2], c.byref(nn),
                                               _shim.ptr(boxes)))
    ms, mn = timed(ctx, run, reps)
    rec = {"op": "ign_find_objects_dev", "workload": name, "what": what, "shape": list(shape), "dtype": "uint32",
           "labels": N, "gpu": gpu, "reps": reps, "ms": round(ms, 3), "min_ms": round(mn, 3),
           "algo_GB": round(n * 4 / 1e9, 3), "boxes_GB": round(N * 24 / 1e9, 3),
           "GBps": round(n * 4 / (ms * 1e-3) / 1e9, 1), "frac_peak": round(n * 4 / (ms * 1e-3) / PEAK, 3)}
    if host and name.startswith("seg"):  # scipy's list for 90 M labels would take tens of GB of host memory
      import scipy.ndimage
      vol = ctx.to_host(d, shape, np.uint32)
      t = time.perf_counter()
      scipy.ndimage.find_objects(vol.T)
      rec["host_scipy_ms"] = round((time.perf_counter() - t) * 1e3, 1)
      del vol
    print(json.dumps(rec), flush=True)
    boxes.free()
    d.free()


if __name__ == "__main__":
  main(host="--no-host" not in sys.argv)
