"""Device-resident micro-benchmark of ign_edt_dev (CUDA events on the ctx stream).

Workloads, uint32 synthetic segmentations (the bench's jittered-grid Voronoi generator, pitch 16,
with membranes of label 0), each with anisotropy (1, 1, 1) and (4, 4, 40), squared output, no
black border:
  seg512     512^3
  seg2k      2048 x 2048 x 256
  seg449     449^3 (SpatialIndexTask's and SkeletonTask's 448^3 + 1 cutout)
Per workload: median and min ms over the timed reps after two warm-ups, and the fraction of
3.35 TB/s on two byte counts:
  algorithmic  the labels read once and 4 B per voxel written;
  pass         what the three passes move at least: pass 1 reads the labels and writes 4 B per
               voxel; passes 2 and 3 each read the labels and 4 B per voxel and write 4 B per
               voxel, plus 8 B written and 8 B read per envelope stack entry (one per voxel of
               finite distance in a run of non-zero label, an upper bound; popped entries are
               read again and not counted).
Beside them, scipy.ndimage.distance_transform_edt on one host core on a 256^3 cutout of seg512:
for one label (the largest) and for all labels (one call per label on its bounding box grown by
one voxel, as tests/edtref.py does).  Prints one JSON line per workload, with the card's name and
power limit."""
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


def synth(ctx, shape, pitch=16):
  n = int(np.prod(shape))
  d = ctx.alloc(n * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d), U32, shape[0], shape[1], shape[2], 0, 0, 0, pitch,
                                        1 << 20, 0, 0))
  ctx.sync()
  return d


def host_scipy(vol):
  """seconds for one label (the largest) and for all labels of vol with scipy on one host core"""
  from scipy import ndimage
  uniq, inv = np.unique(vol, return_inverse=True)
  dense = inv.reshape(vol.shape) + 1
  boxes = ndimage.find_objects(dense)
  sizes = np.bincount(dense.ravel())
  nz = [i for i in range(1, len(uniq) + 1) if uniq[i - 1] != 0]
  big = max(nz, key=lambda i: sizes[i])
  t = time.perf_counter()
  ndimage.distance_transform_edt(dense == big, sampling=(4, 4, 40))
  one = time.perf_counter() - t
  t = time.perf_counter()
  for i in nz:
    sl = tuple(slice(max(0, s.start - 1), min(n, s.stop + 1)) for s, n in zip(boxes[i - 1], vol.shape))
    ndimage.distance_transform_edt(dense[sl] == i, sampling=(4, 4, 40))
  return one, time.perf_counter() - t, len(nz)


def stack_entries(ctx, d, shape):
  """voxels of non-zero label (an upper bound on the stack entries of one line pass)"""
  vol = ctx.to_host(d, shape, np.uint32)
  return int(np.count_nonzero(vol)), vol


def main(reps=10, host=True):
  ctx = _shim.default_context()
  gpu = card()
  for name, shape in (("seg512", (512, 512, 512)), ("seg2k", (2048, 2048, 256)), ("seg449", (449, 449, 449))):
    n = int(np.prod(shape))
    d = synth(ctx, shape)
    out = ctx.alloc(n * 4)
    entries, vol = stack_entries(ctx, d, shape)
    algo = n * 4 + n * 4
    moved = (n * 4 + n * 4) + 2 * (n * 4 + n * 4 + n * 4 + entries * 16)
    for a in ((1.0, 1.0, 1.0), (4.0, 4.0, 40.0)):
      an = (c.c_float * 3)(*a)

      def run():
        _shim.check(ctx.lib.ign_edt_dev(ctx.handle, _shim.ptr(d), U32, shape[0], shape[1], shape[2], an, 0, 1,
                                        _shim.ptr(out)))
      ms, mn = timed(ctx, run, reps)
      rec = {"op": "ign_edt_dev", "workload": name, "shape": list(shape), "dtype": "uint32", "anisotropy": list(a),
             "gpu": gpu, "reps": reps, "ms": round(ms, 3), "min_ms": round(mn, 3),
             "algo_GB": round(algo / 1e9, 3), "pass_GB": round(moved / 1e9, 3),
             "frac_peak_algo": round(algo / (ms * 1e-3) / PEAK, 3),
             "frac_peak_pass": round(moved / (ms * 1e-3) / PEAK, 3),
             "Gvox_s": round(n / (ms * 1e-3) / 1e9, 2)}
      if host and name == "seg512" and a[2] == 40.0:
        one, every, k = host_scipy(np.ascontiguousarray(vol[:256, :256, :256]))
        rec.update({"host_scipy_256_one_label_ms": round(one * 1e3, 1),
                    "host_scipy_256_all_labels_ms": round(every * 1e3, 1), "host_scipy_256_labels": k})
      print(json.dumps(rec), flush=True)
    del vol
    out.free()
    d.free()


if __name__ == "__main__":
  main(host="--no-host" not in sys.argv)
