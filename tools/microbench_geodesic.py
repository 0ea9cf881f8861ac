"""Device-resident micro-benchmark of ign_geodesic_dev (CUDA events on the ctx stream).

Workloads: uint32 synthetic segmentations (the bench's jittered-grid Voronoi generator, pitch 16, with
membranes of label 0), renumbered, one source per label at its first voxel -- what teasar.fields solves:
  seg449     449^3 (SkeletonTask's 448^3 + 1 cutout)
  seg512     512^3
each as a euclidean solve at connectivity 26 and 6 with anisotropy (4, 4, 40), and as a field solve at
connectivity 26 whose weights are a hash of the voxel index in [1, 2).  Per workload: median and min ms
over the timed reps after two warm-ups, the rounds that relaxed a brick, the bricks relaxed over all
rounds, that count per brick of the volume, and the host synchronisations.  Prints one JSON line per
workload with the card's name, power limit, SM clock and throttle reasons read before and after."""
import ctypes as c
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402

U32 = _shim.IGN_U32
BRICK = (32, 8, 8)


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks_throttle_reasons.active",
                      "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
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


def workload(ctx, shape, pitch=16):
  """(renumbered labels, K, first voxel of every label) on the device"""
  n = int(np.prod(shape))
  raw, lab, uniq = ctx.alloc(n * 4), ctx.alloc(n * 4), ctx.alloc(n * 8)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(raw), U32, shape[0], shape[1], shape[2], 0, 0, 0, pitch,
                                        1 << 20, 0, 0))
  k = c.c_uint64(0)
  _shim.check(ctx.lib.ign_renumber_dev(ctx.handle, _shim.ptr(raw), U32, n, _shim.ptr(lab), _shim.ptr(uniq), n,
                                       c.byref(k)))
  ctx.sync()
  raw.free()
  uniq.free()
  K = int(k.value)
  zeros, index, value = ctx.alloc(n * 4), ctx.alloc((K + 1) * 8), ctx.alloc((K + 1) * 4)
  ctx.memset(zeros, 0, n * 4)
  _shim.check(ctx.lib.ign_label_argmax_dev(ctx.handle, _shim.ptr(lab), U32, n, _shim.ptr(zeros), K, _shim.ptr(index),
                                           _shim.ptr(value)))
  ctx.sync()
  zeros.free()
  value.free()
  return lab, K, index


def main(reps=5):
  ctx = _shim.default_context()
  for name, shape in (("seg449", (449, 449, 449)), ("seg512", (512, 512, 512))):
    n = int(np.prod(shape))
    nbricks = int(np.prod([-(-s // b) for s, b in zip(shape, BRICK)]))
    lab, K, index = workload(ctx, shape)
    dist, weights = ctx.alloc(n * 4), ctx.alloc(n * 4)
    i = np.arange(n, dtype=np.uint64)
    ctx.h2d(weights, (1 + ((i * np.uint64(2654435761)) >> np.uint64(9)) % np.uint64(4096) / 4096).astype(np.float32))
    ctx.sync()
    del i
    a = (c.c_float * 3)(4.0, 4.0, 40.0)
    for kind, conn, w in (("euclidean", 26, None), ("euclidean", 6, None), ("field", 26, _shim.ptr(weights))):
      def run():
        _shim.check(ctx.lib.ign_geodesic_dev(ctx.handle, _shim.ptr(lab), U32, shape[0], shape[1], shape[2], conn, a, w,
                                             index.offset(8), K, _shim.ptr(dist), None))
      before = card()
      ms, mn = timed(ctx, run, reps)
      stats = (c.c_uint64 * 3)()
      _shim.check(ctx.lib.ign_geodesic_last_stats(stats))
      print(json.dumps({"op": "ign_geodesic_dev", "workload": name, "shape": list(shape), "labels": K,
                        "weights": kind, "connectivity": conn, "gpu_before": before, "gpu_after": card(),
                        "reps": reps, "ms": round(ms, 3), "min_ms": round(mn, 3), "rounds": int(stats[0]),
                        "brick_visits": int(stats[1]), "visits_per_brick": round(stats[1] / nbricks, 2),
                        "host_syncs": int(stats[2]), "Mvox_s": round(n / (ms * 1e-3) / 1e6, 1)}), flush=True)
    for b in (lab, index, dist, weights):
      b.free()


if __name__ == "__main__":
  main()
