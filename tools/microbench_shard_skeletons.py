"""Micro-benchmark of hashed skeleton shards (host clock unless noted).

  hash     ign_shard_hash_dev on --labels random uint64 labels (default 10^7 and 10^8) with the shard
           parameters compute_shard_params_for_hashed gives them: device time from CUDA events around the
           call alone (labels already on the device), and the host wall time of labelshard.shard_hash with its
           copies.
  task     one ShardedFromUnshardedSkeletonMergeTask on a file:// layer in a temporary directory holding
           --skeletons gzipped precomputed skeletons (random trees of 20-200 vertices, radius and vertex_types),
           all in one shard (min_shards 1, one shard for up to ~700k labels), data and minishard indices
           gzip; phases from tasks.skeleton.last_phase_seconds: labels (.labels read and device order),
           read (file reads and gunzip), device (restrip), gzip, write.
Prints one JSON line per workload with the card's name, power limit and SM clock."""
import argparse
import ctypes
import json
import os
import shutil
import struct
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from igneous_b200 import _shim, labelshard  # noqa: E402
from igneous_b200 import task_creation as tc  # noqa: E402
from igneous_b200._compat import CloudFiles, CloudVolume  # noqa: E402
from igneous_b200.tasks import skeleton as task_module  # noqa: E402


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def bench_hash(ctx, n, rounds):
  rng = np.random.default_rng(n)
  labels = rng.integers(0, 2 ** 64 - 1, n, dtype=np.uint64, endpoint=True)
  sb, mb, ps = tc.compute_shard_params_for_hashed(n)
  runs = min(n, 1 << sb)
  bufs = [ctx.alloc(8 * n) for _ in range(3)] + [ctx.alloc(8 * (runs + 1)), ctx.alloc(8 * runs)]
  ctx.h2d(bufs[0], labels)
  ctx.sync()
  nr = ctypes.c_uint64(0)
  dev = []
  for r in range(rounds + 1):
    ctx.timer_start(0)
    d_in, d_lab, d_loc, d_start, d_shard = (_shim.ptr(b) for b in bufs)
    _shim.check(ctx.lib.ign_shard_hash_dev(ctx.handle, d_in, n, ps, mb, sb, d_lab, d_loc, d_start, d_shard,
                                           ctypes.byref(nr)))
    ctx.timer_stop(0)
    ctx.sync()
    if r:
      dev.append(ctx.timer_ms(0))
  for b in bufs:
    b.free()
  host = []
  for r in range(rounds + 1):
    t = time.perf_counter()
    labelshard.shard_hash(labels, ps, mb, sb, ctx)
    if r:
      host.append(time.perf_counter() - t)
  return {"workload": "hash", "labels": n, "shard_bits": sb, "minishard_bits": mb, "shards": int(nr.value),
          "device_ms": sorted(dev), "device_glabels_per_s": n / (np.median(dev) * 1e6),
          "host_wall_s": sorted(host)}


def skeleton_blob(rng):
  nv = int(rng.integers(20, 200))
  parent = np.array([rng.integers(max(0, i - 5), i) for i in range(1, nv)], np.uint32)
  edges = np.stack([np.arange(1, nv, dtype=np.uint32), parent], axis=1)
  verts = np.cumsum(rng.normal(0, 40, (nv, 3)), axis=0).astype(np.float32)
  return b"".join([struct.pack("<II", nv, nv - 1), verts.tobytes(), edges.tobytes(),
                   rng.uniform(50, 500, nv).astype(np.float32).tobytes(),
                   rng.integers(0, 4, nv).astype(np.uint8).tobytes()])


def bench_task(n, rounds):
  tmp = tempfile.mkdtemp()
  try:
    path = "file://" + os.path.join(tmp, "seg")
    CloudVolume.from_numpy(np.zeros((8, 8, 8), np.uint64), path, resolution=(16, 16, 40), layer_type="segmentation")
    vol = CloudVolume(path)
    vol.info["skeletons"] = "skeletons"
    vol.commit_info()
    rng = np.random.default_rng(0)
    labels = np.unique(rng.integers(1, 10 ** 12, int(n * 1.01)))[:n]
    cf = CloudFiles(CloudVolume(path).skeleton.path)
    for l in labels.tolist():
      cf.put(str(l), skeleton_blob(rng), compress="gzip")
    (task,) = tc.create_sharded_skeletons_from_unsharded_tasks(path, path, skel_dir="sharded")
    out = []
    for r in range(rounds + 1):
      t = time.perf_counter()
      task()
      total = time.perf_counter() - t
      if r:
        out.append(dict(task_module.last_phase_seconds, total=total))
    size = sum(os.path.getsize(os.path.join(tmp, "seg", "sharded", f)) for f in os.listdir(os.path.join(tmp, "seg",
                                                                                                         "sharded"))
               if f.endswith(".shard"))
    return {"workload": "task", "skeletons": n, "shard_bytes": size,
            "phases_s": {k: sorted(o[k] for o in out) for k in out[0]}}
  finally:
    shutil.rmtree(tmp)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--labels", type=int, nargs="*", default=[10 ** 7, 10 ** 8])
  ap.add_argument("--skeletons", type=int, default=50000)
  ap.add_argument("--rounds", type=int, default=3)
  a = ap.parse_args()
  ctx = _shim.default_context()
  c = card()
  for n in a.labels:
    print(json.dumps(dict(bench_hash(ctx, n, a.rounds), card=c)), flush=True)
  if a.skeletons:
    print(json.dumps(dict(bench_task(a.skeletons, a.rounds), card=c)), flush=True)


if __name__ == "__main__":
  main()
