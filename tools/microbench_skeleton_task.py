"""Micro-benchmark of SkeletonTask.execute() on a file:// layer (host clock; every phase ends where the host
already waits for the device or the file system).

Workloads: uint32 synthetic segmentations (the bench's jittered-grid Voronoi generator, pitch 16, with
membranes of label 0, as tools/microbench_skeletonize.py makes them) at 449^3 (a 448^3 task + 1 voxel of
overlap) and 512^3, anisotropy (16, 16, 40), written raw in 128^3 chunks to a layer in a temporary
directory.  One task covers the whole volume; teasar_params scale 4, const 500, dust_threshold 1000,
fix_borders and fix_branching on, the spatial index on.  Both will_postprocess modes: False writes one
precomputed blob per label into the layer's skeleton directory, True one gzipped pickle fragment per
label.  Per workload and mode: median and min seconds of execute() over the timed reps after one warm-up,
and the phases of the last rep (tasks.skeleton.last_phase_seconds: download, teasar, export, writes).
Prints one JSON line per measurement with the card's name, power limit, SM clock and throttle reasons
read before and after.  `--shapes 64` and `--reps 1` make a quick run."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402
from igneous_b200._compat import CloudFiles, CloudVolume  # noqa: E402
from igneous_b200.tasks import SkeletonTask  # noqa: E402
from igneous_b200.tasks import skeleton as task_module  # noqa: E402

PARAMS = {"scale": 4, "const": 500}
ANISO = (16, 16, 40)


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks_throttle_reasons.active",
                      "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def seg(ctx, shape):
  n = int(np.prod(shape))
  raw = ctx.alloc(n * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(raw), _shim.IGN_U32, *shape, 0, 0, 0, 16, 1 << 20, 0,
                                        0))
  out = np.empty(shape, np.uint32, order="F")
  ctx.d2h(out, raw)
  ctx.sync()
  raw.free()
  return out


def make_layer(root, name, vol):
  path = "file://" + os.path.join(root, name)
  CloudVolume.from_numpy(vol, path, resolution=ANISO, chunk_size=(128, 128, 64), layer_type="segmentation")
  return path


def run(path, shape, will_postprocess):
  # a fresh skeleton directory per run, so every rep writes the same files
  shutil.rmtree(os.path.join(path[len("file://"):], "skeletons"), ignore_errors=True)
  SkeletonTask(path, shape, (0, 0, 0), 0, PARAMS, will_postprocess, dust_threshold=1000).execute()


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--shapes", type=int, nargs="+", default=[449, 512])
  ap.add_argument("--reps", type=int, default=3)
  args = ap.parse_args()
  ctx = _shim.default_context()
  root = tempfile.mkdtemp(prefix="skeleton_task_")
  try:
    for side in args.shapes:
      shape = (side, side, side)
      path = make_layer(root, "seg%d" % side, seg(ctx, shape))
      for wp in (False, True):
        before = card()
        run(path, shape, wp)
        ts = []
        for _ in range(args.reps):
          t = time.perf_counter()
          run(path, shape, wp)
          ts.append(time.perf_counter() - t)
        files = len(CloudFiles(path).list("skeletons/"))
        print(json.dumps({"op": "SkeletonTask.execute", "shape": list(shape), "will_postprocess": wp,
                          "params": PARAMS, "anisotropy": ANISO, "gpu_before": before, "gpu_after": card(),
                          "reps": args.reps, "s": round(float(np.median(ts)), 3), "min_s": round(min(ts), 3),
                          "phase_ms_last_rep": {k: round(v * 1e3, 1) for k, v in
                                                task_module.last_phase_seconds.items()},
                          "files": files}), flush=True)
  finally:
    shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
  main()
